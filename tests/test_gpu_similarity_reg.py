"""The k-NN query (knn_points) and the fused similarity regulariser (K43–K46) against the float64 oracle of
oracle/similarity_reg_oracle.py, their determinism, launch counts and host-sync freedom, the reference's recorded module replayed
through B200VanillaMetricsWithSimilarityRegularization and the pytorch3d drop-in, the metric's backward hook, and SegAny's call.

Error model: a neighbour set must equal the oracle's except for queries whose K-th / (K+1)-th gap the oracle marks ambiguous; the
sorted distances must match the oracle's within fp32 rounding of the coordinates in every case.  The fused term's loss and gradient
must lie within max(8 e32, floor) of the float64 oracle, e32 being the distance of the reference's own fp32 torch formula."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import similarity_reg_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def point_set(kind, n, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "uniform":
        p = torch.rand(n, 3, generator=g)
    elif kind == "clustered":
        centers = torch.rand(max(1, n // 500), 3, generator=g) * 10
        p = centers[torch.randint(0, centers.shape[0], (n,), generator=g)] + 0.01 * torch.randn(n, 3, generator=g)
        out = torch.rand(n, generator=g) < 0.01
        p[out] = (torch.rand(int(out.sum()), 3, generator=g) - 0.5) * 1000
    elif kind == "planar":
        p = torch.rand(n, 3, generator=g)
        p[:, 2] = 0.25
    elif kind == "collinear":
        t = torch.rand(n, 1, generator=g)
        p = torch.tensor([[0.5, -1.0, 2.0]]) + t * torch.tensor([[1.0, 2.0, -3.0]])
    elif kind == "duplicated":
        p = torch.rand(n, 3, generator=g)
        half = n // 2
        p[half:] = p[torch.randint(0, max(half, 1), (n - half,), generator=g)]
    else:
        raise ValueError(kind)
    return p.to(DEV)


def outside_queries(p, m, seed):
    g = torch.Generator().manual_seed(seed)
    lo, hi = p.min(0).values.cpu(), p.max(0).values.cpu()
    ext = (hi - lo).clamp_min(1.0)
    d = torch.randn(m, 3, generator=g)
    d = d / d.norm(dim=1, keepdim=True)
    return ((lo + hi) / 2 + d * ext * torch.linspace(0.6, 3.0, m)[:, None]).to(DEV)


def check_knn(q, p, K, dists, idx, allow_ambiguous=True):
    od, oi, gap = O.knn(q, p, K, chunk=max(1, int(2e7 // p.shape[0])))
    S = q.shape[0]
    assert dists.shape == (S, K) and idx.shape == (S, K) and idx.dtype == torch.int64
    assert int(idx.min()) >= 0 and int(idx.max()) < p.shape[0]
    assert (idx.sort(1).values[:, 1:] != idx.sort(1).values[:, :-1]).all(), "a neighbour appears twice"
    assert (dists[:, 1:] >= dists[:, :-1]).all(), "not ascending"
    M = float(torch.cat([q, p]).abs().max())
    dk = ((q.double()[:, None, :] - p.double()[idx]) ** 2).sum(-1)            # float64 distances of the kernel's neighbours
    tol = 1e-6 * od + 6 * 2.0 ** -23 * M * od.sqrt() + 1e-30
    assert ((dists.double() - dk).abs() <= tol).all(), "fp32 distances off"
    assert ((dk.sort(1).values - od).abs() <= tol).all(), "a neighbour set that is not the K nearest"
    amb = gap <= O.AMBIGUOUS
    same = (idx.sort(1).values == oi.sort(1).values).all(1)
    assert (same | amb).all(), int((~(same | amb)).sum())
    if not allow_ambiguous:
        assert float(amb.float().mean()) <= 0.01
    return amb


KINDS = ["uniform", "clustered", "planar", "collinear", "duplicated"]


@pytest.mark.parametrize("K", [1, 2, 16, 17, 32])
@pytest.mark.parametrize("kind", KINDS)
def test_knn_matches_the_oracle(kind, K):
    from b200gs import ops
    for n in sorted({1, K, K + 1, 2000, 200_000}):
        if n < K:
            continue
        p = point_set(kind, n, 10 + n + K)
        queries = [p] if n <= 2000 else []
        g = torch.Generator().manual_seed(n + K)
        queries.append(p[torch.randperm(n, generator=g)[:2048].to(DEV)])
        queries.append(outside_queries(p, 64, n + K))
        for j, q in enumerate(queries):
            d, i = ops.knn_points(q, p, K)
            far = j == len(queries) - 1         # outside the box: seen from afar, a tight cluster's gaps are below fp32 resolution
            check_knn(q, p, K, d, i, allow_ambiguous=(far or kind in ("duplicated", "collinear", "planar") or n <= K + 1))


def test_knn_subset_at_one_million_points():
    from b200gs import ops
    p = point_set("clustered", 1_000_000, 7)
    q = p[torch.randperm(p.shape[0], generator=torch.Generator().manual_seed(8))[:2048].to(DEV)]
    for K in (16, 32):
        d, i = ops.knn_points(q, p, K)
        check_knn(q, p, K, d, i, allow_ambiguous=False)


def test_knn_refusals():
    from b200gs import _lib, ops
    p = point_set("uniform", 10, 1)
    for K in (0, 33, 11):
        with pytest.raises(ValueError):
            ops.knn_points(p, p, K)
    L = _lib.lib()
    ws = torch.empty(int(L.b200gs_knn_workspace_bytes(10)), dtype=torch.uint8, device=DEV)
    d = torch.empty(10, 11, device=DEV)
    i = torch.empty(10, 11, dtype=torch.int64, device=DEV)
    assert L.b200gs_knn_points(10, _lib.ptr(p), 10, _lib.ptr(p), 11, _lib.ptr(d), _lib.ptr(i), _lib.ptr(ws), ws.numel(), None) == -1
    assert b"K exceeds" in L.b200gs_last_error()


# ---- the fused term ------------------------------------------------------------------------------------------------------
def fused_case(S, K, D, seed, n=None, features="randn"):
    from b200gs import ops
    n = n or max(4 * S, K + 1, 64)
    g = torch.Generator().manual_seed(seed)
    pts = (torch.rand(n, 3, generator=g) * 0.2).to(DEV)
    if features == "randn":
        f = torch.randn(n, D, generator=g)
    elif features == "zero":
        f = torch.zeros(n, D)
    elif features == "zero_row":
        f = torch.randn(n, D, generator=g)
    samples = torch.randperm(n, generator=g)[:S].to(DEV)
    dists, idx = ops.knn_points(pts[samples], pts, K)
    f = f.to(DEV)
    if features == "zero_row":
        f[idx[0, 1]] = 0.0
    return f, idx, dists


def bound(got, ref, e32, floor):
    return float((got - ref).abs().max()), max(8 * e32, floor)


def check_fused(f, idx, dists, decay, lam, kind, v=1.0):
    from b200gs import ops
    x = f.clone().requires_grad_(True)
    loss, mean, w = ops.similarity_regularization(x, idx, dists, decay=decay, weight=lam, kind=kind)
    (loss * v).backward()
    l64, m64, g64 = O.similarity_grad(f, idx, dists, decay, lam, kind, torch.float64)
    l32, _, g32 = O.similarity_grad(f, idx, dists, decay, lam, kind, torch.float32)
    pair = lam / (idx.shape[0] * idx.shape[1] * (idx.shape[1] - 1) / 2)       # d loss / d (r w) of one pair
    _, a64 = O.similarity_metric(f, idx, dists, decay, lam, kind, torch.float64, absolute=True)
    err, bar = bound(loss.double(), l64, float((l32.double() - l64).abs()), 1e-6 * lam * abs(float(a64)) + 1e-12)
    assert err <= bar, ("loss", err, bar)
    assert abs(float(mean) * lam - float(loss)) <= 1e-6 * abs(float(loss)) + 1e-12
    assert torch.allclose(w.double(), torch.exp(-decay * dists.double()), rtol=2e-6, atol=1e-30)
    scale = float(g64.abs().max())
    err, bar = bound(x.grad.double() / v, g64, float((g32.double() - g64).abs().max()), 1e-5 * scale + 1e-6 * pair)
    assert err <= bar, ("grad", err, bar, scale)
    return loss, x.grad


@pytest.mark.parametrize("kind", ["cosine", "euclidean"])
@pytest.mark.parametrize("S", [1, 20_480])
@pytest.mark.parametrize("K", [2, 3, 16, 17, 32])
@pytest.mark.parametrize("D", [1, 31, 32, 33, 64, 256])
def test_fused_term_matches_the_oracle(D, K, S, kind):
    f, idx, dists = fused_case(S, K, D, seed=D * 100 + K + S)
    check_fused(f, idx, dists, 200.0, 0.2, kind)


@pytest.mark.parametrize("kind", ["cosine", "euclidean"])
@pytest.mark.parametrize("features", ["zero", "zero_row"])
def test_fused_term_edge_rows(kind, features):
    f, idx, dists = fused_case(256, 16, 64, seed=5, features=features)
    check_fused(f, idx, dists, 200.0, 0.2, kind)


@pytest.mark.parametrize("kind", ["cosine", "euclidean"])
def test_fused_term_underflowing_weights_and_cotangent(kind):
    f, idx, dists = fused_case(512, 16, 64, seed=6)
    loss, g = check_fused(f, idx, dists, 1e9, 0.2, kind)
    check_fused(f, idx, dists, 200.0, 0.2, kind, v=-3.0)


def test_means_and_distances_get_no_gradient():
    from b200gs import ops
    f, idx, dists = fused_case(64, 16, 8, seed=9)
    d = dists.clone().requires_grad_(True)
    x = f.clone().requires_grad_(True)
    loss, mean, w = ops.similarity_regularization(x, idx, d, decay=200.0, weight=0.2, kind="cosine")
    assert not mean.requires_grad and not w.requires_grad
    loss.backward()
    assert d.grad is None and x.grad is not None


def test_repeats_are_bit_identical():
    from b200gs import ops
    p = point_set("clustered", 200_000, 3)
    q = p[torch.randperm(p.shape[0], generator=torch.Generator().manual_seed(4))[:20_480].to(DEV)]
    a, b = ops.knn_points(q, p, 16), ops.knn_points(q, p, 16)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    f = torch.randn(p.shape[0], 64, generator=torch.Generator().manual_seed(5)).to(DEV)
    grads = []
    for _ in range(2):
        x = f.clone().requires_grad_(True)
        loss, _, _ = ops.similarity_regularization(x, a[1], a[0], decay=200.0, weight=0.2, kind="cosine")
        loss.backward()
        grads.append((loss.detach(), x.grad))
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])


def test_no_host_synchronisation_and_launch_counts():
    from b200gs import _lib, ops
    L = _lib.lib()
    n = 300_000
    p = point_set("uniform", n, 11)
    q = p[:20_480].clone()
    x = torch.randn(n, 64, device=DEV).requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        n0 = L.b200gs_launch_count()
        dists, idx = ops.knn_points(q, p, 16)
        n1 = L.b200gs_launch_count()
        loss, _, _ = ops.similarity_regularization(x, idx, dists, decay=200.0, weight=0.2, kind="euclidean")
        n2 = L.b200gs_launch_count()
        loss.backward()
        n3 = L.b200gs_launch_count()
        ops.knn_mean_dist2(p)
        n4 = L.b200gs_launch_count()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert (n1 - n0, n2 - n1, n3 - n2, n4 - n3) == (ops.knn_launches(n), ops.SIMILARITY_FWD_LAUNCHES, ops.similarity_bwd_launches(n),
                                                   ops.knn_launches(n)) == (9, 2, 7, 9)
    assert torch.isfinite(x.grad).all()


# ---- the reference module: recorded values, the plug-in and the drop-in ------------------------------------------------------
GOLDEN_NPZ = os.path.join(GOLDEN, "similarity_reg.npz")
META = json.load(open(os.path.join(GOLDEN, "similarity_reg.json")))
Z = np.load(GOLDEN_NPZ)


class _Model:
    def __init__(self, means, features):
        self.means, self.features = means, features

    def get_means(self):
        return self.means

    def get_appearance_features(self):
        return self.features


class _Module:
    batch_size = 1

    def __init__(self):
        self.on_after_backward_hooks, self.logged = [], []

    def manual_backward(self, loss):
        loss.backward()

    def log(self, name, value, **kwargs):
        self.logged.append((name, value, kwargs))


def golden_tensors(c):
    sys.path.insert(0, GOLDEN)
    try:
        from make_golden_similarity_reg import inputs
    finally:
        sys.path.remove(GOLDEN)
    means, features = inputs(c["n"], c["points"], c["features"], c["seed"])
    return c["key"], means.to(DEV), features.to(DEV)


@pytest.mark.parametrize("c", META["cases"], ids=lambda c: c["key"])
def test_golden_knn_and_term(c):
    """the recorded samples' neighbours (as sets where the recording's K-th gap is ambiguous) and the recorded loss and gradient"""
    from b200gs import ops
    k, means, features = golden_tensors(c)
    samples = torch.from_numpy(Z[f"{k}_samples"]).long().to(DEV)
    dists, idx = ops.knn_points(means[samples], means, c["config"]["n_appearance_nn"])
    amb = check_knn(means[samples], means, idx.shape[1], dists, idx)
    ref_idx = torch.from_numpy(Z[f"{k}_idx"]).long().to(DEV)
    assert ((idx.sort(1).values == ref_idx.sort(1).values).all(1) | amb).all()
    x = features.clone().requires_grad_(True)
    ref_dists = torch.from_numpy(Z[f"{k}_dists"]).to(DEV)
    loss, mean, _ = ops.similarity_regularization(x, ref_idx, ref_dists, decay=c["config"]["distance_weight_decay"],
                                                  weight=c["config"]["similarity_reg_lambda"], kind=c["kind"])
    loss.backward()
    ref_loss, ref_g = float(Z[f"{k}_loss"]), Z[f"{k}_grad"]
    assert abs(float(loss) - ref_loss) <= 1e-5 * abs(ref_loss) + 1e-12, (float(loss), ref_loss)
    assert abs(float(mean) - float(Z[f"{k}_as_r"])) <= 1e-5 * abs(float(Z[f"{k}_as_r"])) + 1e-12
    assert np.abs(x.grad.cpu().numpy() - ref_g).max() <= 1e-4 * np.abs(ref_g).max() + 1e-8


@pytest.mark.parametrize("c", META["cases"], ids=lambda c: c["key"])
def test_golden_hook_through_the_plug_in(c):
    """B200VanillaMetricsWithSimilarityRegularization's training_setup hook at the recorded steps: gating, key and gradient.  The
    plug-in draws its own samples on the device, so its loss is checked against the oracle on those samples."""
    from b200gs import ops
    from b200gs.metrics import B200VanillaMetricsWithSimilarityRegularization
    k, means, features = golden_tensors(c)
    cfg = dict(c["config"])
    cfg["similarity_type"] = {"class_path": c["kind"].capitalize()}
    metric = B200VanillaMetricsWithSimilarityRegularization(**cfg).instantiate()
    pl = _Module()
    metric.training_setup(pl)
    assert len(pl.on_after_backward_hooks) == 1
    for step, called in zip(META["steps"], c["hook_called"]):
        x = features.clone().requires_grad_(True)
        model = _Model(means, x)
        torch.manual_seed(step)
        pl.on_after_backward_hooks[0](None, None, model, step, pl)
        assert (x.grad is not None) == called, step
        if called:
            name, value, kwargs = pl.logged[-1]
            assert name == "train/as_r" and kwargs == META["log_kwargs"]
            torch.manual_seed(step)
            samples = torch.randperm(means.shape[0], device=DEV)[:cfg["n_appearance_samples"]]
            dists, idx = ops.knn_points(means[samples], means, cfg["n_appearance_nn"])      # checked against the oracle above
            check_knn(means[samples], means, idx.shape[1], dists, idx)
            _, m64, g64 = O.similarity_grad(features, idx, dists, cfg["distance_weight_decay"], cfg["similarity_reg_lambda"], c["kind"])
            assert abs(float(value) - float(m64)) <= 1e-5 * abs(float(m64)) + 1e-9
            pair = cfg["similarity_reg_lambda"] / (idx.shape[0] * idx.shape[1] * (idx.shape[1] - 1) / 2)
            assert float((x.grad.double() - g64).abs().max()) <= 1e-4 * float(g64.abs().max()) + 1e-6 * pair


@pytest.mark.parametrize("c", META["cases"], ids=lambda c: c["key"])
def test_golden_reference_call_through_the_drop_in(c):
    """the reference's knn_points call (its shapes, the squeeze, the distance weights) on compat's pytorch3d.ops.knn_points with the
    recorded samples: neighbours and weights against the recording, and the loss of the oracle's fp32 restatement of the reference's
    formula on those neighbours against the recorded loss (the reference tree itself is not imported here)"""
    from b200gs import compat
    compat.install()
    from pytorch3d.ops import knn_points
    k, means, features = golden_tensors(c)
    cfg = c["config"]
    sample_indices = torch.from_numpy(Z[f"{k}_samples"]).long().to(DEV)
    with torch.no_grad():
        knn_results = knn_points(means[sample_indices].unsqueeze(0), means.unsqueeze(0), K=cfg["n_appearance_nn"])
        distance_based_weight = torch.exp(-cfg["distance_weight_decay"] * knn_results.dists.squeeze())
    assert knn_results.knn is None and knn_results.dists.shape == (1, sample_indices.shape[0], cfg["n_appearance_nn"])
    ref_idx = torch.from_numpy(Z[f"{k}_idx"]).long().to(DEV)
    amb = check_knn(means[sample_indices], means, cfg["n_appearance_nn"], knn_results.dists[0], knn_results.idx[0])
    assert ((knn_results.idx[0].sort(1).values == ref_idx.sort(1).values).all(1) | amb).all()
    ref_w = torch.exp(-cfg["distance_weight_decay"] * torch.from_numpy(Z[f"{k}_dists"]).to(DEV))
    assert torch.allclose(distance_based_weight[~amb], ref_w[~amb], rtol=1e-4, atol=1e-30)
    if sample_indices.shape[0] > 1 and not bool(amb.any()):
        loss, mean = O.similarity_metric(features, knn_results.idx.squeeze(), knn_results.dists.squeeze(), cfg["distance_weight_decay"],
                                         cfg["similarity_reg_lambda"], c["kind"], torch.float32)
        assert abs(float(loss) - float(Z[f"{k}_loss"])) <= 1e-5 * abs(float(Z[f"{k}_loss"])) + 1e-12


def test_dropin_refusals():
    from b200gs import compat
    p = point_set("uniform", 64, 1)[None]
    for kwargs in ({"norm": 1}, {"return_nn": True}, {"return_sorted": False}, {"lengths1": torch.tensor([64], device=DEV)}):
        with pytest.raises(NotImplementedError):
            compat.knn_points(p, p, K=4, **kwargs)
    with pytest.raises(NotImplementedError):
        compat.knn_points(p.clone().requires_grad_(True), p, K=4)
    with torch.no_grad():
        r = compat.knn_points(p.clone().requires_grad_(True), p, K=4)
    assert r.idx.shape == (1, 64, 4)
    two = torch.cat([p, p.flip(1)])
    r2 = compat.knn_points(two, two, K=3)
    assert torch.equal(r2.dists[0], r2.dists[1].flip(0)) and r2.idx.shape == (2, 64, 3)


def test_segany_feature_smoothing_call():
    """segany_splatting.py:276-280: knn_points(xyz[None], xyz[None], K=16).idx.squeeze() over every Gaussian"""
    from b200gs import compat
    compat.install()
    import pytorch3d.ops
    xyz = point_set("clustered", 20_000, 12)
    with torch.no_grad():
        nearest_k_idx = pytorch3d.ops.knn_points(xyz.unsqueeze(0), xyz.unsqueeze(0), K=16).idx.squeeze()
    d = ((xyz[:, None, :] - xyz[nearest_k_idx]) ** 2).sum(-1)
    check_knn(xyz, xyz, 16, d, nearest_k_idx)
    assert (nearest_k_idx[:, 0] == torch.arange(20_000, device=DEV)).float().mean() > 0.99   # self first, bar exact duplicates


def test_hook_chain_matches_the_oracle_chain():
    """metric hook on a 200 000-Gaussian clustered scene with 64-dim features at the defaults: gradient against the oracle chain on
    the same device-drawn samples, and within max(8 e32, 1e-5) of the max"""
    from b200gs.metrics import B200VanillaMetricsWithSimilarityRegularization
    means = point_set("clustered", 200_000, 21) * 0.05
    features = torch.randn(200_000, 64, generator=torch.Generator().manual_seed(22)).to(DEV)
    metric = B200VanillaMetricsWithSimilarityRegularization().instantiate()
    pl = _Module()
    metric.training_setup(pl)
    x = features.clone().requires_grad_(True)
    torch.manual_seed(100)
    pl.on_after_backward_hooks[0](None, None, _Model(means, x), 100, pl)
    torch.manual_seed(100)
    samples = torch.randperm(200_000, device=DEV)[:20_480]
    d64, i64, gap = O.knn(means[samples], means, 16, chunk=100)
    assert float((gap <= O.AMBIGUOUS).float().mean()) < 0.01
    _, m64, g64 = O.similarity_grad(features, i64, d64.float(), 200.0, 0.2, "cosine")
    _, m32, g32 = O.similarity_grad(features, i64, d64.float(), 200.0, 0.2, "cosine", torch.float32)
    e32 = float((g32.double() - g64).abs().max())
    assert float((x.grad.double() - g64).abs().max()) <= max(8 * e32, 1e-5 * float(g64.abs().max()))
    assert abs(float(pl.logged[-1][1]) - float(m64)) <= max(8 * abs(float(m32) - float(m64)), 1e-6 * abs(float(m64)))


def test_non_finite_points_and_queries_give_in_range_indices():
    """infinite and NaN reference points stay out of the grid's box and NaN queries find no finite distance: every index is in
    [0, N), the finite queries' neighbours are the oracle's among the finite points, and the similarity term runs on the result"""
    from b200gs import ops
    p = point_set("uniform", 5000, 31)
    p[7] = float("inf")
    p[11, 1] = float("-inf")
    p[13, 2] = float("nan")
    p[4000:4003] = torch.tensor([3e38, -3e38, 3e38], device=DEV)        # finite, but the box's float width overflows
    q = torch.cat([p[:64], torch.full((4, 3), float("nan"), device=DEV)])
    q[0] = float("nan")
    d, i = ops.knn_points(q, p, 16)
    assert int(i.min()) >= 0 and int(i.max()) < p.shape[0]
    assert (i.sort(1).values[:, 1:] != i.sort(1).values[:, :-1]).all()
    nanq = torch.isnan(q).any(1)
    assert torch.equal(i[nanq].sort(1).values, torch.arange(16, device=DEV).expand(int(nanq.sum()), 16))
    good = torch.isfinite(p).all(1) & (p.abs() < 1e30).all(1)
    keep = torch.nonzero(good).squeeze(1)
    fq = ~nanq & torch.isfinite(q).all(1) & (q.abs() < 1e30).all(1)
    od, oi, gap = O.knn(q[fq], p[keep], 16)
    same = (i[fq].sort(1).values == keep[oi].sort(1).values).all(1)
    assert (same | (gap <= O.AMBIGUOUS)).all()
    f = torch.randn(p.shape[0], 8, device=DEV).requires_grad_(True)
    loss, _, _ = ops.similarity_regularization(f, i[fq], d[fq], decay=200.0, weight=0.2)
    loss.backward()
    assert torch.isfinite(loss) and torch.isfinite(f.grad).all()


def test_renderer_metric_and_hook_chain_matches_the_oracle_chain():
    """a training step on a scene with appearance features: B200GSplatAppearanceEmbeddingRenderer render -> the metric's L1 + SSIM
    loss -> backward, then the metric's backward hook at step 0, which adds the similarity gradient on top of the features gradient
    the appearance MLP wrote.  Against the same render and loss backward alone plus the float64 oracle's similarity gradient on the
    hook's own samples and neighbours, within max(8 e32, 1e-5 of the max) plus the render gradient's run-to-run spread."""
    from b200gs import ops
    from b200gs.appearance import B200GSplatAppearanceEmbeddingRenderer, ModelConfig
    from b200gs.metrics import B200VanillaMetricsWithSimilarityRegularization
    from b200gs.scene import SyntheticGaussians, make_ring_cameras, make_scene

    class AppearanceGaussians(SyntheticGaussians):
        def __init__(self, raw):
            super().__init__(raw)
            self.appearance_features = torch.nn.Parameter(torch.randn(raw["means"].shape[0], 64, generator=torch.Generator().manual_seed(9)))

        def get_appearance_features(self):
            return self.appearance_features

    W, H = 256, 192
    cam = make_ring_cameras(W, H)[3].to_device(DEV)
    cam.appearance_id = torch.tensor([1], dtype=torch.int32, device=DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    target = torch.rand(3, H, W, generator=torch.Generator().manual_seed(2)).to(DEV)
    torch.manual_seed(0)
    renderer = B200GSplatAppearanceEmbeddingRenderer(model=ModelConfig(n_appearances=4)).instantiate()
    renderer._setup_model(DEV)
    metric = B200VanillaMetricsWithSimilarityRegularization(n_appearance_samples=2048).instantiate()
    metric.setup("validate", None)

    def step(with_hook):
        pc = AppearanceGaussians(make_scene(8192, 5, mean_scale=0.05)).to(DEV)
        out = renderer(cam, pc, bg, warm_up=False)
        metrics, _ = metric.get_train_metrics(None, pc, 0, (None, ("img", target, None), None), out)
        metrics["loss"].backward()
        if with_hook:
            pl = _Module()
            metric.training_setup(pl)
            torch.manual_seed(5)
            pl.on_after_backward_hooks[0](out, None, pc, 0, pl)
            assert pl.logged[-1][0] == "train/as_r"
        return pc

    render_only, render_only_again, chained = step(False), step(False), step(True)
    g_render = render_only.appearance_features.grad.double()
    spread = float((render_only_again.appearance_features.grad.double() - g_render).abs().max())
    assert float(g_render.abs().max()) > 0
    means = chained.get_means().detach()
    torch.manual_seed(5)
    samples = torch.randperm(means.shape[0], device=DEV)[:2048]
    dists, idx = ops.knn_points(means[samples], means, 16)
    check_knn(means[samples], means, 16, dists, idx)
    f = chained.appearance_features.detach()
    _, _, g64 = O.similarity_grad(f, idx, dists, 200.0, 0.2, "cosine")
    _, _, g32 = O.similarity_grad(f, idx, dists, 200.0, 0.2, "cosine", torch.float32)
    assert float(g64.abs().max()) > 0
    e32 = float((g32.double() - g64).abs().max())
    got = chained.appearance_features.grad.double() - g_render
    bar = max(8 * e32, 1e-5 * float(g64.abs().max())) + spread
    assert float((got - g64).abs().max()) <= bar, (float((got - g64).abs().max()), bar)
