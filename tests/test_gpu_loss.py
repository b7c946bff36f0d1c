"""Fused L1 + SSIM training loss K9/K10 (csrc/loss.cu on the tile engine csrc/ssim.cuh; ops.l1_ssim_loss) on the GPU against the
float64 oracle (oracle/loss_oracle.py, pinned to the reference's internal/utils/ssim.py + vanilla_metrics.py:57-74 by
tests/test_loss_oracle_golden.py) and against the reference's own recorded outputs (tests/golden/loss_*.npz).

Content: the seven kinds of loss_oracle.case: noise, converged, flat, saturated, masked, identical and hdr.  On flat and
near-converged content s = E[x^2] - mu^2 cancels in fp32, so no constant tolerance fits every kind: each quantity's bound is 8x
the distance of the fp32 oracle from float64 on the same input (e32), or a floor.  Gradients are checked on three pixel classes
separately, each against its own largest float64 entry: the 5-pixel image border, the tile seams (x or y % 16 in {0, 15}) and the
interior.  Sizes: every (H, W) in EDGES^2 at C = 2, middle sizes at C in {1, 2, 3, 4, 7}, 1080p, 800x800 and one 2160x3840.  Also:
the exact L1 gradient at lambda 0, the zero cotangent, identical images, symmetry, bit-identical repeats, launch counts, no host
synchronisation, strided inputs, argument errors, the fused_ssim alias, B200VanillaMetrics with a dataset mask and a renderer chain.
"""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import loss_oracle as LO

pytestmark = pytest.mark.gpu
DEV = "cuda"
EDGES = [1, 2, 5, 6, 10, 11, 15, 16, 17, 26, 27, 32, 33]       # around the 16-pixel tile, the 5-pixel halo and the 11-tap window
MIDDLE = [(37, 50), (96, 128), (270, 480), (5, 200), (200, 5)]
CHANNELS = [1, 2, 3, 4, 7]
FLOOR = {"l1": 1e-6, "ssim": 5e-6, "loss": 2e-6}
GRAD_FLOOR = 1e-4                 # x the largest |float64 gradient| of the pixel class
MARGIN = 8.0                      # x e32
RATIOS = {}                       # kind -> [largest error / e32 where 8 e32 is the bound, largest error / bound]


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    for kind, (r, used) in sorted(RATIOS.items()):
        print(f"\nK9/K10 on {kind}: largest kernel error / e32 where 8 e32 > floor: {r:.3g}; largest error / bound: {used:.3g}")


def seed_of(kind, C, H, W):
    """H * 1000 + W for the 3-channel noise pair: the inputs of the earlier fixed-content test"""
    return H * 1000 + W + 7919 * LO.KINDS.index(kind) + 104729 * (C - 3)


def oracle(img, gt, lam, up, dtype, dev="cpu", separable=True):
    """the oracle's l1, ssim, loss and up * d loss / d img (float64, on dev) in dtype on dev; on the GPU without TF32 or cuDNN,
    whose convolution algorithms would make the fp32 error a property of the algorithm chosen"""
    x = img.to(dev, dtype, copy=True).requires_grad_(True)
    with torch.backends.cudnn.flags(enabled=False, allow_tf32=False):
        loss, l1, s = LO.training_loss(x, gt.to(dev, dtype), lam, separable)
        loss.backward(torch.tensor(up, dtype=dtype, device=dev))
    return {"l1": float(l1.detach()), "ssim": float(s.detach()), "loss": float(loss.detach()), "grad": x.grad.double()}


def kernel(img, gt, lam, up):
    from b200gs import ops
    x = img.to(DEV).requires_grad_(True)
    loss, stats = ops.l1_ssim_loss(x, gt.to(DEV), lam)
    loss.backward(torch.tensor(up, device=DEV))
    return {"l1": float(stats[0]), "ssim": float(stats[1]), "loss": float(loss.detach()), "grad": x.grad}


def pixel_classes(H, W, dev):
    y, x = torch.arange(H, device=dev)[:, None], torch.arange(W, device=dev)[None, :]
    border = (x < 5) | (x >= W - 5) | (y < 5) | (y >= H - 5)
    seam = ~border & ((x % 16 == 0) | (x % 16 == 15) | (y % 16 == 0) | (y % 16 == 15))
    return {"border": border, "seam": seam, "interior": ~border & ~seam}


def _note(kind, err, e32, floor):
    r = RATIOS.setdefault(kind, [0.0, 0.0])
    if MARGIN * e32 > floor:
        r[0] = max(r[0], err / e32)
    if max(MARGIN * e32, floor) > 0:
        r[1] = max(r[1], err / max(MARGIN * e32, floor))


def check(kind, img, gt, lam=0.2, up=1.0, dev="cpu", refs=None):
    """kernel against float64: every quantity within max(8 e32, floor); returns the kernel's outputs and the oracle's"""
    r64, r32 = refs or (oracle(img, gt, lam, up, torch.float64, dev), oracle(img, gt, lam, up, torch.float32, dev))
    k = kernel(img, gt, lam, up)
    what = (kind, tuple(img.shape), lam, up)
    assert all(np.isfinite(k[q]) for q in FLOOR) and bool(torch.isfinite(k["grad"]).all()), what
    for q, floor in FLOOR.items():
        err, e32 = abs(k[q] - r64[q]), abs(r32[q] - r64[q])
        _note(kind, err, e32, floor)
        assert err <= max(MARGIN * e32, floor), (what, q, k[q], r64[q], e32)
    g64 = r64["grad"]
    d_k, d_32 = (k["grad"].to(g64.device).double() - g64).abs(), (r32["grad"] - g64).abs()
    for name, m in pixel_classes(img.shape[1], img.shape[2], g64.device).items():
        if not bool(m.any()):
            continue
        m = m.expand_as(g64)
        err, e32, scale = float(d_k[m].max()), float(d_32[m].max()), float(g64.abs()[m].max())
        _note(kind, err, e32, GRAD_FLOOR * scale)
        assert err <= max(MARGIN * e32, GRAD_FLOOR * scale), (what, name, err, e32, scale)
    return k, r64


# ---- sizes ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", EDGES)
def test_tile_edges(H):
    """every width of EDGES at this height, 2 channels: partial tiles, halos that leave the image on both sides, one-pixel images"""
    for W in EDGES:
        img, gt = LO.case("noise", 2, H, W, seed_of("noise", 2, H, W))
        check("noise", img, gt)


@pytest.mark.parametrize("C", [1, 3])
def test_tile_edges_square(C):
    for s in EDGES:
        img, gt = LO.case("noise", C, s, s, seed_of("noise", C, s, s))
        check("noise", img, gt)


@pytest.mark.parametrize("kind", LO.KINDS)
@pytest.mark.parametrize("H,W", MIDDLE)
def test_middle_sizes(H, W, kind):
    for C in CHANNELS:
        img, gt = LO.case(kind, C, H, W, seed_of(kind, C, H, W))
        k, _ = check(kind, img, gt)
        if kind == "identical":
            assert abs(k["ssim"] - 1.0) <= 1e-6
            assert float(k["grad"].abs().max()) <= 1e-4 * 0.2 / img.numel()       # the true gradient is 0


LARGE = ([("1080p", 3, 1080, 1920, kind) for kind in LO.KINDS] + [("1080p", 1, 1080, 1920, "noise"), ("1080p", 4, 1080, 1920, "noise")]
         + [("800", 3, 800, 800, "noise"), ("800", 3, 800, 800, "flat"), ("4k", 3, 2160, 3840, "flat")])


@pytest.mark.parametrize("name,C,H,W,kind", LARGE, ids=[f"{n}-c{c}-{k}" for n, c, _, _, k in LARGE])
def test_large_sizes(name, C, H, W, kind):
    """the float64 and fp32 oracles on the GPU; at 2160x3840 C * H * W > 2^24 and each channel has 135 x 240 CTAs"""
    img, gt = LO.case(kind, C, H, W, seed_of(kind, C, H, W))
    check(kind, img, gt, dev=DEV)


# ---- lambda, the cotangent and exact properties ---------------------------------------------------------------------------
@pytest.mark.parametrize("kind", LO.KINDS)
def test_lambda_and_cotangent(kind):
    C, H, W = 3, 37, 50
    img, gt = LO.case(kind, C, H, W, seed_of(kind, C, H, W))
    a, b = img.numpy(), gt.numpy()
    n = img.numel()
    for lam in (0.0, 0.2, 1.0):
        for up in (1.0, 3.0, -0.5, 0.0):
            k, _ = check(kind, img, gt, lam, up)
            v = k["grad"].cpu().numpy()
            if up == 0.0:
                assert not v.any(), (lam, "a zero cotangent gives exact zeros")
            if lam == 0.0:
                # up * (1 / (C W H)) * sgn(a - b) in the kernel's fp32 order; the reciprocal may be the fast one (1 ulp)
                inv_n = np.float32(1.0) / (np.float32(C) * np.float32(W) * np.float32(H))
                want = (np.float32(up) * inv_n) * np.sign(a - b).astype(np.float32)
                assert (np.abs(v - want) <= np.spacing(np.abs(want))).all(), (up, "the L1 gradient")
                assert not v[a == b].any(), (up, "the subgradient of |a - b| at a == b is 0")
            if kind == "identical":
                assert abs(k["ssim"] - 1.0) <= 1e-6
                assert np.abs(v).max() <= 1e-4 * lam * abs(up) / n, (lam, up)


@pytest.mark.parametrize("kind", LO.KINDS)
def test_ssim_is_symmetric(kind):
    """the SSIM statistic of (a, b) and (b, a): the same within the fp32 bound of the pair"""
    from b200gs import ops
    C, H, W = 3, 96, 128
    img, gt = LO.case(kind, C, H, W, seed_of(kind, C, H, W))
    e32 = abs(oracle(img, gt, 0.2, 1.0, torch.float32)["ssim"] - oracle(img, gt, 0.2, 1.0, torch.float64)["ssim"])
    s_ab = float(ops.l1_ssim_loss(img.to(DEV), gt.to(DEV))[1][1])
    s_ba = float(ops.l1_ssim_loss(gt.to(DEV), img.to(DEV))[1][1])
    assert abs(s_ab - s_ba) <= max(MARGIN * e32, FLOOR["ssim"]), (s_ab, s_ba, e32)


# ---- the reference's recorded outputs ----------------------------------------------------------------------------------------
def _golden_cases():
    from conftest import GOLDEN
    for path in sorted(glob.glob(os.path.join(GOLDEN, "loss_*.npz"))):
        d = np.load(path)
        if "kind" in d:                                      # loss_<kind>_c<C>_<H>x<W>: lambda 0, 0.2 and 1
            seed, C, H, W = (int(x) for x in d["meta"])
            img, gt = LO.case(str(d["kind"]), C, H, W, seed)
            for k, lam in enumerate(d["lambdas"]):
                yield path, img, gt, float(lam), float(d["l1"]), float(d["ssim"]), float(d["loss"][k]), d["grad"][k]
        else:                                                # loss_s<seed>_<H>x<W>: the noise pair, lambda 0.2
            seed, H, W = (int(x) for x in d["meta"])
            img, gt = LO.case("noise", 3, H, W, seed)
            yield path, img, gt, 0.2, float(d["l1"]), float(d["ssim"]), float(d["loss"]), d["grad"]


def test_matches_reference_golden():
    """the reference evaluates a 2-D 11x11 convolution in fp32, which rounds differently from the separable form: e32 here is the
    larger distance from float64 of the fp32 oracle in either form"""
    n = 0
    for path, img, gt, lam, l1, ssim, loss, grad in _golden_cases():
        k = kernel(img, gt, lam, 1.0)
        r64 = oracle(img, gt, lam, 1.0, torch.float64)
        e32s = [oracle(img, gt, lam, 1.0, torch.float32, separable=s) for s in (True, False)]
        for q, want, floor in (("l1", l1, 1e-6), ("ssim", ssim, 1e-5), ("loss", loss, 3e-6)):
            e32 = max(abs(e[q] - r64[q]) for e in e32s)
            assert abs(k[q] - want) <= max(MARGIN * e32, floor), (os.path.basename(path), lam, q, k[q], want)
        g = torch.from_numpy(grad).double()
        e32 = max(float((e["grad"] - r64["grad"]).abs().max()) for e in e32s)
        err = float((k["grad"].cpu().double() - g).abs().max())
        assert err <= max(MARGIN * e32, 1e-3 * float(g.abs().max())), (os.path.basename(path), lam, err)
        n += 1
    assert n >= 4 + 6 * 3


# ---- engineering checks ----------------------------------------------------------------------------------------------------
def test_repeats_are_bit_identical():
    from b200gs import ops
    img, gt = LO.case("flat", 3, 1080, 1920, 5)
    x, t = img.to(DEV).requires_grad_(True), gt.to(DEV)
    runs = []
    for _ in range(2):
        loss, stats = ops.l1_ssim_loss(x, t, 0.2)
        (v,) = torch.autograd.grad(loss, x)
        runs.append((loss.detach(), stats, v))
    (l0, s0, v0), (l1, s1, v1) = runs
    assert torch.equal(l0, l1) and torch.equal(s0, s1) and torch.equal(v0, v1)


def test_launch_counts_and_no_host_synchronisation():
    from b200gs import _lib, ops
    L = _lib.lib()
    img, gt = LO.case("masked", 3, 96, 128, 6)
    x, t = img.to(DEV).requires_grad_(True), gt.to(DEV)
    ops.l1_ssim_loss(x, t)[0].backward()                     # warm-up: library and allocator
    x.grad = None
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        n0 = L.b200gs_launch_count()
        loss, _ = ops.l1_ssim_loss(x, t, 0.2)
        n1 = L.b200gs_launch_count()
        loss.backward()
        n2 = L.b200gs_launch_count()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert (n1 - n0, n2 - n1) == (1, 1)
    assert torch.isfinite(x.grad).all()


def test_strided_input_matches_its_contiguous_copy():
    from b200gs import ops
    g = torch.Generator().manual_seed(8)
    hwc = torch.rand(61, 83, 3, generator=g).to(DEV)
    gt = torch.rand(3, 61, 83, generator=g).to(DEV)
    out = []
    for t in (hwc.permute(2, 0, 1), hwc.permute(2, 0, 1).contiguous()):
        x = t.detach().requires_grad_(True)
        loss, stats = ops.l1_ssim_loss(x, gt, 0.2)
        loss.backward()
        out.append((loss.detach(), stats, x.grad))
    assert not hwc.permute(2, 0, 1).is_contiguous()
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1]) and torch.equal(out[0][2], out[1][2])


def test_bad_arguments_raise():
    from b200gs import ops
    a = torch.rand(3, 20, 30, device=DEV)
    for img, gt in ((a[0], a[0]), (a[None], a[None]), (a, a[:, :, :29]), (a, a[:2]), (a.double(), a), (a, a.half()), (a.cpu(), a),
                    (a, a.cpu())):
        with pytest.raises(ValueError):
            ops.l1_ssim_loss(img, gt)


# ---- the callers -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 3])
def test_fused_ssim_alias(C):
    from b200gs.metrics import fused_ssim
    img, gt = LO.case("converged", C, 61, 83, 4)
    x, y = img.to(DEV).requires_grad_(True), gt.to(DEV).requires_grad_(True)
    s = fused_ssim(x[None], y[None])
    s.backward()
    x64 = img.double().requires_grad_(True)
    ref = LO.ssim(x64, gt.double())
    ref.backward()
    x32 = img.clone().requires_grad_(True)
    ref32 = LO.ssim(x32, gt)
    ref32.backward()
    e32 = abs(float(ref32) - float(ref))
    assert abs(float(s) - float(ref)) <= max(MARGIN * e32, FLOOR["ssim"])
    err, e32 = float((x.grad.cpu().double() - x64.grad).abs().max()), float((x32.grad.double() - x64.grad).abs().max())
    assert err <= max(MARGIN * e32, GRAD_FLOOR * float(x64.grad.abs().max()))
    assert y.grad is None                                     # fused-ssim differentiates img1 only
    with pytest.raises(NotImplementedError):
        fused_ssim(x[None], y[None], padding="valid")
    with pytest.raises(ValueError):
        fused_ssim(torch.stack([x, x]), torch.stack([y, y]))


@pytest.mark.parametrize("fused", [False, True])
def test_vanilla_metrics_with_a_dataset_mask(fused):
    from b200gs.metrics import B200VanillaMetrics
    C, H, W = 3, 96, 128
    g = torch.Generator().manual_seed(21)
    render, gt = LO.case("noise", C, H, W, 21)
    keep = LO.blob_keep_mask(H, W, g)                          # bool [H,W]: False is masked
    metric = B200VanillaMetrics(fused_ssim=fused).instantiate()
    metric.setup("fit", None)
    x = render.to(DEV).requires_grad_(True)
    metrics, pbar = metric.get_train_metrics(None, None, 1000, (None, ("img", gt.to(DEV), keep.to(DEV)), None), {"render": x})
    assert pbar == {"loss": True, "rgb_diff": True, "ssim": True}
    metrics["loss"].backward()
    k = {"l1": float(metrics["rgb_diff"]), "ssim": float(metrics["ssim"]), "loss": float(metrics["loss"]), "grad": x.grad}
    mimg, mgt = render * keep, gt * keep
    r64, r32 = oracle(mimg, mgt, 0.2, 1.0, torch.float64), oracle(mimg, mgt, 0.2, 1.0, torch.float32)
    for q, floor in FLOOR.items():
        assert abs(k[q] - r64[q]) <= max(MARGIN * abs(r32[q] - r64[q]), floor), q
    g64, g32 = r64["grad"] * keep, r32["grad"] * keep                # d loss / d render = d loss / d (render * keep) * keep
    err, e32 = float((k["grad"].cpu().double() - g64).abs().max()), float((g32 - g64).abs().max())
    assert err <= max(MARGIN * e32, GRAD_FLOOR * float(g64.abs().max()))
    assert not x.grad[:, ~keep.to(DEV)].any()                   # the mask's zeros stop the gradient exactly


def test_renderer_metric_chain_matches_the_torch_chain():
    """B200GSplatRenderer -> B200VanillaMetrics -> backward on a sparse scene over a flat background and a flat target: the
    Gaussian-parameter gradients match the same chain with the oracle's loss in fp32 torch within 1e-3 of each tensor's largest
    entry"""
    import types
    from b200gs.metrics import B200VanillaMetrics
    from b200gs.renderers import B200GSplatRenderer
    from b200gs.scene import SyntheticGaussians, make_ring_cameras, make_scene
    H, W = 192, 256
    cam = make_ring_cameras(W, H)[2].to_device(DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    target = (bg[:, None, None] + 0.002 * torch.randn(3, H, W, generator=torch.Generator().manual_seed(3)).to(DEV)).contiguous()
    target[:, 40:101, 70:151] = 0.6
    metric = B200VanillaMetrics().instantiate()
    metric.setup("fit", None)

    def chain(fused):
        pc = SyntheticGaussians(make_scene(256, 5, mean_scale=0.03)).to(DEV)
        outputs = B200GSplatRenderer().to(DEV)(cam, pc, bg)
        if fused:
            loss = metric.get_train_metrics(None, pc, 1000, (types.SimpleNamespace(device=torch.device(DEV)), ("img", target, None), None),
                                            outputs)[0]["loss"]
        else:
            with torch.backends.cudnn.flags(enabled=False, allow_tf32=False):
                loss = LO.training_loss(outputs["render"], target, 0.2)[0]
        loss.backward()
        flat = float(((outputs["render"].detach() - bg[:, None, None]).abs().amax(0) < 1e-6).float().mean())
        return {k: v.grad.detach().clone() for k, v in pc.gaussians.items()}, flat

    (fused, flat), (torch_chain, _) = chain(True), chain(False)
    assert flat > 0.3                                            # the background fills a large part of the render
    assert set(fused) == set(torch_chain)
    for k in fused:
        scale = float(torch_chain[k].abs().max())
        assert scale > 0, k
        assert float((fused[k] - torch_chain[k]).abs().max()) <= 1e-3 * scale, k
