"""Gaussian-regulariser kernels (csrc/gauss_reg.cu, K36-K38) on the GPU: against the float64 oracle (oracle/gaussian_reg_oracle.py)
from N = 1 to 3 M, raw and activated inputs, each term on or off; against the reference formulation run by torch on CUDA (its
torch.sort tie routing included); exact zeros on underflowed and untouched rows and the tied rows; bit-identical repeats; launch
counts and no host synchronisation; the reference modules (tests/golden/gaussian_reg.npz) replayed through the three plug-ins;
and renderer -> metric -> backward chains against the same chains with the torch regulariser."""
import json
import os
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import gaussian_reg_oracle as O
from test_gaussian_reg_cpu import flip_checked_masks

pytestmark = pytest.mark.gpu
DEV = "cuda"
Z = np.load(os.path.join(GOLDEN, "gaussian_reg.npz"))
META = json.load(open(os.path.join(GOLDEN, "gaussian_reg.json")))
SPAN, WRAP = 1024, 2048 * 1024            # one CTA's Gaussians; beyond WRAP the CTAs stride over the rows
SIZES = [1, 2, 31, 32, 33, 255, 256, 257, SPAN - 1, SPAN + 1, WRAP + 5, 1_000_003, 3_000_000]
# "over" and "s_l1" leave out the ratio term, whose gradient on rows with a tiny mid (r / d with d near 1e-8) sets the largest entry
# of every set that has it: there the bars relative to the largest entry say nothing about ordinary rows, which close_rows covers
TERM_SETS = {"all": (0.01, 0.004, 0.05, 0.05), "mcmc": (0.01, 0.01, 0.0, 0.0), "scale": (0.0, 0.0, 0.05, 0.05),
             "ratio": (0.0, 0.0, 0.0, 0.2), "over": (0.0, 0.0, 0.05, 0.0), "s_l1": (0.0, 0.01, 0.0, 0.0)}
V_TERMS = [0.7, -1.3, 2.0, 0.5]


def inputs(n, seed, raw):
    """(kernel opacities, kernel scales, oracle-exact float64 opacities, scales): raw logits / log-scales, or torch's CUDA fp32
    activations of them"""
    o, s = O.scene(n, seed, crafted=n >= 16)
    o_t, s_t = torch.from_numpy(o).to(DEV), torch.from_numpy(s).to(DEV)
    if not raw:
        o_t, s_t = torch.sigmoid(o_t), torch.exp(s_t)
    return o_t, s_t


def fused(o_t, s_t, raw, w, v_terms=V_TERMS, max_ratio=10.0):
    from b200gs.metrics import gaussian_regularizers
    o = o_t.clone().requires_grad_(True)
    s = s_t.clone().requires_grad_(True)
    terms, stats = gaussian_regularizers(o, s, raw=raw, opacity_weight=w[0], scale_weight=w[1], max_scale=O.MAX_SCALE,
                                         max_scale_ratio=max_ratio, scale_lambda=w[2], ratio_lambda=w[3])
    (terms * torch.tensor(v_terms, device=DEV)).sum().backward()
    torch.cuda.synchronize()
    return terms.detach().cpu().double().numpy(), stats.cpu().double().numpy(), o.grad.cpu().double().numpy(), s.grad.cpu().double().numpy()


def torch_cuda(o_t, s_t, raw, w, v_terms=V_TERMS, max_ratio=10.0):
    """the reference formulation in fp32 torch on CUDA, torch.sort as the reference calls it"""
    o = o_t.clone().requires_grad_(True)
    s = s_t.clone().requires_grad_(True)
    terms, stats = O.regularizers(o, s, raw, opacity_weight=w[0], scale_weight=w[1], max_scale=O.MAX_SCALE, max_scale_ratio=max_ratio,
                                  scale_lambda=w[2], ratio_lambda=w[3])
    (terms * torch.tensor(v_terms, device=DEV)).sum().backward()
    grad = lambda t: (t.grad if t.grad is not None else torch.zeros_like(t)).cpu().double().numpy()     # noqa: E731
    return terms.detach().cpu().double().numpy(), stats.cpu().double().numpy(), grad(o), grad(s)


def close_grad(got, ref, what, tol=1e-6):
    scale = max(np.abs(ref).max(), 1e-30)
    assert np.abs(got - ref).max() <= tol * scale, (what, np.abs(got - ref).max(), scale)


def close_rows(got, ref, what, tol=1e-5, skip=None, extra=0.0):
    """each Gaussian's gradient row within tol of that row's largest entry (1e-30 absolute for rows the reference has at 0 or at
    subnormal size), so an error on ordinary rows cannot hide under another row's large entry; rows in skip are left out; extra:
    a per-row relative allowance (O.sigmoid_grad_slack for raw opacities against float64)"""
    got, ref = got.reshape(len(got), -1), ref.reshape(len(ref), -1)
    keep = np.ones(len(ref), bool)
    if skip is not None:
        keep[np.asarray(skip, dtype=np.int64)] = False
    bound = tol * np.abs(ref).max(1, keepdims=True) + np.reshape(extra, (-1, 1)) * np.abs(ref) + 1e-30
    bad = keep[:, None] & (np.abs(got - ref) > bound)
    assert not bad.any(), (what, np.argwhere(bad)[:5].tolist(), got[bad][:5], ref[bad][:5])


@pytest.mark.parametrize("raw", [True, False], ids=["raw", "activated"])
@pytest.mark.parametrize("terms", list(TERM_SETS))
@pytest.mark.parametrize("n", SIZES)
def test_matches_the_oracle(n, terms, raw):
    w = TERM_SETS[terms]
    o_t, s_t = inputs(n, n % 97 + 3, raw)
    got_t, got_s, got_vo, got_vs = fused(o_t, s_t, raw, w)
    masks = flip_checked_masks(s_t, O.MAX_SCALE, 10.0, raw=raw)
    o64 = torch.from_numpy(o_t.cpu().double().numpy()).requires_grad_(True)
    s64 = torch.from_numpy(s_t.cpu().double().numpy()).requires_grad_(True)
    ref_t, ref_s = O.regularizers(o64, s64, raw, *w[:2], max_scale=O.MAX_SCALE, max_scale_ratio=10.0, scale_lambda=w[2],
                                  ratio_lambda=w[3], ties="device", masks=masks)
    (ref_t * torch.tensor(V_TERMS, dtype=torch.float64)).sum().backward()
    ref_t, ref_s = ref_t.detach().numpy(), ref_s.numpy()
    for k in range(4):
        assert abs(got_t[k] - ref_t[k]) <= 2e-6 * abs(ref_t[k]), (O.TERMS[k], got_t[k], ref_t[k])
        if w[k] == 0:
            assert got_t[k] == 0
    assert got_s[0] == ref_s[0] and got_s[1] == ref_s[1]
    assert abs(got_s[4] - ref_s[4]) <= 1e-6 * abs(ref_s[4])
    # the maxima are the fp32 values: torch's CUDA activation and fp32 ratio
    _, t_s, _, _ = torch_cuda(o_t, s_t, raw, w)
    assert got_s[2] == t_s[2] and got_s[3] == t_s[3]
    ref_vo = o64.grad.numpy() if o64.grad is not None else np.zeros(got_vo.shape)
    ref_vs = s64.grad.numpy() if s64.grad is not None else np.zeros(got_vs.shape)
    close_grad(got_vo, ref_vo, "v_opacities")
    close_grad(got_vs, ref_vs, "v_scales")
    close_rows(got_vo, ref_vo, "v_opacities rows", extra=O.sigmoid_grad_slack(o_t.cpu().numpy()) if raw else 0.0)
    close_rows(got_vs, ref_vs, "v_scales rows")


@pytest.mark.parametrize("raw", [True, False], ids=["raw", "activated"])
@pytest.mark.parametrize("terms", ["all", "over", "s_l1"])
@pytest.mark.parametrize("n", [257, 1_000_003, 3_000_000])
def test_matches_torch_on_cuda(n, terms, raw):
    """the production behaviour: the reference formulation as torch runs it on the device, including torch.sort's tie routing"""
    w = TERM_SETS[terms]
    o_t, s_t = inputs(n, 11, raw)
    got = fused(o_t, s_t, raw, w)
    ref = torch_cuda(o_t, s_t, raw, w)
    for k in range(4):
        assert abs(got[0][k] - ref[0][k]) <= 1e-5 * abs(ref[0][k]), O.TERMS[k]
    assert np.array_equal(got[1][:4], ref[1][:4]) and abs(got[1][4] - ref[1][4]) <= 1e-5 * ref[1][4]
    # fp32 against fp32 in another order of operations: a few ulps of the largest entry, and of each row's
    close_grad(got[2], ref[2], "v_opacities", tol=1e-5)
    close_grad(got[3], ref[3], "v_scales", tol=1e-5)
    close_rows(got[2], ref[2], "v_opacities rows")
    close_rows(got[3], ref[3], "v_scales rows")


def test_tie_routing_matches_torch_sort_for_every_pattern():
    """every ordering of three values (the 27 rows over {1, 2, 3}, 13 of them with ties), each row's ratio over the threshold so
    that the "max" and "mid" columns get different gradients: the kernels' and the oracle's routing against torch.sort on the device"""
    import itertools
    rows = torch.tensor(list(itertools.product([1.0, 2.0, 3.0], repeat=3)), device=DEV) * 0.01
    assert torch.equal(torch.sort(rows, dim=-1).indices.cpu(), O.sort_scales(rows.cpu(), "device").indices)
    o = torch.full((len(rows), 1), 0.5, device=DEV)
    w = (0.0, 0.0, 0.0, 0.3)
    got = fused(o, rows, False, w, max_ratio=0.5)
    ref = torch_cuda(o, rows, False, w, max_ratio=0.5)
    assert got[1][1] == len(rows) == ref[1][1]
    np.testing.assert_allclose(got[3], ref[3], rtol=1e-6, atol=0)


def test_exact_zeros_and_tied_rows():
    n, seed = 4099, 5
    o_t, s_t = inputs(n, seed, True)
    at = O.crafted_at(n, seed)
    _, _, vo, vs = fused(o_t, s_t, True, TERM_SETS["all"])
    _, _, tvo, tvs = torch_cuda(o_t, s_t, True, TERM_SETS["all"])
    y = torch.sigmoid(o_t).cpu().numpy()[:, 0]
    e = torch.exp(s_t).cpu().numpy()
    assert (y == 0).sum() >= 2 and not vo[y == 0].any() and not tvo[y == 0].any()
    assert (e == 0).sum() >= 3 and not vs[e == 0].any() and not tvs[e == 0].any()
    # rows under both thresholds get no over-scale or ratio gradient: exact zeros with only those terms on
    _, _, _, vs2 = fused(o_t, s_t, True, TERM_SETS["scale"])
    srt = np.sort(e, axis=1)
    under = (e <= O.MAX_SCALE).all(1) & (srt[:, 2] / (srt[:, 1] + np.float32(1e-8)) <= 10)
    assert under.sum() > 100 and not vs2[under].any()
    # tied min / mid with a ratio > 10: the "mid" gradient goes where torch.sort routes it on the device
    for i in O.TIED_ROWS:
        r = at[i]
        np.testing.assert_allclose(vs[r], tvs[r], rtol=1e-5, atol=0)
        order = O.sort_scales(torch.from_numpy(e[r:r + 1]), "device").indices[0].tolist()
        assert e[r, order[0]] == e[r, order[1]]
        assert vs2[r, order[1]] < 0 and vs2[r, order[0]] == 0      # the mid's gradient is negative; the min gets none


def test_activated_values_match_torch_bit_for_bit():
    from b200gs.metrics import gaussian_regularizers
    x = torch.linspace(-110, 30, 1_000_003, device=DEV)
    o, s = x[:, None].contiguous(), torch.stack([x, x.flip(0), x * 0.5], 1).contiguous()
    raw_t, raw_s = gaussian_regularizers(o, s, raw=True, opacity_weight=1.0, scale_weight=1.0, max_scale=1.0, scale_lambda=1.0,
                                         ratio_lambda=1.0)
    act_t, act_s = gaussian_regularizers(torch.sigmoid(o), torch.exp(s), raw=False, opacity_weight=1.0, scale_weight=1.0,
                                         max_scale=1.0, scale_lambda=1.0, ratio_lambda=1.0)
    assert torch.equal(raw_t, act_t) and torch.equal(raw_s, act_s)


def test_repeats_are_bit_identical():
    o_t, s_t = inputs(3_000_000, 2, True)
    a, b = fused(o_t, s_t, True, TERM_SETS["all"]), fused(o_t, s_t, True, TERM_SETS["all"])
    assert all(np.array_equal(x, y) for x, y in zip(a, b))


def test_no_host_synchronisation_and_launch_counts():
    from b200gs import _lib
    from b200gs.metrics import GAUSSIAN_REG_BWD_LAUNCHES, GAUSSIAN_REG_FWD_LAUNCHES, gaussian_regularizers
    L = _lib.lib()
    o_t, s_t = inputs(100_000, 4, True)
    o, s = o_t.requires_grad_(True), s_t.requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        n0 = L.b200gs_launch_count()
        terms, stats = gaussian_regularizers(o, s, raw=True, opacity_weight=0.01, scale_weight=0.01, max_scale=1.0, scale_lambda=0.05,
                                             ratio_lambda=0.05)
        n1 = L.b200gs_launch_count()
        terms.sum().backward()
        n2 = L.b200gs_launch_count()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert (n1 - n0, n2 - n1) == (GAUSSIAN_REG_FWD_LAUNCHES, GAUSSIAN_REG_BWD_LAUNCHES) == (2, 1)
    assert torch.isfinite(o.grad).all() and torch.isfinite(s.grad).all()


def replay_model(si):
    from b200gs.scene import SyntheticGaussians, make_scene
    n = META["scenes"][si][0]
    sc = make_scene(n, 1)
    sc["opacities"] = torch.from_numpy(Z[f"s{si}_opacities"])
    sc["scales"] = torch.from_numpy(Z[f"s{si}_scales"])
    return SyntheticGaussians(sc).to(DEV)


@pytest.mark.parametrize("c", META["cases"], ids=lambda c: c["key"])
def test_reference_modules_replayed_through_the_plug_ins(c):
    from b200gs import metrics as M
    from oracle.bilagrid_oracle import weyl
    H, W = META["image"]
    seed = META["scenes"][c["scene"]][1]
    cls = {"mcmc": M.B200MCMCMetrics, "scale": M.B200ScaleRegularizationMetrics, "depth": M.B200ScaleRegularizationWithDepthMetrics}
    metric = cls[c["metric"]](**c["config"]).instantiate()
    pl = types.SimpleNamespace(device=torch.device(DEV), trainer=types.SimpleNamespace(datamodule=types.SimpleNamespace(
        dataparser_outputs=types.SimpleNamespace(camera_extent=META["camera_extent"]))))
    metric.setup("fit" if c["stage"] == "train" else "validate", pl)
    metric.psnr = lambda *a: torch.tensor(META["psnr"])
    metric.no_state_dict_models["lpips"] = lambda *a: torch.tensor(META["lpips"])
    model = replay_model(c["scene"])
    render = torch.from_numpy(weyl((3, H, W), seed + 10).astype(np.float32)).to(DEV).requires_grad_(True)
    gt = torch.from_numpy(weyl((3, H, W), seed + 11).astype(np.float32)).to(DEV)
    outputs, extra = {"render": render}, None
    if c["metric"] == "depth":
        outputs["inverse_depth"] = torch.from_numpy(weyl((1, H, W), seed + 12).astype(np.float32)).to(DEV).requires_grad_(True)
        gt_d = torch.from_numpy(weyl((H, W), seed + 13).astype(np.float32))
        extra = types.SimpleNamespace(median=None, mask=None, camera=None, get=lambda device: gt_d.to(device))
    batch = (types.SimpleNamespace(device=torch.device(DEV)), ("img", gt, None), extra)
    if c["stage"] == "train":
        metrics, pbar = metric.get_train_metrics(pl, model, c["step"], batch, outputs)
    else:
        metrics, pbar = metric.get_validate_metrics(pl, model, batch, outputs)
    metrics["loss"].backward()
    assert sorted(metrics) == sorted(c["metrics"]) and pbar == c["pbar"]
    for k, ref in c["metrics"].items():
        assert abs(float(metrics[k]) - ref) <= 2e-5 * max(abs(ref), 1e-3), (k, float(metrics[k]), ref)
    at = O.crafted_at(*META["scenes"][c["scene"]])
    tied = at[list(O.TIED_ROWS)]
    near = []          # rows whose masks the CPU's and the device's fp32 exp may decide differently (DESIGN §2's threshold-flip rule)
    if c["metric"] != "mcmc":
        cfg = {**META["config"][c["metric"]], **c["config"]}
        d_s, d_r = O.threshold_distance(torch.from_numpy(Z[f"s{c['scene']}_scales"]), True, c["resolved_max_scale"], cfg["max_scale_ratio"])
        near = np.flatnonzero((d_s <= 8 * 2.0 ** -23).any(1).numpy() | (d_r <= 8 * 2.0 ** -23).numpy())
        assert len(near) <= 4
    for name in ("opacities", "scales"):
        p = model.gaussians[name]
        got = (p.grad if p.grad is not None else torch.zeros_like(p)).cpu().numpy()
        ref = Z[f"{c['key']}_v_{name}"].copy()
        if name == "scales":
            # the reference recorded on the CPU, whose sort is stable; the kernels route ties as torch.sort does on the GPU:
            # where the two put the "mid" in different columns of a tied pair, their gradients trade places
            for r in tied:
                e = torch.exp(torch.from_numpy(Z[f"s{c['scene']}_scales"][r:r + 1]))
                a, b = O.sort_scales(e, "stable").indices[0, 1].item(), O.sort_scales(e, "device").indices[0, 1].item()
                ref[r, [a, b]] = ref[r, [b, a]]
        close_grad(got, ref, name, tol=1e-5)
        # the CPU's and the device's fp32 sigmoid may differ by an ulp, which y (1 - y) magnifies near y = 1
        extra = O.sigmoid_grad_slack(Z[f"s{c['scene']}_opacities"]) if name == "opacities" else 0.0
        close_rows(got, ref, name + " rows", skip=near, extra=extra)


@pytest.mark.parametrize("kind", ["mcmc", "scale_depth"])
def test_renderer_metric_chain_matches_the_torch_chain(kind):
    """B200GSplatRenderer (fused raw path) -> B200MCMCMetrics, and B200GSplatV1Renderer -> B200ScaleRegularizationWithDepthMetrics
    (l1 depth): every parameter gradient within 1e-5 of its max of the same chain with the torch regulariser"""
    from b200gs import metrics as M
    from b200gs import ops
    from b200gs.renderers import B200GSplatRenderer
    from b200gs.scene import SyntheticGaussians, make_ring_cameras, make_scene
    from b200gs.v1 import B200GSplatV1Renderer
    H, W = 96, 128
    cam = make_ring_cameras(W, H)[2].to_device(DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    target = torch.rand(3, H, W, generator=torch.Generator().manual_seed(2)).to(DEV)
    gt_depth = torch.rand(H, W, generator=torch.Generator().manual_seed(4)).to(DEV)
    depth = types.SimpleNamespace(median=None, mask=None, camera=None, get=lambda device: gt_depth)
    step = 5000
    if kind == "mcmc":
        metric = M.B200MCMCMetrics().instantiate()
        make_renderer, render_types, key = B200GSplatRenderer, None, None
    else:
        metric = M.B200ScaleRegularizationWithDepthMetrics(max_scale=0.05, depth_output_key="inv_depth_alt").instantiate()
        make_renderer, render_types, key = lambda: B200GSplatV1Renderer().instantiate(), ["rgb", "inv_depth_alt"], "inv_depth_alt"
    metric.setup("fit", None)

    def chain(fused):
        pc = SyntheticGaussians(make_scene(4096, 5, mean_scale=0.05)).to(DEV)
        r = make_renderer().to(DEV)
        outputs = r(cam, pc, bg, render_types=render_types) if render_types else r(cam, pc, bg)
        batch = (types.SimpleNamespace(device=torch.device(DEV)), ("img", target, None), depth if key else None)
        if fused:
            loss = metric.get_train_metrics(None, pc, step, batch, outputs)[0]["loss"]
        else:
            loss, _ = ops.l1_ssim_loss(outputs["render"], target, 0.2)
            if kind == "mcmc":
                t, _ = O.regularizers(pc.gaussians["opacities"], pc.gaussians["scales"], True, opacity_weight=0.01, scale_weight=0.01)
                loss = loss + t[0] + t[1]
            else:
                from b200gs.metrics import inverse_depth_loss
                d, _ = inverse_depth_loss(gt_depth, outputs[key].squeeze(0), loss_type="l1")
                loss = loss + d * metric.get_weight(step)
                t, _ = O.regularizers(None, pc.gaussians["scales"], True, max_scale=0.05, max_scale_ratio=10.0, scale_lambda=0.05,
                                      ratio_lambda=0.05)
                loss = loss + t[2] + t[3]
        loss.backward()
        return {k: v.grad.detach().clone() for k, v in pc.gaussians.items() if v.grad is not None}

    got, ref = chain(True), chain(False)
    assert set(got) == set(ref) and {"opacities", "scales"} <= set(got)
    for k in got:
        scale = float(ref[k].abs().max())
        assert scale > 0, k
        assert float((got[k] - ref[k]).abs().max()) <= 1e-5 * scale, k
