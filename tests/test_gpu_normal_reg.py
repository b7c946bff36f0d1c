"""Depth-normal consistency kernels (csrc/normal_reg.cu, K39-K42) on the GPU: the loss, v_normal and depth_to_normal against the
float64 oracle (oracle/normal_reg_oracle.py) at 1080p, 800x800, 37x50, 3x3, 2xW, Hx2 and 1x1 on planes (also against the closed
form), a sphere, noise, flat and zero depth; alpha 0 and 1; a camera far from the origin; a strided normal view; pixels near
F.normalize's 1e-12 floor; bit-identical repeats; launch counts and no host synchronisation; the reference module
(tests/golden/normal_reg.npz) replayed through the plug-in and through the gsplat.utils drop-in; and a v1 renderer -> metric ->
backward chain against the same chain with the oracle's torch loss.

Error model: n_d is compared with the float64 oracle within max(8 e32, 1e-6) (+ 6e-7 for the fp32 coefficient of v_normal), e32
being the largest error of the same origin-free formula evaluated by torch in fp32 on the same input; the loss within
max(8 e32, 2e-6 max(|loss|, weight)), e32 from the fp32 torch chain.  Pixels whose |cross| is below 1e-9 (near the 1e-12 floor)
have their own e32."""
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import normal_reg_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
SIZES = [(1080, 1920), (800, 800), (37, 50), (3, 3), (2, 50), (37, 2), (1, 1)]
WEIGHT, V_LOSS = 0.05, 1.7
FLOOR = 1e-9
Z = np.load(os.path.join(GOLDEN, "normal_reg.npz"))
META = json.load(open(os.path.join(GOLDEN, "normal_reg.json")))


def on_dev(*ts):
    return tuple(t.to(DEV) for t in ts)


def fused(depth, alpha, normal, w2c, K, weight=WEIGHT, v=V_LOSS):
    """(loss, n_d recovered from v_normal) in float64, and the raw loss / v_normal tensors"""
    from b200gs.metrics import normal_consistency_loss
    n = normal.clone().requires_grad_(True)
    loss = normal_consistency_loss(n, depth[None], alpha[None], w2c, K, weight)
    (loss * v).backward()
    H, W = depth.shape
    return loss.detach(), n.grad, n.grad.double() * (-(H * W) / (weight * v))


def dropin(depth, w2c):
    """the reference's call: depth_to_normal(exp_depth.permute(1, 2, 0), torch.linalg.inv(w2c), K)"""
    from b200gs.metrics import depth_to_normal
    return lambda K: depth_to_normal(depth[None].permute(1, 2, 0), torch.linalg.inv(w2c), K)


def bound(got, ref, e32, floor=1e-6, extra=0.0):
    err = float((got - ref).abs().max()) if got.numel() else 0.0
    b = max(8 * e32, floor) + extra
    assert err <= b, (err, e32, b)
    return err


def check(depth, alpha, normal, w2c, K, weight=WEIGHT):
    H, W = depth.shape
    n64 = O.normals_from_depth(depth, w2c, K, alpha)
    n32 = O.origin_free(depth, w2c, K, alpha)
    cn = O.cross_norm(depth, w2c, K)
    inner = torch.zeros(H, W, dtype=torch.bool, device=DEV)
    inner[1:-1, 1:-1] = True
    ordinary, near = inner & (cn >= FLOOR), inner & (cn < FLOOR)
    loss, v_normal, nk = fused(depth, alpha, normal, w2c, K, weight)
    assert torch.isfinite(v_normal).all()
    # outside the interior n_d is exactly 0
    assert float(nk[:, ~inner].abs().sum()) == 0.0
    errs = {}
    for name, sel in (("ordinary", ordinary), ("near_floor", near)):
        e32 = float((n32.double() - n64)[:, sel].abs().max()) if sel.any() else 0.0
        errs[name] = bound(nk[:, sel], n64[:, sel], e32, extra=6e-7)
    # depth_to_normal (alpha 1) as the drop-in is called
    one = torch.ones_like(alpha)
    d2n = dropin(depth, w2c)(K).permute(2, 0, 1).double()
    n64_1, n32_1 = O.normals_from_depth(depth, w2c, K, one), O.origin_free(depth, w2c, K, one)
    assert float(d2n[:, ~inner].abs().sum()) == 0.0
    for sel in (ordinary, near):
        e32 = float((n32_1.double() - n64_1)[:, sel].abs().max()) if sel.any() else 0.0
        bound(d2n[:, sel], n64_1[:, sel], e32, extra=6e-7)
    # the loss
    l64 = float(O.loss(normal, depth, alpha, w2c, K, weight))
    l32 = float((1 - (normal * n32).sum(0)).mean() * weight)
    bound(loss.double(), torch.tensor(l64, dtype=torch.float64, device=DEV), abs(l32 - l64), floor=2e-6 * max(abs(l64), weight))
    return errs, n64, nk


@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("kind", O.KINDS)
def test_kernels_match_the_oracle(kind, size):
    depth, alpha, normal, w2c, K = on_dev(*O.case(kind, *size, 7))
    _, n64, nk = check(depth, alpha, normal, w2c, K)
    if kind == "zero":
        assert float(nk.abs().sum()) == 0.0
    if kind in ("plane", "flat") and min(size) >= 3:
        # the float32 depth map tilts each pixel's plane by ~eps * f
        closed = O.plane_normals(kind, *size, 7).to(DEV) * alpha
        assert float((nk - closed).abs().max()) <= 8 * 2.0 ** -24 * float(K[0, 0]) + 1e-6


@pytest.mark.parametrize("size", [(37, 50), (800, 800)], ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("a", [0.0, 1.0])
def test_alpha_zero_and_one(size, a):
    depth, alpha, normal, w2c, K = on_dev(*O.case("sphere", *size, 3, alpha=a))
    if a == 0.0:
        loss, v_normal, _ = fused(depth, alpha, normal, w2c, K)
        assert float(v_normal.abs().sum()) == 0.0
        assert float(loss) == float(torch.tensor(WEIGHT, dtype=torch.float32))      # mean(1 - 0) * weight, exactly
    else:
        check(depth, alpha, normal, w2c, K)


@pytest.mark.parametrize("translation", [1e3, 1e4, 1e5])
@pytest.mark.parametrize("kind", ["plane", "noise"])
def test_camera_far_from_the_origin(kind, translation):
    """the origin never enters the kernels: their error stays at the origin-free fp32 level, while the reference's fp32 chain loses
    bits to o + depth * ray (a declared difference)"""
    depth, alpha, normal, w2c, K = on_dev(*O.case(kind, 300, 400, 9, translation=translation))
    errs, n64, _ = check(depth, alpha, normal, w2c, K)
    ref32 = O.normals_from_depth(depth, w2c, K, alpha, dtype=torch.float32).double()
    if translation >= 1e4:
        assert float((ref32 - n64)[:, 1:-1, 1:-1].abs().max()) > 10 * errs["ordinary"]


def test_strided_normal_view_is_read_in_place():
    """normal as the v1 renderer hands it over (a channel slice of the permuted [H,W,7] render) gives the bits of a contiguous copy"""
    depth, alpha, normal, w2c, K = on_dev(*O.case("sphere", 123, 217, 4))
    feats = torch.rand(123, 217, 7, device=DEV)
    feats[..., 4:7] = normal.permute(1, 2, 0)
    feats.requires_grad_(True)
    view = feats.permute(2, 0, 1)[4:7]
    assert not view.is_contiguous()
    from b200gs.metrics import normal_consistency_loss
    loss = normal_consistency_loss(view, depth[None], alpha[None], w2c.T.contiguous().T, K, WEIGHT)
    loss.backward()
    l2, g2, _ = fused(depth, alpha, normal.contiguous(), w2c, K, v=1.0)
    assert torch.equal(loss.detach(), l2)
    assert torch.equal(feats.grad[..., 4:7].permute(2, 0, 1), g2) and float(feats.grad[..., :4].abs().sum()) == 0.0


def test_pixels_near_the_normalize_floor():
    """depths scaled so that |cross| straddles F.normalize's 1e-12 floor: n_d = cross / 1e-12 below it"""
    depth, alpha, normal, w2c, K = on_dev(*O.case("noise", 61, 83, 6))
    med = float(O.cross_norm(depth, w2c, K)[1:-1, 1:-1].median())
    depth = (depth * (1e-12 / med) ** 0.5).float()
    cn = O.cross_norm(depth, w2c, K)[1:-1, 1:-1]
    assert float((cn < 1e-12).float().mean()) > 0.2 and float((cn > 1e-12).float().mean()) > 0.2
    errs, n64, nk = check(depth, alpha, normal, w2c, K)
    below = torch.zeros_like(n64[0], dtype=torch.bool)
    below[1:-1, 1:-1] = cn < 1e-12
    assert float(n64.norm(dim=0)[below].max()) < 1.0         # really under the floor: not unit vectors


def test_repeats_are_bit_identical():
    depth, alpha, normal, w2c, K = on_dev(*O.case("noise", 1080, 1920, 8))
    a, b = fused(depth, alpha, normal, w2c, K), fused(depth, alpha, normal, w2c, K)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    from b200gs.metrics import depth_to_normal
    c2w = torch.linalg.inv(w2c)
    assert torch.equal(depth_to_normal(depth[..., None], c2w, K), depth_to_normal(depth[..., None], c2w, K))


def test_no_host_synchronisation_and_launch_counts():
    from b200gs import _lib
    from b200gs.metrics import NORMAL_REG_BWD_LAUNCHES, NORMAL_REG_FWD_LAUNCHES, depth_to_normal, normal_consistency_loss
    L = _lib.lib()
    depth, alpha, normal, w2c, K = on_dev(*O.case("sphere", 200, 300, 1))
    c2w = torch.linalg.inv(w2c)
    n = normal.clone().requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        n0 = L.b200gs_launch_count()
        loss = normal_consistency_loss(n, depth[None], alpha[None], w2c[None], K[None], WEIGHT)
        n1 = L.b200gs_launch_count()
        loss.backward()
        n2 = L.b200gs_launch_count()
        depth_to_normal(depth[..., None], c2w, K)
        n3 = L.b200gs_launch_count()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert (n1 - n0, n2 - n1, n3 - n2) == (NORMAL_REG_FWD_LAUNCHES, NORMAL_REG_BWD_LAUNCHES, 1) == (2, 1, 1)
    assert torch.isfinite(n.grad).all()


def golden_case(c):
    sys.path.insert(0, GOLDEN)
    try:
        from make_golden_normal_reg import inputs
    finally:
        sys.path.remove(GOLDEN)
    return inputs(c["kind"], *c["image"], c["seed"])


def check_golden(c, metrics, pbar, v_render, v_normal, v_scales):
    k = c["key"]
    assert sorted(metrics) == c["metric_keys"] and pbar == c["pbar"]
    for name in ("loss", "rgb_diff", "ssim", "normal_loss", "flatten_loss"):
        ref = float(Z[f"{k}_{name}"])
        assert abs(float(metrics[name]) - ref) <= 2e-5 * max(abs(ref), 1e-3), (name, float(metrics[name]), ref)
    for got, name in ((v_render, "v_render"), (v_normal, "v_normal"), (v_scales, "v_scales")):
        ref = Z[f"{k}_{name}"]
        assert np.abs(got.detach().cpu().numpy() - ref).max() <= 1e-5 * np.abs(ref).max(), name


@pytest.mark.parametrize("c", META["cases"], ids=lambda c: c["key"])
def test_reference_module_replayed_through_the_plug_in(c):
    from b200gs.metrics import B200VanillaWithNormalRegMetrics
    from b200gs.scene import SyntheticGaussians
    render, gt, depth, alpha, normal, w2c, K, scene = golden_case(c)
    model = SyntheticGaussians(scene).to(DEV)
    with torch.no_grad():       # setup's draws come from the CPU generator in the recording: take its result
        model.gaussians["rotations"].copy_(torch.from_numpy(Z[f"{c['key']}_rotations"]))
        model.gaussians["scales"].copy_(torch.from_numpy(Z[f"{c['key']}_scales"]))
    metric = B200VanillaWithNormalRegMetrics(**c["config"]).instantiate()
    metric.setup("validate", None)
    r = render.to(DEV).requires_grad_(True)
    n = normal.to(DEV).requires_grad_(True)
    H, W = c["image"]
    outputs = {"render": r, "alpha": alpha.to(DEV), "exp_depth": depth.to(DEV), "normal": n,
               "preprocessed_camera": (w2c.to(DEV)[None], K.to(DEV)[None], (W, H))}
    metrics, pbar = metric.get_train_metrics(None, model, 0, (None, ("img", gt.to(DEV), None), None), outputs)
    metrics["loss"].backward()
    check_golden(c, metrics, pbar, r.grad, n.grad, model.gaussians["scales"].grad)


@pytest.mark.parametrize("c", META["cases"], ids=lambda c: c["key"])
def test_reference_call_replayed_through_the_drop_in(c):
    """the reference module's normal and flatten terms, restated line for line, on compat's gsplat.utils.depth_to_normal"""
    from b200gs import compat, ops
    compat.install()
    from gsplat.utils import depth_to_normal
    from b200gs.metrics import depth_to_normal as kernel_depth_to_normal
    assert depth_to_normal is kernel_depth_to_normal
    cfg = {**META["config"], **c["config"]}
    render, gt, depth, alpha, normal, w2c, K, scene = golden_case(c)
    scales = torch.from_numpy(Z[f"{c['key']}_scales"]).to(DEV).requires_grad_(True)
    r = render.to(DEV).requires_grad_(True)
    n = normal.to(DEV).requires_grad_(True)
    outputs = {"render": r, "alpha": alpha.to(DEV), "exp_depth": depth.to(DEV), "normal": n,
               "preprocessed_camera": (w2c.to(DEV)[None], K.to(DEV)[None], None)}
    loss, stats = ops.l1_ssim_loss(r, gt.to(DEV), cfg["lambda_dssim"])
    metrics = {"loss": loss, "rgb_diff": stats[0], "ssim": stats[1]}
    pbar = {"loss": True, "rgb_diff": True, "ssim": True}
    # normal_reg.py:27-45
    exp_depth = outputs["exp_depth"]
    w2c_, K_, _ = outputs["preprocessed_camera"]
    normals_from_depth = depth_to_normal(exp_depth.detach().permute(1, 2, 0), torch.linalg.inv(w2c_[0]), K_[0]).permute(2, 0, 1) \
        * outputs["alpha"].squeeze(0).detach()
    normal_error = (1 - (outputs["normal"] * normals_from_depth).sum(dim=0)).mean()
    normal_loss = normal_error * cfg["normal_reg_lambda"]
    flatten_loss = torch.exp(scales)[..., -1].mean() * cfg["flatten_reg"]
    metrics["loss"] = metrics["loss"] + normal_loss + flatten_loss
    metrics["normal_loss"], metrics["flatten_loss"] = normal_loss, flatten_loss
    pbar["normal_loss"] = pbar["flatten_loss"] = False
    metrics["loss"].backward()
    check_golden(c, metrics, pbar, r.grad, n.grad, scales.grad)


def test_renderer_metric_chain_matches_the_oracle_chain():
    """B200GSplatV1Renderer(rgb, alpha, exp_depth, normal) -> B200VanillaWithNormalRegMetrics (after its seeded setup("fit")) ->
    backward, against the same chain with the oracle's float64 torch loss.  The file's error model: every Gaussian-parameter
    gradient within max(8 e32, 1e-5 of its max), e32 being the distance of the reference's own fp32 chain (gsplat's formula with the
    origin, in fp32 torch) from the float64 chain.  That distance includes the blend backward's float-atomic order, which changes
    from run to run; on the H100 it was 2.0e-5 of the max on the scales gradient, so a fixed 1e-5 bar is below what fp32 can do
    here.  The chain without the normal term must lie far outside the bound, so the bound still sees the term."""
    from b200gs import ops
    from b200gs.metrics import B200VanillaWithNormalRegMetrics
    from b200gs.scene import SyntheticGaussians, make_ring_cameras, make_scene
    from b200gs.v1 import B200GSplatV1Renderer
    H, W = 96, 128
    cam = make_ring_cameras(W, H)[2].to_device(DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    target = torch.rand(3, H, W, generator=torch.Generator().manual_seed(2)).to(DEV)
    types_ = ["rgb", "alpha", "exp_depth", "normal"]
    metric = B200VanillaWithNormalRegMetrics().instantiate()

    def chain(arm):
        pc = SyntheticGaussians(make_scene(4096, 5, mean_scale=0.05)).to(DEV)
        torch.manual_seed(3)
        metric.setup("fit", types.SimpleNamespace(gaussian_model=pc))
        r = B200GSplatV1Renderer().instantiate().to(DEV)
        outputs = r(cam, pc, bg, render_types=types_)
        batch = (types.SimpleNamespace(device=torch.device(DEV)), ("img", target, None), None)
        if arm == "kernels":
            metrics, _ = metric.get_train_metrics(None, pc, 100, batch, outputs)
            loss = metrics["loss"]
        else:
            loss, _ = ops.l1_ssim_loss(outputs["render"], target, 0.2)
            w2c, K, _ = outputs["preprocessed_camera"]
            depth, alpha = outputs["exp_depth"][0].detach(), outputs["alpha"][0].detach()
            if arm == "float64":
                loss = loss + O.loss(outputs["normal"], depth, alpha, w2c[0], K[0], 0.05).float()
            elif arm == "reference_fp32":
                n_d = O.normals_from_depth(depth, w2c[0], K[0], alpha, dtype=torch.float32)
                loss = loss + (1 - (outputs["normal"] * n_d).sum(0)).mean() * 0.05
            loss = loss + pc.get_scales()[..., -1].mean() * 0.02
        loss.backward()
        assert float(outputs["alpha"].max()) > 0.1          # the scene covers the view: the normal term has pixels to act on
        return {k: v.grad.detach().clone() for k, v in pc.gaussians.items() if v.grad is not None}

    got, ref, r32, without = chain("kernels"), chain("float64"), chain("reference_fp32"), chain("no_normal_term")
    assert set(got) == set(ref) == set(r32) and {"rotations", "scales", "means"} <= set(got)
    for k in got:
        scale = float(ref[k].abs().max())
        assert scale > 0, k
        e32 = float((r32[k] - ref[k]).abs().max())
        bar = max(8 * e32, 1e-5 * scale)
        assert float((got[k] - ref[k]).abs().max()) <= bar, (k, float((got[k] - ref[k]).abs().max()) / scale, e32 / scale)
        if k in ("means", "opacities", "rotations", "scales"):
            assert float((without[k] - ref[k]).abs().max()) > 100 * bar, k
