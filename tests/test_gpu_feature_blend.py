"""The D-channel blend (b200gs_blend_feat_fwd / _bwd behind ops.rasterize_gaussians for D > 4) against the float64 oracle and
against the <= 4-channel groups of ops.rasterize_binned on the same binning.

A chunk of w channels runs the 8-channel kernels for w <= 8, the 16-channel ones for w <= 16 and the 32-channel ones above.  D
covers each: 5 and 8 (CH = 8), 12 (CH = 16), 17 and 32 (CH = 32), a full chunk plus a 1-channel tail (33, CH = 32 + 8), a full
chunk plus a 16-channel tail (48, CH = 32 + 16) and two full chunks (64).  Features and cotangents follow test_gpu_blend_channels
(channel c of scale 1, 1 or 1e3 by c % 4, cotangent divided by the channel's scale).
"""
import pytest
import torch

from oracle import gs_oracle as O
from test_gpu_blend_channels import ATOMIC_NOISE, _assert_absgrad, _assert_channels, _background, _cotangents, _features, _inside, _oracle, _ring
from test_gpu_parity import _assert_pixels, _projected_inputs, _rel

pytestmark = pytest.mark.gpu

DEV = "cuda"
MODE = O.MODE_GSPLAT
_CACHE = {}


def _scene(name):
    """-> (ref, op, sids, ranges, W, H): blend inputs as the projection hands them over and the full 3-sigma lists"""
    if name not in _CACHE:
        if name == "n256":
            ref, _, op, sids, ranges = _projected_inputs(MODE, 256, 64, 48, 3, 0, 0.05)
            _CACHE[name] = (ref, op, sids, ranges, 64, 48)
        elif name == "n4096":
            ref, _, op, sids, ranges = _projected_inputs(MODE, 4096, 256, 256, 5, 3, 0.05)
            _CACHE[name] = (ref, op, sids, ranges, 256, 256)
        elif name == "inside":
            _CACHE[name] = _inside(MODE)
        else:
            _CACHE[name] = _ring(MODE)
    return _CACHE[name]


def _leaves(ref, op, feats, geometry=True):
    xys, conics, opac = (t.detach().to(DEV).contiguous().requires_grad_(geometry) for t in (ref["xy"], ref["conic"], op[:, None]))
    return xys, conics, feats.to(DEV).requires_grad_(True), opac


def _render(ref, op, xys, conics, colors, opac, bg, W, H, v_img, v_alpha, absgrad=True):
    image, alpha = _rasterize(ref, xys, conics, colors, opac, bg, W, H, absgrad)
    ((image * v_img.permute(1, 2, 0).to(DEV)).sum() + (alpha * v_alpha.to(DEV)).sum()).backward()
    return image.detach(), alpha.detach()


def _rasterize(ref, xys, conics, colors, opac, bg, W, H, absgrad):
    from b200gs import ops
    return ops.rasterize_gaussians(xys, ref["depth"].to(DEV), ref["radii"].to(DEV), conics, ref["tiles"].to(DEV), colors, opac, H, W, 16,
                                   None if bg is None else bg.to(DEV), True, absgrad)


def _check_against_oracle(scene, D, seed, with_bg=True):
    ref, op, sids, ranges, W, H = _scene(scene)
    n = op.shape[0]
    feats = _features(n, D, seed)
    bg = _background(feats) if with_bg else None
    v_img, v_alpha = _cotangents(D, H, W, feats, True, seed + 1)
    o = _oracle(MODE, ref, op, feats, sids, ranges, bg, W, H, v_img, v_alpha)
    xys, conics, colors, opac = _leaves(ref, op, feats)
    image, alpha = _render(ref, op, xys, conics, colors, opac, bg, W, H, v_img, v_alpha)
    what = f"{scene} D={D}"
    assert image.shape == (H, W, D)
    _assert_channels(image.permute(2, 0, 1), o["img"], o["margin"], f"{what} image")
    _assert_pixels(alpha, o["alpha"], f"{what} alpha", o["margin"])
    for name, got, r in (("xys", xys.grad, o["grads"][0]), ("conics", conics.grad, o["grads"][1]), ("opacity", opac.grad[:, 0], o["grads"][2])):
        assert _rel(got, r) < 1e-3, f"{what}: {name} {_rel(got, r):.3e}"
    for c in range(D):
        assert _rel(colors.grad[:, c], o["grads"][3][:, c]) < 1e-3, f"{what}: colors[:, {c}] {_rel(colors.grad[:, c], o['grads'][3][:, c]):.3e}"
    if D <= 32:
        _assert_absgrad(xys.absgrad, o["absgrad"], what)
    return ref, op, feats, bg, v_img, v_alpha, o, colors.grad


@pytest.mark.parametrize("D", [5, 8, 12, 17, 32, 33, 48, 64])
@pytest.mark.parametrize("scene", ["n256", "n4096", "inside"])
def test_feature_blend_matches_oracle_and_channel_groups(scene, D):
    """ops.rasterize_gaussians at D channels: image, alpha, every gradient and (D <= 32) xys.absgrad against the oracle.  On one
    binning the forward is bit-identical to rasterize_binned's 4-channel groups, channel by channel and in alpha; the feature
    gradients of the GEOM and the features-only kernels agree with the groups' to atomic-order noise."""
    from b200gs import ops
    ref, op, feats, bg, v_img, v_alpha, o, _ = _check_against_oracle(scene, D, 100 + D)
    _, _, _, _, W, H = _scene(scene)
    what = f"{scene} D={D}"
    if scene == "inside":
        assert bool(o["side"]["stopped"].any()), f"{what}: no pixel stops at the transmittance cut-off"

    dxy, ddep, drad, dcon, dop = (t.detach().to(DEV).contiguous() for t in (ref["xy"], ref["depth"], ref["radii"], ref["conic"], op))
    dcol, dbg = feats.to(DEV).contiguous(), bg.to(DEV)
    binning = ops.bin_gaussians(MODE, W, H, dxy, ddep, drad, dcon, dop)
    # the composite: bit-identical channel by channel (same fmaf chain per channel, same samples, same order)
    image0, _, _, alpha0 = ops.blend_features_forward(W, H, binning, dxy, dcon, dop, dcol, None)
    image0_g, alpha0_g, _ = ops.rasterize_binned(dxy, dcon, dcol, dop, binning, H, W, None)
    for c in range(D):
        assert torch.equal(image0[..., c], image0_g[..., c]), f"{what}: channel {c} differs from the 4-channel groups"
    assert torch.equal(alpha0, alpha0_g), f"{what}: alpha differs from the 4-channel groups"
    # + T bg: K6 contracts C + T * bg into one FFMA for some channels and rounds T * bg first for others, so the two paths may
    # differ by that one rounding
    image, final_T, n_contrib, alpha = ops.blend_features_forward(W, H, binning, dxy, dcon, dop, dcol, dbg)
    means2d, conics, colors, opac = (t.clone().requires_grad_(True) for t in (dxy, dcon, dcol, dop))
    image_g, alpha_g, _ = ops.rasterize_binned(means2d, conics, colors, opac, binning, H, W, dbg)
    assert torch.equal(alpha, alpha_g.detach()) and torch.equal(alpha, alpha0)
    ulp = 2.0 ** -23 * image_g.detach().abs().amax(dim=(0, 1)).clamp_min(1.0)
    assert bool(((image - image_g.detach()).abs() <= ulp).all()), f"{what}: background term off by more than one rounding"

    dvi, dva = v_img.permute(1, 2, 0).contiguous().to(DEV), v_alpha.to(DEV).contiguous()
    ((image_g * dvi).sum() + (alpha_g * dva).sum()).backward()
    geo = ops.blend_features_backward(W, H, binning, dxy, dcon, dop, dcol, dbg, final_T, n_contrib, dvi, dva, True, False)
    fo = ops.blend_features_backward(W, H, binning, dxy, dcon, dop, dcol, dbg, final_T, n_contrib, dvi, dva, False, False)
    assert fo[0] is None and fo[1] is None and fo[2] is None and fo[4] is None
    assert _rel(geo[3], colors.grad) < ATOMIC_NOISE, f"{what}: GEOM feature gradients vs the groups {_rel(geo[3], colors.grad):.3e}"
    assert _rel(fo[3], geo[3]) < ATOMIC_NOISE, f"{what}: features-only vs GEOM feature gradients {_rel(fo[3], geo[3]):.3e}"
    for name, got, r in (("xy", geo[0], means2d.grad), ("conic", geo[1], conics.grad), ("opacity", geo[2], opac.grad)):
        assert _rel(got, r) < 1e-4, f"{what}: {name} gradient vs the groups {_rel(got, r):.3e}"


@pytest.mark.parametrize("D", [12, 17, 33])
def test_long_tile_lists(D):
    """250x130, 12000 splats: tile lists longer than 512 and pixels compositing past list entry 512, so the forward stages several
    batches and the backward walks several; some samples at the alpha clamp, pixels stopping at T <= 1e-4; no background.  (The
    scene's opaque splats were moved after its lists were built, so it is blended on those lists, not re-binned.)"""
    from b200gs import ops
    ref, op, sids, ranges, W, H = _scene("ring")
    assert int((ranges[:, 1] - ranges[:, 0]).max()) > 2 * 256
    n = op.shape[0]
    feats = _features(n, D, 200 + D)
    v_img, v_alpha = _cotangents(D, H, W, feats, True, 201 + D)
    o = _oracle(MODE, ref, op, feats, sids, ranges, None, W, H, v_img, v_alpha)
    assert int(o["n_contrib"].max()) > 2 * 256
    assert bool(o["side"]["stopped"].any()) and o["side"]["clamped"] > 0
    binning = ops.Binning(sids.to(DEV), ranges.to(torch.int32).to(DEV).contiguous(), int(sids.numel()))
    dxy, dcon, dop, dcol = (t.detach().to(DEV).contiguous() for t in (ref["xy"], ref["conic"], op, feats))
    image, final_T, n_contrib, alpha = ops.blend_features_forward(W, H, binning, dxy, dcon, dop, dcol, None)
    what = f"ring D={D}"
    _assert_channels(image.permute(2, 0, 1), o["img"], o["margin"], f"{what} image")
    _assert_pixels(alpha, o["alpha"], f"{what} alpha", o["margin"])
    image_g, alpha_g, _ = ops.rasterize_binned(dxy, dcon, dcol, dop, binning, H, W, None)
    assert torch.equal(image, image_g) and torch.equal(alpha, alpha_g), f"{what}: differs from the 4-channel groups"
    dvi, dva = v_img.permute(1, 2, 0).contiguous().to(DEV), v_alpha.to(DEV).contiguous()
    v_xy, v_conic, v_op, v_feat, v_abs = ops.blend_features_backward(W, H, binning, dxy, dcon, dop, dcol, None, final_T, n_contrib, dvi, dva,
                                                                     True, D <= 32)
    for name, got, r in (("xy", v_xy, o["grads"][0]), ("conic", v_conic, o["grads"][1]), ("opacity", v_op, o["grads"][2])):
        assert _rel(got, r) < 1e-3, f"{what}: {name} {_rel(got, r):.3e}"
    for c in range(D):
        assert _rel(v_feat[:, c], o["grads"][3][:, c]) < 1e-3, f"{what}: features[:, {c}]"
    if D <= 32:
        _assert_absgrad(v_abs, o["absgrad"], what)
    fo = ops.blend_features_backward(W, H, binning, dxy, dcon, dop, dcol, None, final_T, n_contrib, dvi, dva, False, False)
    assert _rel(fo[3], v_feat) < ATOMIC_NOISE


def test_features_only_backward():
    """Geometry not requiring grad (Feature3DGS projects under no_grad, SegAnyGS trains only the features): the features-only kernel
    runs, xys / conics / opacity get no gradient, the feature gradient equals the full backward's."""
    ref, op, sids, ranges, W, H = _scene("n4096")
    D = 32
    feats = _features(op.shape[0], D, 7)
    bg = _background(feats)
    v_img, v_alpha = _cotangents(D, H, W, feats, True, 8)
    full = _leaves(ref, op, feats)
    _render(ref, op, *full, bg, W, H, v_img, v_alpha)
    frozen = _leaves(ref, op, feats, geometry=False)
    _render(ref, op, *frozen, bg, W, H, v_img, v_alpha)
    assert frozen[0].grad is None and frozen[1].grad is None and frozen[3].grad is None
    assert not hasattr(frozen[0], "absgrad")
    assert _rel(frozen[2].grad, full[2].grad) < ATOMIC_NOISE


def test_noncontiguous_feature_slice():
    """Feature3DGS renders columns [s, s+32) of an [N, 256] parameter: the gradient lands in those columns only and equals the
    gradient of a contiguous copy."""
    ref, op, sids, ranges, W, H = _scene("n256")
    n = op.shape[0]
    param = _features(n, 256, 9).to(DEV).requires_grad_(True)
    s = 96
    v_img, v_alpha = _cotangents(32, H, W, param[:, s:s + 32].detach().cpu(), True, 10)
    xys, conics, opac = (t.detach().to(DEV).contiguous() for t in (ref["xy"], ref["conic"], op[:, None]))
    image, alpha = _render(ref, op, xys, conics, param[:, s:s + 32], opac, None, W, H, v_img, v_alpha, absgrad=False)
    copy = param[:, s:s + 32].detach().clone().requires_grad_(True)
    image_c, _ = _render(ref, op, xys, conics, copy, opac, None, W, H, v_img, v_alpha, absgrad=False)
    assert torch.equal(image, image_c)
    assert _rel(param.grad[:, s:s + 32], copy.grad) < ATOMIC_NOISE
    assert float(param.grad[:, :s].abs().max()) == 0.0 and float(param.grad[:, s + 32:].abs().max()) == 0.0


def _tiny(n, W, H, visible):
    g = torch.Generator().manual_seed(11)
    xy = torch.rand(n, 2, generator=g) * torch.tensor([W, H], dtype=torch.float32)
    conic = torch.tensor([[0.05, 0.01, 0.04]]).repeat(n, 1)
    op = torch.full((n,), 0.7)
    radii = torch.full((n,), 12 if visible else 0, dtype=torch.int32)
    depth = torch.linspace(1.0, 2.0, n)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    rect_min = torch.stack([((xy[:, 0] - radii) / 16).int().clamp(0, gx), ((xy[:, 1] - radii) / 16).int().clamp(0, gy)], dim=1)
    rect_max = torch.stack([((xy[:, 0] + radii) / 16).int().add(1).clamp(0, gx), ((xy[:, 1] + radii) / 16).int().add(1).clamp(0, gy)], dim=1)
    tiles = ((rect_max - rect_min).prod(dim=1) * (radii > 0)).int()
    ref = {"xy": xy, "conic": conic, "depth": depth, "radii": radii, "tiles": tiles}
    keys, ids = O.build_sort_keys(depth.double(), rect_min, rect_max, tiles, gx)
    _, sids, ranges = O.sort_and_ranges(keys, ids, gx * gy)
    return ref, op, sids, ranges


@pytest.mark.parametrize("case", ["one splat", "none visible"])
def test_degenerate_inputs(case):
    """N = 1, and no visible Gaussian (every radius 0: empty lists, the image is the background, every gradient 0)."""
    W, H, D = 40, 36, 33
    ref, op, sids, ranges = _tiny(1 if case == "one splat" else 5, W, H, case == "one splat")
    n = op.shape[0]
    feats = _features(n, D, 12)
    bg = _background(feats)
    v_img, v_alpha = _cotangents(D, H, W, feats, True, 13)
    xys, conics, colors, opac = _leaves(ref, op, feats)
    image, alpha = _render(ref, op, xys, conics, colors, opac, bg, W, H, v_img, v_alpha)
    if case == "none visible":
        assert int(sids.numel()) == 0
        assert torch.equal(image, bg.to(DEV).expand(H, W, D)) and float(alpha.abs().max()) == 0.0
        for t in (xys, conics, colors, opac):
            assert float(t.grad.abs().max()) == 0.0
    else:
        o = _oracle(MODE, ref, op, feats, sids, ranges, bg, W, H, v_img, v_alpha)
        _assert_channels(image.permute(2, 0, 1), o["img"], o["margin"], case)
        _assert_pixels(alpha, o["alpha"], f"{case} alpha", o["margin"])
        assert float(alpha.max()) > 0.5
        for name, got, r in (("xys", xys.grad, o["grads"][0]), ("conics", conics.grad, o["grads"][1]), ("opacity", opac.grad[:, 0], o["grads"][2]),
                             ("colors", colors.grad, o["grads"][3])):
            assert _rel(got, r) < 1e-3, f"{case}: {name} {_rel(got, r):.3e}"
