"""K6 / K7 at 1, 2, 3 and 4 channels, their side channels (has_hit_any_pixels, absgrad), the channel groups of
ops.rasterize_binned and every depth / normal output of the gsplat renderers, against the float64 oracle.

The renderers composite depths, inverse depths and normals through the same kernels as colours, at 1 to 4 channels per
launch.  Those features do not look like colours, so the features here do not either: channel 0 is depth-like (1-60),
channel 1 signed in [-1, 1] as a normal's component, channel 2 the same times 1e3 and channel 3 inverse-depth-like (1/60-1).
Every pixel bar is 1e-4 times max(1, max |channel|), and the image cotangent of channel c is divided by the channel's
scale, so every channel weighs about the same in the geometry gradients (a mistake in a unit channel must not hide
behind the 1e3 one).
"""
import math

import pytest
import torch

from oracle import gs_oracle as O
from test_gpu_parity import AMBIGUOUS, _assert_pixels, _projected_inputs, _rel
from test_inside_scene import _projected, inside_scene

pytestmark = pytest.mark.gpu

DEV = "cuda"
BG_PATTERN = (0.3, -0.5, 0.2, 0.7)      # background of channel c, in units of the channel's scale
ATOMIC_NOISE = 5e-5                     # same terms, other atomic order (test_gpu_parity.test_tile_culling_is_exact)


def _features(n, ch, seed):
    g = torch.Generator().manual_seed(seed)
    cols = []
    for c in range(ch):
        u = torch.rand(n, generator=g, dtype=torch.float64)
        cols.append((1.0 + 59.0 * u, 2.0 * u - 1.0, 1e3 * (2.0 * u - 1.0), 1.0 / (1.0 + 59.0 * u))[c % 4])
    return torch.stack(cols, dim=1).float()


def _scales(feats):
    return feats.abs().max(dim=0).values.clamp_min(1.0).double()


def _background(feats):
    s = _scales(feats)
    return torch.tensor([BG_PATTERN[c % 4] for c in range(feats.shape[1])], dtype=torch.float64).mul(s).float()


def _cotangents(ch, H, W, feats, with_alpha, seed):
    g = torch.Generator().manual_seed(seed)
    v_img = ((torch.rand(ch, H, W, generator=g, dtype=torch.float64) * 2 - 1) / _scales(feats)[:, None, None]).float()
    v_alpha = (torch.rand(H, W, generator=g, dtype=torch.float64) * 2 - 1).float() if with_alpha else None
    return v_img, v_alpha


def _assert_channels(img_chw, ref_chw, margin, what):
    """_assert_pixels per channel, on the channel's own scale."""
    for c in range(ref_chw.shape[0]):
        s = max(1.0, float(ref_chw[c].abs().max()))
        _assert_pixels(img_chw[c].detach().cpu().double() / s, ref_chw[c].detach() / s, f"{what} channel {c}", margin)


def _assert_hits(hits, side, what):
    """Equal to the oracle on every splat whose hit flag is away from every branch; the others are few."""
    got = hits.detach().cpu().bool()
    sure = side["hit_margin"] >= AMBIGUOUS
    assert int((got != side["hit"])[sure].sum()) == 0, f"{what}: {int((got != side['hit'])[sure].sum())} hit flags differ"
    assert int((~sure).sum()) <= max(8, int(side["hit"].sum()) // 20), f"{what}: {int((~sure).sum())} ambiguous hit flags"
    return int((~sure).sum())


def _assert_absgrad(got, ref, what):
    """A sum of magnitudes has no cancellation: elementwise, rtol 1e-3 where the oracle value exceeds 1e-3 of its max,
    1e-3 of the max elsewhere.  Returns the largest error relative to max(|ref|, 1e-3 max)."""
    got, ref = got.detach().cpu().double(), ref.detach().double()
    floor = 1e-3 * float(ref.max())
    assert floor > 0, f"{what}: the oracle's absgrad is zero"
    err = (got - ref).abs() / ref.clamp_min(floor)
    assert float(err.max()) < 1e-3, f"{what}: absgrad off by {float(err.max()):.3e} (relative, at splat {int(err.max(dim=1).values.argmax())})"
    return float(err.max())


REPORT = {}


def _note(key, value):
    REPORT[key] = max(value, REPORT.get(key, 0.0))


def _pixel_err(img_chw, ref_chw, margin):
    """largest error on the channel's scale over the pixels no sample makes ambiguous"""
    e = 0.0
    ok = margin >= AMBIGUOUS
    for c in range(ref_chw.shape[0]):
        s = max(1.0, float(ref_chw[c].abs().max()))
        e = max(e, float(((img_chw[c].detach().cpu().double() - ref_chw[c].detach()).abs() / s)[ok].max()))
    return e


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    print("\n[largest measured errors] " + ", ".join(f"{k}={v:.2e}" for k, v in sorted(REPORT.items())))


# ----------------------------------------------------------------------------------------------------------------------
# scenes: blend inputs as the projection hands them over (fp32), the reference lists of the full 3-sigma rects
# ----------------------------------------------------------------------------------------------------------------------
_SCENE_CACHE = {}


def _with_opaque(mode, ref, op, every=50):
    """Every `every`-th splat made opaque and centred 0.05 px off a pixel centre: that pixel's sample sits at the alpha
    clamp (0.999 / 0.99), clear of the power <= 0 branch.  The depth order and the lists stay as they are."""
    off = 0.5 if mode == O.MODE_GSPLAT else 0.0
    ref = dict(ref)
    ref["xy"] = ref["xy"].clone()
    ref["xy"][::every] = torch.floor(ref["xy"][::every] - off) + off + 0.05
    op = op.clone()
    op[::every] = 1.0
    return ref, op


def _ring(mode):
    """250x130 (partial tiles on both axes), 12000 splats: ~110 tiles list more than 512 splats and some pixels composite
    past list entry 512, so the async forward's double buffer and K7's batch loop take three or more turns."""
    key = ("ring", mode)
    if key not in _SCENE_CACHE:
        W, H = 250, 130
        ref, _, op, sids, ranges = _projected_inputs(mode, 12000, W, H, 3, 1, 0.05)
        _SCENE_CACHE[key] = (*_with_opaque(mode, ref, op), sids, ranges, W, H)
    return _SCENE_CACHE[key]


def _inside(mode):
    """the camera-inside scene of test_inside_scene.py at 128x96: near-plane giants, clamped and off-screen splats, clones;
    every pixel stops at the transmittance cut-off"""
    key = ("inside", mode)
    if key not in _SCENE_CACHE:
        raw, masks, cam = inside_scene(128, 96)
        ref, _, op, sids, ranges = _projected(mode, raw, cam)
        _SCENE_CACHE[key] = (ref, op, sids, ranges, 128, 96)
    return _SCENE_CACHE[key]


SCENES = {"ring": _ring, "inside": _inside}


def _oracle(mode, ref, op, feats, sids, ranges, bg, W, H, v_img, v_alpha):
    """One float64 blend + backward.  -> dict of outputs, margin map, side channels, gradients and absgrad."""
    leaves = [t.detach().double().requires_grad_(True) for t in (ref["xy"], ref["conic"], op, feats)]
    margins, side = [], {}
    img, alpha, nc = O.blend(mode, *leaves, sids, ranges, None if bg is None else bg.double(), W, H, margins=margins, side=side)
    loss = (img * v_img.double()).sum()
    if v_alpha is not None:
        loss = loss + (alpha * v_alpha.double()).sum()
    loss.backward()
    out = {"img": img.detach(), "alpha": alpha.detach(), "n_contrib": nc, "margin": margins[0], "side": side,
           "grads": [t.grad for t in leaves], "absgrad": O.absgrad(side.pop("abs_terms"), feats.shape[0])}
    return out


# ----------------------------------------------------------------------------------------------------------------------
# 1. K6 / K7 directly
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["ring", "inside"])
@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("mode", [O.MODE_VANILLA, O.MODE_GSPLAT])
def test_blend_channels(mode, ch, scene):
    """ops.blend_forward / blend_backward at `ch` channels: planar and interleaved images, with and without a background,
    the synchronous kernel (hit_any=None) and the asynchronous one (a hits buffer), want_abs off and on."""
    from b200gs import ops
    ref, op, sids, ranges, W, H = SCENES[scene](mode)
    n = op.shape[0]
    feats = _features(n, ch, 10 + ch)
    v_img, v_alpha = _cotangents(ch, H, W, feats, mode == O.MODE_GSPLAT, 20 + ch)
    binning = ops.Binning(sids.to(DEV), ranges.to(torch.int32).to(DEV).contiguous(), int(sids.numel()))
    dxy, dcon, dop, dcol = (t.detach().to(DEV).contiguous() for t in (ref["xy"], ref["conic"], op, feats))
    tag = f"mode={mode} ch={ch} {scene}"

    for bg in (_background(feats), None):
        o = _oracle(mode, ref, op, feats, sids, ranges, bg, W, H, v_img, v_alpha)
        side, margin = o["side"], o["margin"]
        # the branches this case exists for
        assert bool(side["stopped"].any()), f"{tag}: no pixel stops at the transmittance cut-off"
        if scene == "ring":      # (the camera-inside view is opaque after a few giants: every pixel stops, nothing clamps)
            assert side["clamped"] > 0, f"{tag}: no sample at the alpha clamp"
            assert int((ranges[:, 1] - ranges[:, 0]).max()) > 2 * 256, f"{tag}: no tile lists more than 512 splats"
            assert int(o["n_contrib"].max()) > 2 * 256, f"{tag}: no pixel composites past list entry 512"
        dbg = None if bg is None else bg.to(DEV)
        what = f"{tag} bg={'yes' if bg is not None else 'NULL'}"

        fwd = {}
        for planar in (True, False):
            for async_hits in (False, True):
                hits = torch.zeros(n, dtype=torch.uint8, device=DEV) if async_hits else None
                image, final_T, n_contrib, a_out = ops.blend_forward(mode, W, H, binning, dxy, dcon, dop, dcol, dbg, planar, True, hits)
                image_chw = image if planar else image.permute(2, 0, 1)
                fwd[(planar, async_hits)] = (image_chw, final_T, n_contrib, a_out)
                if async_hits:
                    _note("hits ambiguous (count)", _assert_hits(hits, side, what))
        image_chw, final_T, n_contrib, a_out = fwd[(True, False)]
        for key, other in fwd.items():      # the two kernels and the two layouts compute the same bits
            for x, y in zip(fwd[(True, False)], other):
                assert torch.equal(x, y), f"{what}: forward {key} differs from the planar synchronous one"
        _assert_channels(image_chw, o["img"], margin, f"{what} image")
        _assert_pixels(a_out, o["alpha"], f"{what} alpha", margin)
        _assert_pixels(final_T, 1.0 - o["alpha"], f"{what} final_T", margin)
        assert int(((n_contrib.cpu() != o["n_contrib"]) & (margin >= AMBIGUOUS)).sum()) == 0, f"{what}: n_contrib"
        _note(f"image ch{ch}", _pixel_err(image_chw, o["img"], margin))
        _note("alpha", _pixel_err(a_out[None], o["alpha"][None], margin))

        dva = v_alpha.to(DEV).contiguous() if v_alpha is not None else None
        runs = {}
        for planar in (True, False):
            v_image = v_img.to(DEV).contiguous() if planar else v_img.permute(1, 2, 0).contiguous().to(DEV)
            for want_abs in (False, True):
                runs[(planar, want_abs)] = ops.blend_backward(mode, W, H, binning, dxy, dcon, dop, dcol, dbg, final_T, n_contrib,
                                                              v_image, dva, planar, (1.0, 1.0), want_abs)
        for (planar, want_abs), (v_xy, v_conic, v_op, v_col, v_abs) in runs.items():
            w = f"{what} planar={planar} want_abs={want_abs}"
            for name, got, r in (("v_xy", v_xy, o["grads"][0]), ("v_conic", v_conic, o["grads"][1]), ("v_opacity", v_op, o["grads"][2])):
                e = _rel(got, r)
                _note(name, e)
                assert e < 1e-3, f"{w}: {name} {e:.3e}"
            for c in range(ch):
                e = _rel(v_col[:, c], o["grads"][3][:, c])
                _note("v_colors", e)
                assert e < 1e-3, f"{w}: v_colors[:, {c}] {e:.3e}"
            base = runs[(planar, False)]
            for x, y in zip(base[:4], (v_xy, v_conic, v_op, v_col)):
                assert _rel(y, x) < ATOMIC_NOISE, f"{w}: gradients move with want_abs"
            if want_abs:
                _note("absgrad", _assert_absgrad(v_abs, o["absgrad"], w))
            else:
                assert v_abs is None


# ----------------------------------------------------------------------------------------------------------------------
# 2. the gsplat v0 compat surface and the channel groups of rasterize_binned
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [1, 2, 3, 4])
def test_rasterize_gaussians_without_background(D):
    """ops.rasterize_gaussians(background=None, return_alpha=True, absgrad=True): image, alpha, gradients of every input
    and xys.absgrad."""
    from b200gs import ops
    mode = O.MODE_GSPLAT
    ref, op, sids, ranges, W, H = _inside(mode)
    n = op.shape[0]
    feats = _features(n, D, 30 + D)
    v_img, v_alpha = _cotangents(D, H, W, feats, True, 40 + D)
    o = _oracle(mode, ref, op, feats, sids, ranges, None, W, H, v_img, v_alpha)
    xys, conics, colors, opac = (t.detach().to(DEV).contiguous().requires_grad_(True) for t in (ref["xy"], ref["conic"], feats, op[:, None]))
    image, alpha = ops.rasterize_gaussians(xys, ref["depth"].to(DEV), ref["radii"].to(DEV), conics, ref["tiles"].to(DEV), colors, opac,
                                           H, W, 16, None, True, True)
    ((image * v_img.permute(1, 2, 0).to(DEV)).sum() + (alpha * v_alpha.to(DEV)).sum()).backward()
    what = f"rasterize_gaussians D={D}"
    _assert_channels(image.permute(2, 0, 1), o["img"], o["margin"], what)
    _assert_pixels(alpha, o["alpha"], f"{what} alpha", o["margin"])
    for name, got, r in (("xys", xys.grad, o["grads"][0]), ("conics", conics.grad, o["grads"][1]), ("opacity", opac.grad[:, 0], o["grads"][2])):
        assert _rel(got, r) < 1e-3, f"{what}: {name} {_rel(got, r):.3e}"
    for c in range(D):
        assert _rel(colors.grad[:, c], o["grads"][3][:, c]) < 1e-3, f"{what}: colors[:, {c}]"
    _note("absgrad", _assert_absgrad(xys.absgrad, o["absgrad"], what))


@pytest.mark.parametrize("D", [5, 7, 8, 9])
def test_rasterize_binned_channel_groups(D):
    """D > 4 channels composite in groups of <= 4 over one binning.  Image and gradients equal ONE D-channel oracle blend
    (so only group 0 may take the alpha cotangent); alpha and hits come from group 0; means2d.absgrad is the sum of every
    group's own absgrad (the documented contract of rasterize_binned, an upper bound of the all-channel value)."""
    from b200gs import ops
    mode = O.MODE_GSPLAT
    ref, op, sids, ranges, W, H = _inside(mode)
    n = op.shape[0]
    feats = _features(n, D, 50 + D)
    bg = _background(feats)
    v_img, v_alpha = _cotangents(D, H, W, feats, True, 60 + D)
    o = _oracle(mode, ref, op, feats, sids, ranges, bg, W, H, v_img, v_alpha)
    ref_abs = torch.zeros(n, 2, dtype=torch.float64)
    for c0 in range(0, D, 4):
        c1 = min(D, c0 + 4)
        og = _oracle(mode, ref, op, feats[:, c0:c1], sids, ranges, bg[c0:c1], W, H, v_img[c0:c1], v_alpha if c0 == 0 else None)
        ref_abs += og["absgrad"]

    dxy, ddep, drad, dcon, dop = (t.detach().to(DEV).contiguous() for t in (ref["xy"], ref["depth"], ref["radii"], ref["conic"], op))
    binning = ops.bin_gaussians(mode, W, H, dxy, ddep, drad, dcon, dop)
    means2d, conics, colors, opac = (t.clone().requires_grad_(True) for t in (dxy, dcon, feats.to(DEV), dop))
    image, alpha, hits = ops.rasterize_binned(means2d, conics, colors, opac, binning, H, W, bg.to(DEV), absgrad=True, want_hits=True)
    ((image * v_img.permute(1, 2, 0).to(DEV)).sum() + (alpha * v_alpha.to(DEV)).sum()).backward()
    what = f"rasterize_binned D={D}"
    _assert_channels(image.permute(2, 0, 1), o["img"], o["margin"], what)
    _assert_pixels(alpha, o["alpha"], f"{what} alpha", o["margin"])
    _assert_hits(hits, o["side"], what)
    for name, got, r in (("means2d", means2d.grad, o["grads"][0]), ("conics", conics.grad, o["grads"][1]), ("opacities", opac.grad, o["grads"][2])):
        assert _rel(got, r) < 1e-3, f"{what}: {name} {_rel(got, r):.3e}"
    for c in range(D):
        assert _rel(colors.grad[:, c], o["grads"][3][:, c]) < 1e-3, f"{what}: colors[:, {c}]"
    _note("absgrad", _assert_absgrad(means2d.absgrad, ref_abs, what))


# ----------------------------------------------------------------------------------------------------------------------
# 3. the renderers: every output, every raw-parameter gradient, the side channels
# ----------------------------------------------------------------------------------------------------------------------
W_R, H_R = 160, 120
RATIO_OUTPUTS = ("acc_depth_inverted", "exp_depth", "exp_depth_inverted")
# exp_depth = acc_depth / alpha and the inverted outputs divide by acc_depth or exp_depth.  Where alpha is small the kernel
# forms alpha = 1 - T from T ~ 1, so its absolute error of a few fp32 ulp of 1 (~1e-7) is a relative error of ~1e-7 / alpha,
# at most ~3e-5 at the smallest non-zero alpha (1/255); acc_depth is a sum of positive terms (relative error ~1e-6) and a
# reciprocal adds one rounding.  An absolute bar would be meaningless after the division, so these outputs are held to 1e-4
# RELATIVE per pixel.  Pixels the oracle marks ambiguous may differ by a whole sample (up to 1/255 of alpha, i.e. any
# relative amount once divided by a small alpha): they are excluded from the bar and their cotangents are zero, so they
# cannot dominate the gradients either.
RATIO_BAR = 1e-4


def _renderer_inputs():
    """A ring scene seen from outside plus one wide, faint backdrop splat behind it: every pixel has alpha > 0.  (Where
    alpha is 0, exp_depth's acc / alpha is 0 / 0 in the branch torch.where discards, and its gradient is NaN in the renderers
    as in the reference's expression; that is not what these tests are about.)"""
    from b200gs.scene import SyntheticGaussians, make_ring_cameras, make_scene
    raw = make_scene(3000, 5, mean_scale=0.05)
    cam = make_ring_cameras(W_R, H_R)[3]
    back = {"means": -2.0 * cam.camera_center[None], "scales": torch.full((1, 3), math.log(4.0)), "rotations": torch.tensor([[1.0, 0, 0, 0]]),
            "opacities": torch.full((1, 1), -1.0), "shs_dc": torch.full((1, 1, 3), 0.2), "shs_rest": torch.zeros(1, 15, 3)}
    raw = {k: torch.cat([v, back[k]]).contiguous() for k, v in raw.items()}
    model = SyntheticGaussians(raw).to(DEV)
    return raw, model, cam, make_ring_cameras(W_R, H_R)[3].to_device(DEV)


def _tie(v32, v64):
    """the value of the renderer's fp32 activation, the float64 gradient of the oracle's"""
    return v32.detach().cpu().double() + (v64 - v64.detach())


def _oracle_passes(raw, act32, cam, passes, hard_lists=None):
    """O.project + O.sh_colors + one O.blend per pass, on the renderer's own fp32 activations.  passes: name -> (feature
    names, background, hard opacities?).  hard_lists: (sorted ids, ranges) the hard-opacity passes composite over instead
    of the full 3-sigma lists.  -> raw leaves, {name: (image, alpha, margin, side)}."""
    rp = {k: v.double().requires_grad_(True) for k, v in raw.items()}
    means = rp["means"]
    scales = _tie(act32["scales"], torch.exp(rp["scales"]))
    rots = _tie(act32["rotations"], torch.nn.functional.normalize(rp["rotations"]))
    opac = _tie(act32["opacities"].reshape(-1), torch.sigmoid(rp["opacities"]).reshape(-1))
    shs = torch.cat((rp["shs_dc"], rp["shs_rest"]), dim=1)
    ov = O.make_view(cam.R, cam.T, float(cam.fx), float(cam.fy), float(cam.cx), float(cam.cy), W_R, H_R)
    p = O.project(O.MODE_GSPLAT, means, scales, rots, ov)
    op = opac * p["comp"]
    # the renderers' hard opacities o + (1 - o.detach()), formed in fp32: value ~1, gradient 1
    o32 = op.detach().float()
    hard = (o32 + (1 - o32)).double() + (op - op.detach())
    q = torch.nn.functional.normalize(rots)
    normals = O.build_rotation_matrix(q)[:, :, 2]
    toward = torch.einsum("ij,ij->i", normals.detach(), (means - ov.camera_center.double()).detach()) > 0
    normals = normals * torch.where(toward, -1.0, 1.0).double()[:, None]
    feats = {"rgb": O.sh_colors(3, shs, means, ov.camera_center.double(), detach_dir=True), "depth": p["depth"][:, None],
             "inv": 1.0 / (p["depth"].clamp_min(0.0) + 1e-8)[:, None], "normal": normals}
    gx, gy = (W_R + 15) // 16, (H_R + 15) // 16
    keys, ids = O.build_sort_keys(p["depth"], p["rect_min"], p["rect_max"], p["tiles"], gx)
    _, sids, ranges = O.sort_and_ranges(keys, ids, gx * gy)
    out = {}
    for name, (fnames, pbg, use_hard) in passes.items():
        f = torch.cat([feats[k] for k in fnames], dim=1)
        margins, side = [], {}
        lists = hard_lists if (use_hard and hard_lists is not None) else (sids, ranges)
        img, alpha, _ = O.blend(O.MODE_GSPLAT, p["xy"], p["conic"], hard if use_hard else op, f, *lists, pbg, W_R, H_R,
                                margins=margins, side=side)
        out[name] = (img, alpha, margins[0], side)
    return rp, out


def _derived(out):
    """the renderers' arithmetic on the blended images (gsplat_v1_renderer.py / gsplat_renderer.py)"""
    acc, alpha = out["acc_depth"], out["alpha"]
    out["acc_depth_inverted"] = torch.where(acc > 0, 1.0 / acc, acc.detach().max())
    exp = torch.where(alpha > 0, acc / alpha, acc.detach().max())
    out["exp_depth"] = exp
    out["exp_depth_inverted"] = torch.where(exp > 0, 1.0 / exp, exp.detach().max())
    return out


def _output_cotangents(names, margin, seed):
    g = torch.Generator().manual_seed(seed)
    cots = {}
    for k in names:
        c = 3 if k in ("render", "normal") else 1
        cots[k] = torch.rand(c, H_R, W_R, generator=g, dtype=torch.float64) * 2 - 1
        if k in RATIO_OUTPUTS:
            cots[k] = cots[k] * (margin >= AMBIGUOUS).double()
    return cots


def _compare_outputs(out, ref, margin_soft, margin_hard, what):
    for k, r in ref.items():
        got = out[k]
        assert got is not None and got.shape == r.shape, f"{what}: {k} shape"
        m = margin_hard if k.startswith("hard") else margin_soft
        if k in RATIO_OUTPUTS:
            ok = (m >= AMBIGUOUS)[None].expand_as(r)
            rel = (got.detach().cpu().double() - r.detach()).abs() / r.detach().abs().clamp_min(1e-30)
            e = float(rel[ok].max())
            assert e < RATIO_BAR, f"{what}: {k} relative error {e:.3e}"
            assert int((~ok).sum()) <= max(8, ok.numel() // 20)
        else:
            _assert_channels(got, r.detach(), m, f"{what} {k}")
            e = _pixel_err(got, r.detach(), m)
        _note(k, e)


def _check_grads(model, rp, what):
    for k in rp:
        e = _rel(model.gaussians[k].grad, rp[k].grad)
        _note(f"grad {k}", e)
        assert e < 1e-3, f"{what}: raw {k} gradient {e:.3e}"


V1_TYPES = ["rgb", "alpha", "acc_depth", "acc_depth_inverted", "exp_depth", "exp_depth_inverted", "inverse_depth", "hard_depth",
            "hard_inverse_depth", "normal"]
V1_KEYS = ["render", "alpha", "acc_depth", "acc_depth_inverted", "exp_depth", "exp_depth_inverted", "inverse_depth", "hard_depth",
           "hard_inverse_depth", "normal"]


@pytest.mark.parametrize("cull", [False, True])
def test_v1_renderer_every_output(cull):
    """B200GSplatV1Renderer with every render type: the 7-channel rgb | acc_depth | normal pass (two channel groups), the
    1-channel inverse, hard and hard-inverse depth passes, the derived outputs, raw-parameter gradients, acc_vis (hits of
    the first pass), has_hit_any_pixels (hits of the LAST pass, as the reference leaves it) and absgrad (rgb groups and
    inverse_depth; the hard passes do not request it).

    With tile_based_culling the lists are culled with the soft opacities, and the hard passes (opacity ~1) reuse them, as
    the reference's renderer does (it hands the same `isects` to every rasterize call): a splat whose soft alpha stays
    below 1/255 over a tile is missing from that tile's hard depth.  The oracle's hard passes then composite over the
    renderer's own lists; every other pass is bit-identical to the full lists and is checked against those."""
    from b200gs.v1 import B200GSplatV1Renderer
    raw, model, cam, cam_d = _renderer_inputs()
    bg = torch.tensor([0.3, 0.1, 0.7])
    r = B200GSplatV1Renderer(tile_based_culling=cull).instantiate().to(DEV)
    out = r(cam_d, model, bg.to(DEV), render_types=V1_TYPES)
    vp = out["viewspace_points"]
    b = out["isects"].binning
    hard_lists = (b.sorted_ids[:b.total].cpu(), b.tile_ranges.cpu().long()) if cull else None

    act32 = {"scales": model.get_scales(), "rotations": model.get_rotations(), "opacities": model.get_opacities()}
    z1, z3 = torch.zeros(1, dtype=torch.float64), torch.zeros(3, dtype=torch.float64)
    passes = {"g0": (("rgb", "depth"), torch.cat([bg.double(), z1]), False), "g1": (("normal",), z3, False),
              "inv": (("inv",), z1, False), "hard": (("depth",), z1, True), "hard_inv": (("inv",), z1, True)}
    rp, res = _oracle_passes(raw, act32, cam, passes, hard_lists)
    g0 = res["g0"][0]
    ref = _derived({"render": g0[0:3], "acc_depth": g0[3:4], "alpha": res["g0"][1][None], "normal": res["g1"][0],
                    "inverse_depth": res["inv"][0], "hard_depth": res["hard"][0], "hard_inverse_depth": res["hard_inv"][0]})
    margin, margin_hard = res["g0"][2], res["hard"][2]
    cots = _output_cotangents(V1_KEYS, margin, 7)
    sum(((ref[k] * cots[k]).sum() for k in V1_KEYS)).backward()
    ref_abs = sum(O.absgrad(res[k][3]["abs_terms"], raw["means"].shape[0]) for k in ("g0", "g1", "inv"))

    sum(((out[k] * cots[k].float().to(DEV)).sum() for k in V1_KEYS)).backward()
    what = f"v1 cull={cull}"
    _compare_outputs(out, {k: ref[k] for k in V1_KEYS}, margin, margin_hard, what)
    _check_grads(model, rp, what)
    _assert_hits(out["acc_vis"], res["g0"][3], f"{what} acc_vis")
    _assert_hits(vp.has_hit_any_pixels, res["hard_inv"][3], f"{what} has_hit_any_pixels")
    _note("absgrad", _assert_absgrad(vp.absgrad, ref_abs, what))

    # inv_depth_alt: consecutive calls alternate between the inverse and the hard inverse depth
    r2 = B200GSplatV1Renderer(tile_based_culling=cull).instantiate().to(DEV)
    with torch.no_grad():
        for k, other in (("inverse_depth", "hard_inverse_depth"), ("hard_inverse_depth", "inverse_depth"), ("inverse_depth", "hard_inverse_depth")):
            o2 = r2(cam_d, model, bg.to(DEV), render_types=["rgb", "inv_depth_alt"])
            assert o2[other] is None and o2[k] is not None, f"{what}: inv_depth_alt gave {k}?"
            assert torch.equal(o2["inv_depth_alt"], o2[k])
            assert torch.equal(o2[k], out[k].detach()), f"{what}: inv_depth_alt {k} differs from the all-outputs render"


V0_TYPES = ["rgb", "alpha", "acc_depth", "acc_depth_inverted", "exp_depth", "exp_depth_inverted", "inverse_depth", "hard_depth",
            "hard_inverse_depth"]
V0_KEYS = ["render", "alpha", "acc_depth", "acc_depth_inverted", "exp_depth", "exp_depth_inverted", "inverse_depth", "hard_depth",
           "hard_inverse_depth"]


def test_v0_renderer_every_output():
    """B200GSplatRenderer(absgrad=True) (the op-by-op path: one rasterize_gaussians per output) with every render type,
    raw-parameter gradients and viewspace_points.absgrad (the rgb pass only)."""
    from b200gs.renderers import B200GSplatRenderer
    raw, model, cam, cam_d = _renderer_inputs()
    bg = torch.tensor([0.3, 0.1, 0.7])
    q = model.get_rotation
    act32 = {"scales": model.get_scaling, "rotations": q / q.norm(dim=-1, keepdim=True), "opacities": model.get_opacity}   # as the renderer
    z1 = torch.zeros(1, dtype=torch.float64)
    passes = {"rgb": (("rgb",), bg.double(), False), "depth": (("depth",), z1, False), "inv": (("inv",), z1, False),
              "hard": (("depth",), z1, True), "hard_inv": (("inv",), z1, True)}
    rp, res = _oracle_passes(raw, act32, cam, passes)
    ref = _derived({"render": res["rgb"][0], "acc_depth": res["depth"][0], "alpha": res["depth"][1][None], "inverse_depth": res["inv"][0],
                    "hard_depth": res["hard"][0], "hard_inverse_depth": res["hard_inv"][0]})
    margin, margin_hard = res["rgb"][2], res["hard"][2]
    cots = _output_cotangents(V0_KEYS, margin, 8)
    sum(((ref[k] * cots[k]).sum() for k in V0_KEYS)).backward()
    ref_abs = O.absgrad(res["rgb"][3]["abs_terms"], raw["means"].shape[0])

    r = B200GSplatRenderer(absgrad=True).to(DEV)
    out = r(cam_d, model, bg.to(DEV), render_types=V0_TYPES)
    vp = out["viewspace_points"]
    sum(((out[k] * cots[k].float().to(DEV)).sum() for k in V0_KEYS)).backward()
    what = "v0"
    _compare_outputs(out, {k: ref[k] for k in V0_KEYS}, margin, margin_hard, what)
    _check_grads(model, rp, what)
    _note("absgrad", _assert_absgrad(vp.absgrad, ref_abs, what))
