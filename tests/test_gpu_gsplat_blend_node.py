"""The gsplat blend node behind ops.rasterize_gaussians and ops.rasterize_binned: the library launches of every call, a warm
rasterize_binned without host synchronisation, the two absgrad policies (rasterize_gaussians replaces `xys.absgrad`,
rasterize_binned adds to it) and the lazy-binning fallback of the K6 / K7 family (the D-channel family's is
test_gpu_feature_boundaries.test_lazy_binning_fallback).  Values are checked elsewhere against the float64 oracle; here the
node is compared with itself."""
import math

import pytest
import torch

from oracle import gs_oracle as O
from test_gpu_blend_channels import ATOMIC_NOISE, _background, _features
from test_gpu_boundaries import _rects
from test_gpu_feature_boundaries import LAZY_PAD, LAZY_SLACK, _lazy_scene
from test_gpu_parity import _rel

pytestmark = pytest.mark.gpu

DEV = "cuda"
GSP = O.MODE_GSPLAT
TILE = 16


def _inputs(D, seed):
    """the 320x240 scene of 3000 splats of the lazy-binning test, D-channel features, a background and cotangents"""
    sp, W, H = _lazy_scene()
    d = {k: v.to(DEV).contiguous() for k, v in sp.items()}
    d["tiles"] = _rects(GSP, sp["xy"], sp["radii"], W, H)[2].to(DEV)
    feats = _features(d["xy"].shape[0], D, seed)
    g = torch.Generator().manual_seed(seed + 1)
    v_img = (torch.rand(H, W, D, generator=g, dtype=torch.float64) * 2 - 1).float().to(DEV)
    v_alpha = (torch.rand(H, W, generator=g, dtype=torch.float64) * 2 - 1).float().to(DEV)
    return d, feats.to(DEV), _background(feats).to(DEV), v_img, v_alpha, W, H


def _forward(entry, d, feats, bg, W, H, binning=None, prior_absgrad=None):
    """ops.rasterize_gaussians ("gaussians") or ops.rasterize_binned ("binned") on fresh leaves, absgrad requested;
    -> (image, alpha, (xys, conics, colors, opacity)).  prior_absgrad: the `absgrad` xys holds before the call."""
    from b200gs import ops
    leaves = xys, conics, colors, opac = tuple(t.clone().requires_grad_(True) for t in (d["xy"], d["conic"], feats, d["opacity"][:, None]))
    if prior_absgrad is not None:
        xys.absgrad = prior_absgrad.clone()
    if entry == "gaussians":
        image, alpha = ops.rasterize_gaussians(xys, d["depth"], d["radii"], conics, d["tiles"], colors, opac, H, W, TILE, bg, True, True)
    else:
        image, alpha, _ = ops.rasterize_binned(xys, conics, colors, opac, binning, H, W, bg, absgrad=True, want_hits=True)
    return image, alpha, leaves


def _render(entry, d, feats, bg, v_img, v_alpha, W, H, binning=None, prior_absgrad=None):
    image, alpha, leaves = _forward(entry, d, feats, bg, W, H, binning, prior_absgrad)
    ((image * v_img).sum() + (alpha * v_alpha).sum()).backward()
    return image.detach(), alpha.detach(), leaves


@pytest.mark.parametrize("D", [1, 3, 4, 5, 33])
def test_launch_counts_and_no_host_synchronisation(D):
    """rasterize_gaussians: the binning's launches plus one K6 (D <= 4) or one D-channel launch per 32 channels, and the same
    for the backward.  rasterize_binned: one K6 and one K7 per group of 4 channels, warm, under sync-debug "error"."""
    from b200gs import _lib, ops
    L = _lib.lib()
    d, feats, bg, v_img, v_alpha, W, H = _inputs(D, 90 + D)
    per_pass = 1 if D <= 4 else math.ceil(D / 32)

    def counted(entry, binning=None):
        n0 = L.b200gs_launch_count()
        image, alpha, _ = _forward(entry, d, feats, bg, W, H, binning)
        n1 = L.b200gs_launch_count()
        ((image * v_img).sum() + (alpha * v_alpha).sum()).backward()
        return n1 - n0, L.b200gs_launch_count() - n1

    counted("gaussians")        # the view's history: the next binning is the lazy one, and its lists fit
    fwd, bwd = counted("gaussians")
    n0 = L.b200gs_launch_count()
    ops.bin_gaussians(GSP, W, H, d["xy"], d["depth"], d["radii"], d["conic"], d["opacity"], lazy=True)
    n_bin = L.b200gs_launch_count() - n0
    assert n_bin > 0
    assert (fwd, bwd) == (n_bin + per_pass, per_pass), f"rasterize_gaussians D={D}"

    binning = ops.bin_gaussians(GSP, W, H, d["xy"], d["depth"], d["radii"], d["conic"], d["opacity"])
    counted("binned", binning)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        fwd, bwd = counted("binned", binning)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert (fwd, bwd) == (math.ceil(D / 4), math.ceil(D / 4)), f"rasterize_binned D={D}"


@pytest.mark.parametrize("D", [3, 5, 33])
def test_absgrad_replaces_or_adds(D):
    """An `xys.absgrad` set before the call is replaced by rasterize_gaussians' and added to by rasterize_binned's (every
    channel group adds: the v1 renderer sums the groups and passes of one render this way)."""
    from b200gs import ops
    d, feats, bg, v_img, v_alpha, W, H = _inputs(D, 70 + D)
    clean = _render("gaussians", d, feats, bg, v_img, v_alpha, W, H)[2][0].absgrad
    assert float(clean.abs().max()) > 0
    got = _render("gaussians", d, feats, bg, v_img, v_alpha, W, H, prior_absgrad=clean)[2][0].absgrad
    assert _rel(got, clean) < ATOMIC_NOISE, f"rasterize_gaussians D={D}: the absgrad held before the call was not replaced"

    binning = ops.bin_gaussians(GSP, W, H, d["xy"], d["depth"], d["radii"], d["conic"], d["opacity"])
    clean = _render("binned", d, feats, bg, v_img, v_alpha, W, H, binning)[2][0].absgrad
    assert float(clean.abs().max()) > 0
    got = _render("binned", d, feats, bg, v_img, v_alpha, W, H, binning, prior_absgrad=clean)[2][0].absgrad
    assert _rel(got, 2 * clean) < ATOMIC_NOISE, f"rasterize_binned D={D}: the absgrad held before the call was not added to"


def test_lazy_binning_fallback_k6():
    """test_gpu_feature_boundaries.test_lazy_binning_fallback at D = 4 (K6 / K7): render once (exact binning), then with the
    view's history set to (100, 100): the lazily sized lists overflow and the forward re-bins exactly.  The image is
    bit-identical, the gradients agree to atomic-order noise, and the history holds the view's real counts again."""
    from b200gs import ops
    d, feats, bg, v_img, v_alpha, W, H = _inputs(4, 77)
    key = (GSP, W, H, d["xy"].shape[0], True)

    def render():
        image, alpha, leaves = _render("gaussians", d, feats, bg, v_img, v_alpha, W, H)
        return image, alpha, [t.grad for t in leaves] + [leaves[0].absgrad]

    ops._last_total.pop(key, None)
    exact = render()
    counts = ops._last_total[key]
    ref = ops.bin_gaussians(GSP, W, H, d["xy"], d["depth"], d["radii"], d["conic"], d["opacity"])
    assert counts == (ref.coarse_pairs, ref.rect_pairs) and ref.rect_pairs > int(100 * LAZY_SLACK) + LAZY_PAD
    ops._last_total[key] = (100, 100)
    again = render()
    assert torch.equal(again[0], exact[0]) and torch.equal(again[1], exact[1]), "the fallback changed the image"
    for x, y in zip(again[2], exact[2]):
        assert _rel(x, y) < ATOMIC_NOISE
    assert ops._last_total[key] == counts, "the history was not repaired"
