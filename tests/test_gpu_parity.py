"""GPU parity tests: every kernel of the hot path, through the C ABI, against the CPU oracle.

Bars (BASELINE.json north_star): forward pixels within 1e-4 abs, gradients within 1e-3 relative (of the tensor's
max magnitude), integer outputs (radii, tiles, sorted ids, ranges) bit-exact — except for Gaussians whose fp32 radius
lands within rounding of an integer, which may differ by one between two fp32 evaluation orders; those are counted and
bounded.
"""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import gs_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _scene(n, seed, ms):
    from b200gs.scene import make_scene, activate
    return activate(make_scene(n, seed, mean_scale=ms))


def _cam(W, H, pose):
    from b200gs.scene import make_ring_cameras
    return make_ring_cameras(W, H)[pose]


def _oview(cam):
    return O.make_view(cam.R, cam.T, float(cam.fx), float(cam.fy), float(cam.cx), float(cam.cy), int(cam.width), int(cam.height))


def _cview(cam, mode, sh_degree=3, sh_stride=16):
    from b200gs.renderers import camera_view, _view_with
    return _view_with(camera_view(cam, mode, cache=False), sh_degree=sh_degree, sh_stride=sh_stride)


AMBIGUOUS = 5e-4   # relative distance of a sample to a branch threshold below which fp32 may legitimately take the other branch


def _assert_pixels(img, ref, what="", margin=None):
    """Forward bar: 1e-4 abs on every pixel — except those the ORACLE marks ambiguous: a sample whose alpha (or remaining T)
    sits within AMBIGUOUS (relative) of the 1/255 (or 1e-4) cut-off may take the other branch in fp32 than in float64 and
    moves that pixel by up to alpha*T*c <= 1/255.  `margin` is the oracle's per-pixel map of that distance (gs_oracle.blend);
    every pixel off by more than 1e-4 must be one of them (no unexplained flips), their error stays below one alpha step,
    and they are rare."""
    err = (img.detach().cpu().double() - ref.detach().cpu().double()).abs()
    per_pixel = err if err.dim() == 2 else err.max(dim=0).values      # [C,H,W] -> [H,W]
    bad = per_pixel > 1e-4
    if margin is not None:
        ambiguous = margin < AMBIGUOUS
        assert int((bad & ~ambiguous).sum()) == 0, f"{what}: {int((bad & ~ambiguous).sum())} pixels off by more than 1e-4 away from any threshold (max {float(per_pixel[~ambiguous].max()):.3e})"
        assert int(ambiguous.sum()) <= max(8, per_pixel.numel() // 20), f"{what}: {int(ambiguous.sum())} ambiguous pixels"
    else:
        assert int(bad.sum()) <= max(4, per_pixel.numel() // 10000), f"{what}: {int(bad.sum())} pixels off by more than 1e-4 (max {float(err.max()):.3e})"
    assert float(err.max()) < 1.0 / 255.0 + 1e-4, f"{what}: max err {float(err.max()):.3e}"
    assert float(err.median()) < 1e-6


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


CASES = [(256, 64, 48, 3, 0, 0.05), (777, 50, 37, 11, 2, 0.05), (4096, 256, 256, 5, 3, 0.05), (30000, 800, 800, 0, 0, 0.01)]


@pytest.mark.parametrize("mode", [O.MODE_VANILLA, O.MODE_GSPLAT])
@pytest.mark.parametrize("n,W,H,seed,pose,ms", CASES)
def test_project_forward(mode, n, W, H, seed, pose, ms):
    from b200gs import ops
    sc = _scene(n, seed, ms)
    cam = _cam(W, H, pose)
    d = {k: v.double() for k, v in sc.items()}
    ref = O.project(mode, d["means"], d["scales"], d["rotations"], _oview(cam))      # float64 evaluation of the formulas
    ref_rgb = O.sh_colors(3, d["shs"], d["means"], cam.camera_center.double(), detach_dir=True)
    g = {k: v.to(DEV) for k, v in sc.items()}
    xy, depth, radii, conic, comp, tiles, cov3d, rgb, clamped = ops.project_forward(
        _cview(cam, mode), g["means"], g["scales"], g["rotations"], g["shs"], want_comp=True, want_cov3d=True)
    radii, tiles = radii.cpu(), tiles.cpu()
    diff = radii != ref["radii"]
    assert int(diff.sum()) <= 1, f"{int(diff.sum())} radii differ"
    same = ~diff
    assert torch.equal(tiles[same], ref["tiles"][same])
    vis = ref["mask"] & same
    assert torch.allclose(xy.cpu().double()[vis], ref["xy"][vis], rtol=2e-7, atol=1e-4)
    assert torch.allclose(depth.cpu().double()[vis], ref["depth"][vis], rtol=2e-7, atol=1e-7)
    assert torch.allclose(conic.cpu().double()[vis], ref["conic"][vis], rtol=1e-6, atol=1e-9)
    if mode == O.MODE_GSPLAT:
        assert torch.allclose(comp.cpu().double()[vis], ref["comp"][vis], rtol=1e-6, atol=1e-7)
    assert torch.allclose(rgb.cpu().double()[vis], ref_rgb[vis], rtol=1e-4, atol=2e-5)   # SH is evaluated in fp32
    up = ref["cov3d"].reshape(-1, 9)[:, [0, 1, 2, 4, 5, 8]]
    assert torch.allclose(cov3d.cpu().double()[vis], up[vis], rtol=1e-6, atol=1e-7 * float(up.abs().max()))
    # culled entries are zero
    inv = ~ref["mask"] & same
    assert float(xy.cpu()[inv].abs().sum()) == 0 and int(radii[inv].abs().sum()) == 0


def test_project_forward_matches_reference_golden():
    """CUDA projection (gsplat mode) directly against the outputs of the reference's own project_gaussians."""
    from b200gs import ops
    for name in ("kat_projection", "scene_n4096_256x256", "scene_n30000_800x800"):
        d = np.load(os.path.join(GOLDEN, name + ".npz"))
        if name == "kat_projection":
            fx, fy, cx, cy, W, H = d["intr"]
            w2c = torch.tensor(d["w2c"])
            view = ops.make_view(1, int(W), int(H), fx=fx, fy=fy, cx=cx, cy=cy, viewmatrix=w2c)
            means, scales, quats = (torch.tensor(d[k]).to(DEV) for k in ("means", "scales", "quats"))
        else:
            n, W, H, seed, pose = [int(x) for x in d["meta"]]
            sc = _scene(n, seed, 0.05 if n <= 4096 else 0.01)
            view = _cview(_cam(W, H, pose), 1)
            means, scales, quats = sc["means"].to(DEV), sc["scales"].to(DEV), sc["rotations"].to(DEV)
        xy, depth, radii, conic, comp, tiles, _, _, _ = ops.project_forward(view, means, scales, quats, None, want_comp=True)
        rr = torch.tensor(d["radii"])
        diff = radii.cpu() != rr
        assert int(diff.sum()) <= 1
        ok = torch.tensor(d["mask"]) & ~diff
        assert torch.equal(tiles.cpu()[~diff], torch.tensor(d["tiles"])[~diff])
        assert torch.allclose(xy.cpu()[ok], torch.tensor(d["xys"])[ok], rtol=1e-5, atol=2e-3)
        assert torch.allclose(conic.cpu()[ok], torch.tensor(d["conic"])[ok], rtol=2e-3, atol=1e-7)
        assert torch.allclose(comp.cpu()[ok], torch.tensor(d["comp"])[ok], rtol=1e-3, atol=1e-5)


@pytest.mark.parametrize("mode", [O.MODE_VANILLA, O.MODE_GSPLAT])
@pytest.mark.parametrize("n,W,H,seed,pose,ms", CASES)
def test_binning_exact(mode, n, W, H, seed, pose, ms):
    """sorted ids / tile ranges bit-exact against the oracle's stable sort of the 64-bit (tile|depth) keys."""
    from b200gs import ops
    sc = _scene(n, seed, ms)
    cam = _cam(W, H, pose)
    ref = O.project(mode, sc["means"], sc["scales"], sc["rotations"], _oview(cam))
    gx, gy = (W + 15) // 16, (H + 15) // 16
    keys, ids = O.build_sort_keys(ref["depth"], ref["rect_min"], ref["rect_max"], ref["tiles"], gx)
    skeys, sids, ranges = O.sort_and_ranges(keys, ids, gx * gy)
    b = ops.bin_gaussians(mode, W, H, ref["xy"].to(DEV), ref["depth"].to(DEV), ref["radii"].to(DEV))
    assert b.total == int(ref["tiles"].sum())
    assert torch.equal(b.sorted_ids[:b.total].cpu(), sids)
    assert torch.equal(b.tile_ranges.cpu().long(), ranges)


# Shapes that drive the hierarchical binning off its common path: huge splats (rects of many coarse cells -> long (rank,row)
# item lists in the emit kernel; 256-entry chunks whose output exceeds the shared-memory staging buffer -> direct-write
# path of the scatter kernel), an image with more than 256 coarse cells (two radix passes over the cell keys), one with more
# than 1024 (the emit kernel's cell histogram and the cell table's chunk search in global memory) and one cell with more than
# 256 chunks of 256 entries (the chunk prefix kernel's loop past its register window).  Every tile after the first listed one
# must have a pair: the library writes an empty tile's range as (0, 0), the oracle as (k, k) at its place in the list.
STRESS = [(1500, 512, 384, 7, 1, 1.0), (2500, 2304, 2304, 9, 4, 0.06), (6000, 4200, 4200, 3, 5, 0.03), (200000, 128, 128, 2, 6, 0.004)]
# (more coarse cells than, more coarse entries in one cell than) each shape must reach, checked on the oracle's tile rects so
# that a change of sizes cannot quietly lose the branch
STRESS_REACH = {STRESS[2]: (1024, 0), STRESS[3]: (0, 256 * 256)}


def _coarse_cover(ref, W, H):
    """(coarse cells of the image, most coarse entries of one cell) of the oracle's tile rects; a cell is 8x8 tiles."""
    cgx, cgy = ((W + 15) // 16 + 7) // 8, ((H + 15) // 16 + 7) // 8
    vis = ref["tiles"] > 0
    c0 = ref["rect_min"][vis].long() // 8
    c1 = (ref["rect_max"][vis].long() - 1) // 8 + 1
    d = torch.zeros(cgy + 1, cgx + 1, dtype=torch.long)     # 2D difference array of the rects in cell units
    for ys, xs, sign in ((c0[:, 1], c0[:, 0], 1), (c0[:, 1], c1[:, 0], -1), (c1[:, 1], c0[:, 0], -1), (c1[:, 1], c1[:, 0], 1)):
        d.index_put_((ys, xs), torch.full_like(ys, sign), accumulate=True)
    return cgx * cgy, int(d.cumsum(0).cumsum(1).max())


@pytest.mark.parametrize("mode", [O.MODE_VANILLA, O.MODE_GSPLAT])
@pytest.mark.parametrize("n,W,H,seed,pose,ms", STRESS)
def test_binning_exact_stress(mode, n, W, H, seed, pose, ms):
    from b200gs import ops
    ref, colors, op, sids, ranges = _projected_inputs(mode, n, W, H, seed, pose, ms)
    if (n, W, H, seed, pose, ms) in STRESS_REACH:
        min_cells, min_cell_entries = STRESS_REACH[(n, W, H, seed, pose, ms)]
        cells, cell_entries = _coarse_cover(ref, W, H)
        assert cells > min_cells and cell_entries > min_cell_entries, (cells, cell_entries)
    dxy, ddep, drad, dcon, dop = (t.detach().to(DEV).contiguous() for t in (ref["xy"], ref["depth"], ref["radii"], ref["conic"], op))
    full = ops.bin_gaussians(mode, W, H, dxy, ddep, drad)
    assert full.total == int(ref["tiles"].sum()) == full.rect_pairs
    assert torch.equal(full.sorted_ids[:full.total].cpu(), sids)
    assert torch.equal(full.tile_ranges.cpu().long(), ranges)
    cul = ops.bin_gaussians(mode, W, H, dxy, ddep, drad, dcon, dop)
    assert 0 < cul.total <= full.total and cul.rect_pairs == full.rect_pairs and cul.coarse_pairs == full.coarse_pairs
    # every tile's culled list is an order-preserving subsequence of the full list
    fr, cr = full.tile_ranges.cpu().tolist(), cul.tile_ranges.cpu().tolist()
    fi, ci = full.sorted_ids.cpu().tolist(), cul.sorted_ids.cpu().tolist()
    for (fs, fe), (cs, ce) in zip(fr, cr):
        it = iter(fi[fs:fe])
        assert all(any(x == y for y in it) for x in ci[cs:ce])
    # the capacity protocol: too small a buffer must be reported, never overrun
    ops._last_total[(mode, W, H, dxy.shape[0], True)] = (max(1, cul.coarse_pairs // 2), max(1, cul.rect_pairs // 2))
    lazy = ops.bin_gaussians(mode, W, H, dxy, ddep, drad, dcon, dop, lazy=True)
    assert lazy.resolve() is False
    ops._last_total[(mode, W, H, dxy.shape[0], True)] = (cul.coarse_pairs, cul.rect_pairs)
    lazy = ops.bin_gaussians(mode, W, H, dxy, ddep, drad, dcon, dop, lazy=True)
    assert lazy.resolve() is True and lazy.total == cul.total
    assert torch.equal(lazy.sorted_ids[:lazy.total], cul.sorted_ids[:cul.total]) and torch.equal(lazy.tile_ranges, cul.tile_ranges)


@pytest.mark.parametrize("mode", [O.MODE_VANILLA, O.MODE_GSPLAT])
@pytest.mark.parametrize("n,W,H,seed,pose,ms", CASES[:3] + STRESS[:1])
def test_tile_culling_is_exact(mode, n, W, H, seed, pose, ms):
    """Exact tile culling drops only pairs no pixel of the tile would have used: per tile the culled list is an
    order-preserving subsequence of the reference list, and the blended image / saved state are BIT-identical."""
    from b200gs import ops
    ref, colors, op, sids, ranges = _projected_inputs(mode, n, W, H, seed, pose, ms)
    dxy, ddep, drad, dcon, dop, dcol = (t.detach().to(DEV).contiguous() for t in
                                        (ref["xy"], ref["depth"], ref["radii"], ref["conic"], op, colors))
    full = ops.bin_gaussians(mode, W, H, dxy, ddep, drad)
    cul = ops.bin_gaussians(mode, W, H, dxy, ddep, drad, dcon, dop)
    assert torch.equal(full.sorted_ids[:full.total].cpu(), sids)
    assert 0 < cul.total < full.total
    fr, cr = full.tile_ranges.cpu().tolist(), cul.tile_ranges.cpu().tolist()
    fi, ci = full.sorted_ids.cpu().tolist(), cul.sorted_ids.cpu().tolist()
    for (fs, fe), (cs, ce) in zip(fr, cr):
        it = iter(fi[fs:fe])
        assert all(any(x == y for y in it) for x in ci[cs:ce])
    bg = torch.tensor([0.1, 0.25, 0.6], device=DEV)
    planar = mode == O.MODE_VANILLA
    a = ops.blend_forward(mode, W, H, full, dxy, dcon, dop, dcol, bg, planar, True)
    b = ops.blend_forward(mode, W, H, cul, dxy, dcon, dop, dcol, bg, planar, True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[3], b[3])
    v_image = (torch.rand(a[0].shape, generator=torch.Generator().manual_seed(3)) * 2 - 1).to(DEV)
    ga = ops.blend_backward(mode, W, H, full, dxy, dcon, dop, dcol, bg, a[1], a[2], v_image, None, planar)
    gb = ops.blend_backward(mode, W, H, cul, dxy, dcon, dop, dcol, bg, b[1], b[2], v_image, None, planar)
    for x, y in zip(ga[:4], gb[:4]):
        assert _rel(x, y) < 5e-5      # same terms, different atomic order (measured up to 1.3e-5 on the large-splat stress case)


def _projected_inputs(mode, n, W, H, seed, pose, ms, dtype=torch.float32):
    sc = _scene(n, seed, ms)
    cam = _cam(W, H, pose)
    ov = _oview(cam)
    ref = O.project(mode, sc["means"], sc["scales"], sc["rotations"], ov)
    colors = O.sh_colors(3, sc["shs"], sc["means"], cam.camera_center, detach_dir=True)
    op = sc["opacities"].reshape(-1)
    if mode == O.MODE_GSPLAT:
        op = op * ref["comp"]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    keys, ids = O.build_sort_keys(ref["depth"], ref["rect_min"], ref["rect_max"], ref["tiles"], gx)
    _, sids, ranges = O.sort_and_ranges(keys, ids, gx * gy)
    return ref, colors, op, sids, ranges


@pytest.mark.parametrize("mode", [O.MODE_VANILLA, O.MODE_GSPLAT])
@pytest.mark.parametrize("n,W,H,seed,pose,ms", CASES[:3])
def test_blend_forward_backward(mode, n, W, H, seed, pose, ms):
    """K6/K7 on identical projected inputs: pixels 1e-4 abs, gradients 1e-3 rel vs autograd through the oracle blend."""
    from b200gs import ops
    ref, colors, op, sids, ranges = _projected_inputs(mode, n, W, H, seed, pose, ms)
    bg = torch.tensor([0.1, 0.25, 0.6])
    xy = ref["xy"].clone().requires_grad_(True)
    conic = ref["conic"].clone().requires_grad_(True)
    opr = op.clone().requires_grad_(True)
    col = colors.clone().requires_grad_(True)
    margins = []
    img, alpha, ncontrib = O.blend(mode, xy, conic, opr, col, sids, ranges, bg, W, H, margins=margins)
    gen = torch.Generator().manual_seed(1)
    cot = torch.rand(3, H, W, generator=gen) * 2 - 1
    cot_a = torch.rand(H, W, generator=gen) * 2 - 1 if mode == O.MODE_GSPLAT else None
    loss = (img * cot).sum() + ((alpha * cot_a).sum() if cot_a is not None else 0.0)
    loss.backward()

    binning = ops.Binning(sids.to(DEV), ranges.to(torch.int32).to(DEV).contiguous(), int(sids.numel()))
    planar = mode == O.MODE_VANILLA
    dxy, dcon, dop, dcol = (t.detach().to(DEV).contiguous() for t in (xy, conic, opr, col))
    image, final_T, n_contrib, a_out = ops.blend_forward(mode, W, H, binning, dxy, dcon, dop, dcol, bg.to(DEV), planar, True)
    image_chw = image if planar else image.permute(2, 0, 1)
    _assert_pixels(image_chw, img, "image", margins[0])
    _assert_pixels(a_out, alpha, "alpha", margins[0])
    assert int(((n_contrib.cpu() != ncontrib) & (margins[0] >= AMBIGUOUS)).sum()) == 0      # same last contributor wherever no sample is ambiguous

    v_image = cot.to(DEV).contiguous() if planar else cot.permute(1, 2, 0).contiguous().to(DEV)
    v_alpha = cot_a.to(DEV) if cot_a is not None else None
    v_xy, v_conic, v_op, v_col, v_abs = ops.blend_backward(mode, W, H, binning, dxy, dcon, dop, dcol, bg.to(DEV), final_T,
                                                           n_contrib, v_image, v_alpha, planar, (1.0, 1.0), True)
    assert _rel(v_xy, xy.grad) < 1e-3
    assert _rel(v_conic, conic.grad) < 1e-3
    assert _rel(v_op, opr.grad) < 1e-3
    assert _rel(v_col, col.grad) < 1e-3
    assert bool((v_abs >= v_xy.abs() - 1e-4 * v_abs.abs().max()).all())


@pytest.mark.parametrize("mode", [O.MODE_VANILLA, O.MODE_GSPLAT])
@pytest.mark.parametrize("n,W,H,seed,pose,ms", CASES[:3])
def test_project_backward(mode, n, W, H, seed, pose, ms):
    """K8 against torch autograd through the oracle projection (+SH), with random cotangents on every output."""
    from b200gs import ops
    sc = _scene(n, seed, ms)
    cam = _cam(W, H, pose)
    ov = _oview(cam)
    ins = {k: sc[k].clone().requires_grad_(True) for k in ("means", "scales", "rotations", "shs")}
    ref = O.project(mode, ins["means"], ins["scales"], ins["rotations"], ov)
    colors = O.sh_colors(3, ins["shs"], ins["means"], cam.camera_center, detach_dir=(mode == O.MODE_GSPLAT))
    gen = torch.Generator().manual_seed(2)
    vis = ref["mask"].float()
    c_xy = torch.randn(n, 2, generator=gen) * vis[:, None]
    c_con = torch.randn(n, 3, generator=gen) * vis[:, None]
    c_rgb = torch.randn(n, 3, generator=gen) * vis[:, None]
    c_dep = torch.randn(n, generator=gen) * vis if mode == O.MODE_GSPLAT else None
    c_comp = torch.randn(n, generator=gen) * vis if mode == O.MODE_GSPLAT else None
    loss = (ref["xy"] * c_xy).sum() + (ref["conic"] * c_con).sum() + (colors * c_rgb).sum()
    if c_dep is not None:
        loss = loss + (ref["depth"] * c_dep).sum() + (ref["comp"] * c_comp).sum()
    loss.backward()

    g = {k: v.detach().to(DEV) for k, v in ins.items()}
    view = _cview(cam, mode)
    xy, depth, radii, conic, comp, tiles, _, rgb, clamped = ops.project_forward(view, g["means"], g["scales"], g["rotations"], g["shs"], True)
    # the kernel consumes vanilla-mode v_xy in dgr's NDC-scaled units
    v_xy_in = c_xy * torch.tensor([1.0, 1.0]) if mode == O.MODE_GSPLAT else c_xy
    if mode == O.MODE_VANILLA:
        # oracle xy is in pixels: dL/dndc = dL/dpix * 0.5*W  ->  feed pixel cotangent scaled the way blend_bwd would
        v_xy_in = c_xy * torch.tensor([0.5 * W, 0.5 * H])
    v_means, v_scales, v_quats, v_shs = ops.project_backward(
        view, g["means"], g["scales"], g["rotations"], g["shs"], radii, clamped, v_xy_in.to(DEV).contiguous(),
        c_dep.to(DEV) if c_dep is not None else None, c_con.to(DEV).contiguous(),
        c_comp.to(DEV) if c_comp is not None else None, c_rgb.to(DEV).contiguous())
    same = (radii.cpu() > 0) == ref["mask"]
    assert int((~same).sum()) <= 1
    s = same
    assert _rel(v_means.cpu()[s], ins["means"].grad[s]) < 1e-3
    assert _rel(v_scales.cpu()[s], ins["scales"].grad[s]) < 1e-3
    assert _rel(v_quats.cpu()[s], ins["rotations"].grad[s]) < 1e-3
    assert _rel(v_shs.cpu()[s], ins["shs"].grad[s]) < 1e-3


def _model_and_cam(n, W, H, seed, pose, ms):
    from b200gs.scene import make_scene, SyntheticGaussians
    raw = make_scene(n, seed, mean_scale=ms)
    return raw, SyntheticGaussians(raw).to(DEV), _cam(W, H, pose)


@pytest.mark.parametrize("mode", [O.MODE_VANILLA, O.MODE_GSPLAT])
@pytest.mark.parametrize("n,W,H,seed,pose,ms", CASES[:3])
def test_renderer_end_to_end(mode, n, W, H, seed, pose, ms):
    """The renderers' static render() (every kernel chained: K1..K8) vs the oracle's end-to-end render + autograd.
    Both sides get bit-identical fp32 activated inputs; the oracle evaluates its formulas in float64."""
    from b200gs.renderers import B200VanillaRenderer, B200GSplatRenderer
    from b200gs.scene import activate
    raw, model, cam = _model_and_cam(n, W, H, seed, pose, ms)
    act = activate(raw)
    bg = torch.tensor([0.3, 0.1, 0.7])
    gen = torch.Generator().manual_seed(1)
    cot = torch.rand(3, H, W, generator=gen) * 2 - 1

    ap = {k: v.double().requires_grad_(True) for k, v in act.items()}
    margins = []
    out_ref = O.render(mode, ap["means"], ap["scales"], ap["rotations"], ap["opacities"], ap["shs"], _oview(cam), bg.double(), margins=margins)
    (out_ref["render"] * cot.double()).sum().backward()

    gp = {k: v.to(DEV).requires_grad_(True) for k, v in act.items()}
    R = B200VanillaRenderer if mode == O.MODE_VANILLA else B200GSplatRenderer
    cam_d = cam.to_device(DEV)
    out = R.render(gp["means"], gp["opacities"], gp["scales"], gp["rotations"], gp["shs"], 3, cam_d, bg.to(DEV))
    out["viewspace_points"].retain_grad()
    (out["render"] * cot.to(DEV)).sum().backward()

    _assert_pixels(out["render"], out_ref["render"], "render", margins[0])
    assert int((out["radii"].cpu() != out_ref["radii"]).sum()) <= 1
    assert torch.equal(out["visibility_filter"].cpu(), out["radii"].cpu() > 0)
    for k in ap:
        assert _rel(gp[k].grad, ap[k].grad) < 1e-3, k
    vs = out["viewspace_points"].grad[:, :2].cpu()
    if mode == O.MODE_GSPLAT:
        assert torch.allclose(out["viewspace_points_grad_scale"].cpu(), 0.5 * torch.tensor([[W, H]], dtype=torch.float32))
    ref_vs = O.viewspace_grad(mode, out_ref["xy"].grad, W, H)
    assert _rel(vs, ref_vs) < 1e-3

    # the plug-in forward(camera, model, bg) — the call the training loop makes — is the same computation on the
    # model's own activations, with gradients reaching the RAW parameters
    renderer = R().to(DEV)
    out2 = renderer(cam_d, model, bg.to(DEV))
    assert float((out2["render"] - out["render"]).abs().max()) < 2e-4      # torch-GPU vs torch-CPU activations differ by ulps
    (out2["render"] * cot.to(DEV)).sum().backward()
    chain = {"means": gp["means"].grad, "scales": gp["scales"].grad * act["scales"].to(DEV),
             "opacities": gp["opacities"].grad * (act["opacities"] * (1 - act["opacities"])).to(DEV)}
    for k, ref_g in chain.items():
        assert _rel(model.gaussians[k].grad, ref_g) < 2e-3, k
    assert set(out2.keys()) >= {"render", "viewspace_points", "visibility_filter", "radii"}


@pytest.mark.parametrize("n,W,H,seed,pose,ms", CASES[:3])
def test_fused_activation_path(n, W, H, seed, pose, ms):
    """B200VanillaRenderer with the activations folded into K1/K8 (raw parameters in) against the float64 oracle fed
    with torch's own activations of the same raw parameters: image 1e-4, raw-parameter gradients 1e-3."""
    from b200gs.renderers import B200VanillaRenderer
    raw, model, cam = _model_and_cam(n, W, H, seed, pose, ms)
    bg = torch.tensor([0.3, 0.1, 0.7])
    cot = torch.rand(3, H, W, generator=torch.Generator().manual_seed(1)) * 2 - 1
    rp = {k: v.double().requires_grad_(True) for k, v in raw.items()}
    out_ref = O.render(O.MODE_VANILLA, rp["means"], torch.exp(rp["scales"]), torch.nn.functional.normalize(rp["rotations"]),
                       torch.sigmoid(rp["opacities"]), torch.cat((rp["shs_dc"], rp["shs_rest"]), dim=1), _oview(cam), bg.double())
    (out_ref["render"] * cot.double()).sum().backward()
    cam_d = cam.to_device(DEV)
    fused = B200VanillaRenderer(fused_activations=True).to(DEV)
    out = fused(cam_d, model, bg.to(DEV))
    out["viewspace_points"].retain_grad()
    (out["render"] * cot.to(DEV)).sum().backward()
    _assert_pixels(out["render"], out_ref["render"], "fused render")
    for k in rp:
        assert _rel(model.gaussians[k].grad, rp[k].grad) < 1e-3, k
    assert _rel(out["viewspace_points"].grad[:, :2], O.viewspace_grad(O.MODE_VANILLA, out_ref["xy"].grad, W, H)) < 1e-3
    # and the unfused plug-in path gives the same picture
    g_fused = {k: p.grad.clone() for k, p in model.gaussians.items()}
    for p_ in model.parameters():
        p_.grad = None
    out_u = B200VanillaRenderer(fused_activations=False).to(DEV)(cam_d, model, bg.to(DEV))
    (out_u["render"] * cot.to(DEV)).sum().backward()
    assert float((out_u["render"] - out["render"]).abs().max()) < 2e-4
    for k in g_fused:
        assert _rel(model.gaussians[k].grad, g_fused[k]) < 2e-3, k


def test_lazy_binning_overflow_falls_back():
    """The sync-free forward sizes its pair buffers from the previous view; when a view needs more than that capacity
    the forward must detect it and redo the binning exactly — same image, same gradients."""
    from b200gs import ops
    from b200gs.renderers import B200VanillaRenderer
    raw, model, cam = _model_and_cam(4096, 256, 256, 5, 3, 0.05)
    cam_d = cam.to_device(DEV)
    bg = torch.tensor([0.3, 0.1, 0.7], device=DEV)
    R = B200VanillaRenderer().to(DEV)
    ops._last_total.clear()
    a = R(cam_d, model, bg)["render"].detach().clone()         # first call: exact (no history)
    b = R(cam_d, model, bg)["render"].detach().clone()         # second call: lazy, capacity from history
    assert torch.equal(a, b)
    assert len(ops._last_total) > 0
    for k in list(ops._last_total):
        ops._last_total[k] = (100, 100)                         # pretend the previous view was almost empty
    out = R(cam_d, model, bg)
    assert torch.equal(a, out["render"].detach())
    out["render"].sum().backward()
    assert bool(torch.isfinite(model.gaussians["means"].grad).all())
    assert all(min(v) > 100 for v in ops._last_total.values())  # history repaired by the fallback


def test_edge_cases():
    """empty scene, everything behind the camera, one huge splat covering all tiles, opaque stack, sh degrees 0..3."""
    from b200gs.renderers import B200VanillaRenderer, B200GSplatRenderer
    from b200gs.scene import make_scene, SyntheticGaussians
    cam = _cam(70, 40, 0).to_device(DEV)
    bg = torch.tensor([0.2, 0.4, 0.6], device=DEV)
    for R in (B200VanillaRenderer(), B200GSplatRenderer()):
        # all Gaussians behind the camera -> background image, zero grads
        raw = make_scene(64, 1, mean_scale=0.05)
        raw["means"] = raw["means"] + torch.tensor([0.0, 0.0, -10.0])
        m = SyntheticGaussians(raw).to(DEV)
        out = R(cam, m, bg)
        assert torch.allclose(out["render"], bg[:, None, None].expand(3, 40, 70))
        assert int(out["radii"].abs().sum()) == 0
        out["render"].sum().backward()
        assert float(m.gaussians["means"].grad.abs().sum()) == 0
        # one huge opaque splat + stack of opaque splats at the centre
        raw = make_scene(40, 2, mean_scale=0.05)
        raw["means"][:] = torch.tensor([0.0, 0.0, 0.0]) + 0.01 * torch.randn(40, 3, generator=torch.Generator().manual_seed(0))
        raw["scales"][0] = 2.0
        raw["opacities"][:] = 8.0
        for deg in range(4):
            m = SyntheticGaussians(raw, active_sh_degree=deg).to(DEV)
            out = R(cam, m, bg)
            assert bool(torch.isfinite(out["render"]).all())
            assert int(out["radii"][0]) > 70
            out["render"].square().sum().backward()
            for p in m.gaussians.values():
                assert bool(torch.isfinite(p.grad).all())


def test_empty_and_single():
    from b200gs import ops
    cam = _cam(64, 48, 0)
    view = _cview(cam, 0)
    for n in (0, 1):
        sc = _scene(max(n, 1), 4, 0.05)
        g = {k: v[:n].to(DEV).contiguous() for k, v in sc.items()}
        xy, depth, radii, conic, comp, tiles, _, rgb, clamped = ops.project_forward(view, g["means"], g["scales"], g["rotations"], g["shs"])
        b = ops.bin_gaussians(0, 64, 48, xy, depth, radii)
        img, fT, nc, _ = ops.blend_forward(0, 64, 48, b, xy, conic, g["opacities"].reshape(-1), rgb, torch.zeros(3, device=DEV), True, False)
        assert img.shape == (3, 48, 64) and bool(torch.isfinite(img).all())
        if n == 0:
            assert float(img.abs().sum()) == 0 and b.total == 0


@pytest.mark.parametrize("mode", [O.MODE_VANILLA, O.MODE_GSPLAT])
def test_full_size_properties(mode):
    """BASELINE config 2 size (1M Gaussians, 1920x1080): size-independent properties, no oracle."""
    from b200gs import ops
    from b200gs.renderers import B200VanillaRenderer, B200GSplatRenderer
    n, W, H = 1_000_000, 1920, 1080
    raw, model, cam = _model_and_cam(n, W, H, 0, 0, 0.01)
    cam = cam.to_device(DEV)
    sc = {k: v for k, v in (("means", model.get_xyz), ("scales", model.get_scaling), ("rot", model.get_rotation))}
    view = _cview(cam, mode)
    xy, depth, radii, conic, comp, tiles, _, _, _ = ops.project_forward(view, sc["means"].detach(), sc["scales"].detach().contiguous(),
                                                                        sc["rot"].detach().contiguous(), None, True)
    if mode == O.MODE_GSPLAT:
        # SURVEY §8d: the generator fixes V and I exactly (reference projection on CPU): V = 656 527, I = 15 119 413
        assert abs(int((radii > 0).sum()) - 656527) <= 2
        assert abs(int(tiles.sum()) - 15119413) <= 200
    b = ops.bin_gaussians(mode, W, H, xy, depth, radii)
    assert b.total == int(tiles.sum())
    r = b.tile_ranges.long()
    lens = r[:, 1] - r[:, 0]
    assert int(lens.sum()) == b.total and bool((lens >= 0).all())
    nz = lens > 0
    starts = r[nz, 0]
    assert bool((starts[1:] == r[nz, 1][:-1]).all()) and int(starts[0]) == 0   # ranges tile [0, I) in tile order
    # depth non-decreasing inside every tile: compare neighbours that are in the same tile
    d = depth[b.sorted_ids[:b.total].long()]
    tile_of = torch.repeat_interleave(torch.arange(r.shape[0], device=DEV), lens)
    same_tile = tile_of[1:] == tile_of[:-1]
    assert bool((d[1:][same_tile] >= d[:-1][same_tile]).all())
    # every pair's tile lies inside the Gaussian's rect -> multiset of ids == repeat(ids, tiles)
    counts = torch.bincount(b.sorted_ids[:b.total].long(), minlength=n)
    assert torch.equal(counts, tiles.long())

    renderer = (B200VanillaRenderer() if mode == O.MODE_VANILLA else B200GSplatRenderer()).to(DEV)
    bg = torch.tensor([0.0, 0.0, 0.0], device=DEV)
    gen = torch.Generator(device="cpu").manual_seed(1)
    cot = (torch.rand(3, H, W, generator=gen) * 2 - 1).to(DEV)

    def run(scale):
        for p in model.parameters():
            p.grad = None
        out = renderer(cam, model, bg)
        (out["render"] * (cot * scale)).sum().backward()
        return out["render"].detach(), {k: p.grad.clone() for k, p in model.gaussians.items()}

    img1, g1 = run(1.0)
    img2, g2 = run(2.0)
    assert torch.equal(img1, img2)                      # forward is deterministic
    assert float(img1.min()) >= 0 and bool(torch.isfinite(img1).all())
    for k in g1:                                        # backward is linear in the cotangent
        assert bool(torch.isfinite(g1[k]).all())
        assert _rel(g2[k], 2 * g1[k]) < 1e-3, k


@pytest.mark.parametrize("mode", [O.MODE_VANILLA, O.MODE_GSPLAT])
@pytest.mark.parametrize("deg", [0, 1, 2, 3, 4])
def test_sh_degrees_values_and_gradients(mode, deg):
    """Every SH degree the reference evaluates (sh_utils.py:57-112, 0..4): colours from K1 and the standalone SH op against the
    float64 oracle, K8 / SH-backward gradients against autograd through it (incl. the view-direction gradient of vanilla mode).
    The coefficient storage is wider than the active degree (max degree 4 model), as during the reference's SH-degree schedule."""
    from b200gs import ops
    n, W, H, K = 1500, 160, 120, 25
    g = torch.Generator().manual_seed(40 + deg)
    from b200gs.scene import make_scene, activate
    sc = activate(make_scene(n, 9, mean_scale=0.05))
    shs = torch.cat([sc["shs"][:, :1], 0.2 * torch.randn(n, K - 1, 3, generator=g)], dim=1).contiguous()
    cam = _cam(W, H, 2)
    ncoef = (deg + 1) ** 2
    ins = {"means": sc["means"].clone().double().requires_grad_(True), "shs": shs.clone().double().requires_grad_(True)}
    ref_rgb = O.sh_colors(deg, ins["shs"][:, :ncoef], ins["means"], cam.camera_center.double(), detach_dir=(mode == O.MODE_GSPLAT))
    c_rgb = torch.randn(n, 3, generator=g)
    proj = O.project(mode, sc["means"].double(), sc["scales"].double(), sc["rotations"].double(), _oview(cam))
    vis = proj["mask"]
    (ref_rgb * (c_rgb * vis[:, None]).double()).sum().backward()

    dev = {k: v.to(DEV) for k, v in sc.items()}
    dshs = shs.to(DEV)
    view = _cview(cam, mode, sh_degree=deg, sh_stride=K)
    xy, depth, radii, conic, comp, tiles, _, rgb, clamped = ops.project_forward(view, dev["means"], dev["scales"], dev["rotations"], dshs, True)
    same = (radii.cpu() > 0) == vis
    ok = vis & same
    assert int((~same).sum()) <= 1
    assert torch.allclose(rgb.cpu().double()[ok], ref_rgb.detach()[ok], rtol=1e-4, atol=3e-5)
    zeros2, zeros3 = torch.zeros(n, 2, device=DEV), torch.zeros(n, 3, device=DEV)
    v_means, v_scales, v_quats, v_shs = ops.project_backward(view, dev["means"], dev["scales"], dev["rotations"], dshs, radii, clamped, zeros2,
                                                             torch.zeros(n, device=DEV) if mode == O.MODE_GSPLAT else None, zeros3,
                                                             torch.zeros(n, device=DEV) if mode == O.MODE_GSPLAT else None, c_rgb.to(DEV).contiguous())
    assert _rel(v_shs.cpu()[same], ins["shs"].grad[same]) < 1e-3
    if ncoef < K:
        assert float(v_shs[:, ncoef:].abs().max()) == 0.0                     # coefficients above the active degree get no gradient
    if mode == O.MODE_VANILLA and deg > 0:
        assert _rel(v_means.cpu()[same], ins["means"].grad[same]) < 1e-3      # dgr back-propagates the view direction into the means
    else:
        assert float(v_means.abs().max()) == 0.0

    # the standalone op (gsplat.sh.spherical_harmonics): no +0.5 / clamp, direction gradient on request
    dirs = (sc["means"] - cam.camera_center).clone()
    d64, s64 = dirs.double().requires_grad_(True), shs.double().requires_grad_(True)
    unit = d64 / d64.norm(dim=-1, keepdim=True)
    ref = O.eval_sh(deg, s64, unit)
    dd, ds = dirs.to(DEV).requires_grad_(True), dshs.clone().requires_grad_(True)
    out = ops.spherical_harmonics(deg, dd, ds)
    (out * c_rgb.to(DEV)).sum().backward()
    (ref * c_rgb.double()).sum().backward()
    assert torch.allclose(out.detach().cpu().double(), ref.detach(), rtol=1e-4, atol=3e-5)
    assert _rel(ds.grad, s64.grad) < 1e-3 and (deg == 0 or _rel(dd.grad, d64.grad) < 1e-3)
