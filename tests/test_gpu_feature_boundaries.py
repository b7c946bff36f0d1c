"""The D-channel feature blend (b200gs_blend_feat_fwd / _bwd: blend_feat_fwd_kernel<CH>, blend_feat_bwd_kernel<CH, GEOM, ABS>) at
the chunk widths, list lengths, stops, clamp and image shapes its code branches on, against the float64 oracle.

test_gpu_feature_blend.py renders projected random scenes, so whether a case lands on a chunk width, a reduction pass, a batch
boundary or the transmittance cut-off is luck.  Here the projected splats are built directly (test_gpu_boundaries.py's
builders), every case first asserts on the CPU, with the oracle only, that it reaches the boundary it was built for
(test_cases_reach_their_boundaries, not GPU-marked: it runs without a device), and the kernels are called twice: directly on the
oracle's lists (ops.blend_features_forward / _backward, geometry on and off) and through ops.rasterize_gaussians, which bins
with culling on and must give the same image bit for bit.

Features follow test_gpu_blend_channels (channel c of scale 1 to 60, 1, 1e3 or 1/60 to 1 by c % 4, cotangents divided by the
channel's scale), so an error in a unit channel cannot hide behind the 1e3 one.  Bars are the repository's: pixels within
1e-4 of each channel's scale away from the oracle's ambiguous samples, every gradient within 1e-3 of its tensor's max, and
exact zeros, bit-identity and integer equality where stated.  The largest error of each bar is printed at the end.
"""
import math

import numpy as np
import pytest
import torch

from oracle import gs_oracle as O
from test_gpu_blend_channels import ATOMIC_NOISE, _assert_absgrad, _background, _cotangents, _features, _oracle, _pixel_err
from test_gpu_boundaries import LENGTHS, _cat, _cutoff_stack, _oracle_lists, _rects, _splats, _stack
from test_gpu_parity import AMBIGUOUS, _assert_pixels, _rel

DEV = "cuda"
GSP = O.MODE_GSPLAT
gpu = pytest.mark.gpu

# The kernels' constants the cases are built against (csrc/blend.cu).
TILE = 16
BATCH = 256                # splats per staging batch of the forward and the backward
GE = 16                    # list entries per reduction group of the backward (its `present` mask has GE bits)
EARLY_OUT = 4              # the forward's warps test for an early exit every 4 list entries
CHUNK = 32                 # channels per chunk: D is blended in chunks of 32 over one binning
WIDTHS = (8, 16, 32)       # the CH instantiations; a chunk of cw channels runs the smallest CH >= cw
EPP = {ch: 32 // ch for ch in WIDTHS}    # list entries per pass of the backward's channel reduction
ALPHA_MIN, ALPHA_MAX = 1.0 / 255.0, 0.999
LAZY_SLACK, LAZY_PAD = 1.15, 4096        # ops: a lazy binning holds LAZY_SLACK x the previous view's pairs + LAZY_PAD

SENTINEL = -777.0
GUARD = 4096               # sentinel elements before and after every guarded output


def _chunks(D):
    """(first channel, width, instantiation) of each chunk of a D-channel blend"""
    return [(c0, min(CHUNK, D - c0), next(w for w in WIDTHS if min(CHUNK, D - c0) <= w)) for c0 in range(0, D, CHUNK)]


REPORT = {}


def _note(key, value):
    REPORT[key] = max(value, REPORT.get(key, 0.0))


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    if REPORT:
        print("\n[largest measured errors] " + ", ".join(f"{k}={v:.2e}" for k, v in sorted(REPORT.items())))


# ----------------------------------------------------------------------------------------------------------------------
# scenes: projected splats built directly; the CPU reach test and the GPU tests share them
# ----------------------------------------------------------------------------------------------------------------------
def _chunk_scene():
    """40x36: 3x3 tiles, the last column and row partial; 160 splats, some centred off-screen."""
    W, H = 40, 36
    gen = torch.Generator().manual_seed(101)
    return _splats(160, W, H, gen, rmax=14.0, lo=(-4.0, -4.0), hi=(W + 4.0, H + 4.0)), W, H


HOLES_LEN = 301                   # entries of the holes tile: more than one batch
HOLES_FLIP = 128                  # a multiple of GE: the holes' phase flips this many entries before the end of the list
HOLE_AT = (8.0, 2.0)              # tile-relative: the pixel corner between warp 0's and warp 1's 8x4 blocks


def _is_hole():
    """bool [HOLES_LEN]: entry i of the holes tile is a hole.  The backward walks the list from its end in groups of GE, bit u of
    a group's `present` mask standing for the entry u before the group's first; counted from the end (k = HOLES_LEN - 1 - i),
    holes sit at odd k in the last HOLES_FLIP entries (the last entry is a contributor, as the walk's first always is) and at
    even k before them, so there every pass of EPP = 2 or 4 entries begins on a hole and holds a contributor."""
    k = HOLES_LEN - 1 - torch.arange(HOLES_LEN)
    return (k % 2 == 1) != (k >= HOLES_FLIP)


def _lengths_scene():
    """One tile per entry of LENGTHS (test_gpu_boundaries.test_blend_list_lengths: wide, faint splats under a 7-pixel radius,
    every entry contributes to every pixel), then a holes tile of HOLES_LEN entries: such wide, faint splats and, at the
    entries _is_hole() marks, holes: faint narrow splats at the corner HOLE_AT.  A hole reaches alpha 1/255 inside the 8x4
    pixel-centre hulls of warps 0 and 1 (so both warps list it) but at none of their pixel centres (so no sample is valid):
    those warps' `present` masks have every other bit set, and where the holes' phase has flipped each reduction pass of the
    8- and 16-channel kernels starts on an unset bit."""
    gen = torch.Generator().manual_seed(3)
    parts = [_stack(L, (16 * k + 8.3, 8.3), gen) for k, L in enumerate(LENGTHS) if L]
    k = len(LENGTHS)
    holes = _stack(HOLES_LEN, (16 * k + 8.3, 8.3), gen)
    h = _is_hole()
    holes["xy"][h] = torch.tensor([16.0 * k + HOLE_AT[0], HOLE_AT[1]])
    holes["conic"][h] = torch.tensor([1.0, 0.0, 1.0])         # sigma 1: alpha 0.0045 exp(-0.25) < 1/255 at the nearest centres
    holes["opacity"][h] = 0.0045
    holes["radii"][h] = 2
    return _cat(*parts, holes), 16 * (k + 1), 16


def _stop_scene():
    """The four stacks of test_gpu_boundaries.test_blend_stop_positions, gsplat rule: tile (0,0) stops on entries 3-5 around the
    every-4 early-out, tile (0,1) on ~240-270 across the batch boundary, tile (1,0) holds a pixel whose T lands exactly on the
    fp32 cut-off, tile (2,0) an opaque stack."""
    gen = torch.Generator().manual_seed(9)
    off = 0.5
    fast = _stack(12, (off - 0.3, 8.0 + off + 0.3), gen, opacity=(0.97, 0.97), radius=2, conic=(0.0012, 0.0, 0.0005))
    slow = _stack(300, (off - 0.3, 24.0 + off + 0.3), gen, opacity=(0.038, 0.038), radius=2, conic=(0.0011, 0.0, 0.0003))
    cutoff = _cutoff_stack(GSP, (24.0 + off, 8.0 + off), gen)
    opaque = _stack(40, (40.0, 8.0), gen, sigma=(10.0, 14.0), opacity=(0.93, 0.97), radius=7)
    opaque["xy"] += 0.3 * torch.randn(40, 2, generator=gen)
    return _cat(fast, slow, cutoff, opaque), 48, 32


CUTOFF_PIXEL = (24, 8)
CLAMP_OPACITIES = [1.0, 0.9915, 0.9935, 0.9955, 0.9975]


def _clamp_scene():
    """test_gpu_boundaries.test_blend_alpha_clamp's splats: opacity 1 and 0.9915-0.9975 with a pixel centre 0.03 px from the
    splat centre, over a wide backdrop.  In gsplat mode only the two opacity-1 samples exceed the 0.999 clamp."""
    gen = torch.Generator().manual_seed(13)
    off = 0.5
    parts = []
    for j in range(2):
        for i, o in enumerate(CLAMP_OPACITIES):
            parts.append(_stack(1, (8.0 + 12 * i + off + 0.03, 8.0 + 16 * j + off), gen, opacity=(o, o), radius=5, conic=(1 / 2.25, 0.0, 1 / 2.25)))
    back = _stack(1, (32.0, 16.0), gen, sigma=(40.0, 40.0), opacity=(0.5, 0.5), radius=40)
    back["depth"][:] = 100.0
    return _cat(*parts, back), 64, 32


CLAMP_IDS = [0, len(CLAMP_OPACITIES)]          # the opacity-1 splats
CLAMP_PIXELS = [(8, 8), (8, 24)]               # (x, y) of their clamped samples

SHAPES = [(1, 1), (17, 1), (1, 300), (15, 17), (4000, 16)]


def _shape_scene(W, H):
    gen = torch.Generator().manual_seed(W * 1000 + H)
    return _splats(max(6, W * H // 24), W, H, gen, rmax=12.0, lo=(-3.0, -3.0), hi=(W + 3.0, H + 3.0)), W, H


def _lazy_scene():
    W, H = 320, 240
    gen = torch.Generator().manual_seed(17)
    return _splats(3000, W, H, gen, rmax=30.0), W, H


def _oracle_fwd(sp, W, H, feats=None, bg=None):
    """float64 forward of the oracle on the oracle's lists -> (image, alpha, n_contrib, margin, side, sids, ranges)"""
    sids, ranges, _ = _oracle_lists(GSP, W, H, sp)
    feats = sp["colors"] if feats is None else feats
    margins, side = [], {}
    with torch.no_grad():
        img, alpha, nc = O.blend(GSP, sp["xy"].double(), sp["conic"].double(), sp["opacity"].double(), feats.double(), sids, ranges,
                                 bg, W, H, margins=margins, side=side)
    return img, alpha, nc, margins[0], side, sids, ranges


def _valid_samples(sp, sids, ranges, W, tile):
    """float64: valid[p, k] <=> pixel p (row-major in the 16x16 tile) has a valid sample (power <= 0, alpha >= 1/255) of entry
    k of the tile's list; -> (valid, ids of the list)"""
    gx = (W + TILE - 1) // TILE
    s, e = ranges[tile].tolist()
    gid = sids[s:e].long()
    ty, tx = divmod(tile, gx)
    yy, xx = torch.meshgrid(torch.arange(16, dtype=torch.float64), torch.arange(16, dtype=torch.float64), indexing="ij")
    px, py = (tx * 16 + xx + 0.5).reshape(-1, 1), (ty * 16 + yy + 0.5).reshape(-1, 1)
    xy, con, op = sp["xy"].double()[gid], sp["conic"].double()[gid], sp["opacity"].double()[gid]
    dx, dy = xy[None, :, 0] - px, xy[None, :, 1] - py
    power = -0.5 * (con[None, :, 0] * dx * dx + con[None, :, 2] * dy * dy) - con[None, :, 1] * dx * dy
    return (power <= 0) & (op[None, :] * power.exp() >= ALPHA_MIN), gid


def _warp_pixels(w):
    """row-major tile pixels of warp w's 8x4 block (csrc/blend.cu pixel_of_thread)"""
    x0, y0 = (w & 1) * 8, (w >> 1) * 4
    return [(y0 + j) * 16 + x0 + i for j in range(4) for i in range(8)]


def _sampled_scene(n, W, H, n_sample=48, seed=5):
    """A benchmark-size gsplat view (test_gpu_fullsize_parity's scene and camera 0): projected splats with opacity x
    compensation, the full lists, and test_gpu_fullsize_parity._oracle_sampled's tile sample (a seeded sample of the non-empty
    tiles, the longest list and the last non-empty tile, a partial one at 1080 rows)."""
    from test_gpu_parity import _cam, _oview, _scene
    sc = _scene(n, 0, 0.01)
    cam = _cam(W, H, 0)
    with torch.no_grad():
        p = O.project(GSP, sc["means"], sc["scales"], sc["rotations"], _oview(cam))
        sp = {"xy": p["xy"].float(), "depth": p["depth"].float(), "radii": p["radii"].to(torch.int32), "conic": p["conic"].float(),
              "opacity": (sc["opacities"].reshape(-1) * p["comp"]).float()}
    sids, ranges, tiles = _oracle_lists(GSP, W, H, sp)
    lens = ranges[:, 1] - ranges[:, 0]
    cand = torch.nonzero(lens > 0).reshape(-1)
    pick = cand[torch.randperm(cand.numel(), generator=torch.Generator().manual_seed(seed))[:n_sample]]
    pick = torch.unique(torch.cat([pick, lens.argmax().reshape(1), cand[-1:].reshape(1)]))
    return sp, sids, ranges, tiles, pick


# ----------------------------------------------------------------------------------------------------------------------
# the CPU reach test
# ----------------------------------------------------------------------------------------------------------------------
D_CHUNKS = [1, 4, 5, 8, 9, 16, 17, 31, 32, 33, 40, 41, 48, 49, 63, 64, 65, 96]
D_LENGTHS = [8, 16, 32, 41]
D_STOPS = [8, 32, 33]
D_CLAMP = [8, 33]
D_SHAPES = [5, 17, 33]
D_ABS = [33, 48, 65]
SAMPLED = [(30_000, 800, 800, 32), (30_000, 800, 800, 33), (1_000_000, 1920, 1080, 32)]


def test_cases_reach_their_boundaries():
    """Each case's boundary, from the constants above and the oracle alone (no device)."""
    # chunk widths: every (chunk 0 / a later chunk) x (CH 8 / 16 / 32) class, D <= 4 too, every pass width of the reduction
    classes = {(c0 > 0, ch) for D in D_CHUNKS for c0, _, ch in _chunks(D)}
    assert classes == {(t, ch) for t in (False, True) for ch in WIDTHS}
    assert min(D_CHUNKS) == 1 and any(D <= 4 for D in D_CHUNKS) and sorted(EPP.values()) == [1, 2, 4]
    tails = {cw for D in D_CHUNKS for c0, cw, _ in _chunks(D) if c0 > 0}
    assert {1, 8, 9, 16, 17, 31, 32} <= tails and any(len(_chunks(D)) == 3 for D in D_CHUNKS)
    assert {_chunks(D)[-1][2] for D in D_LENGTHS} == set(WIDTHS) and _chunks(41)[-1][1] == 9
    sp, W, H = _chunk_scene()
    assert W % TILE and H % TILE
    img, alpha, nc, margin, side, sids, ranges = _oracle_fwd(sp, W, H)
    lens = (ranges[:, 1] - ranges[:, 0])
    assert int(lens.min()) > 0 and int(lens.max()) > GE
    assert float(alpha[-1, :].max()) > 0.5 and float(alpha[:, -1].max()) > 0.5       # the partial row and column are covered

    # list lengths at the group (16), batch (256) boundaries, every entry contributing; the holes tile
    assert {GE - 1, GE, GE + 1, BATCH - 1, BATCH, BATCH + 1, 2 * BATCH - 1, 2 * BATCH, 2 * BATCH + 1} <= set(LENGTHS)
    sp, W, H = _lengths_scene()
    img, alpha, nc, margin, side, sids, ranges = _oracle_fwd(sp, W, H)
    assert (ranges[:, 1] - ranges[:, 0]).tolist() == LENGTHS + [HOLES_LEN]
    for k, L in enumerate(LENGTHS):
        assert bool((nc[:, 16 * k:16 * k + 16] == L).all()), f"tile {k}: not every entry contributes"
    k = len(LENGTHS)
    assert bool((nc[:, 16 * k:] == HOLES_LEN).all()) and float(margin.min()) >= AMBIGUOUS
    valid, gid = _valid_samples(sp, sids, ranges, W, k)
    is_hole = _is_hole()
    assert bool(valid[:, ~is_hole].all()) and not bool(valid[:, is_hole].any())
    # a hole's thresholds (o = 0.0045): alpha = o exp(-q) >= 1/255 <=> q <= ln(255 o); isotropic conic 1: q = d^2 / 2
    hole = gid[is_hole][0]
    assert torch.equal(sp["conic"][hole], torch.tensor([1.0, 0.0, 1.0]))
    q_thresh = math.log(255.0 * float(sp["opacity"][hole]))
    hx, hy = float(sp["xy"][hole, 0]) - 16 * k, float(sp["xy"][hole, 1])
    for w in range(8):                  # distance from the hole to the warp's hull of pixel centres: warps 0 and 1 list it
        x0, y0 = (w & 1) * 8 + 0.5, (w >> 1) * 4 + 0.5
        d = math.hypot(max(x0 - hx, 0.0, hx - x0 - 7.0), max(y0 - hy, 0.0, hy - y0 - 3.0))
        assert (0.5 * d * d < q_thresh - 1e-3) == (w in (0, 1)), w
    # walked from the end, with passes of EPP entries at multiples of EPP (BATCH and GE are multiples of every EPP): before the
    # last HOLES_FLIP entries each pass of EPP 2 and 4 starts on a hole and holds a contributor
    assert HOLES_LEN > BATCH and HOLES_FLIP % GE == 0 and BATCH % GE == 0 and HOLES_LEN - HOLES_FLIP > 4 * GE
    for w in (0, 1):
        present = valid[_warp_pixels(w)].any(dim=0).flip(0)       # by distance from the end of the list
        assert torch.equal(present, ~is_hole.flip(0))
        for epp in (EPP[8], EPP[16]):
            starts = range(HOLES_FLIP, HOLES_LEN - epp + 1, epp)
            assert len(starts) > 8 and all(not present[s] and bool(present[s:s + epp].any()) for s in starts)

    # stops: entries 3-5 and 240-270, the exact cut-off pixel at 13
    sp, W, H = _stop_scene()
    img, alpha, nc, margin, side, sids, ranges = _oracle_fwd(sp, W, H)
    stop_fast, stop_slow = nc[0:16, 0:16] + 1, nc[16:32, 0:16] + 1
    assert bool(side["stopped"][0:32, 0:16].all())
    assert {EARLY_OUT - 1, EARLY_OUT, EARLY_OUT + 1} <= set(stop_fast.unique().tolist())
    assert int(stop_slow.min()) <= 245 and int(stop_slow.max()) >= 265 and int(stop_slow.min()) < BATCH < int(stop_slow.max())
    assert int(nc[CUTOFF_PIXEL[1], CUTOFF_PIXEL[0]]) == 13

    # the clamp: exactly the two opacity-1 samples
    sp, W, H = _clamp_scene()
    img, alpha, nc, margin, side, sids, ranges = _oracle_fwd(sp, W, H)
    assert side["clamped"] == 2
    for i, (x, y) in zip(CLAMP_IDS, CLAMP_PIXELS):
        assert float(sp["opacity"][i]) == 1.0
        dx, dy = float(sp["xy"][i, 0]) - (x + 0.5), float(sp["xy"][i, 1]) - (y + 0.5)
        assert math.exp(-0.5 * (dx * dx + dy * dy) / 2.25) > ALPHA_MAX * (1 + AMBIGUOUS)

    # image shapes: one pixel, one row, one column, partial tiles, 250 tiles in a row
    for W, H in SHAPES:
        sp, _, _ = _shape_scene(W, H)
        _, _, tiles = _rects(GSP, sp["xy"], sp["radii"], W, H)
        assert int((tiles > 0).sum()) > 0
    assert {(1, 1), (4000, 16)} <= set(SHAPES) and any(W % TILE and H % TILE for W, H in SHAPES)

    # lazy binning: the capacity sized from a history of (100, 100) is too small for this view
    sp, W, H = _lazy_scene()
    _, _, tiles = _rects(GSP, sp["xy"], sp["radii"], W, H)
    assert int(tiles.sum()) > int(100 * LAZY_SLACK) + LAZY_PAD

    # benchmark sizes: about 48 sampled tiles, among them the longest list and a border tile
    for n, W, H, _ in SAMPLED[::2]:
        sp, sids, ranges, tiles, pick = _sampled_scene(n, W, H)
        lens = ranges[:, 1] - ranges[:, 0]
        gx = (W + TILE - 1) // TILE
        assert 45 <= pick.numel() <= 50 and int(lens.argmax()) in pick.tolist()
        assert any(t % gx == gx - 1 or t // gx == (H + TILE - 1) // TILE - 1 for t in pick.tolist())
        assert int(lens[pick].max()) > GE


# ----------------------------------------------------------------------------------------------------------------------
# the C ABI with guard bands
# ----------------------------------------------------------------------------------------------------------------------
def _guarded(numel, dtype=torch.float32, inside=None):
    """-> (buffer, its middle numel elements): SENTINEL-filled, the middle set to `inside` when given"""
    buf = torch.full((GUARD + numel + GUARD,), SENTINEL, dtype=dtype, device=DEV)
    if inside is not None:
        buf[GUARD:GUARD + numel] = inside
    return buf, buf[GUARD:GUARD + numel]


def _assert_guards(buf, numel, what):
    head, tail = buf[:GUARD], buf[GUARD + numel:]
    assert bool((head == SENTINEL).all()) and bool((tail == SENTINEL).all()), f"{what}: written outside its rows"


def _abi_blend(W, H, D, binning, dxy, dcon, dop, dfeat, dbg, dvi, dva):
    """b200gs_blend_feat_fwd, then b200gs_blend_feat_bwd with and without the geometry, every output inside a sentinel band."""
    from b200gs import ops
    from b200gs._lib import check, lib, ptr
    L = lib()
    n, P = dxy.shape[0], H * W
    st = ops._stream()
    bi, image = _guarded(P * D)
    bt, final_T = _guarded(P)
    bn, n_contrib = _guarded(P, torch.int32)
    ba, alpha = _guarded(P)
    args = (ptr(binning.tile_ranges), ptr(binning.sorted_ids), ptr(dxy), ptr(dcon), ptr(dop), ptr(dfeat), ptr(dbg))
    check(L.b200gs_blend_feat_fwd(W, H, D, *args, ptr(image), ptr(final_T), ptr(n_contrib), ptr(alpha), st), "b200gs_blend_feat_fwd")
    outs = {}
    for geometry in (True, False):
        bf, v_feat = _guarded(n * D, inside=0.0)
        bufs = [(bf, n * D, "v_features")]
        geo = [None] * 4
        if geometry:
            for k, (name, cols) in enumerate((("v_xy", 2), ("v_conic", 3), ("v_opacity", 1), ("v_abs", 2))):
                b, v = _guarded(n * cols, inside=0.0)
                bufs.append((b, n * cols, name))
                geo[k] = v
        check(L.b200gs_blend_feat_bwd(W, H, D, *args, ptr(final_T), ptr(n_contrib), ptr(dvi), ptr(dva), ptr(v_feat), *(ptr(g) for g in geo), st),
              "b200gs_blend_feat_bwd")
        outs[geometry] = (bufs, geo, v_feat)
    torch.cuda.synchronize()
    for b, numel, name in ((bi, P * D, "image"), (bt, P, "final_T"), (bn, P, "n_contrib"), (ba, P, "alpha")):
        _assert_guards(b, numel, f"D={D} {name}")
    for geometry, (bufs, _, _) in outs.items():
        for b, numel, name in bufs:
            _assert_guards(b, numel, f"D={D} geometry={geometry} {name}")
    fwd = (image.view(H, W, D), final_T.view(H, W), n_contrib.view(H, W), alpha.view(H, W))
    g = outs[True][1]
    geo = (g[0].view(n, 2), g[1].view(n, 3), g[2], outs[True][2].view(n, D), g[3].view(n, 2))
    return fwd, geo, outs[False][2].view(n, D)


# ----------------------------------------------------------------------------------------------------------------------
# one case: the oracle, the direct calls, the 4-channel groups, the C ABI and the autograd wrapper
# ----------------------------------------------------------------------------------------------------------------------
PATTERNS = ["image+alpha", "tail chunks", "alpha only"]


def _cotangent_pattern(D, H, W, feats, pattern, seed):
    """(i) image and alpha; (ii) image cotangent zero on chunk 0's channels and no alpha cotangent: only the later chunks drive
    the geometry gradient; (iii) the alpha cotangent only."""
    v_img, v_alpha = _cotangents(D, H, W, feats, True, seed)
    if pattern == "tail chunks":
        v_img[:CHUNK] = 0.0
        v_alpha = None
    elif pattern == "alpha only":
        v_img.zero_()
    return v_img, v_alpha


def _assert_feature_channels(img_chw, ref_chw, feats, margin, what):
    """_assert_pixels per channel on the channel's own scale: that of its features (test_gpu_blend_channels._scales) or of the
    blended channel, whichever is larger.  On a one-pixel image a 1e3-scale channel can blend to a value near 0, and its fp32
    roundings are those of the 1e3 terms.  -> the largest error away from the ambiguous pixels"""
    e = 0.0
    ok = margin >= AMBIGUOUS
    for c in range(ref_chw.shape[0]):
        s = max(1.0, float(feats[:, c].abs().max()), float(ref_chw[c].abs().max()))
        got, ref = img_chw[c].detach().cpu().double() / s, ref_chw[c].detach() / s
        _assert_pixels(got, ref, f"{what} channel {c}", margin)
        e = max(e, float((got - ref).abs()[ok].max()))
    return e


def _assert_grads(g, o, D, what):
    for name, got, r in (("v_xy", g[0], o["grads"][0]), ("v_conic", g[1], o["grads"][1]), ("v_opacity", g[2], o["grads"][2])):
        e = _rel(got, r)
        _note(name, e)
        assert e < 1e-3, f"{what}: {name} {e:.3e}"
    for c in range(D):
        e = _rel(g[3][:, c], o["grads"][3][:, c])
        _note("v_features", e)
        assert e < 1e-3, f"{what}: v_features[:, {c}] {e:.3e}"


def _run(sp, W, H, D, seed, bg=True, pattern="image+alpha", abi=False, autograd=True, what=""):
    """The full check of one D-channel blend of the splats `sp` on the oracle's lists.  -> dict of the oracle's and the kernels'
    outputs."""
    from b200gs import ops
    n = sp["xy"].shape[0]
    sids, ranges, tiles = _oracle_lists(GSP, W, H, sp)
    feats = _features(n, D, seed)
    bgv = _background(feats) if bg else None
    v_img, v_alpha = _cotangent_pattern(D, H, W, feats, pattern, seed + 1)
    o = _oracle(GSP, {"xy": sp["xy"], "conic": sp["conic"]}, sp["opacity"], feats, sids, ranges, bgv, W, H, v_img, v_alpha)
    margin = o["margin"]
    what = f"{what} D={D} bg={bg} {pattern}"

    total = int(sids.numel())
    binning = ops.Binning((sids if total else torch.zeros(1, dtype=torch.int32)).to(DEV), ranges.to(torch.int32).to(DEV).contiguous(), total)
    dxy, dcon, dop, dfeat = (t.detach().to(DEV).contiguous() for t in (sp["xy"], sp["conic"], sp["opacity"], feats))
    dbg = None if bgv is None else bgv.to(DEV)
    image, final_T, n_contrib, alpha = ops.blend_features_forward(W, H, binning, dxy, dcon, dop, dfeat, dbg)
    assert image.shape == (H, W, D)
    img_chw = image.permute(2, 0, 1)
    _note("pixels", _assert_feature_channels(img_chw, o["img"], feats, margin, f"{what} image"))
    _assert_pixels(alpha, o["alpha"], f"{what} alpha", margin)
    _assert_pixels(final_T, 1.0 - o["alpha"], f"{what} final_T", margin)
    assert int(((n_contrib.cpu() != o["n_contrib"]) & (margin >= AMBIGUOUS)).sum()) == 0, f"{what}: n_contrib"
    _note("alpha", _pixel_err(alpha[None], o["alpha"][None], margin))

    # K6 on the same lists, 4 channels at a time: the same final_T / n_contrib / alpha bits, the same channel bits without a
    # background; with one, K6 may round T * bg before the add where the feature kernel fuses it (one rounding)
    for c0 in range(0, D, 4):
        c1 = min(D, c0 + 4)
        g_img, g_T, g_nc, g_alpha = ops.blend_forward(GSP, W, H, binning, dxy, dcon, dop, dfeat[:, c0:c1].contiguous(),
                                                      None if dbg is None else dbg[c0:c1].contiguous(), False, True)
        assert torch.equal(g_T, final_T) and torch.equal(g_nc, n_contrib) and torch.equal(g_alpha, alpha), f"{what}: K6 group {c0}"
        if dbg is None:
            assert torch.equal(g_img, image[..., c0:c1]), f"{what}: channels {c0}..{c1 - 1} differ from K6's"
        else:
            ulp = 2.0 ** -23 * g_img.abs().amax(dim=(0, 1)).clamp_min(1.0)
            assert bool(((image[..., c0:c1] - g_img).abs() <= ulp).all()), f"{what}: channels {c0}..{c1 - 1}: more than one rounding from K6"

    dvi = v_img.permute(1, 2, 0).contiguous().to(DEV)
    dva = None if v_alpha is None else v_alpha.to(DEV).contiguous()
    geo = ops.blend_features_backward(W, H, binning, dxy, dcon, dop, dfeat, dbg, final_T, n_contrib, dvi, dva, True, True)
    _assert_grads(geo, o, D, what)
    fo = ops.blend_features_backward(W, H, binning, dxy, dcon, dop, dfeat, dbg, final_T, n_contrib, dvi, dva, False, False)
    assert fo[0] is None and fo[1] is None and fo[2] is None and fo[4] is None
    e = _rel(fo[3], geo[3])
    _note("features-only vs GEOM", e)
    assert e < ATOMIC_NOISE, f"{what}: features-only v_features vs the GEOM kernel's {e:.3e}"
    if D <= CHUNK:
        _note("absgrad", _assert_absgrad(geo[4], o["absgrad"], what))

    if abi:
        fwd, g_abi, fo_abi = _abi_blend(W, H, D, binning, dxy, dcon, dop, dfeat, dbg, dvi, dva)
        for x, y in zip(fwd, (image, final_T, n_contrib, alpha)):
            assert torch.equal(x, y), f"{what}: the guarded C ABI forward differs"
        for x, y in zip(g_abi + (fo_abi,), geo + (fo[3],)):
            assert _rel(x, y) < ATOMIC_NOISE, f"{what}: the guarded C ABI backward differs"

    out = {"o": o, "sids": sids, "ranges": ranges, "image": image, "n_contrib": n_contrib.cpu(), "geo": geo, "feats": feats, "bg": bgv,
           "v_img": v_img, "v_alpha": v_alpha}
    if autograd and D > 4:     # rasterize_gaussians: its own binning, culling on
        xys, conics, colors, opac = (t.clone().requires_grad_(True) for t in (dxy, dcon, dfeat, dop[:, None]))
        img_a, alpha_a = ops.rasterize_gaussians(xys, sp["depth"].to(DEV), sp["radii"].to(DEV), conics, tiles.to(DEV), colors, opac, H, W,
                                                 TILE, dbg, True, True)
        assert torch.equal(img_a, image) and torch.equal(alpha_a, alpha), f"{what}: rasterize_gaussians differs from the direct call"
        loss = (img_a * dvi).sum()
        if dva is not None:
            loss = loss + (alpha_a * dva).sum()
        loss.backward()
        for name, got, r in (("xys", xys.grad, geo[0]), ("conics", conics.grad, geo[1]), ("opacity", opac.grad[:, 0], geo[2]),
                             ("colors", colors.grad, geo[3]), ("absgrad", xys.absgrad, geo[4])):
            e = _rel(got, r)
            _note("rasterize_gaussians vs direct", e)
            assert e < ATOMIC_NOISE, f"{what}: rasterize_gaussians {name} vs the direct call {e:.3e}"
        out["absgrad_autograd"] = xys.absgrad
    return out


# ----------------------------------------------------------------------------------------------------------------------
# 1. chunk widths
# ----------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("D", D_CHUNKS)
def test_chunk_widths(D):
    """Every chunk width class in chunk 0 and in a tail chunk, on partial tiles in both axes, with and without a background; for
    D > 32 the three cotangent patterns (a v_alpha reaching more than one chunk, or a tail chunk's term lost, shows in (ii) and
    (iii)).  The C ABI with guard bands for every D."""
    sp, W, H = _chunk_scene()
    patterns = PATTERNS if D > CHUNK else PATTERNS[:1]
    for bg in (True, False):
        for pattern in patterns:
            _run(sp, W, H, D, 300 + D, bg=bg, pattern=pattern, abi=bg and pattern == PATTERNS[0], what="chunk scene")


# ----------------------------------------------------------------------------------------------------------------------
# 2. list lengths and the holes tile
# ----------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("D", D_LENGTHS)
def test_list_lengths(D):
    """Tile lists of LENGTHS entries (the 16-entry group and the 256-splat batch, each +-1) every entry contributing, and the holes
    tile whose warps 0 and 1 see every other entry of their list valid, so that the channel reduction skips passes by its
    `present` mask and, where the holes' phase has flipped, must not skip a pass that starts on a hole."""
    sp, W, H = _lengths_scene()
    out = _run(sp, W, H, D, 400 + D, bg=True, what="lengths")
    k = len(LENGTHS)
    lens = (out["ranges"][:, 1] - out["ranges"][:, 0]).tolist()
    assert lens == LENGTHS + [HOLES_LEN]
    for t, L in enumerate(LENGTHS + [HOLES_LEN]):
        assert bool((out["n_contrib"][:, 16 * t:16 * t + 16] == L).all()), f"tile {t}: n_contrib"
    # every contributing entry of the holes tile carries its feature gradient; the holes carry none
    s, e = out["ranges"][k].tolist()
    ids = out["sids"][s:e].long().to(DEV)
    is_hole = _is_hole().to(DEV)
    v_feat = out["geo"][3]
    assert bool((v_feat[ids[~is_hole]].abs().amax(dim=1) > 0).all())
    assert float(v_feat[ids[is_hole]].abs().max()) == 0.0


# ----------------------------------------------------------------------------------------------------------------------
# 3. stop positions
# ----------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("D", D_STOPS)
def test_stop_positions(D):
    """Stops on entries 3-5 and 240-270 and on the exact fp32 cut-off; n_contrib bit-identical to K6's; every entry behind every
    pixel's stop gets exactly zero gradient in every output, its v_features row included; the entries in front do get one."""
    from b200gs import ops
    sp, W, H = _stop_scene()
    out = _run(sp, W, H, D, 500 + D, bg=True, what="stops")
    nc = out["o"]["n_contrib"]
    assert int(out["n_contrib"][CUTOFF_PIXEL[1], CUTOFF_PIXEL[0]]) == 13
    sids, ranges = out["sids"], out["ranges"]
    binning = ops.Binning(sids.to(DEV), ranges.to(torch.int32).to(DEV).contiguous(), int(sids.numel()))
    d = {k: sp[k].to(DEV).contiguous() for k in ("xy", "conic", "opacity", "colors")}
    k6 = ops.blend_forward(GSP, W, H, binning, d["xy"], d["conic"], d["opacity"], d["colors"], None, False, True)
    assert torch.equal(k6[2].cpu(), out["n_contrib"])
    gx = W // TILE
    for (tx, ty), region in (((0, 0), nc[0:16, 0:16]), ((0, 1), nc[16:32, 0:16]), ((2, 0), nc[0:16, 32:48])):
        s, e = ranges[ty * gx + tx].tolist()
        behind = sids[s + int(region.max()):e].long().to(DEV)
        assert behind.numel() > 0
        for name, gr in zip(("v_xy", "v_conic", "v_opacity", "v_features", "absgrad"), out["geo"]):
            assert float(gr[behind].abs().max()) == 0.0, f"D={D} tile {(tx, ty)}: {name} behind the stop"
        front = sids[s:s + int(region.min())].long().to(DEV)
        assert bool((out["geo"][2][front] != 0).all())


# ----------------------------------------------------------------------------------------------------------------------
# 4. the alpha clamp
# ----------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("D", D_CLAMP)
def test_alpha_clamp(D):
    """Opacity 1 with a pixel centre 0.03 px from the splat centre: alpha clamps at 0.999.  Against the oracle with every cotangent,
    then with the cotangents on the two clamped pixels only: no gradient reaches the clamped splats' geometry or opacity (exact
    zeros), their feature gradient is fac = a T = 0.999 times the pixel's cotangent."""
    from b200gs import ops
    sp, W, H = _clamp_scene()
    out = _run(sp, W, H, D, 600 + D, bg=True, what="clamp")
    assert out["o"]["side"]["clamped"] == 2
    mask = torch.zeros(H, W)
    for x, y in CLAMP_PIXELS:
        mask[y, x] = 1.0
    sids, ranges = out["sids"], out["ranges"]
    binning = ops.Binning(sids.to(DEV), ranges.to(torch.int32).to(DEV).contiguous(), int(sids.numel()))
    dxy, dcon, dop, dfeat = (t.to(DEV).contiguous() for t in (sp["xy"], sp["conic"], sp["opacity"], out["feats"]))
    dbg = out["bg"].to(DEV)
    image, final_T, n_contrib, alpha = ops.blend_features_forward(W, H, binning, dxy, dcon, dop, dfeat, dbg)
    v_img = (out["v_img"] * mask).permute(1, 2, 0).contiguous().to(DEV)
    v_alpha = (out["v_alpha"] * mask).contiguous().to(DEV)
    v_xy, v_conic, v_op, v_feat, v_abs = ops.blend_features_backward(W, H, binning, dxy, dcon, dop, dfeat, dbg, final_T, n_contrib, v_img,
                                                                     v_alpha, True, True)
    ids = torch.tensor(CLAMP_IDS, device=DEV)
    for name, g in (("v_xy", v_xy), ("v_conic", v_conic), ("v_opacity", v_op), ("absgrad", v_abs)):
        assert float(g[ids].abs().max()) == 0.0, f"D={D}: {name} through the clamp"
    for i, (x, y) in zip(CLAMP_IDS, CLAMP_PIXELS):
        want = np.float32(ALPHA_MAX) * v_img[y, x].double()
        e = float((v_feat[i].double() - want).abs().max() / want.abs().max())
        _note("clamp fac", e)
        assert e < 1e-5, f"D={D}: the clamped sample's feature gradient is not 0.999 v ({e:.3e})"
    assert float(v_op.abs().max()) > 0        # the backdrop behind the clamped samples still gets its gradient


# ----------------------------------------------------------------------------------------------------------------------
# 5. image shapes
# ----------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("D", D_SHAPES)
@pytest.mark.parametrize("W,H", SHAPES)
def test_image_shapes(W, H, D):
    """One pixel, one row, one column, partial tiles on both axes and 250 tiles in a row, with a background; the C ABI with guard
    bands (nothing written past the image's last pixel or the last splat's row)."""
    sp, _, _ = _shape_scene(W, H)
    _run(sp, W, H, D, 700 + D, bg=True, abi=True, what=f"{W}x{H}")


# ----------------------------------------------------------------------------------------------------------------------
# 6. the absgrad contract beyond 32 channels
# ----------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("D", D_ABS)
def test_absgrad_chunk_sum(D):
    """absgrad for D > 32 is each 32-channel chunk's own absgrad, summed: the oracle per chunk (that chunk's features, cotangent
    and background, the alpha cotangent on chunk 0 only) summed is the reference, directly and through rasterize_gaussians.  It
    is at least the all-channel value (up to 1e-3 of that value's max), and above it somewhere."""
    sp, W, H = _chunk_scene()
    out = _run(sp, W, H, D, 800 + D, bg=True, what="absgrad")
    sids, ranges = out["sids"], out["ranges"]
    feats, bg, v_img, v_alpha = out["feats"], out["bg"], out["v_img"], out["v_alpha"]
    ref = {"xy": sp["xy"], "conic": sp["conic"]}
    chunked = torch.zeros(sp["xy"].shape[0], 2, dtype=torch.float64)
    for c0, cw, _ in _chunks(D):
        oc = _oracle(GSP, ref, sp["opacity"], feats[:, c0:c0 + cw], sids, ranges, bg[c0:c0 + cw], W, H, v_img[c0:c0 + cw],
                     v_alpha if c0 == 0 else None)
        chunked += oc["absgrad"]
    for name, got in (("direct", out["geo"][4]), ("rasterize_gaussians", out["absgrad_autograd"])):
        _note("absgrad", _assert_absgrad(got, chunked, f"D={D} {name}"))
    full = out["o"]["absgrad"]
    got = out["geo"][4].cpu().double()
    assert bool((got >= full - 1e-3 * float(full.max())).all()), f"D={D}: absgrad below the all-channel value"
    assert bool((chunked > full * (1 + 1e-2)).any()), f"D={D}: the chunk sum never exceeds the all-channel value"


# ----------------------------------------------------------------------------------------------------------------------
# 7. benchmark sizes, sampled
# ----------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("n,W,H,D", SAMPLED)
def test_benchmark_sizes_sampled(n, W, H, D):
    """A benchmark-size frame: the kernels blend the whole frame on the oracle's lists and through rasterize_gaussians; the
    oracle composites the sampled tiles only, the cotangents are zero outside them (and on the ambiguous pixels).  Pixels in
    the sampled tiles and every gradient of the Gaussians listed there match the oracle; every other Gaussian gets exactly zero."""
    from b200gs import ops
    from test_gpu_fullsize_parity import MAX_AMBIGUOUS_FRACTION
    sp, sids, ranges, tiles, pick = _sampled_scene(n, W, H)
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    feats = _features(n, D, 900 + D)
    bg = _background(feats)
    sel = torch.zeros_like(ranges)
    sel[pick] = ranges[pick]
    used = torch.cat([sids[int(ranges[t, 0]):int(ranges[t, 1])].long() for t in pick.tolist()])
    S = torch.unique(used)
    remap = torch.full((n,), -1, dtype=torch.int64)
    remap[S] = torch.arange(S.numel())
    sub_sids = remap[sids.long()].clamp_min(0).to(torch.int32)      # entries outside the sampled tiles are never read
    leaves = [t[S].double().requires_grad_(True) for t in (sp["xy"], sp["conic"], sp["opacity"], feats)]
    margins, side = [], {}
    img, alpha, nc = O.blend(GSP, *leaves, sub_sids, sel, bg.double(), W, H, margins=margins, side=side)
    ref_img = img.detach()
    mask = torch.zeros(gy * TILE, gx * TILE, dtype=torch.bool)
    for t in pick.tolist():
        ty, tx = divmod(t, gx)
        mask[ty * TILE:(ty + 1) * TILE, tx * TILE:(tx + 1) * TILE] = True
    mask = mask[:H, :W]
    ambiguous = (margins[0] < AMBIGUOUS) & mask
    assert int(ambiguous.sum()) <= MAX_AMBIGUOUS_FRACTION * int(mask.sum())
    clear = mask & ~ambiguous
    v_img, v_alpha = _cotangents(D, H, W, feats, True, 901 + D)
    v_img, v_alpha = v_img * clear, v_alpha * clear
    ((img * v_img.double()).sum() + (alpha * v_alpha.double()).sum()).backward()
    what = f"n={n} {W}x{H} D={D}"

    binning = ops.Binning(sids.to(DEV), ranges.to(torch.int32).to(DEV).contiguous(), int(sids.numel()))
    dxy, dcon, dop, dfeat = (t.to(DEV).contiguous() for t in (sp["xy"], sp["conic"], sp["opacity"], feats))
    dbg = bg.to(DEV)
    image, final_T, n_contrib, a_out = ops.blend_features_forward(W, H, binning, dxy, dcon, dop, dfeat, dbg)
    got = image.permute(2, 0, 1).cpu().double()
    for c in range(D):
        s = max(1.0, float(ref_img[c][mask].abs().max()))
        err = (got[c] - ref_img[c]).abs() / s
        _note("pixels (sampled)", float(err[clear].max()))
        assert float(err[clear].max()) < 1e-4, f"{what}: channel {c} off by {float(err[clear].max()):.3e} in the sampled tiles"
        assert float(err[mask].max()) < 1.0 / 255.0 + 1e-4
    assert float((a_out.cpu().double() - alpha.detach()).abs()[clear].max()) < 1e-4
    assert int(((n_contrib.cpu() != nc) & clear).sum()) == 0, f"{what}: n_contrib in the sampled tiles"
    dvi, dva = v_img.permute(1, 2, 0).contiguous().to(DEV), v_alpha.contiguous().to(DEV)
    geo = ops.blend_features_backward(W, H, binning, dxy, dcon, dop, dfeat, dbg, final_T, n_contrib, dvi, dva, True, False)

    xys, conics, colors, opac = (t.clone().requires_grad_(True) for t in (dxy, dcon, dfeat, dop[:, None]))
    img_a, alpha_a = ops.rasterize_gaussians(xys, sp["depth"].to(DEV), sp["radii"].to(DEV), conics, tiles.to(DEV), colors, opac, H, W, TILE,
                                             dbg, True, False)
    assert torch.equal(img_a, image) and torch.equal(alpha_a, a_out), f"{what}: rasterize_gaussians differs from the direct call"
    ((img_a * dvi).sum() + (alpha_a * dva).sum()).backward()

    Sd = S.to(DEV)
    for path, grads in (("direct", geo[:4]), ("rasterize_gaussians", (xys.grad, conics.grad, opac.grad[:, 0], colors.grad))):
        for name, g, r in zip(("v_xy", "v_conic", "v_opacity", "v_features"), grads, leaves):
            e = _rel(g[Sd], r.grad)
            _note(f"{name} (sampled)", e)
            assert e < 1e-3, f"{what} {path}: {name} {e:.3e}"
            outside = g.clone()
            outside[Sd] = 0
            assert float(outside.abs().max()) == 0.0, f"{what} {path}: {name} outside the Gaussians of the sampled tiles"


# ----------------------------------------------------------------------------------------------------------------------
# 8. the lazy-binning fallback of _RasterizeFeatures
# ----------------------------------------------------------------------------------------------------------------------
@gpu
def test_lazy_binning_fallback():
    """Render once (exact binning), then with this view's history set to (100, 100): the lazily sized lists overflow, the forward
    re-bins exactly.  The image is bit-identical, the gradients agree to atomic-order noise, and the history holds the view's
    real counts again."""
    from b200gs import ops
    assert (ops.LAZY_SLACK, int(100 * ops.LAZY_SLACK) + LAZY_PAD) == (LAZY_SLACK, int(100 * LAZY_SLACK) + LAZY_PAD)
    sp, W, H = _lazy_scene()
    n, D = sp["xy"].shape[0], 33
    key = (GSP, W, H, n, True)
    d = {k: v.to(DEV).contiguous() for k, v in sp.items()}
    _, _, tiles = _rects(GSP, sp["xy"], sp["radii"], W, H)
    feats = _features(n, D, 77).to(DEV)
    bg = _background(feats.cpu()).to(DEV)
    v_img, v_alpha = _cotangents(D, H, W, feats.cpu(), True, 78)
    dvi, dva = v_img.permute(1, 2, 0).contiguous().to(DEV), v_alpha.to(DEV)

    def render():
        xys, conics, colors, opac = (t.clone().requires_grad_(True) for t in (d["xy"], d["conic"], feats, d["opacity"][:, None]))
        image, alpha = ops.rasterize_gaussians(xys, d["depth"], d["radii"], conics, tiles.to(DEV), colors, opac, H, W, TILE, bg, True, True)
        ((image * dvi).sum() + (alpha * dva).sum()).backward()
        return image.detach(), alpha.detach(), (xys.grad, conics.grad, opac.grad, colors.grad, xys.absgrad)

    ops._last_total.pop(key, None)
    exact = render()
    counts = ops._last_total[key]
    ref = ops.bin_gaussians(GSP, W, H, d["xy"], d["depth"], d["radii"], d["conic"], d["opacity"])
    assert counts == (ref.coarse_pairs, ref.rect_pairs) and ref.rect_pairs > int(100 * LAZY_SLACK) + LAZY_PAD
    ops._last_total[key] = (100, 100)
    again = render()
    assert torch.equal(again[0], exact[0]) and torch.equal(again[1], exact[1]), "the fallback changed the image"
    for x, y in zip(again[2], exact[2]):
        e = _rel(x, y)
        _note("lazy fallback vs exact", e)
        assert e < ATOMIC_NOISE
    assert ops._last_total[key] == counts, "the history was not repaired"
