"""Binning (K2-K5), blend (K6/K7) and knn_mean_dist2 at the sizes their kernels branch or block on, against the float64 oracle.

The other parity suites render random scenes, so whether a case lands on a block size, a batch boundary or a capacity limit
is luck.  Here the projected splats (xy, depth, radii, conic, opacity, colours) are built directly, so that every count is
exact, and every case first asserts on the CPU that it reaches the boundary it was built for (the STRESS_REACH pattern of
test_gpu_parity.py): a later change of constants cannot quietly turn a case into a no-op.

Bars are the repository's: binning lists bit-exact against the oracle's stable sort of the 64-bit keys with culling off, an
order-preserving subsequence with culling on (and the blended image bit-identical); blend pixels within 1e-4 away from the
oracle's ambiguous samples, n_contrib exact where no sample is ambiguous, every gradient within 1e-3 of its tensor's max.
"""
import math

import numpy as np
import pytest
import torch

from oracle import gs_oracle as O
from test_gpu_parity import AMBIGUOUS, _assert_pixels, _rel

pytestmark = pytest.mark.gpu

DEV = "cuda"
VAN, GSP = O.MODE_VANILLA, O.MODE_GSPLAT
MODES = [VAN, GSP]

# The kernels' block sizes and thresholds the cases are built against (csrc/binning.cu, onesweep.cuh, blend.cu, knn.cu).
DK_BLOCK = 2048            # Gaussians per depth_keys_kernel block (256 threads x DK_ITEMS); ranks per rank_offsets_kernel block
EMIT_BLOCK = 256           # ranks per emit_cells_kernel block
DEPTH_TILE = 4096          # records per onesweep tile of the depth sort (512 threads x DEPTH_IPT)
CELL = 8                   # a coarse cell is CELL x CELL tiles
EMIT_HIST = 1024           # cells counted in shared memory by emit_cells; cells of cell_table's shared chunk table
PACK_IDS, PACK_CELLS = 1 << 24, 255   # pack_ncells: ids below 2^24 and at most 255 cells
RADIX = 256                # cells one partition pass separates
BATCH = 256                # splats per staging batch of K6 / K7
EARLY_OUT = 4              # K6's warps test for an early exit every 4 list entries
KNN_TILE = 4096            # records per onesweep tile of knn's cell sort (512 threads x KNN_IPT)
KNN_AXIS = 1024            # knn grid cells per axis at most


def _grid(W, H):
    gx, gy = (W + 15) // 16, (H + 15) // 16
    return gx, gy, (gx + CELL - 1) // CELL, (gy + CELL - 1) // CELL


def _cell_layout(n, W, H):
    """(coarse cells, pack_ncells, partition passes) that bin_count / bin_sort pick for n Gaussians at W x H."""
    _, _, cgx, cgy = _grid(W, H)
    cells = cgx * cgy
    return cells, n < PACK_IDS and cells <= PACK_CELLS, 2 if cells > RADIX else 1


def _rects(mode, xy, radii, W, H):
    """The tile rects of gs_oracle.project (lines 251-287, both modes) for given xy and radii, in float32 as the kernels
    evaluate them: -> rect_min, rect_max int32 [n,2] and tiles int32 [n] (0 where the radius is not positive)."""
    gx, gy, _, _ = _grid(W, H)
    xy = xy.float()
    r = radii.float()[:, None]
    rmin = ((xy - r) / 16).to(torch.int32)
    rmax = ((xy + r) / 16).to(torch.int32) + 1 if mode == GSP else ((xy + r + 15) / 16).to(torch.int32)
    g = torch.tensor([gx, gy], dtype=torch.int32)
    rmin = torch.minimum(rmin.clamp_min(0), g)
    rmax = torch.minimum(rmax.clamp_min(0), g)
    d = rmax - rmin
    tiles = torch.where(radii > 0, d[:, 0] * d[:, 1], torch.zeros((), dtype=torch.int32)).to(torch.int32)
    return rmin, rmax, tiles


def _oracle_lists(mode, W, H, sp):
    """Reference lists: the oracle's stable sort of the (tile | depth) keys of the rects above."""
    gx, gy, _, _ = _grid(W, H)
    rmin, rmax, tiles = _rects(mode, sp["xy"], sp["radii"], W, H)
    keys, ids = O.build_sort_keys(sp["depth"], rmin, rmax, tiles, gx)
    _, sids, ranges = O.sort_and_ranges(keys, ids, gx * gy)
    return sids, ranges, tiles


def _library_ranges(ranges):
    """The library writes an empty tile's range as (0, 0), the oracle as (k, k) at its place in the list."""
    r = ranges.clone().long()
    r[r[:, 0] == r[:, 1]] = 0
    return r


# ----------------------------------------------------------------------------------------------------------------------
# projected splats, built directly
# ----------------------------------------------------------------------------------------------------------------------
def _conics(sig, theta):
    """conic (inverse covariance, upper triangle) of a 2D Gaussian with std devs sig [n,2] rotated by theta [n]."""
    c, s = theta.cos(), theta.sin()
    s0, s1 = sig[:, 0] ** 2, sig[:, 1] ** 2
    a, b, cc = c * c * s0 + s * s * s1, c * s * (s0 - s1), s * s * s0 + c * c * s1
    det = a * cc - b * b
    return torch.stack([cc / det, -b / det, a / det], dim=-1)


def _splats(count, W, H, gen, rmax=20.0, lo=(0.0, 0.0), hi=None):
    """count splats with centres uniform in [lo, hi) (default: the image), 3-sigma radii up to rmax, random depths."""
    hi = (W, H) if hi is None else hi
    f64 = torch.float64
    xy = torch.tensor(lo, dtype=f64) + torch.rand(count, 2, generator=gen, dtype=f64) * (torch.tensor(hi, dtype=f64) - torch.tensor(lo, dtype=f64))
    sig = 0.5 + torch.rand(count, 2, generator=gen, dtype=f64) * (rmax / 3.0 - 0.5)
    theta = torch.rand(count, generator=gen, dtype=f64) * math.pi
    return {
        "xy": xy.float(),
        "depth": (0.5 + 30.0 * torch.rand(count, generator=gen, dtype=f64)).float(),
        "radii": torch.ceil(3.0 * sig.max(dim=1).values).to(torch.int32),
        "conic": _conics(sig, theta).float(),
        "opacity": (0.05 + 0.9 * torch.rand(count, generator=gen, dtype=f64)).float(),
        "colors": torch.rand(count, 3, generator=gen, dtype=f64).float(),
    }


def _cat(*parts):
    return {k: torch.cat([p[k] for p in parts]) for k in parts[0]}


def _culled(count, W, H, gen):
    """Gaussians that must not be listed: every other one has radius 0, the rest have rects entirely off-screen."""
    sp = _splats(count, W, H, gen)
    sp["radii"][0::2] = 0
    off = torch.tensor([[-5000.0, 0.0], [W + 5000.0, 0.0]])
    sp["xy"][1::2] = sp["xy"][1::2] + off[torch.arange(1, count, 2) % 4 // 2]
    return sp


def _interleave(vis, cul):
    """visible splats at ids 1, 3, 5, ...; the culled ones fill the remaining ids."""
    V, C = vis["xy"].shape[0], cul["xy"].shape[0]
    assert C >= V
    is_vis = torch.zeros(V + C, dtype=torch.bool)
    is_vis[1:2 * V:2] = True
    out = {}
    for k in vis:
        t = torch.empty((V + C,) + tuple(vis[k].shape[1:]), dtype=vis[k].dtype)
        t[is_vis] = vis[k]
        t[~is_vis] = cul[k]
        out[k] = t
    return out


def _device(sp, n=None, at=None):
    """The splats on the device; with `at`, as entries at[i] of n-long arrays whose other entries are culled (radius 0)."""
    if at is None:
        return {k: v.to(DEV).contiguous() for k, v in sp.items()}
    d = {"xy": torch.zeros(n, 2, device=DEV), "depth": torch.ones(n, device=DEV), "radii": torch.zeros(n, dtype=torch.int32, device=DEV),
         "conic": torch.ones(n, 3, device=DEV), "opacity": torch.full((n,), 0.5, device=DEV), "colors": torch.zeros(n, 3, device=DEV)}
    idx = at.to(DEV)
    for k, v in sp.items():
        d[k][idx] = v.to(DEV)
    return d


def _rows(d):
    """[n,12] splat rows (include/b200gs.h column layout) of the device arrays; compensation 1, the opacity column as given."""
    n = d["xy"].shape[0]
    return torch.cat([d["xy"], d["depth"][:, None], d["conic"], torch.ones(n, 1, device=DEV), d["opacity"][:, None], d["colors"],
                      d["radii"].view(torch.float32)[:, None]], dim=1).contiguous()


# ----------------------------------------------------------------------------------------------------------------------
# part 1: binning
# ----------------------------------------------------------------------------------------------------------------------
def _same_lists(a, b, what):
    assert a.total == b.total, f"{what}: {a.total} != {b.total} pairs"
    assert torch.equal(a.sorted_ids[:a.total], b.sorted_ids[:b.total]), f"{what}: sorted ids differ"
    assert torch.equal(a.tile_ranges, b.tile_ranges), f"{what}: tile ranges differ"


def _positions(b):
    """(tile, id) of every listed pair of a Binning, in list order."""
    r = b.tile_ranges.cpu().long()
    tile = torch.repeat_interleave(torch.arange(r.shape[0]), r[:, 1] - r[:, 0])
    return tile, b.sorted_ids[:b.total].cpu().long()


def _assert_subsequence(full, cul, n):
    """Every tile's culled list is an order-preserving subsequence of its full list."""
    ft, fi = _positions(full)
    ct, ci = _positions(cul)
    fk, ck = ft * n + fi, ct * n + ci
    order = torch.argsort(fk)
    skeys = fk[order]
    at = torch.searchsorted(skeys, ck).clamp_max(max(len(skeys) - 1, 0))
    assert len(ck) == 0 or bool((skeys[at] == ck).all()), "a culled pair is not in the full list"
    pos = order[at]
    same = ct[1:] == ct[:-1]
    assert bool((pos[1:] > pos[:-1])[same].all()), "culling reordered a tile's list"


def _check_binning(mode, W, H, sp, n=None, at=None):
    """Full check of one input: oracle lists, both layouts, culling off and on, and the blend of the culled lists."""
    from b200gs import ops
    sids, ranges, tiles = _oracle_lists(mode, W, H, sp)
    if at is not None:
        sids = at[sids.long()].to(torch.int32)      # the oracle saw the visible subset only; `at` is increasing, so ties keep their order
    I = int(tiles.sum())
    d = _device(sp, n, at)
    n = d["xy"].shape[0]
    full = ops.bin_gaussians(mode, W, H, d["xy"], d["depth"], d["radii"])
    assert full.total == I == full.rect_pairs, (full.total, I, full.rect_pairs)
    assert torch.equal(full.sorted_ids[:I].cpu(), sids), "sorted ids differ from the oracle"
    assert torch.equal(full.tile_ranges.cpu().long(), _library_ranges(ranges)), "tile ranges differ from the oracle"
    rows = _rows(d)
    _same_lists(ops.bin_rows(mode, W, H, rows, cull=False), full, "rows, culling off")
    cul = ops.bin_gaussians(mode, W, H, d["xy"], d["depth"], d["radii"], d["conic"], d["opacity"])
    assert cul.rect_pairs == I and cul.coarse_pairs == full.coarse_pairs and cul.total <= I
    _same_lists(ops.bin_rows(mode, W, H, rows, cull=True), cul, "rows, culling on")
    del rows
    _assert_subsequence(full, cul, n)
    bg = torch.tensor([0.1, 0.25, 0.6], device=DEV)
    planar = mode == VAN
    a = ops.blend_forward(mode, W, H, full, d["xy"], d["conic"], d["opacity"], d["colors"], bg, planar, True)
    b = ops.blend_forward(mode, W, H, cul, d["xy"], d["conic"], d["opacity"], d["colors"], bg, planar, True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[3], b[3]), "culling changed the image"
    return full, cul


VISIBLE = [1, 255, 256, 257, 2047, 2048, 2049, 4095, 4096, 4097, 3 * 4096 + 1]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("V", VISIBLE)
def test_binning_visible_count(mode, V):
    """V visible Gaussians at k*B-1, k*B, k*B+1 for the blocks of depth_keys (2048), the depth-sort tiles (4096), rank_offsets
    (2048) and emit_cells (256); V+3 culled Gaussians (radius 0, off-screen rects) interleaved, so n = 2V+3."""
    W, H = 320, 240
    gen = torch.Generator().manual_seed(V)
    sp = _interleave(_splats(V, W, H, gen), _culled(V + 3, W, H, gen))
    _, _, tiles = _rects(mode, sp["xy"], sp["radii"], W, H)
    assert sp["xy"].shape[0] == 2 * V + 3 and int((tiles > 0).sum()) == V
    assert V == 1 or min(abs(V - k * b) for b in (EMIT_BLOCK, DK_BLOCK, DEPTH_TILE) for k in range(1, 4)) <= 1
    _check_binning(mode, W, H, sp)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n", [2047, 2049, 4095, 4097, 6143, 6145])
def test_binning_gaussian_count(mode, n):
    """n itself at 2048 k +- 1 (the depth_keys blocks), half of the Gaussians visible."""
    W, H = 256, 256
    gen = torch.Generator().manual_seed(n)
    V = n // 2
    sp = _interleave(_splats(V, W, H, gen), _culled(n - V, W, H, gen))
    _, _, tiles = _rects(mode, sp["xy"], sp["radii"], W, H)
    assert sp["xy"].shape[0] == n and abs(n - DK_BLOCK * round(n / DK_BLOCK)) == 1 and int((tiles > 0).sum()) == V
    _check_binning(mode, W, H, sp)


DEPTHS = ["equal", "two", "low_byte", "spread", "clones"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", DEPTHS)
def test_binning_depth_keys(mode, kind):
    """Key distributions the radix passes treat differently: all depths bit-equal over more than three sort tiles (every pass
    sees one digit, the order is the id order across tiles), two depths alternating, depths equal in the top three bytes, depths
    spread over 1e-2 .. 1e5, and exact clones (same xy and depth) at far-apart ids."""
    W, H = 512, 384
    V = 3 * DEPTH_TILE + 5
    gen = torch.Generator().manual_seed(11 + DEPTHS.index(kind))
    vis = _splats(V, W, H, gen)
    if kind == "equal":
        vis["depth"][:] = 5.0
    elif kind == "two":
        vis["depth"] = torch.where(torch.arange(V) % 2 == 0, 2.0, 3.0)
    elif kind == "low_byte":
        bits = torch.full((V,), 7.0).view(torch.int32) & ~0xFF
        vis["depth"] = (bits | torch.randint(0, 256, (V,), generator=gen, dtype=torch.int32)).view(torch.float32)
    elif kind == "spread":
        vis["depth"] = torch.pow(10.0, -2.0 + 7.0 * torch.rand(V, generator=gen, dtype=torch.float64)).float()
    else:
        for k in range(64):       # splat V-1-k becomes an exact copy of splat k
            for key in vis:
                vis[key][V - 1 - k] = vis[key][k]
    sp = _interleave(vis, _culled(V + 3, W, H, gen))
    _, _, tiles = _rects(mode, sp["xy"], sp["radii"], W, H)
    on = tiles > 0
    bits = sp["depth"][on].view(torch.int32).long() & 0xFFFFFFFF
    assert int(on.sum()) == V > 3 * DEPTH_TILE
    distinct = int(torch.unique(bits).numel())
    if kind == "equal":
        assert distinct == 1
    elif kind == "two":
        assert distinct == 2
    elif kind == "low_byte":
        assert int(torch.unique(bits >> 8).numel()) == 1 and distinct > 200
    elif kind == "spread":
        d = sp["depth"][on]
        assert float(d.min()) < 2e-2 and float(d.max()) > 5e4
    else:
        ids = torch.nonzero(on).squeeze(1)
        a, b = ids[:64], ids.flip(0)[:64]
        assert torch.equal(sp["xy"][a], sp["xy"][b]) and torch.equal(sp["depth"][a], sp["depth"][b]) and int((b - a).min()) > V
    _check_binning(mode, W, H, sp)


# (width, height) -> (coarse cells, pack_ncells, partition passes, cells counted in shared memory)
GRIDS = {(1920, 2176): (255, True, 1, True), (2048, 2048): (256, False, 1, True), (2048, 2064): (272, False, 2, True),
         (4096, 4096): (1024, False, 2, True), (4096, 4112): (1056, False, 2, False), (1003, 997): (64, True, 1, True)}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("W,H", list(GRIDS))
def test_binning_cell_grid(mode, W, H):
    """Images at the cell-count thresholds: 255 cells (ids packed, one pass), 256 (packing off, one pass), 272 (two passes),
    1024 (shared-memory histogram and chunk table at their limit), 1056 (both in global memory), and a size that is not a
    multiple of 16 in either axis.  A few splats span many cells."""
    gen = torch.Generator().manual_seed(W * 7 + H)
    small = _splats(3000, W, H, gen)
    big = _splats(6, W, H, gen, lo=(0.25 * W, 0.25 * H), hi=(0.75 * W, 0.75 * H))
    r = torch.tensor([150.0, 300.0, 450.0, 600.0, 750.0, 900.0]) * min(W, H) / 4096
    big["radii"] = torch.ceil(r).to(torch.int32)
    big["conic"] = _conics(torch.stack([r / 3, r / 4], dim=1).double(), torch.rand(6, generator=gen, dtype=torch.float64)).float()
    sp = _cat(small, big)
    n = sp["xy"].shape[0]
    cells, pack, passes = _cell_layout(n, W, H)
    assert (cells, pack, passes, cells <= EMIT_HIST) == GRIDS[(W, H)]
    rmin, rmax, tiles = _rects(mode, sp["xy"], sp["radii"], W, H)
    cmin, cmax = rmin // CELL, (rmax - 1) // CELL + 1
    span = (cmax - cmin).prod(dim=1)
    assert int(span.max()) >= 9 and int(tiles.sum()) < 3_000_000
    _check_binning(mode, W, H, sp)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n", [PACK_IDS - 1, PACK_IDS + 5])
def test_binning_id_width(mode, n):
    """n = 2^24 - 1 (ids and cell counts packed in one word) and n = 2^24 + 5 (packing off): the visible Gaussians sit near the
    top of the index range, so ids at or above 2^24 must come back unmasked.  About 1.5 GB of device memory."""
    W, H = 256, 256
    gen = torch.Generator().manual_seed(n)
    at = torch.cat([torch.arange(100) * 997 + 3, torch.arange(n - 2900, n)])
    sp = _splats(at.numel(), W, H, gen)
    cells, pack, _ = _cell_layout(n, W, H)
    assert pack == (n < PACK_IDS) and cells <= PACK_CELLS
    assert bool((at[1:] > at[:-1]).all()) and int(at.max()) == n - 1
    assert (int((at >= PACK_IDS).sum()) > 0) == (n > PACK_IDS)
    _check_binning(mode, W, H, sp, n=n, at=at)
    torch.cuda.empty_cache()


PLACEMENTS = ["first_tile_empty", "bottom_right_only", "cell_boundary", "edges"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", PLACEMENTS)
def test_binning_tile_placement(mode, case):
    gen = torch.Generator().manual_seed(31 + PLACEMENTS.index(case))
    if case == "first_tile_empty":
        W, H = 256, 256
        sp = _splats(2000, W, H, gen)
        r = sp["radii"].float()
        sp["xy"] = torch.maximum(sp["xy"], (16.5 + r)[:, None])           # no rect reaches tile 0
    elif case == "bottom_right_only":
        W, H = 200, 120                                                   # the last tile holds columns 192..199, rows 112..119
        sp = _splats(300, W, H, gen, rmax=3.0, lo=(196.0, 116.0), hi=(199.9, 119.9))
        sp["radii"] = torch.randint(1, 5, (300,), generator=gen, dtype=torch.int32)
    elif case == "cell_boundary":
        W, H = 256, 256
        sp = _splats(1200, W, H, gen)
        r = sp["radii"].float()
        k = torch.arange(1200) % 4
        sp["xy"][k == 0, 0] = 120.0 - r[k == 0]                           # rect ends at tile column 8 = a cell boundary
        sp["xy"][k == 1, 0] = 128.0 + r[k == 1]                           # rect starts at tile column 8
        sp["xy"][k == 2, 1] = 120.0 - r[k == 2]
        sp["xy"][k == 3, 1] = 128.0 + r[k == 3]
    else:
        W, H = 200, 120
        sp = _splats(1200, W, H, gen, lo=(-20.0, -20.0), hi=(W + 20.0, H + 20.0))
    gx, gy, _, _ = _grid(W, H)
    rmin, rmax, tiles = _rects(mode, sp["xy"], sp["radii"], W, H)
    _, ranges, _ = _oracle_lists(mode, W, H, sp)
    lens = ranges[:, 1] - ranges[:, 0]
    on = tiles > 0
    if case == "first_tile_empty":
        assert int(lens[0]) == 0 and int(lens.sum()) > 0
    elif case == "bottom_right_only":
        assert int(lens[-1]) == 300 and int(lens[:-1].sum()) == 0 and W % 16 and H % 16
    elif case == "cell_boundary":
        for axis in (0, 1):
            assert int((on & (rmax[:, axis] == CELL)).sum()) >= 200 and int((on & (rmin[:, axis] == CELL)).sum()) >= 200
    else:
        r = sp["radii"].float()
        for axis, size in ((0, W), (1, H)):
            assert int((on & (sp["xy"][:, axis] - r < 0)).sum()) >= 20 and int((on & (sp["xy"][:, axis] + r > size)).sum()) >= 20
    _check_binning(mode, W, H, sp)


# ---- the capacity protocol at its boundary, through the C ABI ----------------------------------------------------------
SENTINEL = -777
WS_FILL = 0x5A
TAIL = 4096


def _bin_with_capacity(mode, W, H, d, cull, max_coarse, max_pairs):
    """b200gs_bin_count + b200gs_bin_sort with caller-chosen capacities.  sorted_ids and the phase-B workspace carry a
    sentinel-filled tail past their capacity, which must come back untouched.  -> (ids [max_pairs], ranges, phase A counters,
    phase B counters)."""
    from b200gs import ops
    from b200gs._lib import check, lib, ptr
    L = lib()
    n = d["xy"].shape[0]
    gx, gy, _, _ = _grid(W, H)
    st = ops._stream()
    ws_a = torch.empty(int(L.b200gs_bin_count_workspace_bytes(n)), dtype=torch.uint8, device=DEV)
    d_counts = torch.empty(4, dtype=torch.int64, device=DEV)
    host = torch.zeros(8, dtype=torch.int64).pin_memory()
    check(L.b200gs_bin_count(mode, W, H, n, ptr(d["xy"]), ptr(d["depth"]), ptr(d["radii"]), ptr(d["conic"]) if cull else None,
                             ptr(d["opacity"]) if cull else None, ptr(ws_a), ws_a.numel(), ptr(d_counts), host.data_ptr(), 1, st), "b200gs_bin_count")
    wb = int(L.b200gs_bin_sort_workspace_bytes(n, max_coarse, W, H))
    ws_b = torch.full((wb + TAIL,), WS_FILL, dtype=torch.uint8, device=DEV)
    ids = torch.full((max_pairs + TAIL,), SENTINEL, dtype=torch.int32, device=DEV)
    ranges = torch.full((gx * gy, 2), SENTINEL, dtype=torch.int32, device=DEV)
    check(L.b200gs_bin_sort(mode, W, H, n, int(cull), max_coarse, max_pairs, ptr(d_counts), ptr(ws_a), ptr(ws_b), wb, ptr(ids), ptr(ranges),
                            host.data_ptr() + 32, 1, st), "b200gs_bin_sort")
    torch.cuda.synchronize()
    assert bool((ids[max_pairs:] == SENTINEL).all()), "sorted_ids written past max_pairs"
    assert bool((ws_b[wb:] == WS_FILL).all()), "phase-B workspace written past its size"
    assert bool((ranges >= 0).all()) and bool((ranges <= max_pairs).all()) and bool((ranges[:, 0] <= ranges[:, 1]).all())
    return ids[:max_pairs], ranges, host[:4].clone(), host[4:].clone()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cull", [False, True])
def test_binning_capacity_boundary(mode, cull):
    """Exact capacities reproduce exact mode; max_pairs = the listed total (below the rect pairs when culling) loses nothing;
    each capacity at exact - 1 is reported through the counters and never written past."""
    from b200gs import ops
    W, H = 640, 480
    gen = torch.Generator().manual_seed(5 + int(cull))
    sp = _interleave(_splats(5000, W, H, gen, rmax=40.0), _culled(5000, W, H, gen))
    d = _device(sp)
    ref = ops.bin_gaussians(mode, W, H, d["xy"], d["depth"], d["radii"], d["conic"] if cull else None, d["opacity"] if cull else None)
    rect, coarse, total = ref.rect_pairs, ref.coarse_pairs, ref.total
    assert (total < rect) == cull and coarse > 1 and total > 1
    want_ids, want_ranges = ref.sorted_ids[:total], ref.tile_ranges

    def counters_ok(ca, cb, listed):
        assert ca.tolist()[:2] == [rect, coarse] and int(ca[3]) == int(cb[3]) and int(cb[2]) == listed

    for max_coarse, max_pairs in ((coarse, rect), (coarse, total)):           # exact, and the listed total
        ids, ranges, ca, cb = _bin_with_capacity(mode, W, H, d, cull, max_coarse, max_pairs)
        counters_ok(ca, cb, total)
        assert torch.equal(ids[:total], want_ids) and torch.equal(ranges, want_ranges)
    # coarse capacity one short: the counters report it (counts[1] > max_coarse); the lists hold what fitted
    ids, ranges, ca, cb = _bin_with_capacity(mode, W, H, d, cull, coarse - 1, rect)
    assert int(ca[1]) == coarse > coarse - 1 and int(cb[2]) <= total
    got = ids[:int(cb[2])]
    assert bool((got >= 0).all()) and bool((got < d["xy"].shape[0]).all())
    # pair capacity one short of the listed total: counts[2] reports it, everything below the capacity is exact
    ids, ranges, ca, cb = _bin_with_capacity(mode, W, H, d, cull, coarse, total - 1)
    counters_ok(ca, cb, total)
    assert torch.equal(ids, want_ids[:total - 1])
    nz = want_ranges[:, 1] > want_ranges[:, 0]
    assert torch.equal(ranges[nz], want_ranges[nz].clamp_max(total - 1)) and bool((ranges[~nz] == 0).all())


@pytest.mark.parametrize("mode", MODES)
def test_lazy_binning_empty_view_after_pairs(mode):
    """Lazy binning sized from a view with pairs, then a view where nothing is visible: empty lists, the background image, and
    resolve() reports no overflow."""
    from b200gs import ops
    W, H = 333, 222
    gen = torch.Generator().manual_seed(77)
    d = _device(_splats(500, W, H, gen))
    ops._last_total.pop((mode, W, H, 500, True), None)
    first = ops.bin_gaussians(mode, W, H, d["xy"], d["depth"], d["radii"], d["conic"], d["opacity"], lazy=True)
    assert first.resolve() is True and first.total > 0
    empty = torch.zeros_like(d["radii"])
    b = ops.bin_gaussians(mode, W, H, d["xy"], d["depth"], empty, d["conic"], d["opacity"], lazy=True)
    assert b._pending is not None                                      # sized from the previous view, not synchronised
    bg = torch.tensor([0.1, 0.25, 0.6], device=DEV)
    planar = mode == VAN
    image, final_T, n_contrib, alpha = ops.blend_forward(mode, W, H, b, d["xy"], d["conic"], d["opacity"], d["colors"], bg, planar, True)
    assert b.resolve() is True
    assert b.total == 0 and int(b.tile_ranges.abs().sum()) == 0
    want = bg[:, None, None].expand(3, H, W) if planar else bg.expand(H, W, 3)
    assert torch.equal(image, want) and bool((final_T == 1).all()) and int(n_contrib.abs().sum()) == 0 and bool((alpha == 0).all())


# ----------------------------------------------------------------------------------------------------------------------
# part 2: blend, on the oracle's lists, against autograd through O.blend in float64
# ----------------------------------------------------------------------------------------------------------------------
def _check_blend(mode, W, H, sp, seed=0, side=None):
    """K6 through its three stagings (bit-identical) and K7 against the oracle.  -> dict of oracle and kernel outputs."""
    from b200gs import ops
    sids, ranges, tiles = _oracle_lists(mode, W, H, sp)
    bg = torch.tensor([0.1, 0.25, 0.6])
    leaves = {k: sp[k].double().requires_grad_(True) for k in ("xy", "conic", "opacity", "colors")}
    margins = []
    img, alpha, nc = O.blend(mode, leaves["xy"], leaves["conic"], leaves["opacity"], leaves["colors"], sids, ranges, bg.double(), W, H,
                             margins=margins, side=side)
    gen = torch.Generator().manual_seed(seed)
    cot = torch.rand(3, H, W, generator=gen, dtype=torch.float64) * 2 - 1
    cot_a = torch.rand(H, W, generator=gen, dtype=torch.float64) * 2 - 1 if mode == GSP else None
    ((img * cot).sum() + ((alpha * cot_a).sum() if cot_a is not None else 0.0)).backward()

    total = int(sids.numel())
    binning = ops.Binning((sids if total else torch.zeros(1, dtype=torch.int32)).to(DEV), ranges.to(torch.int32).to(DEV).contiguous(), total)
    d = _device(sp)
    planar = mode == VAN
    bgd = bg.float().to(DEV)
    a = ops.blend_forward(mode, W, H, binning, d["xy"], d["conic"], d["opacity"], d["colors"], bgd, planar, True)
    hits = torch.zeros(d["xy"].shape[0], dtype=torch.uint8, device=DEV)
    b = ops.blend_forward(mode, W, H, binning, d["xy"], d["conic"], d["opacity"], d["colors"], bgd, planar, True, hits)
    c = ops.blend_forward_rows(mode, W, H, binning, _rows(d), bgd, planar)
    for k, what in enumerate(("image", "final_T", "n_contrib", "alpha")):     # the staging does not change the per-pixel arithmetic
        assert torch.equal(a[k], b[k]), f"cp.async staging: {what} differs from the synchronous kernel"
        assert k == 3 or torch.equal(a[k], c[k]), f"rows staging: {what} differs from the synchronous kernel"
    image_chw = a[0] if planar else a[0].permute(2, 0, 1)
    _assert_pixels(image_chw, img, "image", margins[0])
    _assert_pixels(a[3], alpha, "alpha", margins[0])
    sure = margins[0] >= AMBIGUOUS
    assert int(((a[2].cpu() != nc) & sure).sum()) == 0, "n_contrib differs away from any threshold"

    v_image = cot.float().to(DEV).contiguous() if planar else cot.float().permute(1, 2, 0).contiguous().to(DEV)
    v_alpha = cot_a.float().to(DEV).contiguous() if cot_a is not None else None
    g = ops.blend_backward(mode, W, H, binning, d["xy"], d["conic"], d["opacity"], d["colors"], bgd, a[1], a[2], v_image, v_alpha, planar)
    for got, k in zip(g[:4], ("xy", "conic", "opacity", "colors")):
        assert _rel(got, leaves[k].grad) < 1e-3, k
    return {"nc": nc, "margin": margins[0], "grads": g[:4], "n_contrib": a[2].cpu(), "ranges": ranges, "sids": sids, "tiles": tiles}


def _stack(L, centre, gen, sigma=(60.0, 60.0), opacity=(0.0043, 0.0055), radius=7, conic=None):
    """L splats at one centre, front to back in id order, with a given radius (which fixes their tile rect) and footprint
    (std devs about `sigma`, randomly rotated, or exactly `conic` for all)."""
    f64 = torch.float64
    theta = torch.rand(L, generator=gen, dtype=f64) * math.pi
    sig = torch.tensor(sigma, dtype=f64).expand(L, 2) * (1.0 + 0.05 * torch.rand(L, 2, generator=gen, dtype=f64))
    return {
        "xy": torch.tensor(centre, dtype=torch.float32).expand(L, 2).clone(),
        "depth": (1.0 + torch.arange(L, dtype=f64) + 0.5 * torch.rand(L, generator=gen, dtype=f64)).float(),
        "radii": torch.full((L,), radius, dtype=torch.int32),
        "conic": _conics(sig, theta).float() if conic is None else torch.tensor(conic, dtype=torch.float32).expand(L, 3).clone(),
        "opacity": (opacity[0] + (opacity[1] - opacity[0]) * torch.rand(L, generator=gen, dtype=f64)).float(),
        "colors": torch.rand(L, 3, generator=gen, dtype=f64).float(),
    }


LENGTHS = [0, 1, 15, 16, 17, 31, 32, 33, 255, 256, 257, 511, 512, 513, 1500]


@pytest.mark.parametrize("mode", MODES)
def test_blend_list_lengths(mode):
    """One row of tiles whose lists hold exactly L splats, L at the list padding (16), the warp (32) and the staging batch (256)
    boundaries and beyond: wide conics under a 7-pixel radius cover each tile evenly at low opacity, so every entry contributes."""
    gen = torch.Generator().manual_seed(3)
    W, H = 16 * len(LENGTHS), 16
    parts = [_stack(L, (16 * k + 8.3, 8.3), gen) for k, L in enumerate(LENGTHS) if L]     # no sample at a centre (power 0)
    sp = _cat(*parts)
    out = _check_blend(mode, W, H, sp, seed=4)
    lens = (out["ranges"][:, 1] - out["ranges"][:, 0]).tolist()
    assert lens == LENGTHS
    for k, L in enumerate(LENGTHS):
        assert bool((out["nc"][:, 16 * k:16 * k + 16] == L).all()), f"tile {k}: not every entry contributes"
    assert float(out["margin"].min()) >= AMBIGUOUS


def _cutoff_stack(mode, centre, gen):
    """14 splats centred on one pixel sample: 13 at opacity 0.5, then one whose alpha takes T to exactly the fp32 cut-off 1e-4f
    (2^-13 (1 - a) = 1e-4f with no rounding), then one more.  vanilla stops when T < 1e-4 (and goes on), gsplat when T <= 1e-4."""
    sp = _stack(15, centre, gen, sigma=(3.0, 3.0), opacity=(0.5, 0.5), radius=7)
    c = np.float32(np.float32(1e-4) * np.float32(8192.0))
    sp["opacity"][13] = float(np.float32(1.0) - c)
    sp["opacity"][14] = 0.3
    assert float(np.float32(2.0 ** -13) * (np.float32(1.0) - np.float32(sp["opacity"][13]))) == float(np.float32(1e-4))
    return sp


@pytest.mark.parametrize("mode", MODES)
def test_blend_stop_positions(mode):
    """The transmittance stop at chosen list positions.  Tile (0,0): alpha falls smoothly across the tile so the per-pixel stop
    lands on entries 3-5, around the every-4 early-out.  Tile (0,1): stops across entries ~240-270, over the 256-splat batch
    boundary and different inside a warp.  Tile (1,0): a pixel whose T lands exactly on the fp32 cut-off.  Tile (2,0): an
    opaque stack of the test_edge_cases kind.  Entries behind every pixel's stop get exactly zero gradient."""
    gen = torch.Generator().manual_seed(9)
    off = 0.5 if mode == GSP else 0.0
    W, H = 48, 32
    # alpha = o exp(-q) with the centre 0.3 px left of column 0: falls along x, barely along y
    fast = _stack(12, (off - 0.3, 8.0 + off + 0.3), gen, opacity=(0.97, 0.97), radius=2, conic=(0.0012, 0.0, 0.0005))
    slow = _stack(300, (off - 0.3, 24.0 + off + 0.3), gen, opacity=(0.038, 0.038), radius=2, conic=(0.0011, 0.0, 0.0003))
    cutoff = _cutoff_stack(mode, (24.0 + off, 8.0 + off), gen)
    # Nearly opaque, but below 0.97: two samples at the vanilla clamp leave T = (1 - 0.99f)^2 = 0.99998e-4 in fp32 and
    # (1 - 0.99)^2 = 1.0000000000000018e-4 in float64, on opposite sides of the cut-off by construction, and a stop that flips
    # after a sample of alpha a moves the pixel by a 1e-4 / (1 - a), above the 1/255 the ambiguous-pixel bar allows when
    # a > 0.975.  The clamp itself is test_blend_alpha_clamp's.
    opaque = _stack(40, (40.0, 8.0), gen, sigma=(10.0, 14.0), opacity=(0.93, 0.97), radius=7)
    opaque["xy"] += 0.3 * torch.randn(40, 2, generator=gen)
    sp = _cat(fast, slow, cutoff, opaque)
    side = {}
    out = _check_blend(mode, W, H, sp, seed=5, side=side)
    nc, stopped = out["nc"], side["stopped"]
    stop_fast = nc[0:16, 0:16] + 1
    stop_slow = nc[16:32, 0:16] + 1
    assert bool(stopped[0:16, 0:16].all()) and bool(stopped[16:32, 0:16].all())
    assert {EARLY_OUT - 1, EARLY_OUT, EARLY_OUT + 1} <= set(stop_fast.unique().tolist()), stop_fast.unique()
    assert int(stop_slow.min()) <= 245 and int(stop_slow.max()) >= 265 and int(stop_slow.min()) < BATCH < int(stop_slow.max())
    assert any(int(stop_slow[y:y + 4, x:x + 8].unique().numel()) > 1 for y in range(0, 16, 4) for x in (0, 8))
    # the exact cut-off pixel: fp32 semantics of the two stop rules
    px, py = 24, 8
    assert int(out["n_contrib"][py, px]) == (14 if mode == VAN else 13)
    # entries behind every pixel's stop: exactly zero gradient
    gx = W // 16
    for (tx, ty), region in (((0, 0), nc[0:16, 0:16]), ((0, 1), nc[16:32, 0:16]), ((2, 0), nc[0:16, 32:48])):
        s, e = out["ranges"][ty * gx + tx].tolist()
        behind = out["sids"][s + int(region.max()):e].long().to(DEV)
        assert behind.numel() > 0
        for gr in out["grads"]:
            assert float(gr[behind].abs().max()) == 0.0
        front = out["sids"][s:s + int(region.min())].long().to(DEV)
        assert bool((out["grads"][2][front] != 0).all())


@pytest.mark.parametrize("mode", MODES)
def test_blend_alpha_clamp(mode):
    """Opacity 1.0 and opacities in [0.99, 0.999] with a pixel sample 0.03 px from the splat centre: alpha sits at the clamp of
    vanilla (0.99, straight-through gradient) and, for opacity 1, of gsplat (0.999, no gradient through the clamp)."""
    gen = torch.Generator().manual_seed(13)
    off = 0.5 if mode == GSP else 0.0
    W, H = 64, 32
    ops_ = [1.0, 0.9915, 0.9935, 0.9955, 0.9975]
    parts = []
    for j in range(2):
        for i, o in enumerate(ops_):
            parts.append(_stack(1, (8.0 + 12 * i + off + 0.03, 8.0 + 16 * j + off), gen, opacity=(o, o), radius=5, conic=(1 / 2.25, 0.0, 1 / 2.25)))
    back = _stack(1, (32.0, 16.0), gen, sigma=(40.0, 40.0), opacity=(0.5, 0.5), radius=40)
    back["depth"][:] = 100.0
    sp = _cat(*parts, back)
    side = {}
    _check_blend(mode, W, H, sp, seed=6, side=side)
    assert side["clamped"] == (10 if mode == VAN else 2)


SHAPES = [(1, 1), (17, 1), (1, 300), (15, 17), (4000, 16)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("W,H", SHAPES)
def test_blend_image_shapes(mode, W, H):
    """Images of one pixel, partial tiles in either axis, and one row of 250 full tiles."""
    gen = torch.Generator().manual_seed(W * 1000 + H)
    count = max(6, W * H // 24)
    sp = _splats(count, W, H, gen, rmax=12.0, lo=(-3.0, -3.0), hi=(W + 3.0, H + 3.0))
    _, _, tiles = _rects(mode, sp["xy"], sp["radii"], W, H)
    assert int((tiles > 0).sum()) > 0
    _check_blend(mode, W, H, sp, seed=7)


# ----------------------------------------------------------------------------------------------------------------------
# part 3: knn_mean_dist2
# ----------------------------------------------------------------------------------------------------------------------
def _knn_ref(p):
    """float64 mean of the squared distances to the 3 nearest other points; with fewer than 3 others the missing distances count
    as 0 (csrc/knn.cu), so a single point gets 0."""
    from scipy.spatial import cKDTree
    p = p.astype(np.float64)
    n = len(p)
    if n == 1:
        return np.zeros(1)
    dist, _ = cKDTree(p).query(p, k=min(4, n))
    return (dist[:, 1:] ** 2).sum(axis=1) / 3.0


def _knn_grid(p):
    """The grid launch_knn_mean_dist2 sizes on the host: (cells per axis before the 1024 cap, cells per axis, cell size)."""
    p = p.astype(np.float32)
    e = (p.max(axis=0) - p.min(axis=0)).astype(np.float64)
    emax = e.max()
    vol = float(np.prod(np.maximum(e, 1e-3 * emax)))
    cs = (vol / (0.5 * len(p))) ** (1.0 / 3.0) if emax > 0 else 1.0
    first = np.floor(e / cs) + 1
    while True:
        g = np.minimum(KNN_AXIS, np.floor(e / cs) + 1)
        if np.prod(g) <= 4 * len(p) + 64 and bool((e / cs < KNN_AXIS).all()):
            return first, g, cs
        cs *= 1.26


def _knn(p):
    from b200gs import ops
    return ops.knn_mean_dist2(torch.from_numpy(p.astype(np.float32)).to(DEV)).cpu().double().numpy()


@pytest.mark.parametrize("n", [1, 2, 4, KNN_TILE - 1, KNN_TILE, KNN_TILE + 1])
def test_knn_sizes(n):
    p = np.random.default_rng(n).random((n, 3)).astype(np.float32)
    got, ref = _knn(p), _knn_ref(p)
    if n == 1:
        assert got.tolist() == [0.0]
    if n == 2:                     # one other point: its squared distance over 3
        d2 = float(((p[0].astype(np.float64) - p[1]) ** 2).sum()) / 3.0
        assert np.allclose(got, [d2, d2], rtol=1e-6)
    np.testing.assert_allclose(got, ref, rtol=1e-4)


def test_knn_sfm_like():
    """300 k points: 60 clusters of different spreads and 2 % uniform outliers, against scipy's cKDTree in float64."""
    rng = np.random.default_rng(0)
    centres = rng.uniform(-10, 10, (60, 3))
    spread = rng.uniform(0.02, 0.8, 60)
    which = rng.integers(0, 60, 294_000)
    pts = centres[which] + rng.normal(size=(294_000, 3)) * spread[which, None]
    pts = np.concatenate([pts, rng.uniform(-60, 60, (6_000, 3))]).astype(np.float32)
    np.testing.assert_allclose(_knn(pts), _knn_ref(pts), rtol=1e-4)


def test_knn_collinear():
    """Points on a line: the grid sizing asks for more than 1024 cells along it and is capped."""
    rng = np.random.default_rng(1)
    t = rng.uniform(0, 100, 50_000)
    pts = np.stack([t, np.zeros_like(t), np.zeros_like(t)], axis=1).astype(np.float32)
    first, g, _ = _knn_grid(pts)
    assert first.max() > KNN_AXIS and g.max() <= KNN_AXIS
    np.testing.assert_allclose(_knn(pts), _knn_ref(pts), rtol=1e-4)


def test_knn_far_outlier():
    """20 k points in a unit cube and one 1e6 away: the inliers all land in one cell."""
    rng = np.random.default_rng(2)
    pts = np.concatenate([rng.random((20_000, 3)), [[1e6, 0.0, 0.0]]]).astype(np.float32)
    _, g, cs = _knn_grid(pts)
    cells = np.floor((pts[:-1] - pts.min(axis=0)) / cs).astype(np.int64)
    assert len({tuple(c) for c in cells}) == 1
    np.testing.assert_allclose(_knn(pts), _knn_ref(pts), rtol=1e-4)
