"""The Gaussian-sharded exchange kernels on ONE GPU, at their capacity, block and camera-count boundaries.

b200gs_project_pack_multi projects one shard into up to B200GS_MAX_VIEWS cameras and stores each camera's visible splats as
[.,12] rows into a fixed-capacity block of `cap` rows of the camera owner's receive buffer (a peer GPU's memory on a real run):
blocks take tickets, compact their visible lanes per warp in shared memory and run one decoupled look-back scan per camera.
Rows at or past `cap` are dropped, d_count[j] reports the true count and row_index is -1 for them.  The multi-GPU test
(test_gpu_distributed.py) needs two devices; here every rank of a W-rank step runs in this process on one device, the receive
buffers are local allocations laid out the way PeerExchange lays them out, and K7 / K8 read them with the pointer shifts of
distributed.py.

1. the pack contract, bit for bit against the single-view rows, at warp / block / ticket boundaries and at every kind of cut
2. the packed rows against the float64 oracle, camera inside the scene among them
3. a simulated W-rank step, forward and backward, against the single-GPU renderer and the float64 oracle, and with empty,
   exactly full and overflowing blocks against the compact rows / the accumulated single-view K8
4. the pack entry point's argument checks, including the int32 bound of row_index
"""
import ctypes
import math

import pytest
import torch

from oracle import gs_oracle as O
from test_gpu_sharded_kernels import COLS, _diff_report, _single_rows
from test_inside_scene import FP32_LIMITED, _ambiguous, _check_forward, _kview, _oview, _per_category, _print_report, activate64, inside_scene

pytestmark = pytest.mark.gpu
DEV = "cuda"
PACK_THREADS = 256                  # Gaussians per ticket of the pack kernel (project.cu PACK_THREADS)
LOOKBACK_WORDS = 32 * 4             # predecessors one look-back step reads at its widest (onesweep.cuh chained_exclusive, DEPTH 4)
GUARD = 40                          # NaN-pattern rows after every block of `cap` rows
GUARD_BITS = 0x7FC0BEEF             # a quiet NaN no kernel produces: any row the pack kernel touches stops matching it
EINVAL = -1


# ----------------------------------------------------------------------------------------------------------------------
# cameras and scenes
# ----------------------------------------------------------------------------------------------------------------------
def _ring(W, H, pose, distance=4.0):
    from b200gs.scene import make_ring_cameras
    return make_ring_cameras(W, H, distance=distance)[pose]


def _posed(W, H, R, T):
    from b200gs.cameras import make_camera
    fx = 0.5 * W / math.tan(math.radians(39.6) * 0.5)
    return make_camera(torch.tensor(R, dtype=torch.float32), torch.tensor(T, dtype=torch.float32), fx, fx, W / 2.0, H / 2.0, W, H)


def _away(W, H):
    """pose 0 turned around: the whole scene (|z| <= extent) lies behind the camera"""
    return _posed(W, H, [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]], [0.0, 0.0, -4.0])


def _up(W, H, height):
    """looks along world +y from (0, height, 0): camera depth = y - height"""
    return _posed(W, H, [[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]], [0.0, 0.0, -height])


def _view(cam, sh_degree, sh_stride):
    from b200gs._lib import MODE_GSPLAT
    return _kview(cam, MODE_GSPLAT, sh_degree, sh_stride, 1.0, 0.3, None)


def _dev(raw):
    return {k: v.to(DEV).contiguous() for k, v in raw.items()}


# ----------------------------------------------------------------------------------------------------------------------
# the pack kernel and its destinations
# ----------------------------------------------------------------------------------------------------------------------
def _guarded(rows):
    return torch.full((rows, 12), GUARD_BITS, dtype=torch.int32, device=DEV).view(torch.float32)


def _stale(rows):
    """what a receive buffer holds behind the valid rows of a block: NaN rows that look visible (radius 5)"""
    t = torch.full((rows, 12), float("nan"), device=DEV)
    t[:, 11] = torch.tensor([5], dtype=torch.int32, device=DEV).view(torch.float32)
    return t


class Packed:
    pass


def _pack(raw, views, cap, dst_ptrs, ws_bytes=None, aa=True):
    """one b200gs_project_pack_multi launch; every output starts as a sentinel so that an entry the call never wrote shows"""
    from b200gs import ops
    from b200gs._lib import lib, ptr
    L = lib()
    n, nv = raw["means"].shape[0], len(views)
    o = Packed()
    o.xy = torch.full((nv * n, 2), float("nan"), device=DEV)
    o.radii = torch.full((nv * n,), -7, dtype=torch.int32, device=DEV)
    o.clamped = torch.full((nv * n,), 0xAB, dtype=torch.uint8, device=DEV)
    o.row_index = torch.full((nv * n,), -7, dtype=torch.int32, device=DEV)
    o.d_count = torch.full((max(nv, 1),), -7, dtype=torch.int64, device=DEV)
    need = int(L.b200gs_project_pack_workspace_bytes(max(nv, 1), n))
    ws = torch.empty(need + 64, dtype=torch.uint8, device=DEV)
    arr = _view_array(views)
    dst_arr = (ctypes.c_void_p * max(len(dst_ptrs), 1))(*dst_ptrs)
    o.rc = int(L.b200gs_project_pack_multi(arr, nv, n, ptr(raw["means"]), ptr(raw["scales"]), ptr(raw["rotations"]),
                                           ptr(raw["opacities"].reshape(-1).contiguous()), ptr(raw["shs_dc"]), ptr(raw["shs_rest"]), int(aa),
                                           ptr(o.xy), ptr(o.radii), ptr(o.clamped), ptr(o.row_index), dst_arr, cap, ptr(ws),
                                           need if ws_bytes is None else ws_bytes, ptr(o.d_count), ops._stream()))
    o.error = L.b200gs_last_error() if o.rc else b""
    torch.cuda.synchronize()
    return o


def _view_array(views):
    from b200gs._lib import B200gsView
    return (B200gsView * max(len(views), 1))(*views)


def _pack_checked(raw, views, cap, dst_ptrs):
    o = _pack(raw, views, cap, dst_ptrs)
    assert o.rc == 0, o.error
    return o


def _expected_row_index(vis, j, cap):
    k = torch.cumsum(vis.to(torch.int64), 0) - 1
    return torch.where(vis & (k < cap), j * cap + k, torch.full_like(k, -1)).to(torch.int32)


def _assert_pack(o, single, cap, dst, n):
    """the pack contract for camera j of launch `o` with destination blocks dst[j] (cap + GUARD rows each)"""
    for j, (rows, rad, cl) in enumerate(single):
        vis = rad > 0
        V = int(vis.sum())
        s = slice(j * n, (j + 1) * n)
        assert int(o.d_count[j]) == V, (j, cap, int(o.d_count[j]), V)
        assert torch.equal(o.radii[s], rad), j
        assert torch.equal(o.clamped[s][vis], cl[vis]) and not bool(o.clamped[s][~vis].any()), j
        assert torch.equal(o.xy[s].view(torch.int32), rows[:, 0:2].contiguous().view(torch.int32)), j
        assert torch.equal(o.row_index[s], _expected_row_index(vis, j, cap)), (j, cap)
        m = min(V, cap)
        bad = _diff_report(dst[j][:m], rows[vis][:m], COLS)
        assert not bad, f"camera {j}, cap {cap}: packed rows differ from the single-view rows: {bad}"
        rest = dst[j][m:].view(torch.int32)
        assert bool((rest == GUARD_BITS).all()), f"camera {j}, cap {cap}: {int((rest != GUARD_BITS).any(1).sum())} rows written at or past row {m}"


# ----------------------------------------------------------------------------------------------------------------------
# 1. pack contract at its boundaries, bit-exact against the single-view rows
# ----------------------------------------------------------------------------------------------------------------------
PACK_N = [1, 31, 255, 256, 257, 20000, 1_000_003]
PACK_W, PACK_H = 320, 240


def _pack_cameras(nv):
    """ordinary ring cameras, one that sees every Gaussian (the scene small in front of it) and one that sees none"""
    cams = [_ring(PACK_W, PACK_H, 0), _ring(PACK_W, PACK_H, 3, distance=14.0), _away(PACK_W, PACK_H)]
    cams += [_ring(PACK_W, PACK_H, p) for p in (7, 11, 20, 26, 30)]
    return cams[:nv], ["ring", "all", "none", "ring", "ring", "ring", "ring", "ring"][:nv]


def _caps(vis_list, n):
    """every cap the launch set uses, and the cuts they make: {cap: [(camera, kind), ...]}.  Per camera: 1, V-1, V, V+1; a cap that
    ends exactly at a block boundary (the visible splats of the first t tickets); one that ends inside a warp's run."""
    caps = {}

    def add(cap, j, kind):
        if cap >= 1:
            caps.setdefault(int(cap), []).append((j, kind))

    tickets = (n + PACK_THREADS - 1) // PACK_THREADS
    for j, vis in enumerate(vis_list):
        V = int(vis.sum())
        add(1, j, "first row" if V > 1 else "other")
        add(V - 1, j, "last row")
        add(V, j, "exactly full")
        add(V + 1, j, "one spare")
        if tickets < 2 or V < 2:
            continue
        cum = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(vis.cpu().to(torch.int64), 0)])
        t = tickets // 2
        at = int(cum[t * PACK_THREADS])
        if 0 < at < V:
            add(at, j, "block boundary")
        for w in range(PACK_THREADS // 32):                # a warp of ticket t with >= 2 visible lanes: keep its first row only
            lo = t * PACK_THREADS + 32 * w
            if lo + 32 <= n and int(cum[lo + 32] - cum[lo]) >= 2:
                add(int(cum[lo]) + 1, j, "inside a warp run")
                break
    return caps


@pytest.mark.parametrize("stride", [16, 25])
@pytest.mark.parametrize("n_views", [1, 2, 8])
@pytest.mark.parametrize("n", PACK_N)
def test_pack_contract_at_boundaries(n, n_views, stride):
    """d_count, row_index, the packed rows (every column, bit for bit, in Gaussian-index order), the guard rows, xy / radii /
    clamped, and the repeatability of the bytes, for every cap of _caps in one launch each."""
    from b200gs.scene import make_scene
    deg = 3 if stride == 16 else 4                 # the pack launcher takes its MC = 25 instantiation for degree 4
    raw = _dev(make_scene(n, 1000 + n, mean_scale=0.03, sh_degree=deg))
    assert 1 + raw["shs_rest"].shape[1] == stride
    cams, kinds = _pack_cameras(n_views)
    views = [_view(c, deg, stride) for c in cams]
    single = [_single_rows(raw, v, True) for v in views]
    vis_list = [s[1] > 0 for s in single]
    for kind, vis in zip(kinds, vis_list):
        if kind == "all":
            assert int(vis.sum()) == n
        elif kind == "none":
            assert int(vis.sum()) == 0

    # what the parameter sets reach
    tickets = (n + PACK_THREADS - 1) // PACK_THREADS
    if n_views == 8:
        assert n_views * PACK_THREADS * 3 * 16 == 96 * 1024          # dynamic shared memory above the 48 KB default
    if n == 1_000_003:
        assert tickets >= 3900 and tickets > 30 * LOOKBACK_WORDS     # the look-back has to widen and walk many windows
    if n in (31, 255, 257, 1_000_003):
        assert n % 32 != 0 and n % PACK_THREADS != 0                 # partial last warp and block
    caps = _caps(vis_list, n)
    reached = {kind for cuts in caps.values() for _, kind in cuts}
    if n >= 20000:
        assert {"block boundary", "inside a warp run", "first row", "exactly full"} <= reached, reached

    for idx, cap in enumerate(sorted(caps)):
        dst = [_guarded(cap + GUARD) for _ in range(n_views)]
        o = _pack_checked(raw, views, cap, [d.data_ptr() for d in dst])
        _assert_pack(o, single, cap, dst, n)
        if idx in (0, len(caps) // 2):
            dst2 = [_guarded(cap + GUARD) for _ in range(n_views)]
            o2 = _pack_checked(raw, views, cap, [d.data_ptr() for d in dst2])
            for a, b in ((o.xy, o2.xy), (o.radii, o2.radii), (o.clamped, o2.clamped), (o.row_index, o2.row_index), (o.d_count, o2.d_count)):
                assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
            for a, b in zip(dst, dst2):
                assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ----------------------------------------------------------------------------------------------------------------------
# 2. the packed rows against the float64 oracle
# ----------------------------------------------------------------------------------------------------------------------
OW, OH = 136, 100                                   # partial border tiles
ORACLE_POSES = [5, 0, 3, 9, 14, 19, 24, 28]          # pose 5 first: the camera of the camera-inside scene
_ORACLE = {}


def _oracle_scene():
    """the camera-inside scene of test_inside_scene.py plus 2500 ring-scene Gaussians around the origin ("ring"), without the
    Gaussians that sit within the decision bands of any of the eight cameras -> (raw, masks, cameras)"""
    if not _ORACLE:
        from b200gs.scene import make_scene
        raw_in, masks_in, cam_in = inside_scene(OW, OH, pose=5)
        ring = make_scene(2500, 17, mean_scale=0.03)
        n_in = raw_in["means"].shape[0]
        raw = {k: torch.cat([raw_in[k], ring[k]]).contiguous() for k in raw_in}
        masks = {k: torch.cat([m, torch.zeros(2500, dtype=torch.bool)]) for k, m in masks_in.items()}
        masks["ring"] = torch.arange(n_in + 2500) >= n_in
        cams = [cam_in] + [_ring(OW, OH, p) for p in ORACLE_POSES[1:]]
        bad = torch.zeros(n_in + 2500, dtype=torch.bool)
        for c in cams:
            bad |= _ambiguous(raw, c, [(O.MODE_GSPLAT, 1.0, 0.3, None)])
        keep = ~bad
        _ORACLE["v"] = ({k: v[keep].contiguous() for k, v in raw.items()}, {k: m[keep] for k, m in masks.items()}, cams)
    return _ORACLE["v"]


def _oracle_rows(raw, cam):
    """float64 oracle of one camera's rows: projection, SH colour, blend opacity (anti-aliased)"""
    ins = activate64(raw)
    p = O.project(O.MODE_GSPLAT, ins["means"], ins["scales"], ins["rotations"], _oview(cam))
    colors = O.sh_colors(3, ins["shs"][:, :16], ins["means"], cam.camera_center.double(), detach_dir=True)
    return p, colors, ins["opacities"].reshape(-1) * p["comp"]


def test_packed_rows_match_float64_oracle_with_the_camera_inside_the_scene():
    """Each camera's packed rows, scattered back to Gaussian order through row_index, against gs_oracle.project + sh_colors with
    _check_forward's tolerances: catches a drift the kernel-against-kernel checks share with the single-view K1."""
    raw, masks, cams = _oracle_scene()
    n = raw["means"].shape[0]
    assert 2500 < n < 5000
    views = [_view(c, 3, 16) for c in cams]
    dst = [_guarded(n + GUARD) for _ in views]
    o = _pack_checked(_dev(raw), views, n, [d.data_ptr() for d in dst])
    for j, cam in enumerate(cams):
        p, colors, blend_op = _oracle_rows(raw, cam)
        s = slice(j * n, (j + 1) * n)
        radii, idx = o.radii[s], o.row_index[s].long()
        vis = radii > 0
        assert int(o.d_count[j]) == int(vis.sum()) and bool((idx[vis] == j * n + torch.arange(int(vis.sum()), device=DEV)).all())
        full = torch.zeros(n, 12, device=DEV)
        full[vis] = dst[j][idx[vis] - j * n]
        r = full.cpu()
        _check_forward(O.MODE_GSPLAT, p, colors, OW, OH, r[:, 0:2], r[:, 2], radii, r[:, 3:6], r[:, 8:11], r[:, 6], r[:, 7], blend_op)
        if j == 0:              # the inside camera sees every category the inside scene builds
            assert all(int((p["mask"] & masks[k]).sum()) > 0 for k in ("near", "near_gs", "clamp", "offscreen", "giant", "ring"))


# ----------------------------------------------------------------------------------------------------------------------
# 3. a simulated W-rank sharded step on one device
# ----------------------------------------------------------------------------------------------------------------------
class Step:
    pass


def _sharded_forward(raw, views, cap, bg, W, H):
    """every rank packs its shard into block r of each owner's receive buffer (stale rows elsewhere); every owner bins and blends
    its buffer with block_counts = min(count, cap), as the fixed-capacity step of distributed.py does"""
    from b200gs import distributed, ops
    from b200gs._lib import MODE_GSPLAT
    world, n = len(views), raw["means"].shape[0]
    st = Step()
    st.world, st.cap = world, cap
    st.recv = [_stale(world * cap) for _ in range(world)]
    st.shards = []
    for r in range(world):
        lo, hi = distributed.shard_range(n, world, r)
        part = {k: v[lo:hi].contiguous() for k, v in raw.items()}
        o = _pack_checked(part, views, cap, [st.recv[j].data_ptr() + r * cap * 48 for j in range(world)])
        st.shards.append((lo, hi, part, o))
    st.counts = torch.stack([o.d_count for *_, o in st.shards])                       # [rank, camera]
    st.out = []
    for j in range(world):
        kept = st.counts[:, j].clamp(max=cap).contiguous()
        binning, (img, T, nc) = ops.bin_and_blend_rows(MODE_GSPLAT, W, H, st.recv[j], bg, True, False, kept, cap)
        st.out.append((binning, img, T, nc))
    return st


def _sharded_backward(st, raw, views, bg, cots, W, H):
    """K7 of every owner into a gradient buffer of the receive buffer's layout, then K8 of every shard for all cameras, reading
    owner j's buffer through the base pointer shifted by rank*cap - j*cap rows.  Rows no K8 may read are poisoned."""
    from b200gs import ops
    from b200gs._lib import MODE_GSPLAT, check, lib, ptr
    L = lib()
    world, cap = st.world, st.cap
    v_recv = []
    for j in range(world):
        binning, img, T, nc = st.out[j]
        v = torch.zeros(world * cap, 12, device=DEV)
        check(L.b200gs_blend_bwd_rows(MODE_GSPLAT, W, H, ptr(binning.tile_ranges), ptr(binning.sorted_ids), ptr(st.recv[j]), ptr(bg), ptr(T),
                                      ptr(nc), ptr(cots[j]), 3, 1, None, 1.0, 1.0, ptr(v), ops._stream()), "b200gs_blend_bwd_rows")
        for r in range(world):
            v[r * cap + int(min(int(st.counts[r, j]), cap)):(r + 1) * cap] = 1e6
        v_recv.append(v)
    grads = []
    for r, (lo, hi, part, o) in enumerate(st.shards):
        m = hi - lo
        out = [torch.full((m, 3), float("nan"), device=DEV), torch.full((m, 3), float("nan"), device=DEV),
               torch.full((m, 4), float("nan"), device=DEV), torch.full((m,), float("nan"), device=DEV),
               torch.full_like(part["shs_dc"], float("nan")), torch.full_like(part["shs_rest"], float("nan"))]
        src = (ctypes.c_void_p * world)(*[v_recv[j].data_ptr() + (r * cap - j * cap) * 48 for j in range(world)])
        check(L.b200gs_project_bwd_rows_multi(_view_array(views), world, m, ptr(part["means"]), ptr(part["scales"]), ptr(part["rotations"]),
                                              ptr(part["opacities"].reshape(-1).contiguous()), ptr(part["shs_dc"]), ptr(part["shs_rest"]), 1,
                                              ptr(o.radii), ptr(o.clamped), ptr(o.row_index), src, *[ptr(t) for t in out], ops._stream()),
              "b200gs_project_bwd_rows_multi")
        grads.append(out)
    torch.cuda.synchronize()
    return v_recv, grads


GRAD_KEYS = ("means", "scales", "rotations", "opacities", "shs_dc", "shs_rest")
# test_inside_scene.py's FP32_LIMITED pairs, and the needles' mean gradient: seen from the seven ring cameras the needles' cov2D is
# as close to rank 1 as from the inside camera, and dL/dmean reaches the conic through the same EWA Jacobian whose fp32 rounding
# turns the thin eigenvector (1.0e-3 of the category's largest entry within one shard, 8 cameras, H100 SXM at 700 W; the single-GPU
# renderer and the sharded step agree to < 1e-4 of each other there, so the error is K8's, not the exchange's)
SHARDED_FP32_LIMITED = FP32_LIMITED + (("needle", "means"),)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_step_matches_single_gpu_renderer_and_float64_oracle(world):
    """cap >= every count: each owner's image is bit-identical to B200GSplatRenderer on the whole model and within the
    _assert_pixels bar of the float64 oracle; each shard's raw-parameter gradients of the summed loss match the matching slice of
    the single-GPU renderer's (< 1e-4 relative) and float64 autograd through the oracle per category (< 1e-3)."""
    from b200gs.renderers import B200GSplatRenderer
    from b200gs.scene import SyntheticGaussians
    from test_gpu_parity import _assert_pixels
    raw, masks, all_cams = _oracle_scene()
    cams = [all_cams[0]] + all_cams[1:world]
    views = [_view(c, 3, 16) for c in cams]
    g = _dev(raw)
    bg = torch.tensor([0.3, 0.1, 0.7])
    gen = torch.Generator().manual_seed(world)
    cots = [torch.rand(3, OH, OW, generator=gen) * 2 - 1 for _ in cams]

    # the counts of a first pass fix cap; a second pass with that cap is the step
    probe = _sharded_forward(g, views, raw["means"].shape[0], bg.to(DEV), OW, OH)
    cap = int(probe.counts.max()) + 37
    st = _sharded_forward(g, views, cap, bg.to(DEV), OW, OH)
    assert bool((st.counts <= cap).all())

    R = B200GSplatRenderer(fused_activations=True).to(DEV)
    model = SyntheticGaussians(raw).to(DEV)
    rp = {k: v.double().requires_grad_(True) for k, v in raw.items()}
    loss_ref = 0.0
    for j, cam in enumerate(cams):
        out = R(cam.to_device(DEV), model, bg.to(DEV))
        (out["render"] * cots[j].to(DEV)).sum().backward()
        img = st.out[j][1].permute(2, 0, 1)
        assert torch.equal(img, out["render"].detach()), f"camera {j}: {float((img - out['render']).abs().max())}"
        margins = []
        ref = O.render(O.MODE_GSPLAT, rp["means"], torch.exp(rp["scales"]), torch.nn.functional.normalize(rp["rotations"]),
                       torch.sigmoid(rp["opacities"]), torch.cat((rp["shs_dc"], rp["shs_rest"]), dim=1), _oview(cam), bg.double(),
                       margins=margins)
        _assert_pixels(img, ref["render"], f"camera {j}", margins[0])
        loss_ref = loss_ref + (ref["render"] * cots[j].double()).sum()
    loss_ref.backward()

    v_images = [c.permute(1, 2, 0).contiguous().to(DEV) for c in cots]
    _, grads = _sharded_backward(st, g, views, bg.to(DEV), v_images, OW, OH)
    for (lo, hi, part, o), got in zip(st.shards, grads):
        for k, t in zip(GRAD_KEYS, got):
            assert bool(torch.isfinite(t).all()), k
            want = model.gaussians[k].grad[lo:hi]
            err = float((t.reshape(want.shape) - want).abs().max() / want.abs().max().clamp_min(1e-30))
            assert err < 1e-4, (k, lo, hi, err)
    # the shards' gradients side by side are the model's: per category over the whole model, as test_inside_scene.py holds them
    report = {}
    for i, k in enumerate(GRAD_KEYS):
        _per_category(torch.cat([got[i].reshape(hi - lo, -1) for (lo, hi, _, _), got in zip(st.shards, grads)]), rp[k].grad, masks, k,
                      report, SHARDED_FP32_LIMITED)
    _print_report(f"sharded step world={world}", report)


def _far_scene():
    """12 000 ring-scene Gaussians around the origin, then 6 000 in a cluster at y = 40 that no ring camera sees; with three ranks
    the last shard is exactly the cluster"""
    from b200gs.scene import make_scene
    main = make_scene(12000, 23, mean_scale=0.03)
    far = make_scene(6000, 24, extent=0.5, mean_scale=0.03)
    far["means"] = far["means"] + torch.tensor([0.0, 40.0, 0.0])
    return {k: torch.cat([main[k], far[k]]).contiguous() for k in main}


@pytest.mark.parametrize("case", ["exactly_full", "overflow", "cap_1"])
def test_sharded_step_with_empty_full_and_overflowing_blocks(case):
    """Three ranks, two ring cameras and one that sees only the far cluster: six of the nine blocks hold rows, three are empty.
    The image of every owner is bit-identical to binning and blending the compact rows that were kept; K8 of every shard, with
    -1 row indices for the dropped splats, equals the single-view K8 accumulated over the cameras with the dropped splats'
    gradient rows set to zero."""
    from b200gs import ops
    from b200gs._lib import MODE_GSPLAT, check, lib, ptr
    L = lib()
    W, H = 256, 192
    raw = _dev(_far_scene())
    n = raw["means"].shape[0]
    cams = [_ring(W, H, 0), _ring(W, H, 9), _up(W, H, 36.0)]
    views = [_view(c, 3, 16) for c in cams]
    bg = torch.tensor([0.2, 0.1, 0.4], device=DEV)
    probe = _sharded_forward(raw, views, n, bg, W, H)
    counts = probe.counts.cpu()
    assert torch.equal(counts == 0, torch.tensor([[False, False, True], [False, False, True], [True, True, False]])), counts
    cap = {"exactly_full": int(counts.max()), "overflow": int(counts[counts > 0].min()) // 2 + 1, "cap_1": 1}[case]
    st = _sharded_forward(raw, views, cap, bg, W, H)
    assert torch.equal(st.counts.cpu(), counts)
    full = counts == cap
    over = counts > cap
    if case == "exactly_full":
        assert bool(full.any()) and not bool(over.any())
    else:
        assert torch.equal(over, counts > 0)             # every block that holds rows overflows

    for j in range(3):
        kept = []
        for lo, hi, part, o in st.shards:
            rows, rad, _ = _single_rows(part, views[j], True)
            kept.append(rows[rad > 0][:cap])
        compact = torch.cat(kept).contiguous()
        _, (img_c, T_c, _) = ops.bin_and_blend_rows(MODE_GSPLAT, W, H, compact, bg, True)
        _, img, T, _ = st.out[j]
        assert torch.equal(T, T_c), f"camera {j}: {float((T - T_c).abs().max())}"
        assert torch.equal(img, img_c), f"camera {j}: {float((img - img_c).abs().max())}"

    gen = torch.Generator().manual_seed(9)
    v_images = [(torch.rand(H, W, 3, generator=gen) * 2 - 1).to(DEV) for _ in cams]
    v_recv, grads = _sharded_backward(st, raw, views, bg, v_images, W, H)
    for r, ((lo, hi, part, o), got) in enumerate(zip(st.shards, grads)):
        m = hi - lo
        ref = [torch.empty_like(t) for t in got]
        ol = part["opacities"].reshape(-1).contiguous()
        for j in range(3):
            idx = o.row_index[j * m:(j + 1) * m].long()
            rows = torch.zeros(m, 12, device=DEV)
            keep = idx >= 0
            rows[keep] = v_recv[j][r * cap + idx[keep] - j * cap]
            check(L.b200gs_project_bwd_rows(ctypes.byref(views[j]), m, ptr(part["means"]), ptr(part["scales"]), ptr(part["rotations"]), ptr(ol),
                                            ptr(part["shs_dc"]), ptr(part["shs_rest"]), 1, ptr(o.radii[j * m:(j + 1) * m].contiguous()),
                                            ptr(o.clamped[j * m:(j + 1) * m].contiguous()), None, ptr(rows), 1 if j > 0 else 0,
                                            *[ptr(t) for t in ref], None, 0, ops._stream()), "b200gs_project_bwd_rows")
        torch.cuda.synchronize()
        for k, a, b in zip(GRAD_KEYS, got, ref):
            assert bool(torch.isfinite(a).all()), (r, k)
            err = float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
            assert err < 2e-5, (r, k, err)


# ----------------------------------------------------------------------------------------------------------------------
# 4. argument checks of the pack entry point
# ----------------------------------------------------------------------------------------------------------------------
def _bad_call_setup():
    from b200gs.scene import make_scene
    raw = _dev(make_scene(256, 5, mean_scale=0.03))
    views = [_view(_ring(PACK_W, PACK_H, p), 3, 16) for p in (0, 3, 6)]
    dst = [_guarded(256) for _ in views]
    return raw, views, dst


def _assert_refused(o, what):
    assert o.rc == EINVAL, (what, o.rc)
    assert int((o.d_count != -7).sum()) == 0, f"{what}: d_count written"
    assert int((o.row_index != -7).sum()) == 0, f"{what}: row_index written"


def test_pack_refuses_bad_arguments_and_writes_nothing():
    from b200gs._lib import lib
    raw, views, dst = _bad_call_setup()
    ptrs = [d.data_ptr() for d in dst]
    need = int(lib().b200gs_project_pack_workspace_bytes(3, 256))
    _assert_refused(_pack(raw, views, 256, ptrs, ws_bytes=need - 1), "workspace one byte short")
    assert b"workspace" in _pack(raw, views, 256, ptrs, ws_bytes=need - 1).error
    _assert_refused(_pack(raw, [], 256, []), "n_views 0")
    nine = views * 3
    _assert_refused(_pack(raw, nine, 256, [dst[0].data_ptr()] * 9), "n_views 9")
    _assert_refused(_pack(raw, views, 256, [ptrs[0], ptrs[1] + 8, ptrs[2]]), "destination 8 bytes off 16-byte alignment")
    _assert_refused(_pack(raw, views, 0, ptrs), "cap 0")
    for d in dst:
        assert bool((d.view(torch.int32) == GUARD_BITS).all())
    # the calls above left no error behind: a valid call still works
    assert _pack(raw, views, 256, ptrs).rc == 0


def test_pack_refuses_row_indices_beyond_int32():
    """row_index is int32: camera j's rows are numbered j*cap + k, so n_views * cap must stay <= 2^31 - 1.  With 3 views and
    cap = 2^30 - 1 the third camera's third visible row would be 2^31.  The kernel only stores rows below min(V, cap), so
    256-row destinations suffice."""
    raw, views, dst = _bad_call_setup()
    cap = (1 << 30) - 1
    assert (len(views) - 1) * cap + cap > 2**31 - 1
    V = [int((_single_rows(raw, v, True)[1] > 0).sum()) for v in views]
    assert V[2] >= 3 and 2 * cap + V[2] - 1 > 2**31 - 1          # a row index that does not fit would be produced
    o = _pack(raw, views, cap, [d.data_ptr() for d in dst])
    wrapped = o.row_index[2 * 256:].tolist() if o.rc == 0 else []
    assert o.rc == EINVAL, f"accepted; camera 2 row_index = {sorted(set(wrapped))[:6]}"
    _assert_refused(o, "n_views * cap > 2^31 - 1")
    assert b"int32" in o.error
    # the largest cap that fits is accepted and numbers camera 2's rows up to 2^31 - 1 at most
    cap = (2**31 - 1) // 3
    o = _pack(raw, views, cap, [d.data_ptr() for d in dst])
    assert o.rc == 0, o.error
    idx = o.row_index[2 * 256:]
    assert int(idx.max()) == 2 * cap + V[2] - 1 and int(idx.min()) == -1
