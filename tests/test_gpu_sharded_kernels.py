"""The three K1 variants must agree BIT FOR BIT on one GPU: the single-view kernel that writes [n,12] rows (b200gs_project_fwd_rows, what the
single-GPU renderers run), the multi-view kernel with separate arrays (b200gs_project_fwd_raw_multi) and the multi-view kernel fused with the
exchange packing (b200gs_project_pack_multi).  That is what makes the Gaussian-sharded image (tests/test_gpu_distributed.py, 2 GPUs)
bit-identical to the single-GPU image; this file pins it where the driver's one-GPU run can see it, column by column.
Reference semantics: internal/renderers/gsplat_distributed_renderer.py:127-217 (project for every camera, exchange, rasterize)."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
COLS = ["x", "y", "depth", "conicA", "conicB", "conicC", "comp", "opacity", "r", "g", "b", "radius"]


# (storage degree, active degree): SH stored with stride 16 or 25.  The multi-view K1 kernels take MC = 25 for an active degree of 4.
SH_DEGREES = pytest.mark.parametrize(("storage_degree", "sh_degree"), [(3, 3), (4, 4), (4, 2)])


def _scene(n, seed, W, H, poses, sh_degree=3, aa=True, storage_degree=3):
    from b200gs import ops
    from b200gs._lib import MODE_GSPLAT
    from b200gs.scene import make_ring_cameras, make_scene
    raw = {k: v.to(DEV).contiguous() for k, v in make_scene(n, seed, mean_scale=0.03, sh_degree=storage_degree).items()}
    cams = [make_ring_cameras(W, H)[p].to_device(DEV) for p in poses]
    stride = int(raw["shs_dc"].shape[1] + raw["shs_rest"].shape[1])
    views = [ops.make_view(MODE_GSPLAT, W, H, fx=float(c.fx), fy=float(c.fy), cx=float(c.cx), cy=float(c.cy), viewmatrix=c.world_to_camera,
                           campos=c.camera_center, sh_degree=sh_degree, sh_stride=stride) for c in cams]
    return raw, views


def _single_rows(raw, view, aa):
    from b200gs import ops
    from b200gs._lib import check, lib, ptr
    n = raw["means"].shape[0]
    rows = torch.empty(n, 12, device=DEV)
    radii = torch.empty(n, dtype=torch.int32, device=DEV)
    clamped = torch.empty(n, dtype=torch.uint8, device=DEV)
    check(lib().b200gs_project_fwd_rows(ctypes.byref(view), n, ptr(raw["means"]), ptr(raw["scales"]), ptr(raw["rotations"]),
                                        ptr(raw["opacities"].reshape(-1).contiguous()), ptr(raw["shs_dc"]), ptr(raw["shs_rest"]), int(aa), ptr(rows),
                                        ptr(radii), ptr(clamped), None, ops._stream()), "b200gs_project_fwd_rows")
    return rows, radii, clamped


def _diff_report(a, b, names):
    bad = []
    for c, name in enumerate(names):
        ne = a[:, c].view(torch.int32) != b[:, c].view(torch.int32)
        if bool(ne.any()):
            bad.append((name, int(ne.sum()), float((a[:, c] - b[:, c]).abs().max())))
    return bad


def _assert_camera_arrays_match_rows(j, n, xy, depth, conic, opac, rgb, radii, clamped, single):
    """Camera j's slice of the camera-major separate arrays of the multi-view K1 against the single-view rows of that camera."""
    rows, rad, cl = single
    s = slice(j * n, (j + 1) * n)
    vis = rad > 0
    assert int(vis.sum()) > 1000
    assert torch.equal(radii[s], rad) and torch.equal(clamped[s][vis], cl[vis])
    multi = torch.cat([xy[s], depth[s, None], conic[s], torch.ones(n, 1, device=DEV), opac[s, None], rgb[s], radii[s, None].view(torch.float32)], 1)
    names = [c for c in COLS if c != "comp"]
    keep = [i for i, c in enumerate(COLS) if c != "comp"]
    bad = _diff_report(multi[vis][:, keep], rows[vis][:, keep], names)
    assert not bad, f"camera {j}: multi-view arrays differ from the single-view rows: {bad}"


@SH_DEGREES
@pytest.mark.parametrize("aa", [True, False])
def test_multi_view_kernels_match_single_view_rows_bitwise(aa, storage_degree, sh_degree):
    from b200gs import ops
    from b200gs._lib import B200gsView, check, lib, ptr
    L = lib()
    n, W, H = 20000, 400, 304
    raw, views = _scene(n, 21, W, H, [0, 3, 4], sh_degree, storage_degree=storage_degree)
    nv = len(views)
    ol = raw["opacities"].reshape(-1).contiguous()
    single = [_single_rows(raw, v, aa) for v in views]

    # --- multi-view, separate arrays
    wn = nv * n
    xy, depth, conic = torch.empty(wn, 2, device=DEV), torch.empty(wn, device=DEV), torch.empty(wn, 3, device=DEV)
    rgb, opac = torch.empty(wn, 3, device=DEV), torch.empty(wn, device=DEV)
    radii = torch.empty(wn, dtype=torch.int32, device=DEV)
    clamped = torch.empty(wn, dtype=torch.uint8, device=DEV)
    arr = (B200gsView * nv)(*views)
    check(L.b200gs_project_fwd_raw_multi(arr, nv, n, ptr(raw["means"]), ptr(raw["scales"]), ptr(raw["rotations"]), ptr(ol), ptr(raw["shs_dc"]),
                                         ptr(raw["shs_rest"]), int(aa), ptr(xy), ptr(depth), ptr(radii), ptr(conic), ptr(rgb), ptr(clamped), ptr(opac),
                                         ops._stream()), "b200gs_project_fwd_raw_multi")
    for j in range(nv):
        _assert_camera_arrays_match_rows(j, n, xy, depth, conic, opac, rgb, radii, clamped, single[j])

    # --- multi-view fused with the packing (local destination blocks)
    cap = n
    dst = torch.zeros(nv * cap, 12, device=DEV)
    xy2 = torch.empty(wn, 2, device=DEV)
    radii2 = torch.empty(wn, dtype=torch.int32, device=DEV)
    clamped2 = torch.empty(wn, dtype=torch.uint8, device=DEV)
    row_index = torch.empty(wn, dtype=torch.int32, device=DEV)
    d_count = torch.zeros(nv, dtype=torch.int64, device=DEV)
    ws = torch.empty(int(L.b200gs_project_pack_workspace_bytes(nv, n)), dtype=torch.uint8, device=DEV)
    dst_arr = (ctypes.c_void_p * nv)(*[dst.data_ptr() + j * cap * 48 for j in range(nv)])
    check(L.b200gs_project_pack_multi(arr, nv, n, ptr(raw["means"]), ptr(raw["scales"]), ptr(raw["rotations"]), ptr(ol), ptr(raw["shs_dc"]),
                                      ptr(raw["shs_rest"]), int(aa), ptr(xy2), ptr(radii2), ptr(clamped2), ptr(row_index), dst_arr, cap, ptr(ws),
                                      ws.numel(), ptr(d_count), ops._stream()), "b200gs_project_pack_multi")
    torch.cuda.synchronize()
    for j in range(nv):
        rows, rad, cl = single[j]
        vis = rad > 0
        V = int(vis.sum())
        assert int(d_count[j]) == V
        s = slice(j * n, (j + 1) * n)
        assert torch.equal(radii2[s], rad) and torch.equal(clamped2[s][vis], cl[vis])
        assert torch.equal(xy2[s][vis].view(torch.int32), rows[vis][:, 0:2].contiguous().view(torch.int32))
        # rows in Gaussian-index order, block-relative numbering j*cap + k
        want_idx = torch.full((n,), -1, dtype=torch.int32, device=DEV)
        want_idx[vis] = (j * cap + torch.arange(V, device=DEV)).to(torch.int32)
        assert torch.equal(row_index[s], want_idx)
        packed = dst[j * cap:j * cap + V]
        bad = _diff_report(packed, rows[vis], COLS)
        assert not bad, f"camera {j}: packed rows differ from the single-view rows: {bad}"


def test_shard_projection_of_more_cameras_than_one_launch_matches_single_view_rows_bitwise():
    """distributed._project_shard with more cameras than one multi-view launch takes (B200GS_MAX_VIEWS): one launch per group of cameras,
    each writing at its offset into the camera-major arrays.  Every camera's slice must equal the single-view rows bit for bit."""
    from b200gs import distributed
    n, W, H = 20000, 400, 304
    raw, views = _scene(n, 21, W, H, list(range(0, 30, 3)))
    nv = len(views)
    assert nv > distributed.MAX_VIEWS
    st = distributed._ShardStep()
    st.views, st.n, st.world, st.sh_degree, st.aa = views, n, nv, 3, True
    distributed._project_shard(st, raw["means"], raw["scales"], raw["rotations"], raw["opacities"].reshape(-1).contiguous(), raw["shs_dc"],
                               raw["shs_rest"])
    for j in range(nv):
        _assert_camera_arrays_match_rows(j, n, st.xy, st.depth, st.conic, st.opac, st.rgb, st.radii, st.clamped, _single_rows(raw, views[j], True))


def test_compacted_and_blocked_rows_render_bit_identically():
    """What a rank of the sharded renderer rasterizes — the visible splats only, compacted in Gaussian-index order, possibly sitting in
    fixed-size blocks with stale rows behind the valid ones — must give the image of the full [n,12] row buffer bit for bit."""
    from b200gs import ops
    from b200gs._lib import MODE_GSPLAT
    n, W, H = 20000, 400, 304
    raw, views = _scene(n, 21, W, H, [3])
    bg = torch.tensor([0.2, 0.1, 0.4], device=DEV)
    rows, rad, _ = _single_rows(raw, views[0], True)
    vis = rad > 0
    V = int(vis.sum())
    _, (img_full, T_full, nc_full) = ops.bin_and_blend_rows(MODE_GSPLAT, W, H, rows, bg, True)
    compact = rows[vis].contiguous()
    _, (img_c, T_c, nc_c) = ops.bin_and_blend_rows(MODE_GSPLAT, W, H, compact, bg, True)
    assert torch.equal(T_c, T_full) and torch.equal(nc_c, nc_full), float((T_c - T_full).abs().max())
    assert torch.equal(img_c, img_full), float((img_c - img_full).abs().max())
    # two fixed-size blocks (as if two ranks had sent their halves), garbage behind the valid rows of each block
    half = int(vis[: n // 2].sum())
    cap = max(half, V - half) + 777
    blocks = torch.full((2 * cap, 12), float("nan"), device=DEV)
    blocks[:, 11] = torch.tensor([5], dtype=torch.int32, device=DEV).view(torch.float32)      # stale rows look visible (radius 5)
    blocks[:half] = compact[:half]
    blocks[cap:cap + V - half] = compact[half:]
    counts = torch.tensor([half, V - half], dtype=torch.int64, device=DEV)
    _, (img_b, T_b, nc_b) = ops.bin_and_blend_rows(MODE_GSPLAT, W, H, blocks, bg, True, False, counts, cap)
    assert torch.equal(T_b, T_full), float((T_b - T_full).abs().max())
    assert torch.equal(img_b, img_full), float((img_b - img_full).abs().max())


def _check_multi_view_backward_against_accumulated_single_view(storage_degree, sh_degree):
    from b200gs import ops
    from b200gs._lib import B200gsView, check, lib, ptr
    L = lib()
    n, W, H = 20000, 400, 304
    raw, views = _scene(n, 21, W, H, [0, 3, 4], sh_degree, storage_degree=storage_degree)
    nv = len(views)
    ol = raw["opacities"].reshape(-1).contiguous()
    single = [_single_rows(raw, v, True) for v in views]
    g = torch.Generator(device="cpu").manual_seed(5)
    v_rows = [(torch.randn(n, 12, generator=g) * 0.1).to(DEV) for _ in range(nv)]
    radii = torch.cat([s[1] for s in single]).contiguous()
    clamped = torch.cat([s[2] for s in single]).contiguous()
    row_index = torch.arange(n, dtype=torch.int32, device=DEV).repeat(nv).contiguous()

    def outs():
        return [torch.empty(n, 3, device=DEV), torch.empty(n, 3, device=DEV), torch.empty(n, 4, device=DEV), torch.empty(n, device=DEV),
                torch.empty_like(raw["shs_dc"]), torch.empty_like(raw["shs_rest"])]

    multi = outs()
    arr = (B200gsView * nv)(*views)
    srcs = (ctypes.c_void_p * nv)(*[t.data_ptr() for t in v_rows])
    check(L.b200gs_project_bwd_rows_multi(arr, nv, n, ptr(raw["means"]), ptr(raw["scales"]), ptr(raw["rotations"]), ptr(ol), ptr(raw["shs_dc"]),
                                          ptr(raw["shs_rest"]), 1, ptr(radii), ptr(clamped), ptr(row_index), srcs, *[ptr(t) for t in multi],
                                          ops._stream()), "b200gs_project_bwd_rows_multi")
    ref = outs()
    for j in range(nv):
        check(L.b200gs_project_bwd_rows(ctypes.byref(views[j]), n, ptr(raw["means"]), ptr(raw["scales"]), ptr(raw["rotations"]), ptr(ol),
                                        ptr(raw["shs_dc"]), ptr(raw["shs_rest"]), 1, ptr(single[j][1]), ptr(single[j][2]), None, ptr(v_rows[j]),
                                        1 if j > 0 else 0, *[ptr(t) for t in ref], None, 0, ops._stream()), "b200gs_project_bwd_rows")
    torch.cuda.synchronize()
    for name, a, b in zip(("means", "scales", "quats", "opacity", "shs_dc", "shs_rest"), multi, ref):
        assert bool(torch.isfinite(a).all())
        err = float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
        assert err < 2e-5, (name, err)


def test_multi_view_backward_matches_accumulated_single_view_backward():
    """K8 for all cameras in one launch (project_bwd_multi_kernel: gradients summed per Gaussian, SH-gradient rows accumulated in the shared-memory
    staging buffer) against the single-view K8 called once per camera with accumulate (b200gs_project_bwd_rows), same gradient rows."""
    _check_multi_view_backward_against_accumulated_single_view(3, 3)


@pytest.mark.parametrize(("storage_degree", "sh_degree"), [(4, 4), (4, 2)])
def test_multi_view_backward_matches_accumulated_single_view_backward_sh_stride_25(storage_degree, sh_degree):
    """The same with SH stored with stride 25: the multi-view K8 takes its MC = 25 instantiation for both active degrees.  At active degree 2
    the single-view K8 evaluates 16 coefficients and writes the wider rows per thread, where accumulate must add to them."""
    _check_multi_view_backward_against_accumulated_single_view(storage_degree, sh_degree)
