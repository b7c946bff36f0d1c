"""torch.autograd.Function wrappers over the C ABI (``libb200gs.so``).

PyTorch is used for device memory (its caching allocator owns every buffer, including workspaces), the current CUDA
stream and autograd bookkeeping only; all arithmetic of the hot path runs in the hand-written kernels.

Functions
  rasterize_vanilla(...)      the whole dgr-semantics pipeline as ONE autograd node (what
                              ``diff_gaussian_rasterization.GaussianRasterizer`` is; vanilla_renderer.py:111-120)
  project_gaussians(...)      gsplat v0 ``project_gaussians``          (gsplat_renderer.py:64-79)
  spherical_harmonics(...)    gsplat ``spherical_harmonics``           (gsplat_renderer.py:105)
  rasterize_gaussians(...)    gsplat v0 ``rasterize_gaussians``        (gsplat_renderer.py:86-99)
  spherical_harmonics_decomposed(...)  gsplat ``sh_decomposed``   (gsplat_v1_renderer.py:124)
  isect_keys / isect_offsets  gsplat v1 ``isect_tiles`` keys / ``isect_offset_encode``   (gsplat_v1_renderer.py:446,458)
  glossy_sh(...)              Glossy-Gaussian view-dependent opacity + SH colour   (glossy_renderer.py get_opacities / get_rgbs)
"""
import ctypes
import os
import threading
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import MODE_GSPLAT, MODE_VANILLA, TILE, B200gsView, check, lib, ptr

ROW_FLOATS = 12   # include/b200gs.h B200GS_ROW_FLOATS


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def _stream() -> int:
    """cudaStream_t of torch's current stream on the current device (raw handle; ~20x cheaper than current_stream())."""
    if _raw_stream is not None:
        return _raw_stream(torch.cuda.current_device())
    return torch.cuda.current_stream().cuda_stream


class StageTimer:
    """Optional per-stage CUDA-event timing on the launching stream (used by bench.py for the roofline numbers)."""

    def __init__(self):
        self.events = {}
        self.calls = {}

    class _Ctx:
        __slots__ = ("timer", "name", "start")

        def __init__(self, timer, name):
            self.timer, self.name = timer, name

        def __enter__(self):
            self.start = torch.cuda.Event(enable_timing=True)
            self.start.record()

        def __exit__(self, *exc):
            end = torch.cuda.Event(enable_timing=True)
            end.record()
            self.timer.events.setdefault(self.name, []).append((self.start, end))
            return False

    def stage(self, name):
        return StageTimer._Ctx(self, name)

    def reset(self):
        self.events.clear()

    def summary_ms(self):
        torch.cuda.synchronize()
        return {k: sum(a.elapsed_time(b) for a, b in v) / len(v) for k, v in self.events.items()}, {k: len(v) for k, v in self.events.items()}


class _Null:
    def __enter__(self):
        return None

    def __exit__(self, *exc):
        return False


_NULL = _Null()
_TIMER: Optional[StageTimer] = None


def set_stage_timer(timer: Optional[StageTimer]):
    global _TIMER
    _TIMER = timer


def _stage(name):
    return _NULL if _TIMER is None else _TIMER.stage(name)


def _f32c(t: torch.Tensor, name: str) -> torch.Tensor:
    if t.dtype != torch.float32:
        raise ValueError(f"{name} must be float32, got {t.dtype}")
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor (b200gs has no CPU path)")
    return t.contiguous()


def make_view(mode: int, width: int, height: int, *, fx: float = 0.0, fy: float = 0.0, cx: float = 0.0, cy: float = 0.0,
              tanfovx: float = 0.0, tanfovy: float = 0.0, viewmatrix=None, projmatrix=None, campos=None,
              sh_degree: int = 0, sh_stride: int = 1, scale_modifier: float = 1.0, eps2d: float = 0.3,
              near_plane: float = -1.0) -> B200gsView:
    """Pack a host-side B200gsView.  ``viewmatrix`` / ``projmatrix`` are the reference's transposed 4x4 tensors
    (Camera.world_to_camera / Camera.full_projection); they are copied to the host here (16 floats)."""
    v = B200gsView()
    v.width, v.height, v.mode = int(width), int(height), int(mode)
    v.sh_degree, v.sh_stride = int(sh_degree), int(sh_stride)
    v.fx, v.fy, v.cx, v.cy = float(fx), float(fy), float(cx), float(cy)
    v.tanfovx, v.tanfovy = float(tanfovx), float(tanfovy)
    v.scale_modifier, v.eps2d, v.near_plane = float(scale_modifier), float(eps2d), float(near_plane)
    if viewmatrix is not None:
        vm = viewmatrix.detach().to("cpu", torch.float32).reshape(-1).tolist()
        v.viewmatrix[:] = vm
    if projmatrix is not None:
        pm = projmatrix.detach().to("cpu", torch.float32).reshape(-1).tolist()
        v.projmatrix[:] = pm
    if campos is not None:
        cp = campos.detach().to("cpu", torch.float32).reshape(-1).tolist()
        v.campos[:] = cp
    return v


def _copy_view(v: B200gsView, **updates) -> B200gsView:
    out = B200gsView()
    ctypes.memmove(ctypes.byref(out), ctypes.byref(v), ctypes.sizeof(B200gsView))
    for k, val in updates.items():
        setattr(out, k, val)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# binning helper (no autograd)
# ----------------------------------------------------------------------------------------------------------------------
class Binning:
    """Result of K2-K5 for one view: depth-sorted per-tile Gaussian id lists.  `rect_pairs` = the reference's pair count
    (every tile of the 3-sigma rects; bounds `total`), `coarse_pairs` = (8x8-tile cell, Gaussian) pairs of the first
    binning level, `total` = number of listed pairs.  In lazy mode the counters arrive asynchronously: rect/coarse are
    None until resolve(), `total` waits for its own copy when first read (see bin_gaussians)."""
    __slots__ = ("sorted_ids", "tile_ranges", "rect_pairs", "coarse_pairs", "_total", "_pending", "_host", "_event_b")

    def __init__(self, sorted_ids, tile_ranges, total=None, host=None, pending=None, event_b=None):
        self.sorted_ids, self.tile_ranges, self._total = sorted_ids, tile_ranges, total
        self.rect_pairs = self.coarse_pairs = None
        self._host, self._pending, self._event_b = host, pending, event_b
        if host is not None and pending is None:
            self.rect_pairs, self.coarse_pairs = int(host[0]), int(host[1])

    @property
    def total(self):
        if self._total is None and self._host is not None:
            if self._event_b is not None:
                self._event_b.synchronize()
            self._total = int(self._host[6])
        return self._total

    def resolve(self) -> bool:
        """Lazy mode: wait for phase A's counters (the GPU is far past that point when this is called after the blend has
        been enqueued).  Returns False when a counter exceeds the capacity the lists were built with — pairs were
        dropped and the caller must re-bin in exact mode.  The check uses the RECT pair count, which bounds the listed
        pairs and is known right after phase A, so it never waits for the binning itself."""
        if self._pending is None:
            return True
        event_a, key, cap_coarse, cap_pairs = self._pending
        self._pending = None
        event_a.synchronize()
        self.rect_pairs, self.coarse_pairs = int(self._host[0]), int(self._host[1])
        with _state_lock:
            _last_total[key] = (self.coarse_pairs, self.rect_pairs)
        return self.coarse_pairs <= cap_coarse and self.rect_pairs <= cap_pairs

    def __del__(self):
        try:
            if self._host is not None:
                _return_host_counts(self._host)
        except Exception:      # interpreter shutdown
            pass


_host_counts_pool = []  # pinned int64[8] buffers: [0:4] phase A's copy of the counters, [4:8] phase B's
_last_total = {}       # key -> (coarse pairs, rect pairs) of the previous view: sizes the next view's buffers in lazy mode
_state_lock = threading.RLock()   # the two process-wide structures above are shared by every thread that renders (trainer + viewer threads)

TILE_CULLING = True    # exact (tile, splat) culling in K3; False reproduces the reference's full 3-sigma-rect pair list
LAZY_SLACK = 1.15      # lazy mode: capacity = slack x previous count


def _host_counts():
    with _state_lock:
        if _host_counts_pool:
            return _host_counts_pool.pop()
    return torch.zeros(8, dtype=torch.int64).pin_memory()


def _return_host_counts(buf):
    with _state_lock:
        if len(_host_counts_pool) < 32:
            _host_counts_pool.append(buf)


def _bin(key, mode, width, height, n, dev, cull, lazy, count_call) -> Binning:
    L = lib()
    st = _stream()
    gx, gy = (width + TILE - 1) // TILE, (height + TILE - 1) // TILE
    ws_a = torch.empty(L.b200gs_bin_count_workspace_bytes(n), dtype=torch.uint8, device=dev)
    d_counts = torch.empty(4, dtype=torch.int64, device=dev)
    ranges = torch.empty(gx * gy, 2, dtype=torch.int32, device=dev)
    host = _host_counts()
    with _state_lock:
        prev = _last_total.get(key) if lazy else None
    sync = prev is None
    with _stage("bin_count"):
        count_call(ptr(ws_a), ws_a.numel(), ptr(d_counts), host.data_ptr(), 1 if sync else 0, st)
    if sync:
        cap_coarse, cap_pairs = int(host[1]), int(host[0])    # exact / an upper bound: cannot overflow
        with _state_lock:
            _last_total[key] = (cap_coarse, cap_pairs)
        pending = None
    else:
        event_a = torch.cuda.Event()
        event_a.record()
        cap_coarse = int(prev[0] * LAZY_SLACK) + 4096
        cap_pairs = int(prev[1] * LAZY_SLACK) + 4096
        pending = (event_a, key, cap_coarse, cap_pairs)
    sorted_ids = torch.empty(max(cap_pairs, 1), dtype=torch.int32, device=dev)
    ws_b = torch.empty(L.b200gs_bin_sort_workspace_bytes(n, cap_coarse, width, height), dtype=torch.uint8, device=dev)
    with _stage("bin_sort"):
        check(L.b200gs_bin_sort(mode, width, height, n, 1 if cull else 0, cap_coarse, cap_pairs, ptr(d_counts), ptr(ws_a), ptr(ws_b),
                                ws_b.numel(), ptr(sorted_ids), ptr(ranges), host.data_ptr() + 32, 1 if sync else 0, st), "b200gs_bin_sort")
    if sync:
        return Binning(sorted_ids, ranges, int(host[6]), host)
    event_b = torch.cuda.Event()
    event_b.record()
    return Binning(sorted_ids, ranges, None, host, pending, event_b)


def bin_gaussians(mode: int, width: int, height: int, xy: torch.Tensor, depth: torch.Tensor, radii: torch.Tensor,
                  conic: Optional[torch.Tensor] = None, opacity: Optional[torch.Tensor] = None, lazy: bool = False) -> Binning:
    """K2-K5.  Passing conic+opacity enables exact tile culling (see include/b200gs.h).

    lazy=False: the counters are read back synchronously (host syncs, like the reference backends) and the buffers can
    never overflow.  lazy=True: buffers are sized from the previous view's counts (x LAZY_SLACK), nothing blocks here;
    call Binning.resolve() once the rest of the forward is enqueued — it returns False in the rare case a capacity was
    exceeded and the forward has to be redone with lazy=False."""
    L = lib()
    if not TILE_CULLING or conic is None or opacity is None:
        conic = opacity = None
    n = xy.shape[0]

    def count_call(ws_a, ws_a_bytes, d_counts, host, sync, st):
        check(L.b200gs_bin_count(mode, width, height, n, ptr(xy), ptr(depth), ptr(radii), ptr(conic), ptr(opacity), ws_a, ws_a_bytes,
                                 d_counts, host, sync, st), "b200gs_bin_count")

    cull = conic is not None
    return _bin((mode, width, height, n, cull), mode, width, height, n, xy.device, cull, lazy, count_call)


def bin_rows(mode: int, width: int, height: int, rows: torch.Tensor, cull: bool = True, lazy: bool = False, block_counts=None,
             block_rows: int = 0) -> Binning:
    """K2-K5 on a [n,12] splat-row buffer read in place (b200gs_bin_count_rows); same lazy protocol as bin_gaussians.
    block_counts (int64 device tensor) / block_rows: the rows come in fixed-size blocks of which only the first block_counts[b] rows
    are valid (the sharded exchange)."""
    L = lib()
    n = rows.shape[0]

    def count_call(ws_a, ws_a_bytes, d_counts, host, sync, st):
        check(L.b200gs_bin_count_rows(mode, width, height, n, ptr(rows), int(cull), ws_a, ws_a_bytes, d_counts, host, sync, st,
                                      ptr(block_counts), int(block_rows) if block_counts is not None else 0), "b200gs_bin_count_rows")

    return _bin(("rows", mode, width, height, bool(cull)), mode, width, height, n, rows.device, bool(cull), lazy, count_call)


def blend_forward_rows(mode, width, height, binning: Binning, rows, bg, planar=False):
    """K6 on rows -> image [H,W,3] (planar: [3,H,W]), final_T, n_contrib."""
    L = lib()
    dev = rows.device
    image = torch.empty((3, height, width) if planar else (height, width, 3), dtype=torch.float32, device=dev)
    final_T = torch.empty(height, width, dtype=torch.float32, device=dev)
    n_contrib = torch.empty(height, width, dtype=torch.int32, device=dev)
    pix_stride, ch_stride = (1, height * width) if planar else (3, 1)
    with _stage("blend_fwd"):
        check(L.b200gs_blend_fwd_rows(mode, width, height, ptr(binning.tile_ranges), ptr(binning.sorted_ids), ptr(rows), ptr(bg), ptr(image),
                                      pix_stride, ch_stride, ptr(final_T), ptr(n_contrib), None, _stream()), "b200gs_blend_fwd_rows")
    return image, final_T, n_contrib


def _bin_then_blend(bin_fn, blend_fn):
    """The lazy (sync-free) binning protocol: bin_fn(lazy=True) sizes the lists from the previous view's counts, blend_fn(binning)
    is enqueued, and only then are the counts checked; in the rare case a capacity was exceeded both are redone exactly."""
    binning = bin_fn(True)
    out = blend_fn(binning)
    if not binning.resolve():
        binning = bin_fn(False)
        out = blend_fn(binning)
    return binning, out


def bin_and_blend_rows(mode, width, height, rows, bg, cull=True, planar=False, block_counts=None, block_rows=0):
    return _bin_then_blend(lambda lazy: bin_rows(mode, width, height, rows, cull, lazy=lazy, block_counts=block_counts, block_rows=block_rows),
                           lambda binning: blend_forward_rows(mode, width, height, binning, rows, bg, planar))


# ----------------------------------------------------------------------------------------------------------------------
# raw stage calls (no autograd) — also used directly by tests
# ----------------------------------------------------------------------------------------------------------------------
def project_forward(view: B200gsView, means, scales, quats, shs=None, want_comp=False, want_cov3d=False):
    L = lib()
    n = means.shape[0]
    dev = means.device
    xy = torch.empty(n, 2, dtype=torch.float32, device=dev)
    depth = torch.empty(n, dtype=torch.float32, device=dev)
    radii = torch.empty(n, dtype=torch.int32, device=dev)
    conic = torch.empty(n, 3, dtype=torch.float32, device=dev)
    tiles = torch.empty(n, dtype=torch.int32, device=dev)
    comp = torch.empty(n, dtype=torch.float32, device=dev) if want_comp else None
    cov3d = torch.empty(n, 6, dtype=torch.float32, device=dev) if want_cov3d else None
    rgb = clamped = None
    if shs is not None:
        rgb = torch.empty(n, 3, dtype=torch.float32, device=dev)
        clamped = torch.empty(n, dtype=torch.uint8, device=dev)
    with _stage("project_fwd"):
        check(L.b200gs_project_fwd(ctypes.byref(view), n, ptr(means), ptr(scales), ptr(quats), ptr(shs), ptr(xy), ptr(depth),
                                   ptr(radii), ptr(conic), ptr(comp), ptr(tiles), ptr(cov3d), ptr(rgb), ptr(clamped), _stream()),
              "b200gs_project_fwd")
    return xy, depth, radii, conic, comp, tiles, cov3d, rgb, clamped


def project_backward(view: B200gsView, means, scales, quats, shs, radii, clamped, v_xy, v_depth, v_conic, v_comp, v_rgb):
    L = lib()
    n = means.shape[0]
    dev = means.device
    v_means = torch.empty(n, 3, dtype=torch.float32, device=dev)
    v_scales = torch.empty(n, 3, dtype=torch.float32, device=dev)
    v_quats = torch.empty(n, 4, dtype=torch.float32, device=dev)
    v_shs = torch.empty_like(shs) if shs is not None else None
    with _stage("project_bwd"):
        check(L.b200gs_project_bwd(ctypes.byref(view), n, ptr(means), ptr(scales), ptr(quats), ptr(shs), ptr(radii), ptr(clamped),
                                   ptr(v_xy), ptr(v_depth), ptr(v_conic), ptr(v_comp), ptr(v_rgb), ptr(v_means), ptr(v_scales),
                                   ptr(v_quats), ptr(v_shs), _stream()), "b200gs_project_bwd")
    return v_means, v_scales, v_quats, v_shs


def blend_forward(mode, width, height, binning: Binning, xy, conic, opacity, colors, bg, planar: bool, want_alpha: bool, hit_any=None):
    """planar=True -> image [C,H,W] (vanilla); else [H,W,C] (gsplat).  hit_any: zero-filled uint8 [N] that receives 1 for every splat
    that contributed to a pixel."""
    L = lib()
    ch = colors.shape[1]
    dev = xy.device
    if planar:
        image = torch.empty(ch, height, width, dtype=torch.float32, device=dev)
        ps, cs = 1, height * width
    else:
        image = torch.empty(height, width, ch, dtype=torch.float32, device=dev)
        ps, cs = ch, 1
    final_T = torch.empty(height, width, dtype=torch.float32, device=dev)
    n_contrib = torch.empty(height, width, dtype=torch.int32, device=dev)
    alpha = torch.empty(height, width, dtype=torch.float32, device=dev) if want_alpha else None
    with _stage("blend_fwd"):
        check(L.b200gs_blend_fwd(mode, width, height, ch, ptr(binning.tile_ranges), ptr(binning.sorted_ids), ptr(xy), ptr(conic),
                                 ptr(opacity), ptr(colors), ptr(bg), ptr(image), ps, cs, ptr(final_T), ptr(n_contrib), ptr(alpha),
                                 ptr(hit_any), _stream()), "b200gs_blend_fwd")
    return image, final_T, n_contrib, alpha


def blend_backward(mode, width, height, binning: Binning, xy, conic, opacity, colors, bg, final_T, n_contrib, v_image, v_alpha,
                   planar: bool, xy_scale=(1.0, 1.0), want_abs: bool = False):
    L = lib()
    n, ch = colors.shape
    dev = xy.device
    # one zero-filled slab for all atomically accumulated outputs
    width_cols = 2 + 3 + 1 + ch + (2 if want_abs else 0)
    slab = torch.zeros(n * width_cols, dtype=torch.float32, device=dev)
    o = 0
    v_xy = slab[o:o + 2 * n].view(n, 2); o += 2 * n
    v_conic = slab[o:o + 3 * n].view(n, 3); o += 3 * n
    v_opacity = slab[o:o + n]; o += n
    v_colors = slab[o:o + ch * n].view(n, ch); o += ch * n
    v_abs = slab[o:o + 2 * n].view(n, 2) if want_abs else None
    ps, cs = (1, height * width) if planar else (ch, 1)
    with _stage("blend_bwd"):
        check(L.b200gs_blend_bwd(mode, width, height, ch, ptr(binning.tile_ranges), ptr(binning.sorted_ids), ptr(xy), ptr(conic),
                                 ptr(opacity), ptr(colors), ptr(bg), ptr(final_T), ptr(n_contrib), ptr(v_image), ps, cs,
                                 ptr(v_alpha), float(xy_scale[0]), float(xy_scale[1]), ptr(v_xy), ptr(v_conic), ptr(v_opacity),
                                 ptr(v_colors), ptr(v_abs), _stream()), "b200gs_blend_bwd")
    return v_xy, v_conic, v_opacity, v_colors, v_abs


def blend_features_forward(width, height, binning: Binning, xy, conic, opacity, features, bg):
    """Gsplat-mode blend of [N, D] features, any D >= 1 (b200gs_blend_feat_fwd: chunks of 32 channels over one binning)
    -> image [H,W,D], final_T, n_contrib, alpha."""
    L = lib()
    d = features.shape[1]
    dev = xy.device
    image = torch.empty(height, width, d, dtype=torch.float32, device=dev)
    final_T = torch.empty(height, width, dtype=torch.float32, device=dev)
    n_contrib = torch.empty(height, width, dtype=torch.int32, device=dev)
    alpha = torch.empty(height, width, dtype=torch.float32, device=dev)
    with _stage("blend_feat_fwd"):
        check(L.b200gs_blend_feat_fwd(width, height, d, ptr(binning.tile_ranges), ptr(binning.sorted_ids), ptr(xy), ptr(conic), ptr(opacity),
                                      ptr(features), ptr(bg), ptr(image), ptr(final_T), ptr(n_contrib), ptr(alpha), _stream()),
              "b200gs_blend_feat_fwd")
    return image, final_T, n_contrib, alpha


def blend_features_backward(width, height, binning: Binning, xy, conic, opacity, features, bg, final_T, n_contrib, v_image, v_alpha,
                            geometry: bool = True, want_abs: bool = False):
    """Backward of blend_features_forward -> (v_xy, v_conic, v_opacity, v_features, v_abs).  geometry=False runs the features-only
    kernels: v_xy / v_conic / v_opacity / v_abs are None and no geometry gradient is computed."""
    L = lib()
    n, d = features.shape
    dev = xy.device
    cols = d + ((2 + 3 + 1 + (2 if want_abs else 0)) if geometry else 0)
    slab = torch.zeros(n * cols, dtype=torch.float32, device=dev)     # one zero-filled slab for all atomically accumulated outputs
    v_feat = slab[:n * d].view(n, d)
    v_xy = v_conic = v_opacity = v_abs = None
    if geometry:
        o = n * d
        v_xy = slab[o:o + 2 * n].view(n, 2); o += 2 * n
        v_conic = slab[o:o + 3 * n].view(n, 3); o += 3 * n
        v_opacity = slab[o:o + n]; o += n
        v_abs = slab[o:o + 2 * n].view(n, 2) if want_abs else None
    with _stage("blend_feat_bwd"):
        check(L.b200gs_blend_feat_bwd(width, height, d, ptr(binning.tile_ranges), ptr(binning.sorted_ids), ptr(xy), ptr(conic), ptr(opacity),
                                      ptr(features), ptr(bg), ptr(final_T), ptr(n_contrib), ptr(v_image), ptr(v_alpha), ptr(v_feat), ptr(v_xy),
                                      ptr(v_conic), ptr(v_opacity), ptr(v_abs), _stream()), "b200gs_blend_feat_bwd")
    return v_xy, v_conic, v_opacity, v_feat, v_abs


# ----------------------------------------------------------------------------------------------------------------------
# vanilla: one autograd node for the whole pipeline (diff_gaussian_rasterization semantics)
# ----------------------------------------------------------------------------------------------------------------------
class _RasterizeVanilla(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, shs, colors_precomp, opacities, scales, rotations, bg, view: B200gsView):
        n = means3D.shape[0]
        means3D = _f32c(means3D, "means3D")
        scales = _f32c(scales, "scales")
        rotations = _f32c(rotations, "rotations")
        opac = _f32c(opacities, "opacities").reshape(-1)
        bg = _f32c(bg, "bg")
        use_sh = shs is not None
        if use_sh:
            shs = _f32c(shs, "shs")
            view = _copy_view(view, sh_stride=int(shs.shape[1]))
        else:
            colors_precomp = _f32c(colors_precomp, "colors_precomp")
        W, H = view.width, view.height
        xy, depth, radii, conic, _, tiles, _, rgb, clamped = project_forward(view, means3D, scales, rotations, shs if use_sh else None)
        colors = rgb if use_sh else colors_precomp
        binning, (image, final_T, n_contrib, _) = _bin_then_blend(
            lambda lazy: bin_gaussians(MODE_VANILLA, W, H, xy, depth, radii, conic, opac, lazy=lazy),
            lambda binning: blend_forward(MODE_VANILLA, W, H, binning, xy, conic, opac, colors, bg, True, False))
        ctx.view = view
        ctx.use_sh = use_sh
        ctx.binning = binning
        ctx.means2D_shape = tuple(means2D.shape)
        ctx.opac_shape = tuple(opacities.shape)
        ctx.save_for_backward(means3D, scales, rotations, shs if use_sh else colors_precomp, opac, bg, xy, conic, radii,
                              clamped if use_sh else None, rgb if use_sh else None, final_T, n_contrib)
        ctx.mark_non_differentiable(radii)
        return image, radii

    @staticmethod
    def backward(ctx, v_image, _v_radii):
        means3D, scales, rotations, sh_or_col, opac, bg, xy, conic, radii, clamped, rgb, final_T, n_contrib = ctx.saved_tensors
        view = ctx.view
        W, H = view.width, view.height
        use_sh = ctx.use_sh
        colors = rgb if use_sh else sh_or_col
        v_image = _f32c(v_image, "grad_image")
        # dgr stores dL/dmean2D in NDC-scaled units: pixel gradient x (0.5 W, 0.5 H)
        v_xy, v_conic, v_opacity, v_colors, _ = blend_backward(MODE_VANILLA, W, H, ctx.binning, xy, conic, opac, colors, bg,
                                                              final_T, n_contrib, v_image, None, True, (0.5 * W, 0.5 * H))
        v_means, v_scales, v_quats, v_shs = project_backward(view, means3D, scales, rotations, sh_or_col if use_sh else None,
                                                             radii, clamped, v_xy, None, v_conic, None, v_colors if use_sh else None)
        n = means3D.shape[0]
        v_means2D = torch.zeros(ctx.means2D_shape, dtype=torch.float32, device=means3D.device)
        v_means2D[:, :2] = v_xy
        return (v_means, v_means2D, v_shs if use_sh else None, None if use_sh else v_colors, v_opacity.reshape(ctx.opac_shape),
                v_scales, v_quats, None, None)


def rasterize_vanilla(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, bg, view: B200gsView):
    """-> (color [3,H,W], radii int32 [N]).  Exactly one of shs / colors_precomp."""
    if (shs is None) == (colors_precomp is None):
        raise ValueError("Please provide exactly one of either SHs or precomputed colors!")
    if scales is None or rotations is None:
        raise NotImplementedError("cov3D_precomp is not supported by b200gs; pass scales and rotations")
    return _RasterizeVanilla.apply(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, bg, view)


# ----------------------------------------------------------------------------------------------------------------------
# activations fused: the renderer step fed with the model's RAW parameter tensors (b200gs_project_*_rows)
# ----------------------------------------------------------------------------------------------------------------------
class _RasterizeRaw(torch.autograd.Function):
    """The whole renderer step as ONE autograd node on the model's RAW parameters, either constant set: K1 (activations + SH fused)
    writes one [N,12] row per Gaussian, K2-K6 read the rows in place; backward: K7 accumulates [N,12] gradient rows (128-bit
    reductions), K8 reads them in place.  `means2D` is the viewspace-points tensor of the renderer contract ([N,3] zeros in vanilla
    mode, [N,2] in gsplat mode where it is also filled with the projected means): its `.grad` receives d loss / d mean2D."""

    @staticmethod
    def forward(ctx, mode, means3D, means2D, shs_dc, shs_rest, opacity_logits, log_scales, raw_quats, bg, view: B200gsView, anti_aliased):
        means3D = _f32c(means3D, "means3D")
        log_scales = _f32c(log_scales, "scales")
        raw_quats = _f32c(raw_quats, "rotations")
        ol = _f32c(opacity_logits, "opacities").reshape(-1)
        shs_dc = _f32c(shs_dc, "shs_dc")
        shs_rest = _f32c(shs_rest, "shs_rest")
        bg = _f32c(bg, "bg")
        view = _copy_view(view, sh_stride=int(shs_dc.shape[1] + shs_rest.shape[1]))
        W, H = view.width, view.height
        n, dev = means3D.shape[0], means3D.device
        rows = torch.empty(n, ROW_FLOATS, dtype=torch.float32, device=dev)
        radii = torch.empty(n, dtype=torch.int32, device=dev)
        clamped = torch.empty(n, dtype=torch.uint8, device=dev)
        with _stage("project_fwd"):
            check(lib().b200gs_project_fwd_rows(ctypes.byref(view), n, ptr(means3D), ptr(log_scales), ptr(raw_quats), ptr(ol), ptr(shs_dc),
                                                ptr(shs_rest), int(bool(anti_aliased)), ptr(rows), ptr(radii), ptr(clamped), None, _stream()),
                  "b200gs_project_fwd_rows")
        binning, (image, final_T, n_contrib) = bin_and_blend_rows(mode, W, H, rows, bg, True, mode == MODE_VANILLA)
        if mode == MODE_GSPLAT:
            means2D.detach()[:, :2].copy_(rows[:, 0:2])     # the gsplat renderers hand the projected means out as `viewspace_points`
        ctx.view, ctx.mode, ctx.aa = view, mode, bool(anti_aliased)
        ctx.binning = binning
        ctx.means2D_shape = tuple(means2D.shape)
        ctx.opac_shape = tuple(opacity_logits.shape)
        ctx.save_for_backward(means3D, log_scales, raw_quats, ol, shs_dc, shs_rest, bg, rows, radii, clamped, final_T, n_contrib)
        ctx.mark_non_differentiable(radii)
        return image, radii

    @staticmethod
    def backward(ctx, v_image, _v_radii):
        means3D, log_scales, raw_quats, ol, shs_dc, shs_rest, bg, rows, radii, clamped, final_T, n_contrib = ctx.saved_tensors
        view, mode = ctx.view, ctx.mode
        W, H = view.width, view.height
        v_image = _f32c(v_image, "grad_image")
        n = means3D.shape[0]
        dev = means3D.device
        v_rows = torch.zeros(n, ROW_FLOATS, dtype=torch.float32, device=dev)
        L = lib()
        if mode == MODE_VANILLA:      # [3,H,W] image, mean2D gradient in NDC units (the vanilla rasterizer's convention)
            pix_stride, ch_stride, gsx, gsy = 1, H * W, 0.5 * W, 0.5 * H
        else:                         # [H,W,3] image, mean2D gradient in pixels
            pix_stride, ch_stride, gsx, gsy = 3, 1, 1.0, 1.0
        with _stage("blend_bwd"):
            check(L.b200gs_blend_bwd_rows(mode, W, H, ptr(ctx.binning.tile_ranges), ptr(ctx.binning.sorted_ids), ptr(rows), ptr(bg), ptr(final_T),
                                          ptr(n_contrib), ptr(v_image), pix_stride, ch_stride, None, gsx, gsy, ptr(v_rows), _stream()),
                  "b200gs_blend_bwd_rows")
        v_means = torch.empty(n, 3, dtype=torch.float32, device=dev)
        v_ls = torch.empty(n, 3, dtype=torch.float32, device=dev)
        v_q = torch.empty(n, 4, dtype=torch.float32, device=dev)
        v_ol = torch.empty(n, dtype=torch.float32, device=dev)
        v_dc, v_rest = torch.empty_like(shs_dc), torch.empty_like(shs_rest)
        # d loss / d mean2D (`viewspace_points.grad`): K8 writes it while it has the gradient row in registers
        cols = int(ctx.means2D_shape[1])
        v_means2D = torch.empty(n, cols, dtype=torch.float32, device=dev) if (ctx.needs_input_grad[2] and cols in (2, 3)) else None
        with _stage("project_bwd"):
            check(L.b200gs_project_bwd_rows(ctypes.byref(view), n, ptr(means3D), ptr(log_scales), ptr(raw_quats), ptr(ol), ptr(shs_dc), ptr(shs_rest),
                                            int(ctx.aa), ptr(radii), ptr(clamped), None, ptr(v_rows), 0, ptr(v_means), ptr(v_ls), ptr(v_q), ptr(v_ol),
                                            ptr(v_dc), ptr(v_rest), ptr(v_means2D), cols if v_means2D is not None else 0, _stream()),
                  "b200gs_project_bwd_rows")
        if v_means2D is None and ctx.needs_input_grad[2]:
            v_means2D = torch.zeros(ctx.means2D_shape, dtype=torch.float32, device=dev)
            v_means2D[:, :2] = v_rows[:, 0:2]
        return None, v_means, v_means2D, v_dc, v_rest, v_ol.reshape(ctx.opac_shape), v_ls, v_q, None, None, None


def rasterize_vanilla_raw(means3D, means2D, shs_dc, shs_rest, opacity_logits, log_scales, raw_quats, bg, view: B200gsView):
    """Fused-activation variant of rasterize_vanilla: inputs are the model's RAW parameters
    (means, shs_dc [N,1,3], shs_rest [N,K-1,3], opacity logits, log-scales, un-normalised quaternions)."""
    return _RasterizeRaw.apply(MODE_VANILLA, means3D, means2D, shs_dc, shs_rest, opacity_logits, log_scales, raw_quats, bg, view, False)


def rasterize_gsplat_raw(means3D, means2D, shs_dc, shs_rest, opacity_logits, log_scales, raw_quats, bg, view: B200gsView, anti_aliased=True):
    """The gsplat-semantics counterpart: -> ([H,W,3] image, radii); `means2D` [N,2] receives the projected means (values) and
    d loss / d mean2D in pixels (`.grad`)."""
    return _RasterizeRaw.apply(MODE_GSPLAT, means3D, means2D, shs_dc, shs_rest, opacity_logits, log_scales, raw_quats, bg, view, anti_aliased)


# ----------------------------------------------------------------------------------------------------------------------
# gsplat v0 surface
# ----------------------------------------------------------------------------------------------------------------------
class _ProjectGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3d, scales, quats, view: B200gsView):
        means3d = _f32c(means3d, "means3d")
        scales = _f32c(scales, "scales")
        quats = _f32c(quats, "quats")
        xy, depth, radii, conic, comp, tiles, cov3d, _, _ = project_forward(view, means3d, scales, quats, None, True, True)
        ctx.view = view
        ctx.save_for_backward(means3d, scales, quats, radii)
        ctx.mark_non_differentiable(radii, tiles, cov3d)
        return xy, depth, radii, conic, comp, tiles, cov3d

    @staticmethod
    def backward(ctx, v_xy, v_depth, _v_radii, v_conic, v_comp, _v_tiles, _v_cov3d):
        means3d, scales, quats, radii = ctx.saved_tensors
        n = means3d.shape[0]
        dev = means3d.device

        def z(t, shape):
            return torch.zeros(shape, dtype=torch.float32, device=dev) if t is None else _f32c(t, "grad")

        v_means, v_scales, v_quats, _ = project_backward(ctx.view, means3d, scales, quats, None, radii, None, z(v_xy, (n, 2)),
                                                         z(v_depth, (n,)), z(v_conic, (n, 3)), z(v_comp, (n,)), None)
        return v_means, v_scales, v_quats, None


def project_gaussians(means3d, scales, glob_scale, quats, viewmat, fx, fy, cx, cy, img_height, img_width, block_width=16,
                      clip_thresh=0.01, filter_2d_kernel_size=0.3, view: Optional[B200gsView] = None):
    """gsplat v0 ``project_gaussians``: -> (xys [N,2], depths [N], radii int32 [N], conics [N,3], compensation [N],
    num_tiles_hit int32 [N], cov3d [N,6]).  ``viewmat`` is the standard [3|4,4] world-to-camera (rows R|t), i.e.
    ``camera.world_to_camera.T[:3,:]`` as the reference passes it (gsplat_renderer.py:69)."""
    if block_width != TILE:
        raise ValueError(f"b200gs supports block_width {TILE} only (the reference default, gsplat_renderer.py:7)")
    if view is None:
        vm = torch.eye(4, dtype=torch.float32)
        vm[:viewmat.shape[0], :] = viewmat.detach().to("cpu", torch.float32)
        view = make_view(MODE_GSPLAT, img_width, img_height, fx=fx, fy=fy, cx=cx, cy=cy, viewmatrix=vm.T.contiguous(),
                         scale_modifier=glob_scale, eps2d=filter_2d_kernel_size, near_plane=clip_thresh)
    return _ProjectGaussians.apply(means3d, scales, quats, view)


class _SphericalHarmonics(torch.autograd.Function):
    @staticmethod
    def forward(ctx, degree: int, dirs, coeffs):
        dirs = _f32c(dirs, "dirs")
        coeffs = _f32c(coeffs, "coeffs")
        n, k = coeffs.shape[0], coeffs.shape[1]
        rgb = torch.empty(n, 3, dtype=torch.float32, device=coeffs.device)
        check(lib().b200gs_sh_fwd(int(degree), k, n, ptr(dirs), ptr(coeffs), ptr(rgb), _stream()), "b200gs_sh_fwd")
        ctx.degree = int(degree)
        ctx.save_for_backward(dirs, coeffs)
        return rgb

    @staticmethod
    def backward(ctx, v_rgb):
        dirs, coeffs = ctx.saved_tensors
        n, k = coeffs.shape[0], coeffs.shape[1]
        v_rgb = _f32c(v_rgb, "grad")
        v_coeffs = torch.empty_like(coeffs)
        v_dirs = torch.empty_like(dirs) if ctx.needs_input_grad[1] else None
        check(lib().b200gs_sh_bwd(ctx.degree, k, n, ptr(dirs), ptr(coeffs), ptr(v_rgb), ptr(v_coeffs), ptr(v_dirs), _stream()),
              "b200gs_sh_bwd")
        return None, v_dirs, v_coeffs


def spherical_harmonics(degrees_to_use: int, dirs: torch.Tensor, coeffs: torch.Tensor, masks: Optional[torch.Tensor] = None) -> torch.Tensor:
    """gsplat ``spherical_harmonics(deg, dirs[N,3], coeffs[N,K,3], masks=None) -> [N,3]`` (directions normalised inside).  `masks`
    (gsplat skips the masked-out rows) is accepted for call compatibility; every row is evaluated, the caller only reads the visible ones."""
    if coeffs.shape[-1] != 3 or coeffs.dim() != 3:
        raise ValueError("coeffs must be [N, K, 3]")
    return _SphericalHarmonics.apply(degrees_to_use, dirs, coeffs)


class _SphericalHarmonicsSplit(torch.autograd.Function):
    @staticmethod
    def forward(ctx, degree: int, dirs, dc, rest, mask):
        dirs, dc, rest = _f32c(dirs, "dirs"), _f32c(dc, "dc"), _f32c(rest, "coeffs")
        n, k_rest = dc.shape[0], rest.shape[1]
        rgb = torch.empty(n, 3, dtype=torch.float32, device=dc.device)
        check(lib().b200gs_sh_split_fwd(int(degree), k_rest, n, ptr(dirs), ptr(dc), ptr(rest), ptr(mask), ptr(rgb), _stream()),
              "b200gs_sh_split_fwd")
        ctx.degree = int(degree)
        ctx.save_for_backward(dirs, dc, rest, mask)
        return rgb

    @staticmethod
    def backward(ctx, v_rgb):
        dirs, dc, rest, mask = ctx.saved_tensors
        n, k_rest = dc.shape[0], rest.shape[1]
        v_rgb = _f32c(v_rgb, "grad")
        v_dc, v_rest = torch.empty_like(dc), torch.empty_like(rest)
        v_dirs = torch.empty_like(dirs) if ctx.needs_input_grad[1] else None
        check(lib().b200gs_sh_split_bwd(ctx.degree, k_rest, n, ptr(dirs), ptr(dc), ptr(rest), ptr(mask), ptr(v_rgb), ptr(v_dc), ptr(v_rest),
                                        ptr(v_dirs), _stream()), "b200gs_sh_split_bwd")
        return None, v_dirs, v_dc, v_rest, None


def spherical_harmonics_decomposed(degrees_to_use: int, dirs: torch.Tensor, dc: torch.Tensor, coeffs: torch.Tensor,
                                   masks: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``spherical_harmonics_decomposed(deg, dirs[N,3], dc[N,1,3], coeffs[N,K-1,3], masks[N]=None) -> [N,3]`` of yzslab's gsplat fork:
    SH on dc | rest read in place (no concatenation).  Rows with masks[i] false read no coefficient and get rgb = 0 and zero
    gradients; the other rows are bit-identical to spherical_harmonics on torch.cat((dc, coeffs), 1)."""
    n = dc.shape[0]
    if dc.shape != (n, 1, 3) or coeffs.dim() != 3 or coeffs.shape[0] != n or coeffs.shape[2] != 3 or dirs.shape != (n, 3):
        raise ValueError("expected dirs [N,3], dc [N,1,3] and coeffs [N,K-1,3]")
    mask = None
    if masks is not None:
        if masks.shape != (n,) or masks.device != dc.device:
            raise ValueError("masks must be [N] on the device of the coefficients")
        mask = (masks if masks.dtype == torch.bool else masks != 0).contiguous().view(torch.uint8)
    return _SphericalHarmonicsSplit.apply(degrees_to_use, dirs, dc, coeffs, mask)


# ---- Glossy-Gaussian view-dependent opacity and colour (csrc/glossy.cu) -------------------------------------------------------
GLOSSY_FWD_LAUNCHES = 1     # K47
GLOSSY_BWD_LAUNCHES = 1     # K48


def _f32_in_place(t: torch.Tensor, name: str) -> torch.Tensor:
    """A float32 CUDA tensor the kernels read in place: refused, never copied, when it is not contiguous."""
    _f32c(t, name)
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous (read in place)")
    return t


class _GlossySH(torch.autograd.Function):
    @staticmethod
    def forward(ctx, degree, split, mask, means, campos, op_dc, op_rest, shs, shs_rest):
        n, dev = means.shape[0], means.device
        colour = shs is not None
        stride = (shs.shape[1] + (shs_rest.shape[1] if split else 0)) if colour else 0
        opacity = torch.empty(n, dtype=torch.float32, device=dev)
        rgb = torch.empty(n, 3, dtype=torch.float32, device=dev) if colour else None
        clamped = torch.empty(n, dtype=torch.uint8, device=dev)
        check(lib().b200gs_glossy_sh_fwd(degree, n, ptr(means), ptr(campos), ptr(op_dc), ptr(op_rest), op_rest.shape[1], ptr(shs),
                                         ptr(shs_rest), stride, int(split), ptr(mask), ptr(opacity), ptr(rgb), ptr(clamped), _stream()),
              "b200gs_glossy_sh_fwd")
        ctx.degree, ctx.split, ctx.stride, ctx.colour = degree, split, stride, colour
        ctx.shapes = (op_dc.shape, op_rest.shape, shs.shape if colour else None, shs_rest.shape if colour and split else None)
        ctx.save_for_backward(means, campos, clamped)
        return rgb, opacity

    @staticmethod
    def backward(ctx, v_rgb, v_opacity):
        means, campos, clamped = ctx.saved_tensors
        n, dev = means.shape[0], means.device
        dc_shape, rest_shape, shs_shape, shs_rest_shape = ctx.shapes
        v_opacity = _f32c(v_opacity, "grad") if v_opacity is not None else torch.zeros(n, dtype=torch.float32, device=dev)
        colour = ctx.colour and v_rgb is not None
        v_rgb = _f32c(v_rgb, "grad") if colour else None
        v_op_dc = torch.empty(dc_shape, dtype=torch.float32, device=dev)
        v_op_rest = torch.empty(rest_shape, dtype=torch.float32, device=dev)
        v_shs = torch.empty(shs_shape, dtype=torch.float32, device=dev) if colour else None
        v_shs_rest = torch.empty(shs_rest_shape, dtype=torch.float32, device=dev) if colour and ctx.split else None
        check(lib().b200gs_glossy_sh_bwd(ctx.degree, n, ptr(means), ptr(campos), rest_shape[1], ctx.stride, int(ctx.split), ptr(clamped),
                                         ptr(v_opacity), ptr(v_rgb), ptr(v_op_dc), ptr(v_op_rest), ptr(v_shs), ptr(v_shs_rest), _stream()),
              "b200gs_glossy_sh_bwd")
        return None, None, None, None, None, v_op_dc, v_op_rest, v_shs, v_shs_rest


def glossy_sh(degree: int, means: torch.Tensor, campos: torch.Tensor, op_dc: torch.Tensor, op_rest: torch.Tensor, *,
              shs_dc: Optional[torch.Tensor] = None, shs_rest: Optional[torch.Tensor] = None, features: Optional[torch.Tensor] = None,
              mask: Optional[torch.Tensor] = None) -> Tuple[Optional[torch.Tensor], torch.Tensor]:
    """Glossy-Gaussian view-dependent opacity and SH colour on one kernel each way: returns ``(rgb, opacity)``.

    The view direction of Gaussian i is ``F.normalize(means[i] - campos)``, detached (no gradient reaches ``means``); ``campos`` is
    the camera centre, 3 floats on the device.  ``opacity`` [N] = ``clamp(SH_degree(op_dc | op_rest) + 0.5, 0, 1)`` for every row,
    from the model's ``[N,1,1]`` dc and ``[N,R,1]`` rest, R >= (degree+1)^2 - 1.  ``rgb`` [N,3] = ``clamp(SH_degree(colour) + 0.5,
    min=0)`` on the rows where ``mask`` ([N] bool, None: all) is set and 0.5 on the others; the colour is ``shs_dc`` [N,1,3] with
    ``shs_rest`` [N,K-1,3], or ``features`` [N,K,3], K >= (degree+1)^2; without either, no colour is computed and rgb is None.
    Every tensor is read in place: non-float32, non-CUDA or non-contiguous inputs are refused with a ValueError."""
    degree = int(degree)
    if not 0 <= degree <= 4:
        raise ValueError(f"degree must be 0..4, got {degree}")
    n, need = means.shape[0], (degree + 1) ** 2
    if means.shape != (n, 3):
        raise ValueError("means must be [N, 3]")
    if op_dc.shape != (n, 1, 1) or op_rest.dim() != 3 or op_rest.shape[0] != n or op_rest.shape[2] != 1:
        raise ValueError("expected op_dc [N,1,1] and op_rest [N,R,1]")
    if op_rest.shape[1] + 1 < need:
        raise ValueError(f"op_rest has {op_rest.shape[1]} rows, degree {degree} needs {need - 1}")
    if features is not None and (shs_dc is not None or shs_rest is not None):
        raise ValueError("pass either features or shs_dc and shs_rest, not both")
    if (shs_dc is None) != (shs_rest is None):
        raise ValueError("shs_dc and shs_rest go together")
    split = shs_dc is not None
    shs = shs_dc if split else features
    if split:
        if shs_dc.shape != (n, 1, 3) or shs_rest.dim() != 3 or shs_rest.shape[0] != n or shs_rest.shape[2] != 3:
            raise ValueError("expected shs_dc [N,1,3] and shs_rest [N,K-1,3]")
        if shs_rest.shape[1] + 1 < need:
            raise ValueError(f"shs_rest has {shs_rest.shape[1]} rows, degree {degree} needs {need - 1}")
    elif features is not None:
        if features.dim() != 3 or features.shape[0] != n or features.shape[2] != 3:
            raise ValueError("expected features [N,K,3]")
        if features.shape[1] < need:
            raise ValueError(f"features has {features.shape[1]} coefficients, degree {degree} needs {need}")
    means = _f32_in_place(means.detach(), "means")
    op_dc, op_rest = _f32_in_place(op_dc, "op_dc"), _f32_in_place(op_rest, "op_rest")
    if shs is not None:
        shs = _f32_in_place(shs, "shs_dc" if split else "features")
        shs_rest = _f32_in_place(shs_rest, "shs_rest") if split else None
    campos = _f32c(campos, "campos").reshape(-1)
    if campos.numel() != 3 or campos.device != means.device:
        raise ValueError("campos must be 3 floats on the device of means")
    m = None
    if mask is not None and shs is not None:
        if mask.shape != (n,) or mask.device != means.device:
            raise ValueError("mask must be [N] on the device of means")
        m = (mask if mask.dtype == torch.bool else mask != 0).contiguous().view(torch.uint8)
    return _GlossySH.apply(degree, split, m, means, campos, op_dc, op_rest, shs, shs_rest)


def _check_channels(colors, background):
    if colors.dim() != 2 or colors.shape[1] < 1:
        raise ValueError("colors must be [N, D] with D >= 1")
    if background is not None and background.shape[0] != colors.shape[1]:
        raise ValueError("background must have one entry per colour channel")


class _RasterizeGsplat(torch.autograd.Function):
    """The gsplat-mode blend of [N, D] colours behind rasterize_gaussians and rasterize_binned.

    binning: a Binning computed beforehand, or None to bin here from depths / radii with the lazy protocol (_bin_then_blend).
    D <= 4 runs K6 / K7; wider D the D-channel kernels, whose backward skips the geometry gradients when none of xys, conics and
    opacity needs one.  want_hits (K6 only): also return uint8 [N] has-hit flags.  absgrad: after the backward, `xys.absgrad`
    holds this blend's value, or with sum_absgrad, that value added to the one it already holds (so the channel groups and the
    passes of one render accumulate)."""

    @staticmethod
    def forward(ctx, xys, conics, colors, opacity, background, depths, radii, binning, hw, absgrad, sum_absgrad, want_hits):
        xys = _f32c(xys, "xys")
        conics = _f32c(conics, "conics")
        colors = _f32c(colors, "colors")
        opac = _f32c(opacity, "opacity").reshape(-1)
        bg = _f32c(background, "background") if background is not None else None
        H, W = hw
        features = colors.shape[1] > 4

        def blend(binning):
            if features:
                return (*blend_features_forward(W, H, binning, xys, conics, opac, colors, bg), None)
            hits = torch.zeros(xys.shape[0], dtype=torch.uint8, device=xys.device) if want_hits else None
            return (*blend_forward(MODE_GSPLAT, W, H, binning, xys, conics, opac, colors, bg, False, True, hits), hits)

        if binning is None:
            depths, radii = _f32c(depths, "depths"), radii.contiguous()
            binning, out = _bin_then_blend(lambda lazy: bin_gaussians(MODE_GSPLAT, W, H, xys, depths, radii, conics, opac, lazy=lazy), blend)
        else:
            out = blend(binning)
        image, final_T, n_contrib, alpha, hits = out
        ctx.binning, ctx.hw, ctx.features, ctx.opac_shape = binning, hw, features, tuple(opacity.shape)
        ctx.absgrad, ctx.sum_absgrad = absgrad, sum_absgrad
        ctx.save_for_backward(xys, conics, colors, opac, bg, final_T, n_contrib)
        ctx.xys_ref = xys
        if hits is None:
            return image, alpha
        ctx.mark_non_differentiable(hits)
        return image, alpha, hits

    @staticmethod
    def backward(ctx, v_image, v_alpha, *_):
        xys, conics, colors, opac, bg, final_T, n_contrib = ctx.saved_tensors
        H, W = ctx.hw
        need = ctx.needs_input_grad
        v_image = _f32c(v_image, "grad_image")
        v_alpha = _f32c(v_alpha, "grad_alpha") if v_alpha is not None else None
        if ctx.features:
            geometry = need[0] or need[1] or need[3]
            grads = blend_features_backward(W, H, ctx.binning, xys, conics, opac, colors, bg, final_T, n_contrib, v_image, v_alpha,
                                            geometry, geometry and ctx.absgrad)
        else:
            grads = blend_backward(MODE_GSPLAT, W, H, ctx.binning, xys, conics, opac, colors, bg, final_T, n_contrib, v_image, v_alpha,
                                   False, (1.0, 1.0), ctx.absgrad)
        v_xy, v_conic, v_opacity, v_colors, v_abs = grads
        if v_abs is not None:
            prev = getattr(ctx.xys_ref, "absgrad", None) if ctx.sum_absgrad else None
            ctx.xys_ref.absgrad = v_abs if prev is None else prev + v_abs
        return (v_xy if need[0] else None, v_conic if need[1] else None, v_colors if need[2] else None,
                v_opacity.reshape(ctx.opac_shape) if need[3] else None) + (None,) * 8


def rasterize_gaussians(xys, depths, radii, conics, num_tiles_hit, colors, opacity, img_height, img_width, block_width=16,
                        background=None, return_alpha=False, absgrad=False):
    """gsplat v0 ``rasterize_gaussians`` -> [H,W,D] (and alpha [H,W] when return_alpha), any D >= 1.  D <= 4 runs K6 / K7; wider
    feature maps run the D-channel kernels in chunks of 32 channels over one binning.  `xys.absgrad` is exact for D <= 32; beyond,
    it is the sum of each 32-channel chunk's value (an upper bound of gsplat's all-channel value)."""
    if block_width != TILE:
        raise ValueError(f"b200gs supports block_width {TILE} only")
    _check_channels(colors, background)
    image, alpha = _RasterizeGsplat.apply(xys, conics, colors, opacity, background, depths, radii, None, (int(img_height), int(img_width)),
                                          bool(absgrad), False, False)
    return (image, alpha) if return_alpha else image


def rasterize_binned(means2d, conics, colors, opacities, binning: Binning, img_height: int, img_width: int, background=None,
                     absgrad: bool = False, want_hits: bool = False):
    """K6 / K7 on a binning computed beforehand (gsplat v1: isect_tiles + isect_offset_encode once, rasterize_to_pixels several
    times with different colour sets — gsplat_v1_renderer.py:176-196,326-352).
    -> (image [H,W,D], alpha [H,W], hits uint8 [N] or None) for any D >= 1: the channels are composited in groups of <= 4 over the
    same per-tile lists (alpha / hits come from the first group; `means2d.absgrad`, when requested, accumulates every group's: |.|
    per group, an upper bound of gsplat's all-channel value when D > 4).  The groups stay on K6 / K7 even when D > 4: only K6
    writes hits, and with a background the D-channel kernels round the background term differently (see csrc/blend.cu)."""
    _check_channels(colors, background)
    D = colors.shape[1]
    images, alpha, hits = [], None, None
    for c0 in range(0, D, 4):
        c1 = min(D, c0 + 4)
        out = _RasterizeGsplat.apply(means2d, conics, colors[:, c0:c1], opacities, None if background is None else background[c0:c1], None,
                                     None, binning, (int(img_height), int(img_width)), bool(absgrad), True, want_hits and c0 == 0)
        images.append(out[0])
        if c0 == 0:
            alpha = out[1]
            hits = out[2] if want_hits else None
    return (images[0] if len(images) == 1 else torch.cat(images, dim=-1)), alpha, hits


def isect_keys(binning: Binning, depths: torch.Tensor) -> torch.Tensor:
    """gsplat's sorted ``isect_ids`` of a binning (b200gs_isect_keys): int64 [binning.total], (tile << 32) | float_bits(depth)
    in list order, for every tile of binning.tile_ranges.  Reads binning.total, i.e. waits for the counts of a lazy binning."""
    depths = _f32c(depths, "depths")
    n_tiles = binning.tile_ranges.shape[0]
    total = int(binning.total)
    keys = torch.empty(total, dtype=torch.int64, device=depths.device)
    with _stage("isect_keys"):
        check(lib().b200gs_isect_keys(int(n_tiles), ptr(binning.tile_ranges), ptr(binning.sorted_ids), total, ptr(depths), ptr(keys), _stream()),
              "b200gs_isect_keys")
    return keys


def isect_offsets(keys: torch.Tensor, n_tiles: int) -> torch.Tensor:
    """gsplat's ``isect_offset_encode`` for one camera (b200gs_isect_offsets): int32 [n_tiles], offsets[t] = index of the first
    of the sorted keys whose tile is >= t."""
    if keys.dtype != torch.int64 or keys.dim() != 1 or not keys.is_cuda:
        raise ValueError("isect_ids must be a 1-D int64 CUDA tensor")
    keys = keys.contiguous()
    offsets = torch.empty(int(n_tiles), dtype=torch.int32, device=keys.device)
    with _stage("isect_offsets"):
        check(lib().b200gs_isect_offsets(keys.shape[0], ptr(keys), int(n_tiles), ptr(offsets), _stream()), "b200gs_isect_offsets")
    return offsets


def knn_mean_dist2(points: torch.Tensor) -> torch.Tensor:
    """``simple_knn._C.distCUDA2(points [N,3]) -> [N]``: mean squared distance to the 3 nearest neighbours (vanilla_gaussian.py:122-125)."""
    pts = _f32c(points, "points")
    if pts.dim() != 2 or pts.shape[1] != 3:
        raise ValueError("points must be [N, 3]")
    L = lib()
    n = pts.shape[0]
    out = torch.empty(n, dtype=torch.float32, device=pts.device)
    ws = torch.empty(max(int(L.b200gs_knn_workspace_bytes(n)), 256), dtype=torch.uint8, device=pts.device)
    check(L.b200gs_knn_mean_dist2(n, ptr(pts), ptr(out), ptr(ws), ws.numel(), _stream()), "b200gs_knn_mean_dist2")
    return out


KNN_MAX_K = 32


def knn_launches(n: int) -> int:
    """library launches of one knn_points or knn_mean_dist2 call over n points: bounds, grid, cell keys, histogram, the radix passes
    over the cell keys (< 4n + 64 cells), gather, search"""
    bits = max(1, (4 * max(n, 1) + 63).bit_length())
    return 6 + (bits + 7) // 8


def knn_points(queries: torch.Tensor, points: torch.Tensor, K: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The K nearest of ``points`` [N,3] for every query of ``queries`` [S,3] (float32 CUDA, one device), a query that is itself one
    of the points included: (dists [S,K] squared distances, idx [S,K] int64), ascending.  pytorch3d's ``knn_points`` for one batch
    entry with norm 2.  Exact up to ties.  No host synchronisation; not differentiable (both reference callers run it under
    ``no_grad``).  1 <= K <= min(32, N)."""
    q, pts = _f32c(queries, "queries"), _f32c(points, "points")
    if q.dim() != 2 or q.shape[1] != 3 or pts.dim() != 2 or pts.shape[1] != 3:
        raise ValueError(f"queries and points must be [S, 3] and [N, 3], got {tuple(q.shape)} and {tuple(pts.shape)}")
    if q.device != pts.device:
        raise ValueError("queries and points must be on one device")
    K = int(K)
    if not 1 <= K <= KNN_MAX_K or K > pts.shape[0]:
        raise ValueError(f"K must be 1..{KNN_MAX_K} and at most the number of points ({pts.shape[0]}), got {K}")
    L = lib()
    s, n = q.shape[0], pts.shape[0]
    dists = torch.empty((s, K), dtype=torch.float32, device=q.device)
    idx = torch.empty((s, K), dtype=torch.int64, device=q.device)
    ws = torch.empty(max(int(L.b200gs_knn_workspace_bytes(n)), 256), dtype=torch.uint8, device=q.device)
    check(L.b200gs_knn_points(s, ptr(q), n, ptr(pts), K, ptr(dists), ptr(idx), ptr(ws), ws.numel(), _stream()), "b200gs_knn_points")
    return dists, idx


SIMILARITY_KINDS = {"cosine": 0, "euclidean": 1}
SIMILARITY_FWD_LAUNCHES = 2     # library launches of one similarity_regularization forward: per-sample sums, reduce


def similarity_bwd_launches(n: int) -> int:
    """library launches of one similarity_regularization backward over n Gaussians: entries, histogram, radix passes, run table,
    sums"""
    bits = max(1, (n - 1).bit_length())
    return 4 + (bits + 7) // 8


class _SimilarityRegularization(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, idx, dists, decay, weight, kind):
        n, d = features.shape
        s, k = idx.shape
        L = lib()
        nbytes = int(L.b200gs_similarity_reg_workspace_bytes(n, s, k, d, 0))          # the per-sample sums only
        ws = torch.empty(nbytes, dtype=torch.uint8, device=features.device)
        out = torch.empty(2, dtype=torch.float32, device=features.device)
        weights = torch.empty((s, k), dtype=torch.float32, device=features.device)
        check(L.b200gs_similarity_reg_fwd(n, d, ptr(features), s, k, ptr(idx), ptr(dists), kind, decay, weight, ptr(ws), nbytes, ptr(out),
                                          ptr(weights), _stream()), "b200gs_similarity_reg_fwd")
        ctx.save_for_backward(features, idx, dists)
        ctx.args = (decay, weight, kind)
        mean = out[1]
        ctx.mark_non_differentiable(mean, weights)
        return out[0], mean, weights

    @staticmethod
    def backward(ctx, v_loss, _v_mean, _v_weights):
        features, idx, dists = ctx.saved_tensors
        decay, weight, kind = ctx.args
        n, d = features.shape
        s, k = idx.shape
        L = lib()
        nbytes = int(L.b200gs_similarity_reg_workspace_bytes(n, s, k, d, 1))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=features.device)
        v = v_loss.reshape(1).to(torch.float32).contiguous()
        v_features = torch.empty_like(features)
        check(L.b200gs_similarity_reg_bwd(n, d, ptr(features), s, k, ptr(idx), ptr(dists), kind, decay, weight, ptr(ws), nbytes,
                                              ptr(v), ptr(v_features), _stream()), "b200gs_similarity_reg_bwd")
        return v_features, None, None, None, None, None


def similarity_regularization(features: torch.Tensor, idx: torch.Tensor, dists: torch.Tensor, *, decay: float, weight: float,
                              kind: str = "cosine"):
    """``SimilarityRegularizationMixin.get_similarity_metric``'s term after ``knn_points`` (K43/K44, backward K45, the onesweep sort
    and K46), without its [S,K,K,D] broadcast:
        m = mean_{s, i<j} r_sij exp(-decay dists[s,j]),   loss = weight m,
        "cosine": r = -n_i . n_j with n = F.normalize(f),   "euclidean": r = |f_i - f_j|,   f_i = features[idx[s,i]].
    The forward allocates only the S per-sample sums; the backward its own S K (4 D + 16) + 8 N bytes.
    features float32 CUDA [N,D] (D <= 256), idx int64 [S,K] (2 <= K <= 32, values in [0, N)), dists float32 [S,K].  Returns
    (loss, m, w): device scalars and the weights [S,K]; the gradient goes to ``features`` only, densely and deterministically.  No
    host synchronisation."""
    if kind not in SIMILARITY_KINDS:
        raise NotImplementedError(f"similarity kind {kind!r}: only {sorted(SIMILARITY_KINDS)} are provided")
    if features.dim() != 2 or idx.dim() != 2 or tuple(dists.shape) != tuple(idx.shape):
        raise ValueError(f"features must be [N, D] and idx, dists [S, K], got {tuple(features.shape)}, {tuple(idx.shape)}, "
                         f"{tuple(dists.shape)}")
    n, d = features.shape
    s, k = idx.shape
    if not 1 <= d <= 256 or not 2 <= k <= KNN_MAX_K or s < 1 or n < 1:
        raise ValueError(f"need 1 <= D <= 256, 2 <= K <= {KNN_MAX_K}, S >= 1 and N >= 1, got D={d}, K={k}, S={s}, N={n}")
    if features.dtype != torch.float32 or dists.dtype != torch.float32 or idx.dtype != torch.int64:
        raise ValueError("features and dists must be float32 and idx int64")
    if not (features.is_cuda and idx.device == features.device and dists.device == features.device):
        raise ValueError("features, idx and dists must be CUDA tensors on one device")
    return _SimilarityRegularization.apply(features.contiguous(), idx.detach().contiguous(), dists.detach().contiguous(), float(decay),
                                           float(weight), SIMILARITY_KINDS[kind])


# ----------------------------------------------------------------------------------------------------------------------
# fused L1 + SSIM loss (csrc/loss.cu; the metric the reference computes right after the renderer, vanilla_metrics.py:57-80)
# ----------------------------------------------------------------------------------------------------------------------
class _L1SSIMLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, target, lambda_dssim):
        L = lib()
        image, target = _f32c(image, "image"), _f32c(target, "target")
        if image.dim() != 3 or image.shape != target.shape:
            raise ValueError("image and target must both be [C,H,W]")
        C, H, W = image.shape
        dev = image.device
        blocks = int(L.b200gs_loss_blocks(C, W, H))
        dmaps = torch.empty(3, C, H, W, dtype=torch.float32, device=dev)
        partials = torch.empty(blocks, 2, dtype=torch.float32, device=dev)
        with _stage("loss_fwd"):
            check(L.b200gs_loss_fwd(C, W, H, ptr(image), ptr(target), ptr(dmaps), ptr(partials), _stream()), "b200gs_loss_fwd")
        sums = partials.sum(dim=0) / float(C * H * W)                   # [mean |a-b|, mean SSIM]; fixed summation order
        loss = (1.0 - lambda_dssim) * sums[0] + lambda_dssim * (1.0 - sums[1])
        ctx.save_for_backward(image, target, dmaps)
        ctx.lambda_dssim = float(lambda_dssim)
        ctx.mark_non_differentiable(sums)
        return loss, sums

    @staticmethod
    def backward(ctx, v_loss, _v_sums):
        L = lib()
        image, target, dmaps = ctx.saved_tensors
        C, H, W = image.shape
        v_image = torch.empty_like(image)
        v = _f32c(v_loss.reshape(1), "grad_loss")
        with _stage("loss_bwd"):
            check(L.b200gs_loss_bwd(C, W, H, ptr(image), ptr(target), ptr(dmaps), ctx.lambda_dssim, ptr(v), ptr(v_image), _stream()),
                  "b200gs_loss_bwd")
        return v_image, None, None


def l1_ssim_loss(image: torch.Tensor, target: torch.Tensor, lambda_dssim: float = 0.2):
    """(1 - lambda) * L1 + lambda * (1 - SSIM) of `VanillaMetricsImpl._get_basic_metrics` (vanilla_metrics.py:57-74) in two
    kernels; returns (loss, stats) with stats = [mean |image - target|, mean SSIM].  image/target: [C,H,W] fp32 CUDA."""
    return _L1SSIMLoss.apply(image, target, float(lambda_dssim))


# ---- appearance-embedding colour pass (csrc/appearance.cu) ---------------------------------------------------------------------
APPEARANCE_FWD_LAUNCHES = 1     # library launches of one appearance_mlp / appearance_colors forward
APPEARANCE_BWD_LAUNCHES = 2     # and of its backward: the MLP backward and the reduction of the per-CTA weight-gradient blocks


def appearance_supported(feat_dim: int, n_freq: int, n_neurons: int, n_layers: int, n_out: int) -> bool:
    """Whether the appearance kernels take this network (no device needed)."""
    return int(lib().b200gs_appearance_mlp_workspace_bytes(feat_dim, n_freq, n_neurons, n_layers, n_out)) > 0


def _appearance_offsets(feat_dim, n_freq, n_neurons, n_layers, n_out):
    """[(offset, rows, cols)] of each layer's weight, then [(offset, rows)] of each bias, in b200gs_appearance_mlp_bwd's v_params."""
    pe = 0 if n_freq < 0 else 3 * (2 * n_freq + 1)
    k0p = (feat_dim + pe + 7) // 8 * 8
    shapes = [(n_out if l == n_layers - 1 else n_neurons, k0p if l == 0 else n_neurons) for l in range(n_layers)]
    o, ws, bs = 0, [], []
    for r, c in shapes:
        ws.append((o, r, c))
        o += r * c
    for r, _ in shapes:
        bs.append((o, r))
        o += r
    return ws, bs, o


class _AppearanceMlp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cfg, features, mask, base_rgb, dirs, cam, raw_opacity, embed_cols, *params):
        n_freq, normalize, normalize_dirs, epilogue = cfg
        n, feat_dim = features.shape
        weights, biases = params[0::2], params[1::2]
        n_layers, n_neurons, n_out = len(weights), weights[0].shape[0], weights[-1].shape[0]
        m = _lib.B200gsAppearanceMlp(feat_dim, n_freq, n_neurons, n_layers, n_out, int(normalize), int(normalize_dirs), int(epilogue),
                                     weights[0].shape[1], feat_dim + embed_cols)
        for l in range(n_layers):
            m.weights[l], m.biases[l] = weights[l].data_ptr(), biases[l].data_ptr()
        dev = features.device
        with_opacity = epilogue and n_out == 4
        out = torch.empty(n, 3 if epilogue else n_out, dtype=torch.float32, device=dev)
        offsets = torch.empty(n, dtype=torch.float32, device=dev) if with_opacity else None
        opacities = torch.empty(n, dtype=torch.float32, device=dev) if with_opacity else None
        check(lib().b200gs_appearance_mlp_fwd(ctypes.byref(m), n, ptr(features), ptr(mask), ptr(base_rgb), ptr(dirs), ptr(cam),
                                              ptr(raw_opacity), ptr(out), ptr(offsets), ptr(opacities), _stream()), "b200gs_appearance_mlp_fwd")
        ctx.m, ctx.cfg, ctx.embed_cols = m, cfg, embed_cols
        ctx.save_for_backward(features, mask, base_rgb, dirs, cam, raw_opacity, *params)
        if not epilogue:
            return out
        return (out, opacities, offsets) if with_opacity else out

    @staticmethod
    def backward(ctx, v_out, v_opacities=None, v_offsets=None):
        features, mask, base_rgb, dirs, cam, raw_opacity, *params = ctx.saved_tensors
        m, (n_freq, _, _, epilogue) = ctx.m, ctx.cfg
        n, feat_dim = features.shape
        with_opacity = epilogue and m.n_out == 4
        dev, L_ = features.device, lib()
        ws, bs, total = _appearance_offsets(feat_dim, n_freq, m.n_neurons, m.n_layers, m.n_out)
        v_out = _f32c(v_out, "grad")
        v_opacities = _f32c(v_opacities, "grad") if v_opacities is not None else None
        v_offsets = _f32c(v_offsets, "grad") if v_offsets is not None else None
        v_base = torch.empty_like(base_rgb) if epilogue else None
        v_features = torch.empty_like(features) if ctx.needs_input_grad[1] else None
        v_raw = torch.empty_like(raw_opacity) if with_opacity else None
        ws_bytes = int(L_.b200gs_appearance_mlp_workspace_bytes(feat_dim, n_freq, m.n_neurons, m.n_layers, m.n_out))
        workspace = torch.empty(ws_bytes // 4, dtype=torch.float32, device=dev)
        v_params = torch.empty(total, dtype=torch.float32, device=dev)
        check(L_.b200gs_appearance_mlp_bwd(ctypes.byref(m), n, ptr(features), ptr(mask), ptr(base_rgb), ptr(dirs), ptr(cam), ptr(raw_opacity),
                                           ptr(v_out), ptr(v_opacities), ptr(v_offsets), ptr(v_base), ptr(v_features), ptr(v_raw),
                                           ptr(workspace), ws_bytes, ptr(v_params), _stream()), "b200gs_appearance_mlp_bwd")
        grads = []
        for l, ((wo, r, c), (bo, _)) in enumerate(zip(ws, bs)):
            v_w = v_params[wo:wo + r * c].view(r, c)
            if l == 0:      # the kernel's columns are features | view direction; the embedding's columns get theirs through biases[0]
                pe = 0 if n_freq < 0 else 3 * (2 * n_freq + 1)
                full = torch.zeros_like(params[0])
                full[:, :feat_dim] = v_w[:, :feat_dim]
                if pe:
                    full[:, feat_dim + ctx.embed_cols:] = v_w[:, feat_dim:feat_dim + pe]
                v_w = full
            grads += [v_w, v_params[bo:bo + r]]
        return (None, v_features, None, v_base, None, None, v_raw, None, *grads)


def appearance_mlp(features, embedding, weights, biases, *, dirs=None, cam=None, n_freq=-1, normalize=False, normalize_dirs=False,
                   mask=None, base_rgb=None, raw_opacity=None):
    """The appearance network of the reference's GSplatAppearanceEmbeddingRenderer on one kernel each way.

    ``features`` [N, F]; ``embedding`` [E], the image's (already normalised, when the model normalises) embedding row; ``weights`` /
    ``biases`` the Linear layers, ``weights[0]`` [H, F + E (+ PE)].  The embedding is the same for every row, so it is folded into the
    first bias here (``b0 + W0[:, F:F+E] @ embedding``, torch, differentiable) and the kernel never sees it.  ``dirs`` [N, 3] minus
    ``cam`` [3] (optional) is the view direction when ``n_freq >= 0``.  ``mask`` bool [N] (None: every row) selects the rows.

    Without ``base_rgb``: returns the sigmoid outputs [N, 3 | 4] (zeros in unmasked rows).  With ``base_rgb`` [N, 3] (SH colours before
    the + 0.5): returns ``rgbs`` [N, 3] = clamp(base + 0.5 + 2 s - 1, 0, 1), zeros in unmasked rows, and, for a 4-output network,
    ``(rgbs, opacities, opacity_offsets)`` with ``opacities = min(raw_opacity + offset, 1)``.  Gradients reach features, base_rgb,
    raw_opacity, the embedding and every weight and bias; none reaches dirs or cam."""
    feat_dim, e = features.shape[1], embedding.shape[0]
    w0 = weights[0]
    b0 = torch.addmv(biases[0], w0[:, feat_dim:feat_dim + e], embedding)
    params = []
    for l, (w, b) in enumerate(zip(weights, biases)):
        params += [_f32c(w, "weight"), _f32c(b0 if l == 0 else b, "bias")]
    if mask is not None:
        mask = (mask if mask.dtype == torch.bool else mask != 0).contiguous().view(torch.uint8)
    epilogue = base_rgb is not None
    cfg = (int(n_freq), bool(normalize), bool(normalize_dirs), epilogue)
    return _AppearanceMlp.apply(cfg, _f32c(features, "features"), mask, _f32c(base_rgb, "base_rgb") if epilogue else None,
                                _f32c(dirs, "dirs") if n_freq >= 0 else None, _f32c(cam.reshape(-1), "cam") if cam is not None and n_freq >= 0 else None,
                                _f32c(raw_opacity, "raw_opacity") if raw_opacity is not None else None, e, *params)


# ---- transient visibility map (csrc/visibility.cu; the visibility MLP runs on the appearance kernels) ------------------------------
UV_GRID_FWD_LAUNCHES = 1        # library launches of one uv_grid_encode forward (K32)
UV_GRID_BWD_LAUNCHES = 1        # and of its backward (K33)
VISIBILITY_MLP_FWD_LAUNCHES = 1
VISIBILITY_MLP_BWD_LAUNCHES = 2
VISIBILITY_LOSS_FWD_LAUNCHES = 1    # K34
VISIBILITY_LOSS_BWD_LAUNCHES = 1    # K35


def uv_grid_params(n_levels: int = 8, base_resolution: int = 16, per_level_scale: float = 1.405) -> int:
    """Floats of one DenseGrid of the given config (tcnn's ``n_params``; 121760 for the defaults), 0 when not supported."""
    return int(lib().b200gs_uv_grid_params(ctypes.byref(_lib.B200gsUvGrid(n_levels, base_resolution, per_level_scale))))


_GRID_TABLES = {}


def _grid_table(grids, device) -> torch.Tensor:
    """int64 [n] device table of the grids' addresses, built once per set of addresses: the kernels pick the row on the device."""
    key = (str(device),) + tuple(g.data_ptr() for g in grids)
    t = _GRID_TABLES.get(key)
    if t is None:
        if len(_GRID_TABLES) >= 16:
            _GRID_TABLES.clear()
        t = _GRID_TABLES[key] = torch.tensor(key[1:], dtype=torch.int64).to(device)
    return t


class _UvGridEncode(torch.autograd.Function):
    @staticmethod
    def forward(ctx, grid, width, height, uv, table, id_dev, host_id, selected):
        n = width * height if uv is None else uv.shape[0]
        enc = torch.empty(n, 2 * grid.n_levels, dtype=torch.float32, device=table.device)
        check(lib().b200gs_uv_grid_fwd(ctypes.byref(grid), width, height, ptr(uv), n, ptr(table), table.shape[0], ptr(id_dev), host_id,
                                       ptr(enc), _stream()), "b200gs_uv_grid_fwd")
        ctx.grid, ctx.size = grid, (width, height, n)
        ctx.save_for_backward(uv)
        return enc

    @staticmethod
    def backward(ctx, v_enc):
        (uv,) = ctx.saved_tensors
        width, height, n = ctx.size
        v_enc = _f32c(v_enc, "grad")
        v_params = torch.empty(int(lib().b200gs_uv_grid_params(ctypes.byref(ctx.grid))), dtype=torch.float32, device=v_enc.device)
        check(lib().b200gs_uv_grid_bwd(ctypes.byref(ctx.grid), width, height, ptr(uv), n, ptr(v_enc), ptr(v_params), _stream()),
              "b200gs_uv_grid_bwd")
        return None, None, None, None, None, None, None, v_params


def uv_grid_encode(grids, appearance_id, *, width=None, height=None, uv=None, selected=None, n_levels=8, base_resolution=16,
                   per_level_scale=1.405):
    """tiny-cuda-nn's 2-D ``DenseGrid`` encoding (linear interpolation, 2 features per level) on K32/K33: enc [n, 2 n_levels].

    ``grids``: the per-image flat parameter vectors (tcnn layout, ``uv_grid_params`` floats each); the one used is
    ``grids[appearance_id]``, with ``appearance_id`` an int, a CPU tensor or a one-element CUDA tensor read on the device (an id out of
    range gives NaN).  Coordinates: ``uv`` [n, 2], or, when None, the pixel grid of a ``width`` x ``height`` image (row-major, u =
    x / (width - 1), v = y / (height - 1), both sizes >= 2).  The gradient goes to ``grids[selected]`` (default: the host id), the
    pixel grid's without atomics, so two backwards are bit-identical.  With a CUDA ``appearance_id`` the caller passes ``selected``,
    which must be the value that tensor holds: the kernels read the grid the device id names, and autograd can only route the
    gradient to a tensor named on the host (``visibility.host_appearance_id`` reads and caches it per camera)."""
    grid = _lib.B200gsUvGrid(int(n_levels), int(base_resolution), float(per_level_scale))
    if not grids or any(g.dtype != torch.float32 or not g.is_cuda or not g.is_contiguous() for g in grids):
        raise ValueError("grids must be contiguous float32 CUDA tensors")
    if any(g.numel() != uv_grid_params(n_levels, base_resolution, per_level_scale) for g in grids):
        raise ValueError(f"every grid must hold {uv_grid_params(n_levels, base_resolution, per_level_scale)} floats")
    device = grids[0].device
    if isinstance(appearance_id, torch.Tensor) and appearance_id.is_cuda:
        if appearance_id.numel() != 1 or appearance_id.is_floating_point():
            raise ValueError("appearance_id must be one integer")
        id_dev, host_id = appearance_id.reshape(1).to(device=device, dtype=torch.int64), 0
    else:
        id_dev, host_id = None, int(appearance_id)
        selected = host_id if selected is None else selected
    if uv is None:
        if width is None or height is None or int(width) < 2 or int(height) < 2:
            raise ValueError("the pixel grid needs width and height >= 2")
        width, height = int(width), int(height)
    else:
        uv = _f32c(uv, "uv")
        if uv.dim() != 2 or uv.shape[1] != 2:
            raise ValueError("uv must be [n, 2]")
        width = height = 0
    if selected is None or not 0 <= selected < len(grids):
        if torch.is_grad_enabled() and any(g.requires_grad for g in grids):
            raise ValueError("the grid that receives the gradient is unknown: pass `selected` with a CUDA appearance_id")
        target = grids[0].detach()
    else:
        target = grids[selected]
    return _UvGridEncode.apply(grid, width, height, uv, _grid_table(grids, device), id_dev, host_id, target)


def visibility_supported(feat_dim: int, n_neurons: int, n_layers: int) -> bool:
    """Whether the visibility MLP kernels take this network (no device needed)."""
    return int(lib().b200gs_visibility_mlp_workspace_bytes(feat_dim, n_neurons, n_layers)) > 0


class _VisibilityMlp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, enc, *params):
        n, feat_dim = enc.shape
        weights, biases = params[0::2], params[1::2]
        n_layers, n_neurons = len(weights), weights[0].shape[0]
        m = _lib.B200gsAppearanceMlp(feat_dim, -1, n_neurons, n_layers, 1, 0, 0, 0, weights[0].shape[1], weights[0].shape[1])
        for l in range(n_layers):
            m.weights[l], m.biases[l] = weights[l].data_ptr(), biases[l].data_ptr()
        out = torch.empty(n, dtype=torch.float32, device=enc.device)
        check(lib().b200gs_visibility_mlp_fwd(ctypes.byref(m), n, ptr(enc), ptr(out), _stream()), "b200gs_visibility_mlp_fwd")
        ctx.m = m
        ctx.save_for_backward(enc, *params)
        return out

    @staticmethod
    def backward(ctx, v_out):
        enc, *params = ctx.saved_tensors
        m, L_ = ctx.m, lib()
        n, feat_dim = enc.shape
        ws, bs, total = _appearance_offsets(feat_dim, -1, m.n_neurons, m.n_layers, 1)
        v_out = _f32c(v_out, "grad")
        v_enc = torch.empty_like(enc) if ctx.needs_input_grad[0] else None
        ws_bytes = int(L_.b200gs_visibility_mlp_workspace_bytes(feat_dim, m.n_neurons, m.n_layers))
        workspace = torch.empty(ws_bytes // 4, dtype=torch.float32, device=enc.device)
        v_params = torch.empty(total, dtype=torch.float32, device=enc.device)
        check(L_.b200gs_visibility_mlp_bwd(ctypes.byref(m), n, ptr(enc), ptr(v_out), ptr(v_enc), ptr(workspace), ws_bytes, ptr(v_params),
                                           _stream()), "b200gs_visibility_mlp_bwd")
        grads = []
        for l, ((wo, r, c), (bo, _)) in enumerate(zip(ws, bs)):
            v_w = v_params[wo:wo + r * c].view(r, c)
            if l == 0:      # the encoding's columns; the embedding's get theirs through biases[0]
                full = torch.zeros_like(params[0])
                full[:, :feat_dim] = v_w
                v_w = full
            grads += [v_w, v_params[bo:bo + r]]
        return (v_enc, *grads)


def visibility_mlp(enc, embedding, weights, biases):
    """The reference's ``visibility_network`` on ``[enc | embedding]`` rows: sigmoid outputs [n].  ``enc`` [n, F] (F = 8, 16, 24 or 32),
    ``embedding`` [E] the image's transient embedding, ``weights[0]`` [H, F + E].  The embedding is the same for every row, so it is
    folded into the first bias here (torch, differentiable) and the kernels see F inputs.  Gradients reach enc, the embedding and
    every weight and bias."""
    feat_dim, e = enc.shape[1], embedding.shape[0]
    b0 = torch.addmv(biases[0], weights[0][:, feat_dim:feat_dim + e], embedding)
    params = []
    for l, (w, b) in enumerate(zip(weights, biases)):
        params += [_f32c(w, "weight"), _f32c(b0 if l == 0 else b, "bias")]
    return _VisibilityMlp.apply(_f32c(enc, "enc"), *params)


class _VisibilityLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, gt, visibility, mask, lambda_dssim, vis_reg_factor):
        _, H, W = image.shape
        L_ = lib()
        vis_grad = ctx.needs_input_grad[2]
        nbytes = int(L_.b200gs_vis_loss_workspace_bytes(W, H, int(vis_grad)))
        ws = torch.empty(nbytes // 4, dtype=torch.float32, device=image.device)
        with _stage("vis_loss_fwd"):
            check(L_.b200gs_vis_loss_fwd(W, H, ptr(image), ptr(gt), ptr(visibility), ptr(mask), int(vis_grad), ptr(ws), nbytes, _stream()),
                  "b200gs_vis_loss_fwd")
        blocks = int(L_.b200gs_vis_loss_blocks(W, H))
        sums = ws[nbytes // 4 - 3 * blocks:].view(blocks, 3).sum(dim=0)     # fixed summation order
        stats = torch.stack([sums[0] / float(3 * H * W), sums[1] / float(3 * H * W), sums[2] * (vis_reg_factor / float(H * W))])
        loss = (1.0 - lambda_dssim) * stats[0] + lambda_dssim * (1.0 - stats[1]) + stats[2]
        ctx.save_for_backward(image, gt, visibility, mask, ws)
        ctx.args = (float(lambda_dssim), float(vis_reg_factor), vis_grad)
        ctx.mark_non_differentiable(stats)
        return loss, stats

    @staticmethod
    def backward(ctx, v_loss, _v_stats):
        image, gt, visibility, mask, ws = ctx.saved_tensors
        lambda_dssim, vis_reg_factor, vis_grad = ctx.args
        _, H, W = image.shape
        v = _f32c(v_loss.reshape(1), "grad_loss")
        v_image = torch.empty_like(image)
        v_vis = torch.empty_like(visibility) if vis_grad else None
        with _stage("vis_loss_bwd"):
            check(lib().b200gs_vis_loss_bwd(W, H, ptr(image), ptr(gt), ptr(visibility), ptr(mask), ptr(ws), ws.numel() * 4, lambda_dssim,
                                            vis_reg_factor, ptr(v), ptr(v_image), ptr(v_vis), _stream()), "b200gs_vis_loss_bwd")
        return v_image, None, v_vis, None, None, None


def visibility_l1_ssim_loss(image, gt, visibility, mask=None, lambda_dssim: float = 0.2, vis_reg_factor: float = 0.2):
    """``VisibilityMapMetricsImpl.get_train_metrics``' loss of one view in two kernels: with w = visibility * mask,
    (1 - lambda) mean|w image - w gt| + lambda (1 - SSIM(w image, w gt)) + vis_reg_factor mean((1 - visibility)^2), the SSIM of
    ``l1_ssim_loss``.  image, gt [3,H,W], visibility [1,H,W] or [H,W], float32 CUDA; mask None or [H,W] / [1,H,W] (bool or uint8,
    nonzero keeps; a [C,H,W] mask is read at channel 0).  Gradients reach image and visibility (none to gt).  Returns (loss, stats),
    stats = [mean |a' - b'|, mean SSIM, the weighted regulariser]."""
    image, gt = _f32c(image, "image"), _f32c(gt, "gt").detach()
    if image.dim() != 3 or image.shape[0] != 3 or image.shape != gt.shape:
        raise ValueError(f"image and gt must both be [3,H,W], got {tuple(image.shape)} and {tuple(gt.shape)}")
    _, H, W = image.shape
    vis = _f32c(visibility, "visibility")
    if tuple(vis.shape[-2:]) != (H, W) or vis.numel() != H * W:
        raise ValueError(f"visibility must be [1,H,W] or [H,W] of the image's size, got {tuple(vis.shape)}")
    vis = vis.reshape(H, W)
    if mask is not None:
        if mask.dim() == 3:
            mask = mask[0]
        if tuple(mask.shape) != (H, W) or mask.dtype not in (torch.bool, torch.uint8) or mask.device != image.device:
            raise ValueError(f"mask must be bool or uint8 [H,W] on the image's device, got {mask.dtype} {tuple(mask.shape)}")
        mask = (mask != 0).contiguous().view(torch.uint8)
    return _VisibilityLoss.apply(image, gt, vis, mask, float(lambda_dssim), float(vis_reg_factor))


# ---- SWAG in-the-wild appearance (csrc/swag.cu K49/K50; the MLP runs on the appearance kernels with epilogue 2) -------------------
HASH_GRID_FWD_LAUNCHES = 1      # library launches of one hash_grid_encode forward (K49 without colour)
HASH_GRID_BWD_LAUNCHES = 1      # and of its backward (K50; the table gradient is zeroed with a memset)
SWAG_FWD_LAUNCHES = 2           # swag_colours_and_opacities forward: K49, K20
SWAG_BWD_LAUNCHES = 3           # and backward: K21, K22, K50
HASH_GRID_DEFAULTS = dict(n_levels=8, n_features_per_level=4, log2_hashmap_size=19, base_resolution=16, per_level_scale=2.0)
HASH_GRID_SUPPORTED = ("n_levels 1..16, n_features_per_level 2 or 4, log2_hashmap_size 1..24, base_resolution >= 1 and "
                       "per_level_scale >= 1 (every level's scale below 2^30)")


def _hash_grid(n_levels=8, n_features_per_level=4, log2_hashmap_size=19, base_resolution=16, per_level_scale=2.0) -> _lib.B200gsHashGrid:
    return _lib.B200gsHashGrid(int(n_levels), int(n_features_per_level), int(log2_hashmap_size), int(base_resolution),
                               float(per_level_scale))


def hash_grid_params(**grid) -> int:
    """Floats of one 3-D hash grid (tiny-cuda-nn's ``n_params``; 11681792 for the defaults), 0 when the grid is not supported."""
    return int(lib().b200gs_hash_grid_params(ctypes.byref(_hash_grid(**grid))))


def _check_table(table: torch.Tensor, grid: _lib.B200gsHashGrid) -> int:
    n = int(lib().b200gs_hash_grid_params(ctypes.byref(grid)))
    if n == 0:
        raise NotImplementedError(f"b200gs HashGrid supports {HASH_GRID_SUPPORTED}")
    if table.dtype != torch.float32 or not table.is_cuda or not table.is_contiguous() or table.numel() != n:
        raise ValueError(f"the grid table must be a contiguous float32 CUDA tensor of {n} floats")
    return n


class _HashGridEncode(torch.autograd.Function):
    @staticmethod
    def forward(ctx, grid, table, x):
        n, width = x.shape[0], grid.n_levels * grid.n_features_per_level
        enc = torch.empty(n, width, dtype=torch.float32, device=x.device)
        check(lib().b200gs_swag_inputs_fwd(ctypes.byref(grid), 0, n, ptr(x), None, None, None, 0, 0, None, ptr(table), width, ptr(enc),
                                           None, _stream()), "b200gs_swag_inputs_fwd")
        ctx.grid = grid
        ctx.save_for_backward(x, table)
        return enc

    @staticmethod
    def backward(ctx, v_enc):
        x, table = ctx.saved_tensors
        v_enc = _f32c(v_enc, "grad")
        v_table = torch.empty_like(table)
        check(lib().b200gs_swag_inputs_bwd(ctypes.byref(ctx.grid), 0, x.shape[0], ptr(x), None, None, None, 0, 0, None, None, ptr(v_enc),
                                           v_enc.shape[1], None, None, None, ptr(v_table), _stream()), "b200gs_swag_inputs_bwd")
        return None, v_table, None


def hash_grid_encode(params: torch.Tensor, x: torch.Tensor, **grid) -> torch.Tensor:
    """tiny-cuda-nn's 3-D ``HashGrid`` encoding (linear interpolation) of the points ``x`` [n, 3] (any values: points outside [0, 1]
    wrap as in tcnn) with the flat table ``params`` (tcnn layout, ``hash_grid_params(**grid)`` floats): enc [n, n_levels F].  The
    gradient reaches ``params`` only (tcnn's input gradient is not provided), scattered with vector float atomics: not
    bit-reproducible.  ``grid``: n_levels, n_features_per_level, log2_hashmap_size, base_resolution, per_level_scale."""
    g = _hash_grid(**{**HASH_GRID_DEFAULTS, **grid})
    _check_table(params, g)
    x = _f32c(x.detach(), "x")
    if x.dim() != 2 or x.shape[1] != 3:
        raise ValueError("x must be [n, 3]")
    return _HashGridEncode.apply(g, params, x)


def swag_supported(in_dim: int, n_neurons: int, n_layers: int) -> bool:
    """Whether the SWAG MLP kernels take a network on ``in_dim`` real input columns (no device needed)."""
    return int(lib().b200gs_swag_mlp_workspace_bytes((in_dim + 7) // 8 * 8, n_neurons, n_layers)) > 0


class _SwagColoursAndOpacities(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cfg, means, campos, shs, shs_rest, bbox, table, base_opacity, u, *params):
        grid, degree, split, stride, in_dim, row, temperature, eps = cfg
        n, dev, L_ = means.shape[0], means.device, lib()
        weights, biases = params[0::2], params[1::2]
        x0 = torch.empty(n, row, dtype=torch.float32, device=dev)
        clamped = torch.empty(n, dtype=torch.uint8, device=dev)
        check(L_.b200gs_swag_inputs_fwd(ctypes.byref(grid), degree, n, ptr(means), ptr(campos), ptr(shs), ptr(shs_rest), stride, int(split),
                                        ptr(bbox), ptr(table), row, ptr(x0), ptr(clamped), _stream()), "b200gs_swag_inputs_fwd")
        m = _lib.B200gsAppearanceMlp(row, -1, weights[0].shape[0], len(weights), 4, 0, 0, 2, weights[0].shape[1], weights[0].shape[1])
        for l in range(len(weights)):
            m.weights[l], m.biases[l] = weights[l].data_ptr(), biases[l].data_ptr()
        colour = torch.empty(n, 3, dtype=torch.float32, device=dev)
        opacity = torch.empty(n, dtype=torch.float32, device=dev)
        check(L_.b200gs_swag_mlp_fwd(ctypes.byref(m), in_dim, n, ptr(x0), ptr(base_opacity), ptr(u), temperature, eps, ptr(colour),
                                     ptr(opacity), _stream()), "b200gs_swag_mlp_fwd")
        ctx.cfg, ctx.m = cfg, m
        ctx.save_for_backward(means, campos, shs, shs_rest, bbox, table, base_opacity, u, x0, clamped, *params)
        return colour, opacity

    @staticmethod
    def backward(ctx, v_colour, v_opacity):
        means, campos, shs, shs_rest, bbox, table, base_opacity, u, x0, clamped, *params = ctx.saved_tensors
        grid, degree, split, stride, in_dim, row, temperature, eps = ctx.cfg
        m, L_ = ctx.m, lib()
        n, dev = means.shape[0], means.device
        v_colour = _f32c(v_colour, "grad") if v_colour is not None else torch.zeros(n, 3, dtype=torch.float32, device=dev)
        v_opacity = _f32c(v_opacity, "grad") if v_opacity is not None else None
        ws, bs, total = _appearance_offsets(row, -1, m.n_neurons, m.n_layers, 4)
        v_x0 = torch.empty_like(x0)
        v_base = torch.empty_like(base_opacity)
        ws_bytes = int(L_.b200gs_swag_mlp_workspace_bytes(row, m.n_neurons, m.n_layers))
        workspace = torch.empty(ws_bytes // 4, dtype=torch.float32, device=dev)
        v_params = torch.empty(total, dtype=torch.float32, device=dev)
        check(L_.b200gs_swag_mlp_bwd(ctypes.byref(m), in_dim, n, ptr(x0), ptr(base_opacity), ptr(u), temperature, eps, ptr(v_colour),
                                     ptr(v_opacity), ptr(v_x0), ptr(v_base), ptr(workspace), ws_bytes, ptr(v_params), _stream()),
              "b200gs_swag_mlp_bwd")
        v_shs, v_shs_rest = torch.empty_like(shs), (torch.empty_like(shs_rest) if split else None)
        v_means = torch.empty_like(means)
        v_table = torch.empty_like(table)
        check(L_.b200gs_swag_inputs_bwd(ctypes.byref(grid), degree, n, ptr(means), ptr(campos), ptr(shs), ptr(shs_rest), stride, int(split),
                                        ptr(bbox), ptr(clamped), ptr(v_x0), row, ptr(v_shs), ptr(v_shs_rest), ptr(v_means), ptr(v_table),
                                        _stream()), "b200gs_swag_inputs_bwd")
        grads = []
        for l, ((wo, r, c), (bo, _)) in enumerate(zip(ws, bs)):
            v_w = v_params[wo:wo + r * c].view(r, c)
            if l == 0:      # the row's real columns; the embedding's get theirs through biases[0]
                full = torch.zeros_like(params[0])
                full[:, :in_dim] = v_w[:, :in_dim]
                v_w = full
            grads += [v_w, v_params[bo:bo + r]]
        return (None, v_means, None, v_shs, v_shs_rest, None, v_table, v_base, None, *grads)


def swag_colours_and_opacities(degree: int, means: torch.Tensor, campos: torch.Tensor, base_opacity: torch.Tensor, u: torch.Tensor,
                               table: torch.Tensor, embedding: torch.Tensor, weights, biases, *, bbox: Optional[torch.Tensor] = None,
                               shs_dc: Optional[torch.Tensor] = None, shs_rest: Optional[torch.Tensor] = None,
                               features: Optional[torch.Tensor] = None, temperature: float = 0.1, eps: float = 1e-8,
                               **grid) -> Tuple[torch.Tensor, torch.Tensor]:
    """SWAG's image-conditioned colours and opacities (swag_renderer.py:47-56) as one autograd node: returns ``(colours [N, 3],
    opacities [N])``.

    Per Gaussian: rgb = clamp_min(SH_degree(colour; normalize(means - campos)) + 0.5, 0) from ``shs_dc`` [N,1,3] with ``shs_rest``
    [N,K-1,3] or ``features`` [N,K,3]; enc = the hash grid ``table`` (``hash_grid_params(**grid)`` floats) at ``(means - bbox[:3]) /
    bbox[3:]`` (``bbox`` 6 floats on the device: the box's minimum and size; None: the means themselves); o = the network
    ``weights`` / ``biases`` (Linear layers, ReLU between them, no output activation, ``weights[0]`` [H, 3 + enc + E]) on
    ``[rgb | enc | embedding]``, the image ``embedding`` [E] folded into the first bias; colours = sigmoid(o[:3]) and opacities =
    clamp_min(base_opacity - sigmoid((log(|o3| + eps) + log(u + eps) - log(1 - u + eps)) / temperature), 0), ``base_opacity`` [N] the
    activated opacity and ``u`` a one-element device tensor (no host read).  Forward K49 + K20, backward K21 + K22 + K50: no host
    synchronisation.  Gradients reach the SH coefficients, ``means`` (through the view direction only, as in the reference), the
    table, ``base_opacity``, the embedding and every weight and bias."""
    degree = int(degree)
    if not 0 <= degree <= 4:
        raise ValueError(f"degree must be 0..4, got {degree}")
    g = _hash_grid(**{**HASH_GRID_DEFAULTS, **grid})
    _check_table(table, g)
    n, need = means.shape[0], (degree + 1) ** 2
    if means.dim() != 2 or means.shape[1] != 3:
        raise ValueError("means must be [N, 3]")
    if features is not None and (shs_dc is not None or shs_rest is not None):
        raise ValueError("pass either features or shs_dc and shs_rest, not both")
    split = shs_dc is not None
    if split:
        if shs_rest is None or shs_dc.shape != (n, 1, 3) or shs_rest.dim() != 3 or shs_rest.shape[0] != n or shs_rest.shape[2] != 3:
            raise ValueError("expected shs_dc [N,1,3] and shs_rest [N,K-1,3]")
        stride = 1 + shs_rest.shape[1]
        shs, shs_rest = _f32_in_place(shs_dc, "shs_dc"), _f32_in_place(shs_rest, "shs_rest")
    else:
        if features is None or features.dim() != 3 or features.shape[0] != n or features.shape[2] != 3:
            raise ValueError("expected features [N,K,3] (or shs_dc and shs_rest)")
        stride = features.shape[1]
        shs, shs_rest = _f32_in_place(features, "features"), None
    if stride < need:
        raise ValueError(f"the SH colour has {stride} coefficients, degree {degree} needs {need}")
    enc_dim = g.n_levels * g.n_features_per_level
    in_dim, e = 3 + enc_dim, embedding.shape[0]
    row = (in_dim + 7) // 8 * 8
    if weights[0].shape[1] != in_dim + e or weights[-1].shape[0] != 4:
        raise ValueError(f"weights[0] must be [H, {in_dim + e}] (3 colour + {enc_dim} encoding + {e} embedding columns) and the output 4 wide")
    if not swag_supported(in_dim, weights[0].shape[0], len(weights)):
        raise NotImplementedError(f"b200gs SWAG network: {len(weights)} layers of {weights[0].shape[0]} neurons on {in_dim} inputs is not "
                                  "supported (n_neurons 64 or 128, n_layers 2..4)")
    means = _f32_in_place(means, "means")
    campos = _f32c(campos, "campos").reshape(-1)
    base_opacity = _f32c(base_opacity.reshape(-1), "base_opacity")
    u = _f32c(u.reshape(-1), "u")
    if campos.numel() != 3 or u.numel() != 1 or base_opacity.numel() != n:
        raise ValueError("campos must be 3 floats, u one float and base_opacity [N]")
    if bbox is not None:
        bbox = _f32c(bbox.reshape(-1), "bbox")
        if bbox.numel() != 6:
            raise ValueError("bbox must be 6 floats: the minimum, then the size")
    b0 = torch.addmv(biases[0], weights[0][:, in_dim:in_dim + e], embedding)
    params = []
    for l, (w, b) in enumerate(zip(weights, biases)):
        params += [_f32c(w, "weight"), _f32c(b0 if l == 0 else b, "bias")]
    cfg = (g, degree, split, stride, in_dim, row, float(temperature), float(eps))
    return _SwagColoursAndOpacities.apply(cfg, means, campos, shs, shs_rest, bbox, table, base_opacity, u, *params)


# ---- 4DGS deformation (csrc/gs4d.cu K51/K52): forward only ------------------------------------------------------------------------
GS4D_FWD_LAUNCHES = 1           # library launches of one gs4d_deform (K51)
GS4D_HEADS = ("dx", "ds", "dr", "dshs")
GS4D_HEAD_OUT = {"dx": 3, "ds": 3, "dr": 4, "dshs": 48}
GS4D_SUPPORTED = ("grid_dimensions 2 and input_coordinate_dim 4, output_coordinate_dim 16 or 32, 1..4 levels (multires), every plane "
                  "resolution 1..16384 with each plane below 2^31 floats, net_width 64 or 128, defor_depth 0..2, any combination of "
                  "no_dx / no_ds / no_dr / no_dshs / apply_rotation, and no_grid, static_mlp and empty_voxel off with grid_pe 0")


def _gs4d_struct(n_levels, channels, net_width, defor_depth, flags, resolution) -> _lib.B200gsGs4d:
    g = _lib.B200gsGs4d()
    g.n_levels, g.channels, g.net_width, g.defor_depth, g.flags = int(n_levels), int(channels), int(net_width), int(defor_depth), int(flags)
    for l, r in enumerate(resolution[:4]):
        for d in range(4):
            g.resolution[l][d] = int(r[d])
    return g


def gs4d_supported(n_levels: int, channels: int, net_width: int, defor_depth: int, resolution=None) -> bool:
    """Whether K51 takes this HexPlane field and network (no device needed).  ``resolution``: per level the (x, y, z, t) nodes
    (None: 64, 64, 64, 25 at every level)."""
    if resolution is None:
        resolution = [(64, 64, 64, 25)] * max(int(n_levels), 0)
    if len(resolution) != int(n_levels):
        return False
    return int(lib().b200gs_gs4d_plane_floats(ctypes.byref(_gs4d_struct(n_levels, channels, net_width, defor_depth, 0, resolution)))) > 0


class Gs4dPlanes:
    """A HexPlane field repacked channel-last by K52: ``planes`` float32 [b200gs_gs4d_plane_floats], ``resolution`` the (x, y, z, t)
    nodes of each level, ``channels`` C.  Made by ``gs4d_repack_planes``; read by every ``gs4d_deform`` call."""

    def __init__(self, planes: torch.Tensor, resolution, channels: int):
        self.planes, self.resolution, self.channels = planes, [tuple(r) for r in resolution], int(channels)

    @property
    def n_levels(self) -> int:
        return len(self.resolution)


def gs4d_repack_planes(grids) -> Gs4dPlanes:
    """Repack the reference's ``HexPlaneField.grids`` (L levels of 6 planes [1, C, res_b, res_a], plane k = (a, b) of (0,1), (0,2),
    (0,3), (1,2), (1,3), (2,3)) into K51's channel-last layout, once per model (K52, one launch).  The planes are only read."""
    grids = [list(level) for level in grids]
    if not 1 <= len(grids) <= 4:
        raise NotImplementedError(f"{len(grids)} HexPlane levels (multires) is not supported: b200gs 4DGS takes {GS4D_SUPPORTED}")
    channels, resolution, flat = None, [], []
    for level in grids:
        if len(level) != 6:
            raise NotImplementedError(f"a level of {len(level)} planes is not supported (grid_dimensions 2, input_coordinate_dim 4 give 6)")
        if any(p.dim() != 4 or p.shape[0] != 1 for p in level):
            raise ValueError("every plane must be [1, C, res_b, res_a]")
        c = int(level[0].shape[1])
        channels = c if channels is None else channels
        r = (int(level[0].shape[3]), int(level[0].shape[2]), int(level[1].shape[2]), int(level[2].shape[2]))
        for (a, b), p in zip(((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)), level):
            if tuple(p.shape[1:]) != (channels, r[b], r[a]):
                raise ValueError(f"plane ({a},{b}) is {tuple(p.shape)}, expected [1, {channels}, {r[b]}, {r[a]}]")
            flat.append(_f32c(p.detach(), "plane"))
        resolution.append(r)
    g = _gs4d_struct(len(grids), channels, 64, 0, 0, resolution)
    total = int(lib().b200gs_gs4d_plane_floats(ctypes.byref(g)))
    if total == 0:
        raise NotImplementedError(f"HexPlane field with output_coordinate_dim {channels} and resolutions {resolution} is not supported: "
                                  f"b200gs 4DGS takes {GS4D_SUPPORTED}")
    planes = torch.empty(total, dtype=torch.float32, device=flat[0].device)
    src = (ctypes.c_void_p * len(flat))(*[p.data_ptr() for p in flat])
    check(lib().b200gs_gs4d_repack_planes(ctypes.byref(g), src, ptr(planes), _stream()), "b200gs_gs4d_repack_planes")
    return Gs4dPlanes(planes, resolution, channels)


def _aligned16(t: torch.Tensor) -> torch.Tensor:
    return t if t.data_ptr() % 16 == 0 else t.clone()


def gs4d_deform(means: torch.Tensor, log_scales: torch.Tensor, quats: torch.Tensor, time, planes: Gs4dPlanes, aabb: torch.Tensor,
                trunk, heads, *, shs_dc: Optional[torch.Tensor] = None, shs_rest: Optional[torch.Tensor] = None,
                apply_rotation: bool = False):
    """The 4DGS deformation of VanillaGS4DRenderer.forward (Deformation.forward_dynamic with mask 1) in one kernel (K51), forward only:
    returns ``(means', log_scales', quats', shs_dc', shs_rest')`` of the raw parameters ``means`` / ``log_scales`` [N,3] and ``quats``
    [N,4] (not normalised) at time ``time`` (a float or a one-element tensor, used as given).

    ``planes``: the repacked HexPlane field (``gs4d_repack_planes``); ``aabb`` [2, 3]: the reference's ``grid.aabb`` (row 0 xyz_max,
    row 1 xyz_min).  ``trunk``: the (weight, bias) of ``feature_out``'s Linear layers (one, or two for defor_depth 2); ``heads``: for
    each enabled head of ``GS4D_HEADS`` its ((hidden weight, bias), (output weight, bias)).  A head left out is off (no_dx ...): its
    parameter passes through.  With ``dshs`` on, ``shs_dc`` [N,1,3] and ``shs_rest`` [N,15,3] get dshs; otherwise they are returned
    as they are.  ``apply_rotation``: quats' = normalize(quats * dr) instead of quats + dr.

    There is no autograd node: while grad is enabled, an input that requires grad raises.  Shapes outside ``GS4D_SUPPORTED`` raise
    NotImplementedError."""
    heads = dict(heads)
    unknown = set(heads) - set(GS4D_HEADS)
    if unknown:
        raise ValueError(f"unknown heads {sorted(unknown)}: the heads are {GS4D_HEADS}")
    trunk = list(trunk)
    tensors = [means, log_scales, quats, aabb, shs_dc, shs_rest, planes.planes, time] + [t for wb in trunk for t in wb] + \
        [t for h in heads.values() for wb in h for t in wb]
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in tensors):
        raise RuntimeError("ops.gs4d_deform is forward only (the 4DGS deformation has no autograd node) and an input requires grad: "
                           "call it under torch.no_grad() or pass detached tensors")
    n = means.shape[0]
    if means.dim() != 2 or means.shape[1] != 3 or log_scales.shape != (n, 3) or quats.shape != (n, 4):
        raise ValueError("expected means [N,3], log_scales [N,3] and quats [N,4]")
    if not 1 <= len(trunk) <= 2:
        raise NotImplementedError(f"a trunk of {len(trunk)} Linear layers is not supported (defor_depth 0..2): b200gs 4DGS takes "
                                  f"{GS4D_SUPPORTED}")
    width, k0 = int(trunk[0][0].shape[0]), planes.channels * planes.n_levels
    if width not in (64, 128):
        raise NotImplementedError(f"net_width {width} is not supported: b200gs 4DGS takes {GS4D_SUPPORTED}")
    g = _gs4d_struct(planes.n_levels, planes.channels, width, len(trunk), 0, planes.resolution)
    keep = []

    def layer(i, wb, rows, cols, what):
        w, b = wb
        if tuple(w.shape) != (rows, cols) or tuple(b.shape) != (rows,):
            raise ValueError(f"{what} must be a Linear({cols}, {rows}), got weight {tuple(w.shape)} and bias {tuple(b.shape)}")
        w, b = _aligned16(_f32c(w.detach(), what)), _f32c(b.detach(), what)
        keep.extend((w, b))
        g.weights[i], g.biases[i] = w.data_ptr(), b.data_ptr()

    layer(0, trunk[0], width, k0, "the first trunk layer")
    if len(trunk) == 2:
        layer(1, trunk[1], width, width, "the second trunk layer")
    for h, name in enumerate(GS4D_HEADS):
        if name in heads:
            g.flags |= 1 << h
            hidden, out = heads[name]
            layer(2 + 2 * h, hidden, width, width, f"the {name} head's hidden layer")
            layer(3 + 2 * h, out, GS4D_HEAD_OUT[name], width, f"the {name} head's output layer")
    if apply_rotation:
        g.flags |= 16
    if int(lib().b200gs_gs4d_plane_floats(ctypes.byref(g))) != planes.planes.numel():
        raise NotImplementedError(f"net_width {width} with defor_depth {len(trunk)} on {planes.n_levels} levels of "
                                  f"{planes.channels} channels is not supported: b200gs 4DGS takes {GS4D_SUPPORTED}")
    dev = means.device
    means, log_scales = _f32c(means.detach(), "means"), _f32c(log_scales.detach(), "log_scales")
    quats = _aligned16(_f32c(quats.detach(), "quats"))
    aabb = _f32c(aabb.detach().reshape(-1), "aabb")
    if aabb.numel() != 6:
        raise ValueError("aabb must be [2, 3]: xyz_max, then xyz_min")
    t = time.detach().reshape(-1).to(device=dev, dtype=torch.float32) if isinstance(time, torch.Tensor) else \
        torch.tensor([float(time)], dtype=torch.float32).to(dev, non_blocking=True)
    if t.numel() != 1:
        raise ValueError("time must be one value")
    if planes.planes.device != dev:
        raise ValueError("planes must be on the means' device")
    dshs = "dshs" in heads
    if dshs:
        if shs_dc is None or shs_rest is None or shs_dc.shape != (n, 1, 3) or shs_rest.shape != (n, 15, 3):
            raise ValueError("the dshs head needs shs_dc [N,1,3] and shs_rest [N,15,3] (SH degree 3: 16 coefficients)")
        shs_dc, shs_rest = _f32c(shs_dc.detach(), "shs_dc"), _f32c(shs_rest.detach(), "shs_rest")
    means_out, scales_out = torch.empty_like(means), torch.empty_like(log_scales)
    quats_out = torch.empty_like(quats)
    dc_out, rest_out = (torch.empty_like(shs_dc), torch.empty_like(shs_rest)) if dshs else (shs_dc, shs_rest)
    check(lib().b200gs_gs4d_deform_fwd(ctypes.byref(g), n, ptr(planes.planes), ptr(aabb), ptr(t), ptr(means), ptr(log_scales), ptr(quats),
                                       ptr(shs_dc) if dshs else None, ptr(shs_rest) if dshs else None, ptr(means_out), ptr(scales_out),
                                       ptr(quats_out), ptr(dc_out) if dshs else None, ptr(rest_out) if dshs else None, _stream()),
          "b200gs_gs4d_deform_fwd")
    return means_out, scales_out, quats_out, dc_out, rest_out
