"""CPU oracle for the differentiable 3D-Gaussian rasterizer hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` may be imported by the product package
(``gaussian-splatting-lightning_b200`` / ``b200gs``); only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs use it, and only as the checker / the CPU timing arm.

What it restates (all citations relative to the reference repository):

* projection / EWA / blur / compensation / conic / radius / tile rect in "gsplat" constants:
  ``internal/utils/gaussian_projection.py:6-138`` (cov3D ``:235-254``, rotation ``:211-232``, cov2D ``:257-287``).
  PINNED: ``tests/golden/*.npz`` hold outputs and autograd gradients of that very file, imported from the
  reference in the authoring container by ``tests/golden/make_golden.py``; ``tests/test_oracle_golden.py`` checks
  this restatement against them, and against the known-answer fixture of ``tests/gaussian_projection_test.py:30-113``.
* SH evaluation: ``internal/utils/sh_utils.py:57-112`` (constants ``:26-54``).  PINNED the same way.
* (tile | depth) sort keys: ``internal/utils/gaussian_projection.py:173-208``.  PINNED the same way.
* camera conventions: ``internal/cameras/cameras.py:142-192``.
* "vanilla" constants (diff-gaussian-rasterization@59f5f77, the backend of ``internal/renderers/vanilla_renderer.py:62-120``)
  and the alpha-blend forward for both modes: the arithmetic lives in pip git dependencies that are NOT under
  the reference repository (``requirements/common.txt:10``, ``requirements/gsplat.txt:1``) and are not installable offline.
  They are restated here from their published algorithm (SURVEY.md §8c constant table, Appendix B).
  **PARITY UNPINNED** for: vanilla-mode projection constants, blend forward, blend backward.  The backward of
  everything is obtained by torch autograd through this differentiable restatement (sort order and the
  alpha<1/255, T<1e-4, power>0 branches are piecewise constant), so it is an independent check of the
  hand-derived CUDA backward.

All functions are dtype-generic (float32 mimics the reference's arithmetic; float64 gives a tighter truth).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch

MODE_VANILLA = 0
MODE_GSPLAT = 1

BLOCK = 16

# --------------------------------------------------------------------------------------------------------------------
# SH  (internal/utils/sh_utils.py:26-112)
# --------------------------------------------------------------------------------------------------------------------
C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435]
C4 = [2.5033429417967046, -1.7701307697799304, 0.9461746957575601, -0.6690465435572892, 0.10578554691520431,
      -0.6690465435572892, 0.47308734787878004, -1.7701307697799304, 0.6258357354491761]


def sh_basis(deg: int, dirs: torch.Tensor) -> torch.Tensor:
    """[N,3] unit dirs -> [N,(deg+1)^2] real SH basis with the signs of sh_utils.py:74-111."""
    assert 0 <= deg <= 4
    x, y, z = dirs[:, 0], dirs[:, 1], dirs[:, 2]
    b = [torch.full_like(x, C0)]
    if deg > 0:
        b += [-C1 * y, C1 * z, -C1 * x]
    if deg > 1:
        xx, yy, zz = x * x, y * y, z * z
        xy, yz, xz = x * y, y * z, x * z
        b += [C2[0] * xy, C2[1] * yz, C2[2] * (2.0 * zz - xx - yy), C2[3] * xz, C2[4] * (xx - yy)]
    if deg > 2:
        b += [C3[0] * y * (3 * xx - yy), C3[1] * xy * z, C3[2] * y * (4 * zz - xx - yy),
              C3[3] * z * (2 * zz - 3 * xx - 3 * yy), C3[4] * x * (4 * zz - xx - yy),
              C3[5] * z * (xx - yy), C3[6] * x * (xx - 3 * yy)]
    if deg > 3:
        b += [C4[0] * xy * (xx - yy), C4[1] * yz * (3 * xx - yy), C4[2] * xy * (7 * zz - 1),
              C4[3] * yz * (7 * zz - 3), C4[4] * (zz * (35 * zz - 30) + 3), C4[5] * xz * (7 * zz - 3),
              C4[6] * (xx - yy) * (7 * zz - 1), C4[7] * xz * (xx - 3 * yy),
              C4[8] * (xx * (xx - 3 * yy) - yy * (3 * xx - yy))]
    return torch.stack(b, dim=-1)


def eval_sh(deg: int, shs: torch.Tensor, dirs: torch.Tensor) -> torch.Tensor:
    """shs [N,K,3] (the layout of GaussianModel.get_features, models/gaussian.py:250-254), unit dirs [N,3] -> [N,3].

    Same polynomial as sh_utils.eval_sh (which takes [N,3,K]); no +0.5, no clamp.
    """
    basis = sh_basis(deg, dirs)  # [N,k]
    k = basis.shape[-1]
    return (basis[:, :, None] * shs[:, :k, :]).sum(dim=1)


def sh_colors(deg: int, shs: torch.Tensor, means: torch.Tensor, campos: torch.Tensor, detach_dir: bool) -> torch.Tensor:
    """colour = max(SH(dir)+0.5, 0).  vanilla: dir differentiable (dgr computeColorFromSH); gsplat renderers
    detach it (gsplat_renderer.py:104, pypreprocess_gsplat_renderer.py:35-36)."""
    d = (means.detach() if detach_dir else means) - campos[None, :]
    d = d / d.norm(dim=-1, keepdim=True)
    return torch.clamp_min(eval_sh(deg, shs, d) + 0.5, 0.0)


# --------------------------------------------------------------------------------------------------------------------
# camera  (internal/cameras/cameras.py:142-192)
# --------------------------------------------------------------------------------------------------------------------
@dataclass
class View:
    width: int
    height: int
    fx: float
    fy: float
    cx: float
    cy: float
    world_to_camera: torch.Tensor  # [4,4] transposed: translation in the last row (cameras.py:147-153)
    full_projection: torch.Tensor  # [4,4] = world_to_camera @ P^T            (cameras.py:164-189)
    camera_center: torch.Tensor  # [3]                                       (cameras.py:191-192)
    tanfovx: float
    tanfovy: float

    def to(self, dtype):
        return View(self.width, self.height, self.fx, self.fy, self.cx, self.cy, self.world_to_camera.to(dtype),
                    self.full_projection.to(dtype), self.camera_center.to(dtype), self.tanfovx, self.tanfovy)


def make_view(R: torch.Tensor, T: torch.Tensor, fx: float, fy: float, cx: float, cy: float, width: int, height: int) -> View:
    """Build the derived camera quantities exactly as Cameras.__post_init__ does (float32 arithmetic)."""
    R = R.to(torch.float32)
    T = T.to(torch.float32)
    fx_t = torch.tensor(fx, dtype=torch.float32)
    fy_t = torch.tensor(fy, dtype=torch.float32)
    w_t = torch.tensor(width, dtype=torch.int32)
    h_t = torch.tensor(height, dtype=torch.int32)
    fov_x = 2 * torch.atan((w_t / 2) / fx_t)
    fov_y = 2 * torch.atan((h_t / 2) / fy_t)
    w2c = torch.zeros(4, 4)
    w2c[:3, :3] = R
    w2c[:3, 3] = T
    w2c[3, 3] = 1.0
    w2c = w2c.T.contiguous()
    zfar, znear = 100.0, 0.01
    tan_y = torch.tan(fov_y / 2)
    tan_x = torch.tan(fov_x / 2)
    top = tan_y * znear
    bottom = -top
    right = tan_x * znear
    left = -right
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (right - left)
    P[1, 1] = 2.0 * znear / (top - bottom)
    P[0, 2] = (right + left) / (right - left)
    P[1, 2] = (top + bottom) / (top - bottom)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    full = w2c @ P.T
    center = torch.linalg.inv(w2c)[3, :3]
    return View(int(width), int(height), float(fx_t), float(fy_t), float(cx), float(cy), w2c, full.contiguous(),
                center.contiguous(), math.tan(float(fov_x) * 0.5), math.tan(float(fov_y) * 0.5))


# --------------------------------------------------------------------------------------------------------------------
# projection
# --------------------------------------------------------------------------------------------------------------------
def build_rotation_matrix(q: torch.Tensor) -> torch.Tensor:
    """gaussian_projection.py:211-232 — wxyz, used as given (no normalisation)."""
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    rows = [
        1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y),
    ]
    return torch.stack(rows, dim=-1).reshape(-1, 3, 3)


def compute_cov_3d(scales: torch.Tensor, scale_modifier: float, quats: torch.Tensor) -> torch.Tensor:
    """gaussian_projection.py:235-254 — Sigma = (R S)(R S)^T."""
    Rm = build_rotation_matrix(quats)
    M = Rm * (scales * scale_modifier)[:, None, :]
    return M @ M.transpose(1, 2)


def compute_cov_2d(t, tan_fovx, tan_fovy, focal_x, focal_y, cov_3d, world_to_camera, dgr_clamp_grad: bool = False) -> torch.Tensor:
    """gaussian_projection.py:257-287 (same arithmetic as dgr computeCov2D before the +0.3).

    dgr_clamp_grad: the published dgr backward (computeCov2DCUDA) zeroes dL/dt_x when the +-1.3 tan(fov) clamp is active
    and does NOT propagate the clamped value's dependence on t_z; torch.clamp autograd (gsplat mode / the reference's
    python) does.  Forward values are identical."""
    limx = 1.3 * tan_fovx
    limy = 1.3 * tan_fovy
    txtz = t[:, 0] / t[:, 2]
    tytz = t[:, 1] / t[:, 2]
    cx_ = torch.clamp(txtz, min=-limx, max=limx) * t[:, 2]
    cy_ = torch.clamp(tytz, min=-limy, max=limy) * t[:, 2]
    if dgr_clamp_grad:
        cx_ = torch.where((txtz < -limx) | (txtz > limx), cx_.detach(), cx_)
        cy_ = torch.where((tytz < -limy) | (tytz > limy), cy_.detach(), cy_)
    tz = t[:, 2]
    zero = torch.zeros_like(tz)
    J = torch.stack([
        focal_x / tz, zero, -(focal_x * cx_) / (tz * tz),
        zero, focal_y / tz, -(focal_y * cy_) / (tz * tz),
        zero, zero, zero], dim=-1).reshape(-1, 3, 3)
    Wm = world_to_camera[:3, :3].T
    Tm = J @ Wm[None]
    cov = Tm @ cov_3d @ Tm.transpose(1, 2)
    return cov[:, :2, :2]


def _extent_from_cov(a, b, c, det):
    """3 sqrt(largest eigenvalue): the radius before it is rounded up to whole pixels."""
    mid = 0.5 * (a + c)
    sq = torch.sqrt(torch.clamp_min(mid * mid - det, 0.1))  # gaussian_projection.py:98-105 / dgr max(0.1, ...)
    lam = torch.maximum(mid + sq, mid - sq)
    return 3.0 * torch.sqrt(lam)


def _radius_from_cov(a, b, c, det):
    return torch.ceil(_extent_from_cov(a, b, c, det)).to(torch.int32)


def project(mode: int, means: torch.Tensor, scales: torch.Tensor, quats: torch.Tensor, view: View,
            scale_modifier: float = 1.0, eps2d: float = 0.3, block: int = BLOCK,
            min_depth: Optional[float] = None) -> Dict[str, torch.Tensor]:
    """Per-Gaussian projection.  Returns a dict of (differentiable where it makes sense) tensors:

    xy [N,2] pixel coordinates (vanilla: ((ndc+1)S-1)/2, i.e. pixel-index space; gsplat: K t/(t_z+1e-6), no +0.5),
    depth [N], radii int32 [N], conic [N,3], comp [N] (gsplat; ones in vanilla), tiles int32 [N],
    rect_min / rect_max int32 [N,2], mask bool [N], cov3d [N,3,3].  Entries of culled Gaussians are zero.
    Unmasked, for tests that keep their scenes away from the culling decisions: t [N,3] camera-space means,
    xy_all [N,2], extent [N] (3 sqrt(largest eigenvalue), the radius before it is rounded up).
    """
    dt = means.dtype
    v = view.to(dt)
    W2C = v.world_to_camera
    t = means @ W2C[:3, :3] + W2C[3, :3]
    cov3d = compute_cov_3d(scales, scale_modifier, quats)
    grid_x = (v.width + block - 1) // block
    grid_y = (v.height + block - 1) // block

    if mode == MODE_GSPLAT:
        # gaussian_projection.py:41-136
        near = 0.01 if min_depth is None else min_depth
        with torch.no_grad():
            front = t[:, 2] >= near
        tanx = (0.5 * v.width) / v.fx
        tany = (0.5 * v.height) / v.fy
        cov2d = compute_cov_2d(t, tanx, tany, v.fx, v.fy, cov3d, W2C)
        det0 = cov2d[:, 0, 0] * cov2d[:, 1, 1] - cov2d[:, 0, 1] * cov2d[:, 1, 0]
        a = cov2d[:, 0, 0] + eps2d
        b = cov2d[:, 0, 1]
        b2 = cov2d[:, 1, 0]
        c = cov2d[:, 1, 1] + eps2d
        det = a * c - b * b2
        comp = torch.sqrt(torch.clamp_min(det0 / det, 0.0))
        inv = 1.0 / det
        conic = torch.stack([c * inv, -b * inv, a * inv], dim=-1)
        pn = t / (t[:, 2:] + 1e-6)
        xy = torch.stack([pn[:, 0] * v.fx + pn[:, 2] * v.cx, pn[:, 1] * v.fy + pn[:, 2] * v.cy], dim=-1)
        radius = _radius_from_cov(a, b, c, det)
        with torch.no_grad():
            rf = radius.to(dt)[:, None]
            rmin = ((xy - rf) / block).to(torch.int32)
            rmax = ((xy + rf) / block).to(torch.int32) + 1
            det_ok = torch.ones_like(front)
    else:
        # diff-gaussian-rasterization@59f5f77 preprocessCUDA (PARITY UNPINNED; SURVEY §8c constant table)
        with torch.no_grad():
            front = t[:, 2] > 0.2
        FP = v.full_projection
        ph = means @ FP[:3, :] + FP[3, :]
        pw = 1.0 / (ph[:, 3] + 1e-7)
        ndc = ph[:, :2] * pw[:, None]
        focal_x = v.width / (2.0 * v.tanfovx)
        focal_y = v.height / (2.0 * v.tanfovy)
        cov2d = compute_cov_2d(t, v.tanfovx, v.tanfovy, focal_x, focal_y, cov3d, W2C, dgr_clamp_grad=True)
        a = cov2d[:, 0, 0] + 0.3
        b = cov2d[:, 0, 1]
        c = cov2d[:, 1, 1] + 0.3
        det = a * c - b * b
        with torch.no_grad():
            det_ok = det != 0
        inv = 1.0 / det
        conic = torch.stack([c * inv, -b * inv, a * inv], dim=-1)
        comp = torch.ones_like(det)
        S = torch.tensor([v.width, v.height], dtype=dt)
        xy = ((ndc + 1.0) * S - 1.0) * 0.5
        radius = _radius_from_cov(a, b, c, det)
        with torch.no_grad():
            rf = radius.to(dt)[:, None]
            rmin = ((xy - rf) / block).to(torch.int32)
            rmax = ((xy + rf + (block - 1)) / block).to(torch.int32)

    with torch.no_grad():
        g = torch.tensor([grid_x, grid_y], dtype=torch.int32)
        rmin = torch.minimum(torch.clamp_min(rmin, 0), g)
        rmax = torch.minimum(torch.clamp_min(rmax, 0), g)
        d = rmax - rmin
        tiles = d[:, 0] * d[:, 1]
        mask = front & det_ok & (tiles > 0)
    inv_mask = ~mask
    z = torch.zeros((), dtype=dt)
    return {
        "xy": torch.where(inv_mask[:, None], z, xy),
        "depth": torch.where(inv_mask, z, t[:, 2]),
        "radii": torch.where(inv_mask, torch.zeros((), dtype=torch.int32), radius),
        "conic": torch.where(inv_mask[:, None], z, conic),
        "comp": torch.where(inv_mask, z, comp),
        "tiles": torch.where(inv_mask, torch.zeros((), dtype=torch.int32), tiles),
        "cov3d": torch.where(inv_mask[:, None, None], z, cov3d),
        "mask": mask,
        "rect_min": rmin,
        "rect_max": rmax,
        "t": t,
        "xy_all": xy,
        "extent": _extent_from_cov(a, b, c, det),
    }


# --------------------------------------------------------------------------------------------------------------------
# binning  (gaussian_projection.py:173-208, vectorised; sort = what cub::DeviceRadixSort::SortPairs does: stable)
# --------------------------------------------------------------------------------------------------------------------
def build_sort_keys(depth: torch.Tensor, rect_min: torch.Tensor, rect_max: torch.Tensor, tiles: torch.Tensor,
                    grid_x: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """key = (tile_id << 32) | bitcast<int32>(float32 depth), emitted Gaussian-major, row-major inside the rect."""
    n = depth.shape[0]
    tiles = tiles.to(torch.int64)
    ids = torch.repeat_interleave(torch.arange(n, dtype=torch.int64), tiles)
    total = int(tiles.sum())
    if total == 0:
        return torch.zeros(0, dtype=torch.int64), torch.zeros(0, dtype=torch.int32)
    start = torch.cumsum(tiles, 0) - tiles
    local = torch.arange(total, dtype=torch.int64) - start[ids]
    w = (rect_max[:, 0] - rect_min[:, 0]).to(torch.int64)[ids]
    ty = rect_min[:, 1].to(torch.int64)[ids] + local // w
    tx = rect_min[:, 0].to(torch.int64)[ids] + local % w
    tile_id = ty * grid_x + tx
    dbits = depth.detach().to(torch.float32).contiguous().view(torch.int32).to(torch.int64)[ids]
    return (tile_id << 32) | dbits, ids.to(torch.int32)


def sort_and_ranges(keys: torch.Tensor, ids: torch.Tensor, n_tiles: int):
    """Stable sort by key; ranges[t] = [start, end) of tile t in the sorted list."""
    if keys.numel() == 0:
        return keys, ids, torch.zeros(n_tiles, 2, dtype=torch.int64)
    skeys, perm = torch.sort(keys, stable=True)
    sids = ids[perm]
    tile_of = skeys >> 32
    counts = torch.bincount(tile_of, minlength=n_tiles)
    end = torch.cumsum(counts, 0)
    start = end - counts
    return skeys, sids, torch.stack([start, end], dim=-1)


# --------------------------------------------------------------------------------------------------------------------
# blend  (PARITY UNPINNED: restated from the published dgr / gsplat kernels; SURVEY Appendix B)
# --------------------------------------------------------------------------------------------------------------------
def blend(mode: int, xy: torch.Tensor, conic: torch.Tensor, opacity: torch.Tensor, colors: torch.Tensor,
          sorted_ids: torch.Tensor, ranges: torch.Tensor, bg: Optional[torch.Tensor], width: int, height: int,
          block: int = BLOCK, margins: Optional[list] = None, side: Optional[dict] = None):
    """Per-tile front-to-back compositing.  xy [N,2], conic [N,3], opacity [N], colors [N,D].

    Returns image [D,H,W], alpha [H,W] (= 1 - T_final), n_contrib int32 [H,W] (1-based index, inside the tile's
    list, of the last splat that contributed — dgr's n_contrib), all on CPU.  Differentiable wrt xy/conic/opacity/colors.

    margins: pass an empty list to receive ONE [H,W] tensor: per pixel, the smallest relative distance of any of its
    (pixel, splat) samples to a branch threshold of the loop (alpha vs 1/255, remaining T vs 1e-4, power vs 0, alpha vs the
    clamp of the gsplat backward).  A sample closer to a threshold than fp32 resolves may take the other branch in a
    float32 implementation; tests use this map to tell such pixels from real errors.

    side: pass an empty dict to receive the side channels below; the returned values are the same with or without it.
      "hit"         bool [N]: the splat is active (weight a * T_excl > 0) in at least one pixel: gsplat's has_hit_any_pixels.
      "hit_margin"  [N]: how far "hit" is from flipping, in the units of `margins`.  A splat that is hit stays hit while one of
                    its active samples keeps its branches: the largest margin of its active samples.  A splat that is not
                    hit becomes hit if any sample the loop reaches flips: the smallest margin of those (inf when no pixel
                    reaches it).  An fp32 implementation can only disagree with "hit" where this is small.  A pixel whose
                    stop is ambiguous does not lower the margin of the splats behind it: if fp32 keeps it alive, the next
                    valid sample (alpha >= 1/255) takes T below the cut-off and stops it with weight 0.
      "stopped"     bool [H,W]: the pixel stopped at the 1e-4 transmittance cut-off.
      "clamped"     int: the number of active samples whose alpha sits at the clamp (0.999 / 0.99).
      "abs_terms"   list of (ids [L], dx [P,L], dy [P,L]) per non-empty tile: mean - pixel centre of every (pixel, splat) sample
                    of the tile's list.  When xy requires grad they retain their gradient: after backward(), dx.grad[p, j] is
                    pixel p's own contribution to the x gradient of splat ids[j], and absgrad() sums their magnitudes.
    """
    dt = xy.dtype
    D = colors.shape[1]
    gx = (width + block - 1) // block
    gy = (height + block - 1) // block
    off = 0.5 if mode == MODE_GSPLAT else 0.0
    amax = 0.999 if mode == MODE_GSPLAT else 0.99
    img = torch.zeros(height, width, D, dtype=dt)
    alpha_img = torch.zeros(height, width, dtype=dt)
    ncontrib = torch.zeros(height, width, dtype=torch.int32)
    if side is not None:
        n_splats = xy.shape[0]
        side["hit"] = torch.zeros(n_splats, dtype=torch.bool)
        side["hit_margin"] = torch.full((n_splats,), float("inf"), dtype=dt)
        witness = torch.full((n_splats,), float("-inf"), dtype=dt)
        side["clamped"] = 0
        side["abs_terms"] = []
        stopped_rows = []
    img_rows = []
    for ty in range(gy):
        row_tiles = []
        for tx in range(gx):
            s, e = int(ranges[ty * gx + tx, 0]), int(ranges[ty * gx + tx, 1])
            x0, y0 = tx * block, ty * block
            x1, y1 = min(x0 + block, width), min(y0 + block, height)
            px = torch.arange(x0, x1, dtype=dt) + off
            py = torch.arange(y0, y1, dtype=dt) + off
            PX = px[None, :].expand(y1 - y0, x1 - x0).reshape(-1)
            PY = py[:, None].expand(y1 - y0, x1 - x0).reshape(-1)
            npx = PX.shape[0]
            tile_margin = torch.full((npx,), float("inf"), dtype=dt)
            stopped = torch.zeros(npx, dtype=torch.bool)
            if e <= s:
                C = torch.zeros(npx, D, dtype=dt)
                Tf = torch.ones(npx, dtype=dt)
                last = torch.zeros(npx, dtype=torch.int32)
            else:
                gid = sorted_ids[s:e].to(torch.int64)
                mxy, con, op, col = xy[gid], conic[gid], opacity[gid], colors[gid]
                dx = mxy[None, :, 0] - PX[:, None]
                dy = mxy[None, :, 1] - PY[:, None]
                if side is not None:
                    if dx.requires_grad:
                        dx.retain_grad()
                        dy.retain_grad()
                    side["abs_terms"].append((gid, dx, dy))
                power = -0.5 * (con[None, :, 0] * dx * dx + con[None, :, 2] * dy * dy) - con[None, :, 1] * dx * dy
                G = torch.exp(power)
                raw = op[None, :] * G
                if mode == MODE_GSPLAT:
                    a = torch.clamp(raw, max=amax)  # true clamp: no grad to geometry/opacity when saturated
                else:
                    a = raw + (torch.clamp(raw, max=amax) - raw).detach()  # dgr backward is straight-through
                with torch.no_grad():
                    valid = (power <= 0) & (a >= 1.0 / 255.0)
                    a_eff = torch.where(valid, a, torch.zeros((), dtype=dt))
                    testT = torch.cumprod(1.0 - a_eff, dim=1)
                    alive = (testT > 1e-4) if mode == MODE_GSPLAT else (testT >= 1e-4)
                    active = valid & alive
                    if margins is not None or side is not None:
                        reach = torch.cat([torch.ones(npx, 1, dtype=torch.bool), alive[:, :-1]], dim=1)   # the sample is evaluated at all
                        big = torch.full((), float("inf"), dtype=dt)
                        m_alpha = torch.where(reach & (power <= 0), (raw - 1.0 / 255.0).abs() * 255.0, big)
                        m_T = torch.where(reach & valid, (testT - 1e-4).abs() / 1e-4, big)
                        m_pow = torch.where(reach, power.abs() / 1e-3, big)          # power > 0 is skipped: absolute scale 1e-3
                        m_clamp = torch.where(reach & valid, (raw - amax).abs() / amax, big)
                        m_sample = torch.minimum(torch.minimum(m_alpha, m_T), torch.minimum(m_pow, m_clamp))
                        tile_margin = m_sample.min(dim=1).values
                    if side is not None:
                        stopped = (reach & valid & ~alive).any(dim=1)
                        witness.scatter_reduce_(0, gid, torch.where(active, m_sample, -big).max(dim=0).values, "amax")
                        side["hit_margin"].scatter_reduce_(0, gid, m_sample.min(dim=0).values, "amin")
                        side["hit"][gid[active.any(dim=0)]] = True
                        side["clamped"] += int((active & (raw > amax)).sum())
                    idx = torch.arange(1, e - s + 1, dtype=torch.int32)[None, :].expand_as(active)
                    last = torch.where(active, idx, torch.zeros((), dtype=torch.int32)).max(dim=1).values
                a_act = torch.where(active, a, torch.zeros((), dtype=dt))
                one_m = 1.0 - a_act
                Tincl = torch.cumprod(one_m, dim=1)
                Texcl = torch.cat([torch.ones(npx, 1, dtype=dt), Tincl[:, :-1]], dim=1)
                w = a_act * Texcl
                C = w @ col
                Tf = Tincl[:, -1]
            if bg is not None:
                C = C + Tf[:, None] * bg.to(dt)[None, :]
            row_tiles.append((C.reshape(y1 - y0, x1 - x0, D), (1.0 - Tf).reshape(y1 - y0, x1 - x0),
                              last.reshape(y1 - y0, x1 - x0), tile_margin.detach().reshape(y1 - y0, x1 - x0),
                              stopped.reshape(y1 - y0, x1 - x0)))
        img_rows.append(tuple(torch.cat([r[k] for r in row_tiles], dim=1) for k in range(5)))
    img = torch.cat([r[0] for r in img_rows], dim=0)
    alpha_img = torch.cat([r[1] for r in img_rows], dim=0)
    ncontrib = torch.cat([r[2] for r in img_rows], dim=0)
    if margins is not None:
        margins.append(torch.cat([r[3] for r in img_rows], dim=0))
    if side is not None:
        side["stopped"] = torch.cat([r[4] for r in img_rows], dim=0)
        side["hit_margin"] = torch.where(side["hit"], witness, side["hit_margin"])
    return img.permute(2, 0, 1), alpha_img, ncontrib


def absgrad(abs_terms: list, n: int) -> torch.Tensor:
    """gsplat's means2d.absgrad [n,2] from blend(side=...)["abs_terms"] after backward(): sum over pixels of |dL_pixel/dmean2d|."""
    out = torch.zeros(n, 2, dtype=torch.float64)
    for gid, dx, dy in abs_terms:
        if dx.grad is not None:
            out[:, 0].index_add_(0, gid, dx.grad.abs().sum(dim=0).to(out.dtype))
        if dy.grad is not None:
            out[:, 1].index_add_(0, gid, dy.grad.abs().sum(dim=0).to(out.dtype))
    return out


# --------------------------------------------------------------------------------------------------------------------
# full render
# --------------------------------------------------------------------------------------------------------------------
def render(mode: int, means: torch.Tensor, scales: torch.Tensor, quats: torch.Tensor, opacities: torch.Tensor,
           shs: Optional[torch.Tensor], view: View, bg: Optional[torch.Tensor], sh_degree: int = 3,
           scale_modifier: float = 1.0, colors_precomp: Optional[torch.Tensor] = None, anti_aliased: bool = True,
           eps2d: float = 0.3, margins: Optional[list] = None):
    """End-to-end oracle of VanillaRenderer.forward (vanilla_renderer.py:25-129) / GSPlatRenderer.forward's rgb path
    (gsplat_renderer.py:58-108) on activated parameters.  opacities [N,1] or [N]."""
    proj = project(mode, means, scales, quats, view, scale_modifier, eps2d)
    if colors_precomp is not None:
        colors = colors_precomp
    else:
        colors = sh_colors(sh_degree, shs, means, view.camera_center.to(means.dtype), detach_dir=(mode == MODE_GSPLAT))
    op = opacities.reshape(-1)
    if mode == MODE_GSPLAT and anti_aliased:
        op = op * proj["comp"]
    gx = (view.width + BLOCK - 1) // BLOCK
    gy = (view.height + BLOCK - 1) // BLOCK
    keys, ids = build_sort_keys(proj["depth"], proj["rect_min"], proj["rect_max"], proj["tiles"], gx)
    skeys, sids, ranges = sort_and_ranges(keys, ids, gx * gy)
    xy = proj["xy"]
    if xy.requires_grad:
        xy.retain_grad()
    img, alpha, ncontrib = blend(mode, xy, proj["conic"], op, colors, sids, ranges, bg, view.width, view.height, margins=margins)
    return {
        "render": img, "alpha": alpha, "n_contrib": ncontrib, "xy": xy, "radii": proj["radii"], "proj": proj,
        "colors": colors, "sorted_keys": skeys, "sorted_ids": sids, "ranges": ranges,
    }


def viewspace_grad(mode: int, xy_grad: torch.Tensor, width: int, height: int) -> torch.Tensor:
    """What the density controller reads from outputs["viewspace_points"].grad[:, :2]
    (vanilla_density_controller.py:101-123).  dgr stores dL/dmean2D in NDC-scaled units (pixel grad x 0.5W, 0.5H);
    gsplat stores pixel units and the renderer hands over viewspace_points_grad_scale (gsplat_renderer.py:198)."""
    if mode == MODE_VANILLA:
        return xy_grad * torch.tensor([0.5 * width, 0.5 * height], dtype=xy_grad.dtype)
    return xy_grad
