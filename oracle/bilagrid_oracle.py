"""float64 restatement of bilateral-grid slicing and its total variation (Wang et al., "Bilateral Guided Radiance Field
Processing", 2024), written from the contract of internal/output_processors/bilagrid.py and torch's grid_sample(mode='bilinear',
align_corners=True, padding_mode='border') on 5-D input:

  per pixel (x, y, rgb) of batch row b, with G = grids[grid_idx[b]] of shape (12, L, Hg, Wg):
      gray = rgb . w,  w = float32 (0.299, 0.587, 0.114)
      ix = ((2 (x - 0.5) + 1) / 2) (Wg - 1),  iy likewise with Hg,  iz = ((2 gray - 1 + 1) / 2) (L - 1)
      each clipped to [0, size - 1];  A[c] = sum over the 8 corners (z0 + kz, y0 + ky, x0 + kx) inside the grid of
      wx wy wz G[c, corner],  wx = 1 - fx or fx etc.;  out_i = sum_j A[4i + j] rgb_j + A[4i + 3]
  gradients: the grid of row b gets sum over its pixels of w_corner dL/dA[c]; rgb gets the affine part plus, through the guidance,
      dL/dgray = sum_c dL/dA[c] dA[c]/diz (L - 1), where a clipped iz (including one exactly on 0 or L - 1: grid_sample's border
      rule) passes nothing.  dA/diz is piecewise constant in iz: it jumps where iz crosses an integer, so a sample whose iz lies
      within a rounding error of an integer strictly inside the clip range is ambiguous between two values (``ambiguous``).
  total variation of grids (N, C, L, Hg, Wg):
      sum over the axes L, Hg, Wg of sum (x[.., i + 1, ..] - x[.., i, ..])^2 / max(numel per grid of the difference, 1), over N.
"""
import builtins

import numpy as np

GRAY_WEIGHTS = np.array([0.299, 0.587, 0.114], dtype=np.float32).astype(np.float64)


def _axis(coord, size):
    """unnormalised coordinate (unclipped), clipped coordinate, and 1 where the clip passes gradient"""
    i = ((coord + 1.0) / 2.0) * (size - 1)
    return i, np.clip(i, 0.0, size - 1), ((i > 0) & (i < size - 1)).astype(np.float64)


def _footprint(grids, xy, rgb, grid_idx):
    grids, xy, rgb = (np.asarray(a, np.float64) for a in (grids, xy, rgb))
    B, H, W = rgb.shape[:3]
    _, _, L, gh, gw = grids.shape
    idx = np.broadcast_to(np.asarray(grid_idx, np.int64).reshape(-1), (B,))
    g = np.repeat(idx, H * W)
    x, y, c = xy[..., 0].reshape(-1), xy[..., 1].reshape(-1), rgb.reshape(-1, 3)
    gray = c @ GRAY_WEIGHTS
    _, ix, _ = _axis((x - 0.5) * 2, gw)
    _, iy, _ = _axis((y - 0.5) * 2, gh)
    iz_raw, iz, zpass = _axis(gray * 2 - 1, L)
    lo = [np.floor(v).astype(np.int64) for v in (ix, iy, iz)]
    frac = [v - l for v, l in zip((ix, iy, iz), lo)]
    corners = []
    for k in range(8):
        kx, ky, kz = k & 1, (k >> 1) & 1, (k >> 2) & 1
        cx, cy, cz = lo[0] + kx, lo[1] + ky, lo[2] + kz
        inside = (cx < gw) & (cy < gh) & (cz < L)
        wxy = (frac[0] if kx else 1 - frac[0]) * (frac[1] if ky else 1 - frac[1])
        wz = frac[2] if kz else 1 - frac[2]
        corners.append((np.minimum(cx, gw - 1), np.minimum(cy, gh - 1), np.minimum(cz, L - 1), inside, wxy, wz, kz))
    return dict(grids=grids, g=g, rgb=c, corners=corners, iz_raw=iz_raw, zpass=zpass, L=L, shape=(B, H, W))


def _affine(fp):
    """A [P, 12] and dA/diz [P, 12]; corners outside the grid contribute nothing"""
    P = fp["g"].shape[0]
    A, dA = np.zeros((P, 12)), np.zeros((P, 12))
    valid = _valid(fp)
    g = np.where(valid, fp["g"], 0)
    for cx, cy, cz, inside, wxy, wz, kz in fp["corners"]:
        V = fp["grids"][g, :, cz, cy, cx] * inside[:, None]
        A += (wxy * wz)[:, None] * V
        dA += ((wxy if kz else -wxy))[:, None] * V
    return A, dA


def _valid(fp):
    return (fp["g"] >= 0) & (fp["g"] < fp["grids"].shape[0])


def slice(grids, xy, rgb, grid_idx):
    """out [B, H, W, 3]; a row whose grid index is out of range is NaN"""
    fp = _footprint(grids, xy, rgb, grid_idx)
    A, _ = _affine(fp)
    M = A.reshape(-1, 3, 4)
    out = np.einsum("pij,pj->pi", M[:, :, :3], fp["rgb"]) + M[:, :, 3]
    out[~_valid(fp)] = np.nan
    return out.reshape(*fp["shape"], 3)


def slice_vjp(grids, xy, rgb, grid_idx, v_out):
    """(v_grids [N, 12, L, Hg, Wg], v_rgb [B, H, W, 3]) for the cotangent v_out [B, H, W, 3]"""
    fp = _footprint(grids, xy, rgb, grid_idx)
    A, dA = _affine(fp)
    go = np.asarray(v_out, np.float64).reshape(-1, 3)
    r1 = np.concatenate([fp["rgb"], np.ones((go.shape[0], 1))], axis=1)
    dL_dA = (go[:, :, None] * r1[:, None, :]).reshape(-1, 12)         # c = 4 i + j
    dL_dgray = (dL_dA * dA).sum(1) * (fp["L"] - 1) * fp["zpass"]
    M = A.reshape(-1, 3, 4)
    v_rgb = np.einsum("pi,pij->pj", go, M[:, :, :3]) + dL_dgray[:, None] * GRAY_WEIGHTS[None, :]
    valid = _valid(fp)
    v_rgb[~valid] = np.nan
    N, _, L, gh, gw = fp["grids"].shape
    v_grids = np.zeros(fp["grids"].size)
    for cx, cy, cz, inside, wxy, wz, kz in fp["corners"]:
        m = inside & valid
        for c in range(12):
            flat = (((fp["g"][m] * 12 + c) * L + cz[m]) * gh + cy[m]) * gw + cx[m]
            v_grids += np.bincount(flat, weights=(wxy * wz * dL_dA[:, c])[m], minlength=v_grids.size)
    return v_grids.reshape(fp["grids"].shape), v_rgb.reshape(*fp["shape"], 3)


def guidance_distances(rgb, L):
    """Per pixel: distance of iz (unclipped, float64) to the nearest integer, and its signed distance to the clip range
    (> 0 strictly inside, <= 0 on or outside a bound)."""
    gray = np.asarray(rgb, np.float64).reshape(-1, 3) @ GRAY_WEIGHTS
    iz, _, _ = _axis(gray * 2 - 1, L)
    return np.abs(iz - np.round(iz)), np.minimum(iz, (L - 1) - iz)


def ambiguous(rgb, L, eps=1e-5):
    """Samples whose guidance gradient a float32 evaluation may take from the neighbouring cell: iz within eps of an integer
    while strictly inside the clip range (exactly on a bound, as for black pixels, is unambiguous: both sides clip)."""
    d_int, d_bound = guidance_distances(rgb, L)
    return ((d_int < eps) & (d_bound > 0)).reshape(np.asarray(rgb).shape[:-1])


def weyl(shape, seed):
    """Deterministic values in [0, 1): u_k = frac(a k + frac(b k^2) + c seed) on the flat index k.  Only float64 multiplies, adds
    and fmod, which every IEEE platform evaluates alike, so test inputs can be rebuilt rather than stored."""
    k = np.arange(int(np.prod(shape)), dtype=np.float64)
    return np.mod(0.6180339887498949 * k + np.mod(0.41421356237309515 * k * k, 1.0) + 0.2247448713915890 * seed, 1.0).reshape(shape)


def golden_inputs(n, grid, image, seed):
    """The inputs of the cases of tests/golden/bilagrid.npz: float32 grids [n,12,L,Hg,Wg] (grid = (Wg, Hg, L)) equal to the
    identity plus up to +-0.2, a meshgrid xy [1,H,W,2] in [0,1], rgb [1,H,W,3] in [-0.2, 1.2] and a cotangent v_out in [-1, 1].
    Images of 26 pixels or more get 7 black pixels (gray = 0 exactly, on the clip bound), 4 white ones, one with a zero red, and
    xy outside [0, 1] at pixels 20-25."""
    gw, gh, L = grid
    H, W = image
    identity = np.array([1., 0, 0, 0, 0, 1., 0, 0, 0, 0, 1., 0]).reshape(1, 12, 1, 1, 1)
    grids = (identity + 0.4 * weyl((n, 12, L, gh, gw), seed) - 0.2).astype(np.float32)
    gx = (np.arange(W, dtype=np.float64) / max(W - 1, 1)).astype(np.float32)
    gy = (np.arange(H, dtype=np.float64) / max(H - 1, 1)).astype(np.float32)
    xy = np.stack(np.broadcast_arrays(gx[None, :], gy[:, None]), -1)[None].copy()
    rgb = (1.4 * weyl((1, H, W, 3), seed + 1) - 0.2).astype(np.float32)
    v_out = (2.0 * weyl((1, H, W, 3), seed + 2) - 1.0).astype(np.float32)
    if H * W >= 26:
        flat_rgb, flat_xy = rgb.reshape(-1, 3), xy.reshape(-1, 2)
        flat_rgb[:7] = 0.0
        flat_rgb[7:11] = 1.0
        flat_rgb[11, 0] = 0.0
        flat_xy[20:26] = [[-0.3, 0.5], [1.4, 0.2], [0.5, -2.0], [0.1, 1.7], [-1.0, -1.0], [2.0, 2.0]]
    return grids, xy, rgb, v_out


def golden_index(size):
    """Flat entries kept of a recorded array of `size` entries: all of a small one; of a large one the first 192 (the pixels with
    black, white, zero-red colours and out-of-range xy) and every 29th (29 divides no grid or image extent used, so the kept
    entries run through all channels, levels, cells and pixels)."""
    if size <= 2048:
        return np.arange(size)
    return np.union1d(np.arange(192), np.arange(0, size, 29))


def processor_inputs(seed, n=3, image=(37, 50)):
    """grids and render [3,H,W] of the processor case of tests/golden/bilagrid.npz: the default 16x16x8 grids of golden_inputs and
    a render in [0, 1) with a black 2x3 corner."""
    H, W = image
    render = weyl((3, H, W), seed + 1).astype(np.float32)
    render[:, :2, :3] = 0.0
    return golden_inputs(n, (16, 16, 8), (1, 1), seed)[0], render


def total_variation(grids):
    x = np.asarray(grids, np.float64)
    n = x.shape[0]
    tv = 0.0
    for ax in range(2, x.ndim):
        d = np.diff(x, axis=ax)
        tv += (d ** 2).sum() / max(float(np.prod(d.shape[1:])), 1.0)
    return tv / n


def total_variation_grad(grids):
    x = np.asarray(grids, np.float64)
    n = x.shape[0]
    g = np.zeros_like(x)
    for ax in range(2, x.ndim):
        d = np.diff(x, axis=ax)
        w = 2.0 / (max(float(np.prod(d.shape[1:])), 1.0) * n)
        lo = [builtins.slice(None)] * x.ndim
        hi = [builtins.slice(None)] * x.ndim
        lo[ax], hi[ax] = builtins.slice(0, -1), builtins.slice(1, None)
        g[tuple(lo)] -= w * d
        g[tuple(hi)] += w * d
    return g

