"""float64 restatement of the reference's transient visibility map (internal/renderers/gsplat_appearance_embedding_visibility_map_
renderer.py: Model.visibility_forward :140-157) and its masked loss (internal/metrics/visibility_map_metrics.py).  Plain torch,
differentiable by autograd; the GPU tests compare the kernels against it, and tests/test_visibility_golden_cpu.py compares it
against recordings of the unmodified reference modules (tests/golden/visibility.npz), which ran with ``encode`` standing in for
tcnn: they pin everything around the grid, not the grid.

PARITY UNPINNED: the grid.  The reference encodes the pixel grid with tiny-cuda-nn's ``Encoding`` (``otype: DenseGrid``), which
cannot be installed here.  ``encode`` restates tcnn's published grid encoding (2-D, linear interpolation, 2 features per level):
    scale_l = exp2f(l log2f(per_level_scale)) base - 1 (fp32), res_l = ceil(scale_l) + 1, size_l = next_multiple(res_l^2, 8);
    pos = fmaf(scale_l, u, 0.5f), cell = floor(pos), frac = pos - cell (fp32); corners k = 0..3, bit 0 along x, weight
    (frac or 1 - frac along x) * (.. along y); vertex (cell_x + k&1 + (cell_y + k>>1) res_l) % size_l, so the last pixel column and
    row, which reach corner res_l on levels whose scale has a fractional part >= 0.5 (or none), wrap into the next row or the start.
Cell selection is done in fp32 exactly as the kernels do; the interpolation is float64."""
import math

import numpy as np
import torch

from . import loss_oracle
from .appearance_oracle import mlp


def levels(n_levels=8, base_resolution=16, per_level_scale=1.405):
    """[(scale_l (fp32), res_l, size_l, offset_l)] in vertices; the grid holds 2 (offset_last + size_last) floats."""
    lg = np.float32(math.log2(float(np.float32(per_level_scale))))
    out, offset = [], 0
    for l in range(n_levels):
        e = np.float32(np.float32(l) * lg)
        scale = np.float32(np.float32(2.0 ** float(e)) * np.float32(base_resolution)) - np.float32(1.0)
        res = int(math.ceil(float(scale))) + 1
        size = (res * res + 7) // 8 * 8
        out.append((np.float32(scale), res, size, offset))
        offset += size
    return out


def n_params(n_levels=8, base_resolution=16, per_level_scale=1.405):
    lv = levels(n_levels, base_resolution, per_level_scale)
    return 2 * (lv[-1][3] + lv[-1][2])


def pixel_uv(width, height):
    """fp32 (u [H*W], v [H*W]) of the row-major pixel grid: x / (W - 1), y / (H - 1), as the reference's meshgrid and division."""
    u = np.arange(width, dtype=np.float32) / np.float32(width - 1)
    v = np.arange(height, dtype=np.float32) / np.float32(height - 1)
    return np.tile(u, height), np.repeat(v, width)


def _axis(scale, u):
    # fmaf(scale, u, 0.5f): the product of two fp32 values is exact in float64, then one rounding to fp32 after the add
    pos = (np.float64(scale) * u.astype(np.float64) + 0.5).astype(np.float32)
    cell = np.floor(pos)
    return cell.astype(np.int64), (pos - cell).astype(np.float64)


def corners(u, v, lv):
    """Per level: (vertex index into the flat [vertices, 2] grid [n, 4], weight [n, 4] float64)."""
    out = []
    for scale, res, size, offset in lv:
        cx, fx = _axis(scale, u)
        cy, fy = _axis(scale, v)
        idx, w = [], []
        for k in range(4):
            kx, ky = k & 1, k >> 1
            idx.append(((cx + kx) + (cy + ky) * res) % size + offset)
            w.append((fx if kx else 1.0 - fx) * (fy if ky else 1.0 - fy))
        out.append((torch.from_numpy(np.stack(idx, 1)), torch.from_numpy(np.stack(w, 1))))
    return out


def encode(params, u, v, n_levels=8, base_resolution=16, per_level_scale=1.405):
    """DenseGrid encoding [n, 2 n_levels] of fp32 numpy coordinates u, v [n] with the flat grid ``params`` (any float dtype)."""
    table = params.reshape(-1, 2)
    cols = []
    for idx, w in corners(u, v, levels(n_levels, base_resolution, per_level_scale)):
        cols.append((table[idx] * w.to(params.dtype).unsqueeze(-1)).sum(1))
    return torch.cat(cols, dim=1)


def visibility(params, embedding_row, weights, biases, width, height, **grid):
    """The reference's visibility_forward: sigmoid(network([uv encoding | transient embedding])) [H, W]."""
    u, v = pixel_uv(width, height)
    enc = encode(params, u, v, **grid)
    return mlp(enc, embedding_row, weights, biases).reshape(height, width)


def masked_loss(image, gt, vis, mask=None, lambda_dssim=0.2, vis_reg_factor=0.2):
    """VisibilityMapMetricsImpl.get_train_metrics' loss: (loss, rgb_diff, ssim, vis_reg) with w = vis * mask on image and gt [3,H,W],
    vis [1,H,W] or [H,W], mask None or [H,W]."""
    H, W = image.shape[-2:]
    w = vis.reshape(1, H, W)
    if mask is not None:
        w = w * mask.reshape(1, H, W).to(vis.dtype)
    loss, l1, s = loss_oracle.training_loss(image * w, gt * w, lambda_dssim)
    reg = ((1.0 - vis) ** 2).mean() * vis_reg_factor
    return loss + reg, l1, s, reg


# ---- deterministic parameters and inputs of the recorded reference cases (tests/golden/make_golden_visibility.py) -------------
def _seed(name):
    return sum((i + 1) * b for i, b in enumerate(name.encode())) % 9973


def golden_param(name, shape):
    """float32 value of the reference Model's parameter `name` in the recordings, rebuilt from weyl: embeddings in [-1.5, 1.5),
    grids in [-0.5, 0.5) (far above tcnn's 1e-4 start, so the encoding matters), Linear weights and biases in +-2 / sqrt(fan_in)."""
    from .bilagrid_oracle import weyl
    w = weyl(tuple(shape), _seed(name)) * 2.0 - 1.0
    if "embedding" in name:
        w = w * 1.5
    elif "uv_encodings" in name:
        w = w * 0.5
    else:
        fan_in = shape[1] if len(shape) == 2 else shape[0]
        w = w * 2.0 / math.sqrt(fan_in)
    return torch.from_numpy(w.astype(np.float32))


def golden_inputs(width, height, seed):
    """float32 render, gt [3,H,W] in [0, 1) and a bool keep-mask [H,W] (about 80 % kept) of a recorded case"""
    from .bilagrid_oracle import weyl
    render = torch.from_numpy(weyl((3, height, width), seed).astype(np.float32))
    gt = torch.from_numpy(weyl((3, height, width), seed + 1).astype(np.float32))
    mask = torch.from_numpy(weyl((height, width), seed + 2) < 0.8)
    return render, gt, mask


def golden_probe(n):
    """float64 probe vector: the recordings hold the grid gradient's dot product with it (the grid itself is not pinned)"""
    from .bilagrid_oracle import weyl
    return torch.from_numpy(weyl((n,), 77) - 0.5)
