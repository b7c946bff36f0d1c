"""float64 restatement of the reference's SWAG in-the-wild appearance (internal/renderers/swag_renderer.py: SWAGRenderer.forward
:32-66 with internal/models/swag_model.py: SWAGModel).  Plain torch, differentiable by autograd; the GPU tests compare K49/K50 and
the SWAG MLP against it, and tests/test_swag_cpu.py compares it against recordings of the unmodified reference modules
(tests/golden/swag.npz), which ran with ``encode`` standing in for tinycudann: they pin everything around the grid, not the grid.

    rgb     = clamp_min(SH_deg(features; (xyz - campos) / |xyz - campos|) + 0.5, 0)        eval_gaussian_model_sh (xyz not detached)
    x       = (xyz.detach() - bbox_min) / bbox_size                                          fp32, as torch divides
    o       = theta([rgb | HashGrid(x) | embedding])                                         Linear-ReLU-..-Linear, no output activation
    colour  = sigmoid(o[:, :3])
    opacity = clamp_min(base_opacity - sigmoid((log(|o3| + eps) + log(u + eps) - log(1 - u + eps)) / temperature), 0)

PARITY UNPINNED: the grid.  The reference encodes with tiny-cuda-nn's ``Encoding`` (``otype: HashGrid``), which cannot be installed
here.  ``encode`` restates tcnn's published grid encoding for 3-D inputs with linear interpolation:
    scale_l = exp2f(l log2f(per_level_scale)) base - 1 (fp32), res_l = ceil(scale_l) + 1,
    size_l = min(next_multiple(res_l^3, 8), 2^log2_hashmap_size) vertices of F floats, the levels one after the other;
    pos = fmaf(scale_l, x, 0.5f), cell = (uint32)(int)floor(pos), frac = pos - floor(pos) per axis (fp32);
    corner k = 0..7, bit d on axis d, weight prod_d (bit ? frac_d : 1 - frac_d);
    vertex = grid_index(cell + bits): in uint32, index = sum_d c_d stride_d with stride_0 = 1 and stride_{d+1} = stride_d res_l
    while stride_d <= size_l; when the final stride exceeds size_l, index = c_0 ^ c_1 * 2654435761 ^ c_2 * 805459861 (coherent prime
    hash); then index % size_l.  Points outside [0, 1] wrap through the same uint32 arithmetic (negative cells included).
Cell selection is done in fp32 exactly as the kernels do; the interpolation is float64.

The trap of swag_model.GridEncodingConfig: ``n_levels = 12`` there has no annotation, so it only sets a class attribute and the
dataclass field keeps its inherited default of 8.  The effective grid is 8 levels x 4 features, log2_hashmap_size 19, base 16,
per_level_scale 2.0: a 32-wide encoding, a 59-wide network input and 4096 + 32768 + 262144 + 5 x 524288 = 2920448 vertices,
11681792 floats."""
import math

import numpy as np
import torch

from oracle.gs_oracle import sh_basis

DEFAULT_GRID = dict(n_levels=8, n_features_per_level=4, log2_hashmap_size=19, base_resolution=16, per_level_scale=2.0)
PRIMES = (1, 2654435761, 805459861)


def levels(n_levels=8, n_features_per_level=4, log2_hashmap_size=19, base_resolution=16, per_level_scale=2.0):
    """[(scale_l (fp32), res_l, size_l, offset_l)], sizes and offsets in vertices."""
    lg = np.float32(math.log2(float(np.float32(per_level_scale))))
    cap = 1 << int(log2_hashmap_size)
    out, offset = [], 0
    for l in range(int(n_levels)):
        e = np.float32(np.float32(l) * lg)
        scale = np.float32(np.float32(2.0 ** float(e)) * np.float32(base_resolution)) - np.float32(1.0)
        res = int(math.ceil(float(scale))) + 1
        size = min((res ** 3 + 7) // 8 * 8, cap)
        out.append((np.float32(scale), res, size, offset))
        offset += size
    return out


def n_params(**grid):
    g = {**DEFAULT_GRID, **grid}
    lv = levels(**g)
    return g["n_features_per_level"] * (lv[-1][3] + lv[-1][2])


def grid_index(c, res, size):
    """tcnn's grid_index of uint32 corner coordinates c [n, 3] (numpy uint64 holding uint32 values)."""
    M = np.uint64(0xFFFFFFFF)
    stride, index = np.uint64(1), np.zeros(c.shape[0], dtype=np.uint64)
    for d in range(3):
        if int(stride) > size:
            break
        index = (index + c[:, d] * stride) & M
        stride = (stride * np.uint64(res)) & M
    if size < int(stride):
        index = np.zeros(c.shape[0], dtype=np.uint64)
        for d in range(3):
            index ^= (c[:, d] * np.uint64(PRIMES[d])) & M
    return (index % np.uint64(size)).astype(np.int64)


def _axis(scale, x):
    # fmaf(scale, x, 0.5f): the product of two fp32 values is exact in float64, then one rounding to fp32 after the add
    pos = (np.float64(scale) * x.astype(np.float64) + 0.5).astype(np.float32)
    fl = np.floor(pos)
    cell = (fl.astype(np.int64) & 0xFFFFFFFF).astype(np.uint64)          # (uint32)(int)floor(pos)
    return cell, (pos - fl).astype(np.float64)


def corners(x, **grid):
    """Per level: (vertex index into the flat [vertices, F] table [n, 8], weight [n, 8] float64) of fp32 points x [n, 3]."""
    g = {**DEFAULT_GRID, **grid}
    x = np.asarray(x, dtype=np.float32)
    out = []
    for scale, res, size, offset in levels(**g):
        ax = [_axis(scale, x[:, d]) for d in range(3)]
        idx, w = [], []
        for k in range(8):
            c = np.stack([ax[d][0] + np.uint64((k >> d) & 1) for d in range(3)], 1) & np.uint64(0xFFFFFFFF)
            wt = np.ones(x.shape[0])
            for d in range(3):
                wt = wt * (ax[d][1] if (k >> d) & 1 else 1.0 - ax[d][1])
            idx.append(grid_index(c, res, size) + offset)
            w.append(wt)
        out.append((torch.from_numpy(np.stack(idx, 1)), torch.from_numpy(np.stack(w, 1))))
    return out


def encode(params, x, **grid):
    """HashGrid encoding [n, n_levels F] of fp32 numpy points x [n, 3] with the flat table ``params`` (any float dtype)."""
    g = {**DEFAULT_GRID, **grid}
    table = params.reshape(-1, g["n_features_per_level"])
    cols = []
    for idx, w in corners(x, **g):
        cols.append((table[idx] * w.to(params.dtype).unsqueeze(-1)).sum(1))
    return torch.cat(cols, dim=1)


def normalized_xyz(means, bbox_min, bbox_size):
    """(means - bbox_min) / bbox_size in fp32 (numpy), as the reference's _get_normalized_xyz and K49 compute it."""
    m = np.asarray(means, dtype=np.float32)
    return (m - np.asarray(bbox_min, dtype=np.float32)) / np.asarray(bbox_size, dtype=np.float32)


def sh_colour(degree, means, campos, features):
    """eval_gaussian_model_sh: clamp_min(SH + 0.5, 0) with dir = (means - campos) / |means - campos| (means differentiable);
    features [N, K, 3]."""
    d = means - campos.reshape(1, 3)
    d = d / d.norm(dim=1, keepdim=True)
    B = sh_basis(degree, d)
    ncoef = (degree + 1) ** 2
    rgb = (B.unsqueeze(-1) * features[:, :ncoef]).sum(1) + 0.5
    return torch.clamp_min(rgb, 0.0), rgb


def network(x, weights, biases):
    """theta: Linear layers with ReLU between them and no output activation."""
    h = x
    for l, (w, b) in enumerate(zip(weights, biases)):
        h = h @ w.T + b
        if l < len(weights) - 1:
            h = torch.relu(h)
    return h


def epilogue(o, base_opacity, u, temperature=0.1, eps=1e-8):
    """(colour [N,3], opacity [N]) from the network outputs o [N, 4]."""
    colour = torch.sigmoid(o[:, :3])
    u = torch.as_tensor(u, dtype=o.dtype)
    z = 1 / temperature * (torch.log(torch.abs(o[:, 3]) + eps) + torch.log(u + eps) - torch.log(1 - u + eps))
    return colour, torch.clamp_min(base_opacity - torch.sigmoid(z), 0)


def swag(degree, means, campos, features, table, embedding_row, weights, biases, base_opacity, u, bbox_min, bbox_size,
         temperature=0.1, eps=1e-8, **grid):
    """The whole per-view computation: (colour [N,3], opacity [N]).  ``means`` is differentiable through the SH colour only."""
    rgb, _ = sh_colour(degree, means, campos, features)
    x = normalized_xyz(means.detach().float().numpy(), bbox_min, bbox_size)
    enc = encode(table, x, **grid)
    e = embedding_row.reshape(1, -1).expand(means.shape[0], -1)
    o = network(torch.cat([rgb, enc.to(rgb.dtype), e.to(rgb.dtype)], dim=1), weights, biases)
    return epilogue(o, base_opacity, u, temperature, eps)
