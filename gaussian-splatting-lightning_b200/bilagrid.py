"""Bilateral-grid colour correction (the reference's ``configs/bilagrid.yaml`` / ``configs/bilagrid_fused.yaml``) on the b200gs
kernels.  ``b200gs.compat.install()`` registers this module's three names as ``fused_bilagrid``, the import of
``BilagridProcessor(fused=True)`` (internal/output_processors/bilagrid.py:38-43), so the reference's processor runs unmodified:

    BilateralGrid(num, grid_X=16, grid_Y=16, grid_W=8)   the per-image grids: parameter ``grids`` [num,12,L,H,W] and buffer
                                                         ``rgb2gray_weight``, the state_dict of lib_bilagrid.BilateralGrid
    slice(bil_grids, xy, rgb, grid_idx)                  {"rgb": colour-corrected rgb} on the slice kernels
    total_variation_loss(grids)                          the grids' total variation on the TV kernels

Differences from lib_bilagrid: ``slice`` takes the 4-D ``[B,H,W,.]`` inputs of the processor only; ``xy`` gets no gradient; the
returned dict has no ``"rgb_affine_mats"`` (12 floats per pixel, 100 MB at 1080p, which no caller reads); the guidance uses the
BT.601 weights the buffer holds at construction; ``BilateralGrid.forward`` (the direct 5-D ``grid_sample`` path) is not provided.
"""
import torch
import torch.nn as nn

from ._lib import check, lib, ptr
from .ops import _f32c, _stream


class BilateralGrid(nn.Module):
    """``num`` bilateral grids of ``grid_W`` guidance levels x ``grid_Y`` x ``grid_X`` cells, each cell a 3x4 affine colour
    matrix, initialised to the identity."""

    def __init__(self, num, grid_X=16, grid_Y=16, grid_W=8):
        super().__init__()
        self.grid_width, self.grid_height, self.grid_guidance = grid_X, grid_Y, grid_W
        identity = torch.tensor([1., 0, 0, 0, 0, 1., 0, 0, 0, 0, 1., 0]).view(1, 12, 1, 1, 1)
        self.grids = nn.Parameter(identity.repeat(num, 1, grid_W, grid_Y, grid_X))     # (N, 12, L, H, W)
        self.register_buffer("rgb2gray_weight", torch.tensor([[0.299, 0.587, 0.114]]))

    def tv_loss(self):
        return total_variation_loss(self.grids)

    def forward(self, grid_xy, rgb, idx=None):
        raise NotImplementedError("b200gs.bilagrid.BilateralGrid is sliced through slice(bil_grids, xy, rgb, grid_idx); "
                                  "the direct grid_sample path is not provided")


def _grid_dims(grids: torch.Tensor):
    if grids.dim() != 5 or grids.shape[1] != 12:
        raise ValueError(f"grids must be [N, 12, L, H, W], got {tuple(grids.shape)}")
    return grids.shape[0], grids.shape[2], grids.shape[3], grids.shape[4]


def _same_layout(a: torch.Tensor, b: torch.Tensor) -> bool:
    """a and b address their elements alike (the stride of a size-1 dimension is never used)."""
    return all(sa == sb for sa, sb, n in zip(a.stride(), b.stride(), a.shape) if n > 1)


class _Slice(torch.autograd.Function):
    @staticmethod
    def forward(ctx, grids, xy, rgb, grid_idx):
        n, L, gh, gw = _grid_dims(grids)
        B, H, W = rgb.shape[:3]
        out = torch.empty_like(rgb)
        if not _same_layout(out, rgb):          # not a dense layout: the kernels read and write one set of strides
            rgb = rgb.contiguous()
            out = torch.empty_like(rgb)
        check(lib().b200gs_bilagrid_slice_fwd(n, L, gh, gw, ptr(grids), B, H, W, ptr(xy), ptr(rgb), *rgb.stride(), ptr(grid_idx),
                                              grid_idx.numel(), ptr(out), _stream()), "b200gs_bilagrid_slice_fwd")
        ctx.save_for_backward(grids, xy, rgb, grid_idx)
        return out

    @staticmethod
    def backward(ctx, v_out):
        grids, xy, rgb, grid_idx = ctx.saved_tensors
        n, L, gh, gw = _grid_dims(grids)
        B, H, W = rgb.shape[:3]
        if not _same_layout(v_out, rgb):
            v_out = torch.empty_like(rgb).copy_(v_out)
        v_grids = torch.zeros_like(grids) if ctx.needs_input_grad[0] else None
        v_rgb = torch.empty_like(rgb) if ctx.needs_input_grad[2] else None
        check(lib().b200gs_bilagrid_slice_bwd(n, L, gh, gw, ptr(grids), B, H, W, ptr(xy), ptr(rgb), *rgb.stride(), ptr(grid_idx),
                                              grid_idx.numel(), ptr(v_out), ptr(v_rgb), ptr(v_grids), _stream()),
              "b200gs_bilagrid_slice_bwd")
        return v_grids, None, v_rgb, None


def slice(bil_grids, xy, rgb, grid_idx):
    """Colour-correct ``rgb`` [B,H,W,3] with the grids of ``bil_grids`` (a :class:`BilateralGrid`) sampled at ``xy`` [B,H,W,2]
    (in [0,1]) and the gray of each pixel.  ``grid_idx`` names one grid for every row (one element, as the processor's
    ``appearance_id[None, None]``) or one per row (its first element per row is used, as lib_bilagrid does).  An index outside
    the grids gives NaN in that row.  Returns ``{"rgb": out}``, ``out`` laid out like ``rgb`` (a permuted view of a CHW render
    gives an output whose inverse permutation is contiguous)."""
    grids = bil_grids.grids
    if rgb.dim() != 4 or xy.dim() != 4 or rgb.shape[-1] != 3 or xy.shape[-1] != 2 or xy.shape[:3] != rgb.shape[:3]:
        raise ValueError(f"slice takes xy [B,H,W,2] and rgb [B,H,W,3], got {tuple(xy.shape)} and {tuple(rgb.shape)}")
    if xy.requires_grad:
        raise ValueError("xy gets no gradient from the fused slice; pass it without requires_grad")
    if grids.dtype != torch.float32 or rgb.dtype != torch.float32 or not (grids.is_cuda and rgb.is_cuda):
        raise ValueError(f"grids and rgb must be float32 CUDA tensors, got {grids.dtype} on {grids.device}, {rgb.dtype} on {rgb.device}")
    B = rgb.shape[0]
    if grid_idx.numel() == 1:
        idx = grid_idx.reshape(1)
    elif grid_idx.dim() >= 1 and grid_idx.shape[0] == B:
        idx = grid_idx.reshape(B, -1)[:, 0]
    else:
        raise ValueError(f"grid_idx must have one element or one row per batch row ({B}), got {tuple(grid_idx.shape)}")
    idx = idx.to(device=rgb.device, dtype=torch.int64).contiguous()
    return {"rgb": _Slice.apply(grids.contiguous(), _f32c(xy, "xy"), rgb, idx)}


class _TotalVariation(torch.autograd.Function):
    @staticmethod
    def forward(ctx, grids):
        n, c, L, gh, gw = grids.shape
        L_ = lib()
        partials = torch.empty(int(L_.b200gs_bilagrid_tv_blocks(n, c, L, gh, gw)), dtype=torch.float32, device=grids.device)
        check(L_.b200gs_bilagrid_tv_fwd(n, c, L, gh, gw, ptr(grids), ptr(partials), _stream()), "b200gs_bilagrid_tv_fwd")
        ctx.save_for_backward(grids)
        return partials.sum()                                    # fixed summation order

    @staticmethod
    def backward(ctx, v_tv):
        (grids,) = ctx.saved_tensors
        n, c, L, gh, gw = grids.shape
        v_tv = v_tv.to(torch.float32).contiguous()
        v_grids = torch.empty_like(grids)
        check(lib().b200gs_bilagrid_tv_bwd(n, c, L, gh, gw, ptr(grids), ptr(v_tv), ptr(v_grids), _stream()), "b200gs_bilagrid_tv_bwd")
        return v_grids


def total_variation_loss(grids: torch.Tensor) -> torch.Tensor:
    """lib_bilagrid's total_variation_loss of 5-D ``grids`` [N,C,L,H,W]: over the L, H and W axes, the summed squared
    differences of neighbours divided by their count per grid, all divided by N."""
    if grids.dim() != 5:
        raise ValueError(f"total_variation_loss takes [N, C, L, H, W] grids, got {tuple(grids.shape)}")
    return _TotalVariation.apply(_f32c(grids, "grids"))
