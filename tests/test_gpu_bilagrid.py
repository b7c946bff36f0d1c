"""Bilateral-grid kernels (csrc/bilagrid.cu) on the GPU against the float64 oracle (oracle/bilagrid_oracle.py) and the reference's
own outputs (tests/golden/bilagrid.npz): slice forward and both gradients at 1080p, 800x800 and the golden sizes, in the contiguous
HWC layout and as a permuted CHW view, one grid for the batch or one per row; the shared-memory and global-atomic branches of the
backward; the total variation; out-of-range grid indices; the processor's call replayed through ``fused_bilagrid``; and no host
synchronisation."""
import json
import os
import sys

import numpy as np
import pytest
import torch
from torch.utils._python_dispatch import TorchDispatchMode

from conftest import GOLDEN
from oracle import bilagrid_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
Z = np.load(os.path.join(GOLDEN, "bilagrid.npz"))
META = json.load(open(os.path.join(GOLDEN, "bilagrid.json")))


def make_grids(n, grid, seed):
    from b200gs.bilagrid import BilateralGrid
    bg = BilateralGrid(n, *grid)
    with torch.no_grad():
        bg.grids.add_(0.2 * torch.randn(bg.grids.shape, generator=torch.Generator().manual_seed(seed)))
    return bg.to(DEV)


def meshgrid_xy(B, H, W):
    gy, gx = torch.meshgrid(torch.linspace(0, 1., H), torch.linspace(0, 1., W), indexing="ij")
    return torch.stack([gx, gy], dim=-1)[None].expand(B, H, W, 2).contiguous()


def make_rgb(B, H, W, layout, seed):
    """rgb in [-0.1, 1.1] with black and white pixels, as a contiguous [B,H,W,3] or a permuted [B,3,H,W] render"""
    g = torch.Generator().manual_seed(seed)
    chw = torch.rand(B, 3, H, W, generator=g) * 1.2 - 0.1
    black = torch.rand(B, 1, H, W, generator=g) < 0.05
    white = torch.rand(B, 1, H, W, generator=g) < 0.002
    chw = torch.where(black, 0.0, torch.where(white, 1.0, chw))
    if layout == "hwc":
        return chw.permute(0, 2, 3, 1).contiguous().to(DEV)
    return chw.to(DEV).permute(0, 2, 3, 1)


def run(bg, xy, rgb, idx, v_out):
    from b200gs.bilagrid import slice
    rgb = rgb.detach().requires_grad_(True)
    bg.zero_grad()
    out = slice(bg, xy, rgb, idx)["rgb"]
    assert out.stride() == rgb.stride() or rgb.shape[0] == 1
    out.backward(v_out)
    torch.cuda.synchronize()
    return out.detach().cpu().double().numpy(), bg.grids.grad.cpu().double().numpy(), rgb.grad.cpu().double().numpy()


def check_against_oracle(bg, xy, rgb, idx, seed, ambiguous_share=0.01):
    v_out = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(seed)).to(DEV)
    out, v_grids, v_rgb = run(bg, xy, rgb, idx, v_out)
    G, XY, RGB, V = (t.detach().cpu().double().numpy() for t in (bg.grids, xy, rgb, v_out))
    I = idx.reshape(-1).cpu().numpy()
    ref = O.slice(G, XY, RGB, I)
    assert np.abs(out - ref).max() <= 1e-5
    ref_vg, ref_vr = O.slice_vjp(G, XY, RGB, I, V)
    assert np.abs(v_grids - ref_vg).max() <= 1e-4 * np.abs(ref_vg).max()
    unused = [i for i in range(G.shape[0]) if i not in set(I.tolist())]
    assert not v_grids[unused].any()
    amb = O.ambiguous(RGB, G.shape[2])
    assert amb.mean() <= ambiguous_share
    assert np.abs(v_rgb[~amb] - ref_vr[~amb]).max() <= 1e-5 * np.abs(ref_vr).max()


FULL = [((1080, 1920), 1, "chw"), ((1080, 1920), 1, "hwc"), ((800, 800), 2, "chw"), ((800, 800), 2, "hwc")]


@pytest.mark.parametrize("image,B,layout", FULL, ids=[f"{h}x{w}-B{b}-{lay}" for (h, w), b, lay in FULL])
def test_slice_matches_the_oracle_at_full_size(image, B, layout):
    H, W = image
    bg = make_grids(3, (16, 16, 8), seed=1)
    idx = torch.tensor([[2]]) if B == 1 else torch.tensor([[2], [0]])
    check_against_oracle(bg, meshgrid_xy(B, H, W).to(DEV), make_rgb(B, H, W, layout, seed=H + B), idx.to(DEV), seed=5)


GOLDEN_SIZES = [(tuple(c["grid"]), tuple(c["image"])) for c in META["cases"]]


@pytest.mark.parametrize("grid,image", GOLDEN_SIZES, ids=[f"{g}-{i}" for g, i in GOLDEN_SIZES])
@pytest.mark.parametrize("layout", ["chw", "hwc"])
def test_slice_matches_the_oracle_at_the_golden_sizes(grid, image, layout):
    bg = make_grids(3, grid, seed=2)
    H, W = image
    xy = meshgrid_xy(2, H, W)
    if H * W > 1:
        xy.view(-1, 2)[:4] = torch.tensor([[-0.3, 0.5], [1.4, 0.2], [0.5, -2.0], [2.0, 2.0]])      # outside [0, 1]: clipped
    check_against_oracle(bg, xy.to(DEV), make_rgb(2, H, W, layout, seed=7), torch.tensor([1, 2]).to(DEV), seed=3,
                         ambiguous_share=0.05 if H * W > 1 else 1.0)


def recorded(key, shape):
    """a recorded array at full shape, NaN at the entries the golden file does not keep (oracle.golden_index)"""
    size = int(np.prod(shape))
    full = np.full(size, np.nan)
    full[O.golden_index(size)] = Z[key]
    return full.reshape(shape)


def max_err(a, ref):
    kept = ~np.isnan(ref)
    assert kept.any()
    return np.abs(a[kept] - ref[kept]).max()


@pytest.mark.parametrize("case", META["cases"], ids=lambda c: c["key"])
def test_slice_reproduces_the_reference(case):
    """the reference's lib_bilagrid outputs and autograd gradients (float32 on the CPU), ambiguous guidance gradients excluded"""
    from b200gs.bilagrid import BilateralGrid
    k = case["key"]
    grids, xy, rgb, v_out = O.golden_inputs(META["n_grids"], case["grid"], case["image"], case["seed"])
    bg = BilateralGrid(grids.shape[0], grids.shape[4], grids.shape[3], grids.shape[2]).to(DEV)
    with torch.no_grad():
        bg.grids.copy_(torch.from_numpy(grids))
    out, v_grids, v_rgb = run(bg, torch.from_numpy(xy).to(DEV), torch.from_numpy(rgb).to(DEV),
                              torch.tensor([[case["grid_idx"]]]).to(DEV), torch.from_numpy(v_out).to(DEV))
    assert max_err(out, recorded(f"{k}_out", rgb.shape)) <= 1e-5
    ref_vg, ref_vr = recorded(f"{k}_v_grids", grids.shape), recorded(f"{k}_v_rgb", rgb.shape)
    assert max_err(v_grids, ref_vg) <= 1e-4 * max(np.nanmax(np.abs(ref_vg)), 1e-30)
    amb = O.ambiguous(rgb, grids.shape[2])
    assert max_err(v_rgb[~amb], ref_vr[~amb]) <= 1e-5 * max(np.nanmax(np.abs(ref_vr)), 1e-30)


def test_scattered_coordinates_take_the_global_atomic_branch():
    """Shuffled meshgrid coordinates: every 16x16 CTA touches cells all over the 16x16 plane, 16 * 16 * 8 * 12 floats, more than
    the 4096 of the shared box, so the backward adds every pixel's terms to global memory."""
    H, W = 800, 800
    bg = make_grids(3, (16, 16, 8), seed=4)
    xy = meshgrid_xy(1, H, W).view(-1, 2)
    xy = xy[torch.randperm(H * W, generator=torch.Generator().manual_seed(0))].view(1, H, W, 2)
    check_against_oracle(bg, xy.contiguous().to(DEV), make_rgb(1, H, W, "chw", seed=9), torch.tensor([[0]]).to(DEV), seed=11)


@pytest.mark.parametrize("n", [1, 3, 64])
def test_total_variation_matches_the_oracle(n):
    from b200gs.bilagrid import total_variation_loss
    grids = make_grids(n, (16, 16, 8), seed=n).grids
    tv = total_variation_loss(grids)
    (10.0 * tv).backward()
    G = grids.detach().cpu().double().numpy()
    assert abs(float(tv.detach()) - O.total_variation(G)) <= 1e-5 * O.total_variation(G)
    ref = 10.0 * O.total_variation_grad(G)
    assert np.abs(grids.grad.cpu().double().numpy() - ref).max() <= 1e-5 * np.abs(ref).max()


def test_out_of_range_grid_index_gives_nan_rows_and_reads_no_other_memory():
    """Rows with indices n and -1 against n = 3 grids stored between two sentinel grids of 1e6: a read past either end would put
    a finite value of about 1e6 in the row, and a write past either end would change a sentinel or its gradient."""
    from b200gs import _lib
    from b200gs.ops import _stream
    n, (gx, gy, gl), H, W = 3, (16, 16, 8), 64, 48
    buf = torch.full((n + 2, 12, gl, gy, gx), 1e6, device=DEV)
    buf[1:n + 1] = make_grids(n, (gx, gy, gl), seed=6).grids.detach()
    grids = buf[1:n + 1]
    v_buf = torch.zeros_like(buf)
    xy = meshgrid_xy(3, H, W).to(DEV)
    rgb = make_rgb(3, H, W, "hwc", seed=8)
    idx = torch.tensor([1, n, -1], device=DEV)
    out, v_rgb = torch.empty_like(rgb), torch.empty_like(rgb)
    v_out = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(1)).to(DEV)
    L = _lib.lib()
    _lib.check(L.b200gs_bilagrid_slice_fwd(n, gl, gy, gx, grids.data_ptr(), 3, H, W, xy.data_ptr(), rgb.data_ptr(), *rgb.stride(),
                                           idx.data_ptr(), 3, out.data_ptr(), _stream()), "slice_fwd")
    _lib.check(L.b200gs_bilagrid_slice_bwd(n, gl, gy, gx, grids.data_ptr(), 3, H, W, xy.data_ptr(), rgb.data_ptr(), *rgb.stride(),
                                           idx.data_ptr(), 3, v_out.data_ptr(), v_rgb.data_ptr(), v_buf[1:n + 1].data_ptr(), _stream()),
               "slice_bwd")
    torch.cuda.synchronize()
    assert torch.isnan(out[1:]).all() and torch.isnan(v_rgb[1:]).all()
    assert torch.isfinite(out[0]).all() and torch.isfinite(v_rgb[0]).all()
    ref = O.slice(grids.cpu().double().numpy(), xy[:1].cpu().double().numpy(), rgb[:1].cpu().double().numpy(), [1])
    assert np.abs(out[:1].cpu().double().numpy() - ref).max() <= 1e-5
    assert not v_buf[0].any() and not v_buf[n + 1].any() and not v_buf[1].any() and not v_buf[3].any()
    assert v_buf[2].abs().max() > 0 and (buf[0] == 1e6).all() and (buf[n + 1] == 1e6).all()


class _OpLog(TorchDispatchMode):
    def __init__(self):
        super().__init__()
        self.ops = []

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        self.ops.append(str(func))
        return func(*args, **(kwargs or {}))


def test_processor_call_replayed_through_fused_bilagrid():
    """The recorded call of the reference's BilagridProcessorModule.forward (bilagrid.py:115-124), replayed with its recorded
    layouts through sys.modules["fused_bilagrid"], gives the processor's golden render; the processed render is a contiguous
    [3,H,W] that no copy produced; tv_loss reproduces the recorded metric."""
    from b200gs import compat
    compat.install()
    fb = sys.modules["fused_bilagrid"]
    p = META["processor"]
    (call,) = p["calls"]
    H, W = p["image"]
    grids, render = (torch.from_numpy(a) for a in O.processor_inputs(p["seed"], META["n_grids"], (H, W)))
    bgrid = fb.BilateralGrid(num=grids.shape[0], grid_X=grids.shape[4], grid_Y=grids.shape[3], grid_W=grids.shape[2]).to(DEV)
    with torch.no_grad():
        bgrid.grids.copy_(grids)
    rgb = render.to(DEV).permute(1, 2, 0).unsqueeze(0)
    assert list(rgb.shape) == call["rgb"]["shape"] and list(rgb.stride())[1:] == call["rgb"]["stride"][1:]
    xy = meshgrid_xy(1, H, W).to(DEV)
    assert list(xy.stride()) == call["xy"]["stride"]
    grid_idx = torch.tensor(p["appearance_id"], device=DEV)[None, None]
    assert list(grid_idx.shape) == call["grid_idx"]["shape"] and str(grid_idx.dtype) == call["grid_idx"]["dtype"]
    with _OpLog() as log:
        res = fb.slice(bgrid, xy=xy, rgb=rgb, grid_idx=grid_idx)["rgb"]
        out = res.squeeze(0).permute(2, 0, 1)
    assert not [op for op in log.ops if "copy" in op or "clone" in op or "contiguous" in op], log.ops
    assert out.shape == (3, H, W) and out.is_contiguous() and out.data_ptr() == res.data_ptr()
    assert max_err(out.detach().cpu().double().numpy(), recorded("proc_out", (3, H, W))) <= 1e-5
    tv = p["tv_loss_weight"] * fb.total_variation_loss(bgrid.grids)
    assert abs(float(tv.detach()) - float(Z["proc_tv"])) <= 1e-5 * float(Z["proc_tv"])


def test_slice_and_tv_forward_backward_do_not_synchronise():
    from b200gs.bilagrid import slice, total_variation_loss
    bg = make_grids(4, (16, 16, 8), seed=3)
    H, W = 96, 128
    xy = meshgrid_xy(1, H, W).to(DEV)
    render = make_rgb(1, H, W, "chw", seed=2)[0].permute(2, 0, 1).contiguous().requires_grad_(True)
    idx = torch.tensor(3, device=DEV)[None, None]
    cot = torch.rand(3, H, W, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = slice(bg, xy, render.permute(1, 2, 0).unsqueeze(0), idx)["rgb"].squeeze(0).permute(2, 0, 1)
        loss = (out * cot).sum() + 10.0 * total_variation_loss(bg.grids)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.isfinite(render.grad).all() and torch.isfinite(bg.grids.grad).all()
