"""Argument validation of the bilateral-grid entry points without a GPU: every bad argument is rejected before any CUDA call,
and empty work is a no-op."""
import ctypes
import os

import pytest


@pytest.fixture(scope="module")
def L():
    from b200gs import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


D = ctypes.c_void_p(16)    # non-NULL dummy; never dereferenced here
GRID = (3, 8, 16, 16)      # n_grids, L, grid_h, grid_w
STRIDES = (3 * 64 * 64, 64, 1, 64 * 64)


def slice_fwd(L, grid=GRID, image=(1, 64, 64), strides=STRIDES, n_idx=1, ptrs=(D,) * 5):
    g, xy, rgb, idx, out = ptrs
    return L.b200gs_bilagrid_slice_fwd(*grid, g, *image, xy, rgb, *strides, idx, n_idx, out, None)


def slice_bwd(L, grid=GRID, image=(1, 64, 64), strides=STRIDES, n_idx=1, ptrs=(D,) * 5, v_rgb=D, v_grids=D):
    g, xy, rgb, idx, v_out = ptrs
    return L.b200gs_bilagrid_slice_bwd(*grid, g, *image, xy, rgb, *strides, idx, n_idx, v_out, v_rgb, v_grids, None)


@pytest.mark.parametrize("call", [slice_fwd, slice_bwd], ids=["fwd", "bwd"])
def test_slice_rejects_bad_arguments(L, call):
    for k in range(4):
        grid = list(GRID)
        grid[k] = 0
        assert call(L, grid=grid) == -1 and b"grid sizes" in L.b200gs_last_error()
    assert call(L, grid=(1, 1 << 12, 1 << 12, 1 << 8)) == -1 and b"too large" in L.b200gs_last_error()
    for k in range(3):
        image = [1, 64, 64]
        image[k] = -1
        assert call(L, image=image) == -1 and b"negative image size" in L.b200gs_last_error()
    assert call(L, strides=(0, 64, 1, -1)) == -1 and b"negative stride" in L.b200gs_last_error()
    for n_idx in (0, 3):
        assert call(L, image=(2, 64, 64), n_idx=n_idx) == -1 and b"n_idx" in L.b200gs_last_error()
    for k in range(5):
        ptrs = [D] * 5
        ptrs[k] = None
        assert call(L, ptrs=ptrs) == -1 and b"NULL" in L.b200gs_last_error()
    for image in ((0, 64, 64), (1, 0, 64), (1, 64, 0)):      # no pixel: nothing is read, no launch
        assert call(L, image=image, n_idx=1, ptrs=(None,) * 5) == 0


def test_slice_bwd_without_outputs_is_a_no_op(L):
    before = L.b200gs_launch_count()
    assert slice_bwd(L, v_rgb=None, v_grids=None) == 0
    assert L.b200gs_launch_count() == before


def test_tv_rejects_bad_arguments(L):
    for k in range(5):
        dims = [3, 12, 8, 16, 16]
        dims[k] = -1
        assert L.b200gs_bilagrid_tv_fwd(*dims, D, D, None) == -1 and b"negative" in L.b200gs_last_error()
        assert L.b200gs_bilagrid_tv_bwd(*dims, D, D, D, None) == -1 and b"negative" in L.b200gs_last_error()
        assert L.b200gs_bilagrid_tv_blocks(*dims) == 0
    assert L.b200gs_bilagrid_tv_fwd(3, 12, 8, 16, 16, None, D, None) == -1 and b"NULL" in L.b200gs_last_error()
    assert L.b200gs_bilagrid_tv_fwd(3, 12, 8, 16, 16, D, None, None) == -1 and b"NULL" in L.b200gs_last_error()
    for k in range(3):
        ptrs = [D] * 3
        ptrs[k] = None
        assert L.b200gs_bilagrid_tv_bwd(3, 12, 8, 16, 16, *ptrs, None) == -1 and b"NULL" in L.b200gs_last_error()
    assert L.b200gs_bilagrid_tv_blocks(3, 12, 8, 16, 16) == (3 * 12 * 8 * 16 * 16 + 255) // 256
    assert L.b200gs_bilagrid_tv_fwd(0, 12, 8, 16, 16, None, None, None) == 0
    assert L.b200gs_bilagrid_tv_bwd(3, 12, 0, 16, 16, None, None, None, None) == 0
