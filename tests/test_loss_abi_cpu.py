"""Argument validation of the L1 + SSIM loss entry points (K9/K10) without a GPU: sizes the launch grid cannot take and NULL
pointers are rejected before any CUDA call, and the partial-block count follows the grid."""
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
C, W, H = 3, 50, 37
MAX_C, MAX_H, MAX_W = 65535, 65535 * 16, 2 ** 31 - 16


def fwd(L, size=(C, W, H), ptrs=(D,) * 4):
    return L.b200gs_loss_fwd(*size, *ptrs, None)


def bwd(L, size=(C, W, H), ptrs=(D,) * 4):
    return L.b200gs_loss_bwd(*size, ptrs[0], ptrs[1], ptrs[2], 0.2, None, ptrs[3], None)


@pytest.mark.parametrize("call", [fwd, bwd], ids=["fwd", "bwd"])
def test_loss_rejects_bad_arguments(L, call):
    before = L.b200gs_launch_count()
    for size in ((0, W, H), (C, 0, H), (C, W, 0), (-1, W, H), (C, -5, H), (C, W, -16)):
        assert call(L, size=size) == -1 and b"bad size" in L.b200gs_last_error()
    assert call(L, size=(MAX_C + 1, W, H)) == -1 and b"too many channels" in L.b200gs_last_error()
    assert call(L, size=(C, W, MAX_H + 1)) == -1 and b"too tall" in L.b200gs_last_error()
    for w in (MAX_W + 1, 2 ** 31 - 1):
        assert call(L, size=(1, w, 1)) == -1 and b"too wide" in L.b200gs_last_error()
    for k in range(4):
        ptrs = [D] * 4
        ptrs[k] = None
        assert call(L, ptrs=ptrs) == -1 and b"NULL" in L.b200gs_last_error()
    assert L.b200gs_launch_count() == before


def test_blocks_follow_the_grid_up_to_each_limit(L):
    def expect(c, w, h):
        return c * ((w + 15) // 16) * ((h + 15) // 16)
    for size in ((C, W, H), (1, 1, 1), (2, 16, 16), (2, 17, 33), (3, 1920, 1080), (MAX_C, 1, 1), (1, 1, MAX_H), (1, MAX_W, 1),
                 (MAX_C, MAX_W, MAX_H)):
        assert L.b200gs_loss_blocks(*size) == expect(*size), size
    for size in ((0, W, H), (C, 0, H), (C, W, 0), (-1, W, H), (MAX_C + 1, 1, 1), (1, 1, MAX_H + 1), (1, MAX_W + 1, 1),
                 (1, 2 ** 31 - 1, 1)):
        assert L.b200gs_loss_blocks(*size) == 0, size
