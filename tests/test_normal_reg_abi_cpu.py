"""Argument validation of the depth-normal entry points (b200gs_normal_reg_fwd / _bwd, b200gs_depth_to_normal) without a GPU: bad
sizes, NULL pointers, negative strides and short workspaces are rejected before any CUDA call, and the workspace size follows the
documented layout (a 4-float head, then one partial per 16x16 tile)."""
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
H, W = 37, 50
BAD_SIZES = ((0, W), (H, 0), (-1, W), (H, -5))
LARGE = ((65535 * 16 + 1, 4), (1 << 16, 1 << 16))


def fwd(L, size=(H, W), ptrs=(D,) * 6, mstrides=(4, 1, 3, 1), nstrides=(H * W, W, 1), ws=None):
    ws = L.b200gs_normal_reg_workspace_bytes(H, W) if ws is None else ws
    normal, depth, alpha, cam, K, out = ptrs
    return L.b200gs_normal_reg_fwd(*size, normal, *nstrides, depth, alpha, cam, *mstrides[:2], K, *mstrides[2:], 0.05, D, ws, out, None)


def bwd(L, size=(H, W), ptrs=(D,) * 6, mstrides=(4, 1, 3, 1), nstrides=None, ws=None):
    ws = L.b200gs_normal_reg_workspace_bytes(H, W) if ws is None else ws
    v_loss, depth, alpha, cam, K, out = ptrs
    return L.b200gs_normal_reg_bwd(*size, depth, alpha, cam, *mstrides[:2], K, *mstrides[2:], D, ws, v_loss, out, None)


def d2n(L, size=(H, W), ptrs=(D,) * 6, mstrides=(4, 1, 3, 1), nstrides=None, ws=None):
    _, depth, _, cam, K, out = ptrs
    return L.b200gs_depth_to_normal(*size, depth, cam, *mstrides[:2], K, *mstrides[2:], out, None)


def test_workspace_bytes(L):
    for (h, w) in ((1, 1), (16, 16), (17, 16), (H, W), (1080, 1920)):
        tiles = -(-h // 16) * -(-w // 16)
        assert L.b200gs_normal_reg_workspace_bytes(h, w) == 4 * (4 + tiles)
    for size in BAD_SIZES + LARGE:
        assert L.b200gs_normal_reg_workspace_bytes(*size) == 0


@pytest.mark.parametrize("call", [fwd, bwd, d2n], ids=["fwd", "bwd", "depth_to_normal"])
def test_normal_entry_points_reject_bad_arguments(L, call):
    before = L.b200gs_launch_count()
    for size in BAD_SIZES:
        assert call(L, size=size) == -1 and b"image size" in L.b200gs_last_error()
    for size in LARGE:
        assert call(L, size=size) == -1 and b"too large" in L.b200gs_last_error()
    for k in range(4):
        ms = [4, 1, 3, 1]
        ms[k] = -1
        assert call(L, mstrides=ms) == -1 and b"negative matrix stride" in L.b200gs_last_error()
    # every pointer the entry point reads or writes (d2n takes no alpha and no first pointer)
    used = {fwd: range(6), bwd: range(6), d2n: (1, 3, 4, 5)}[call]
    for k in used:
        ptrs = [D] * 6
        ptrs[k] = None
        assert call(L, ptrs=ptrs) == -1 and b"NULL" in L.b200gs_last_error(), k
    if call is not d2n:
        assert call(L, ws=L.b200gs_normal_reg_workspace_bytes(H, W) - 4) == -3 and b"workspace too small" in L.b200gs_last_error()
        assert call(L, ws=0) == -3
    if call is fwd:
        for k in range(3):
            ns = [H * W, W, 1]
            ns[k] = -ns[k]
            assert call(L, nstrides=ns) == -1 and b"negative normal stride" in L.b200gs_last_error()
    assert L.b200gs_launch_count() == before
