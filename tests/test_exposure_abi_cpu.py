"""Argument validation of the exposure entry points without a GPU: every bad argument is rejected before any CUDA call, and the
workspace size follows the documented layout."""
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
H, W, S = 37, 50, 16
STRIDES = (H * W, W, 1)


def ws_bytes(L, backward, size=(H, W), s=S):
    return L.b200gs_exposure_workspace_bytes(*size, s, backward)


def fwd(L, channels=3, size=(H, W), strides=STRIDES, n_app=5, n_params=7, s=S, ptrs=(D,) * 4, ws=None):
    render, params, shade, out = ptrs
    ws = ws_bytes(L, 0) if ws is None else ws
    return L.b200gs_exposure_fwd(channels, *size, render, *strides, n_app, n_params, params, None, 2, s, shade, 5.0, 5.0, D, ws, out,
                                 None)


def bwd(L, channels=3, size=(H, W), strides=STRIDES, n_app=5, n_params=7, s=S, ptrs=(D,) * 4, ws=None, grads=(D,) * 3):
    render, params, shade, v_out = ptrs
    ws = ws_bytes(L, 1) if ws is None else ws
    return L.b200gs_exposure_bwd(channels, *size, render, *strides, n_app, n_params, params, D, 0, s, shade, 5.0, 5.0, D, ws, v_out,
                                 *grads, None)


@pytest.mark.parametrize("call", [fwd, bwd], ids=["fwd", "bwd"])
def test_exposure_rejects_bad_arguments(L, call):
    for c in (1, 4, 0):
        assert call(L, channels=c) == -1 and b"channels must be 3" in L.b200gs_last_error()
    for size in ((0, W), (H, 0), (-1, W), (H, -5)):
        assert call(L, size=size) == -1 and b"image size" in L.b200gs_last_error()
    assert call(L, size=(65535 * 8 + 1, 4)) == -1 and b"too large" in L.b200gs_last_error()
    assert call(L, s=-1) == -1 and b"negative shade_size" in L.b200gs_last_error()
    assert call(L, strides=(H * W, -W, 1)) == -1 and b"negative stride" in L.b200gs_last_error()
    assert call(L, n_app=0) == -1 and b"n_appearances" in L.b200gs_last_error()
    for n_params in (3, 5, 6, 8):
        assert call(L, n_params=n_params) == -1 and b"n_params" in L.b200gs_last_error()
    for k in range(4):
        ptrs = [D] * 4
        ptrs[k] = None
        assert call(L, ptrs=ptrs) == -1 and b"NULL" in L.b200gs_last_error()
    # without shade correction a NULL map passes the pointer checks; an empty workspace does not
    assert call(L, ptrs=(D, D, None, D), s=0, ws=0) == -3 and b"workspace too small" in L.b200gs_last_error()


def test_exposure_bwd_rejects_null_gradients(L):
    for k in range(3):
        grads = [D] * 3
        grads[k] = None
        assert bwd(L, grads=grads) == -1 and b"NULL" in L.b200gs_last_error()
    before = L.b200gs_launch_count()
    assert bwd(L, grads=(D, D, None), s=-1) == -1        # rejected before any launch
    assert L.b200gs_launch_count() == before


def test_workspace_size_follows_the_layout(L):
    head = 16
    blocks = ((W + 31) // 32) * ((H + 7) // 8)
    assert ws_bytes(L, 0) == 4 * (head + S * S)
    assert ws_bytes(L, 1) == 4 * (head + S * S + 8 * blocks + H * W)
    assert ws_bytes(L, 0, s=0) == 4 * head
    assert ws_bytes(L, 1, s=0) == 4 * (head + 8 * blocks)
    for size, s in (((0, W), S), ((H, -1), S), ((H, W), -1), ((H, W), 4097), ((1 << 16, 1 << 16), S)):
        assert ws_bytes(L, 0, size=size, s=s) == 0 and ws_bytes(L, 1, size=size, s=s) == 0
    for call in (fwd, bwd):
        need = ws_bytes(L, int(call is bwd))
        before = L.b200gs_launch_count()
        assert call(L, ws=need - 4) == -3 and b"workspace too small" in L.b200gs_last_error()
        assert L.b200gs_launch_count() == before
