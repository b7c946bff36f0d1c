"""CPU-only checks of the D-channel blend entry points (b200gs_blend_feat_fwd / _bwd): bad channel counts, image sizes and NULL
pointers are rejected with B200GS_EINVAL and a message before any CUDA call."""
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


D16 = ctypes.c_void_p(16)   # a non-NULL dummy: never dereferenced, every call below fails validation first


def _fwd_args(W=64, H=48, D=32, **null):
    names = ["tile_ranges", "sorted_ids", "xy", "conic", "opacity", "features", "bg", "image", "final_T", "n_contrib", "alpha"]
    ptrs = [None if null.get(k) else D16 for k in names]
    return [W, H, D] + ptrs + [None]


def _bwd_args(W=64, H=48, D=32, **null):
    names = ["tile_ranges", "sorted_ids", "xy", "conic", "opacity", "features", "bg", "final_T", "n_contrib", "v_image", "v_alpha",
             "v_features", "v_xy", "v_conic", "v_opacity", "v_xy_abs"]
    ptrs = [None if null.get(k) else D16 for k in names]
    return [W, H, D] + ptrs + [None]


@pytest.mark.parametrize("D", [0, -1, -32])
def test_rejects_channel_counts_below_one(L, D):
    for fn, args in ((L.b200gs_blend_feat_fwd, _fwd_args(D=D)), (L.b200gs_blend_feat_bwd, _bwd_args(D=D))):
        assert fn(*args) == -1
        assert b"channels" in L.b200gs_last_error()


@pytest.mark.parametrize("W,H", [(0, 48), (64, 0), (-16, 48)])
def test_rejects_bad_image_sizes(L, W, H):
    for fn, args in ((L.b200gs_blend_feat_fwd, _fwd_args(W=W, H=H)), (L.b200gs_blend_feat_bwd, _bwd_args(W=W, H=H))):
        assert fn(*args) == -1
        assert b"size" in L.b200gs_last_error()


@pytest.mark.parametrize("name", ["tile_ranges", "sorted_ids", "xy", "conic", "opacity", "features", "image", "final_T", "n_contrib"])
def test_forward_rejects_null_required_pointers(L, name):
    assert L.b200gs_blend_feat_fwd(*_fwd_args(**{name: True})) == -1
    assert b"NULL" in L.b200gs_last_error()


@pytest.mark.parametrize("name", ["tile_ranges", "sorted_ids", "xy", "conic", "opacity", "features", "final_T", "n_contrib", "v_image",
                                  "v_features"])
def test_backward_rejects_null_required_pointers(L, name):
    assert L.b200gs_blend_feat_bwd(*_bwd_args(**{name: True})) == -1
    assert b"NULL" in L.b200gs_last_error()


@pytest.mark.parametrize("missing", [("v_xy",), ("v_conic",), ("v_opacity",), ("v_conic", "v_opacity")])
def test_backward_geometry_gradients_come_together(L, missing):
    assert L.b200gs_blend_feat_bwd(*_bwd_args(**{k: True for k in missing})) == -1
    assert b"all given or all NULL" in L.b200gs_last_error()


def test_backward_absgrad_needs_the_geometry_gradients(L):
    assert L.b200gs_blend_feat_bwd(*_bwd_args(v_xy=True, v_conic=True, v_opacity=True)) == -1
    assert b"v_xy_abs" in L.b200gs_last_error()
