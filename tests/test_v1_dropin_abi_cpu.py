"""CPU checks of the gsplat v1 drop-in: the new C ABI entry points are bound and reject bad arguments before any CUDA call, every
name the reference's GSplatV1Renderer imports resolves after install(), and every option without a b200gs implementation raises."""
import ctypes
import importlib
import json
import os
import sys

import pytest
import torch

from conftest import GOLDEN


@pytest.fixture(scope="module")
def lib():
    from b200gs import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def test_new_exports_are_bound_and_validate_without_gpu(lib):
    d = ctypes.c_void_p(16)
    for name in ("b200gs_sh_split_fwd", "b200gs_sh_split_bwd", "b200gs_isect_keys", "b200gs_isect_offsets"):
        assert hasattr(lib, name)
    assert lib.b200gs_sh_split_fwd(5, 35, 10, d, d, d, None, d, None) == -1 and b"degree" in lib.b200gs_last_error()
    assert lib.b200gs_sh_split_fwd(3, 14, 10, d, d, d, None, d, None) == -1 and b"k_rest" in lib.b200gs_last_error()
    assert lib.b200gs_sh_split_fwd(3, 15, 10, d, d, None, None, d, None) == -1 and b"NULL" in lib.b200gs_last_error()
    assert lib.b200gs_sh_split_bwd(3, 15, 10, d, d, d, None, d, d, None, None, None) == -1 and b"NULL" in lib.b200gs_last_error()
    assert lib.b200gs_sh_split_fwd(3, 15, 0, None, None, None, None, None, None) == 0          # n = 0: a no-op
    assert lib.b200gs_sh_split_fwd(0, 0, 0, None, None, None, None, None, None) == 0
    assert lib.b200gs_isect_keys(-1, d, d, 0, d, d, None) == -1 and b"bad size" in lib.b200gs_last_error()
    assert lib.b200gs_isect_keys(4, d, None, 5, d, d, None) == -1 and b"NULL" in lib.b200gs_last_error()
    assert lib.b200gs_isect_keys(4, ctypes.c_void_p(12), d, 5, d, d, None) == -1 and b"aligned" in lib.b200gs_last_error()
    assert lib.b200gs_isect_keys(4, d, None, 0, None, None, None) == 0
    assert lib.b200gs_isect_offsets(1 << 31, d, 4, d, None) == -1 and b"bad size" in lib.b200gs_last_error()
    assert lib.b200gs_isect_offsets(0, None, 4, None, None) == -1 and b"NULL" in lib.b200gs_last_error()
    assert lib.b200gs_isect_offsets(5, None, 4, d, None) == -1 and b"NULL" in lib.b200gs_last_error()
    assert lib.b200gs_isect_offsets(0, None, 0, None, None) == 0


def test_every_recorded_import_resolves_after_install(monkeypatch):
    imported = []
    for name in ("dropin_v1.json", "dropin_v1_appearance.json"):     # GSplatV1Renderer, GSplatAppearanceEmbeddingRenderer
        with open(os.path.join(GOLDEN, name)) as f:
            imported += [tuple(x) for x in json.load(f)["imported"]]
    assert ("gsplat.v0_interfaces", "rasterize_to_pixels") in imported and ("gsplat.sh_decomposed", "spherical_harmonics_decomposed") in imported
    for name in [m for m in list(sys.modules) if m == "gsplat" or m.startswith("gsplat.")]:
        monkeypatch.delitem(sys.modules, name)
    from b200gs import compat
    from b200gs.compat import gsplat_v0, gsplat_v1
    compat.install()
    for mod, attr in imported:
        if mod.startswith("gsplat"):
            assert callable(getattr(importlib.import_module(mod), attr)), (mod, attr)
    # what install() registered before is unchanged
    v0 = sys.modules["gsplat.v0_interfaces"]
    assert v0.project_gaussians is gsplat_v0.project_gaussians and v0.rasterize_gaussians is gsplat_v0.rasterize_gaussians
    assert sys.modules["gsplat"].spherical_harmonics is gsplat_v0.spherical_harmonics
    assert sys.modules["gsplat.cuda._wrapper"].isect_tiles is gsplat_v1.isect_tiles
    exec("from gsplat.cuda._wrapper import fully_fused_projection, isect_offset_encode, isect_tiles, spherical_harmonics", {})
    exec("from gsplat.cuda.isect_tiles_tile_based_culling import isect_tiles_tile_based_culling, isect_offset_encode_tile_based_culling", {})


def _proj_args(**kw):
    a = dict(means=torch.zeros(4, 3), covars=None, quats=torch.zeros(4, 4), scales=torch.zeros(4, 3), viewmats=torch.eye(4)[None],
             Ks=torch.eye(3)[None], width=32, height=32, eps2d=0.3)
    a.update(kw)
    return a


@pytest.mark.parametrize("bad", [
    dict(covars=torch.zeros(4, 6)), dict(packed=True), dict(sparse_grad=True), dict(camera_model="fisheye"), dict(camera_model="ortho"),
    dict(radius_clip=1.0), dict(far_plane=100.0), dict(viewmats=torch.eye(4)[None].requires_grad_(True)),
    dict(Ks=torch.eye(3)[None].requires_grad_(True))])
def test_projection_options_without_an_implementation_raise(bad):
    from b200gs.compat import gsplat_v1 as G
    with pytest.raises(NotImplementedError):
        G.fully_fused_projection(**_proj_args(**bad))


def test_isect_and_rasterize_options_without_an_implementation_raise():
    from b200gs.compat import gsplat_v1 as G
    xy, r, d = torch.zeros(1, 4, 2), torch.zeros(1, 4, dtype=torch.int32), torch.ones(1, 4)
    with pytest.raises(ValueError):
        G.isect_tiles(xy, r, d, 8, 4, 4)
    with pytest.raises(NotImplementedError):
        G.isect_tiles(xy, r, d, 16, 4, 4, packed=True)
    with pytest.raises(NotImplementedError):
        G.isect_tiles(xy.expand(2, 4, 2), r.expand(2, 4), d.expand(2, 4), 16, 4, 4, n_cameras=2)
    with pytest.raises(NotImplementedError):
        G.isect_tiles_tile_based_culling(xy.expand(2, 4, 2), r.expand(2, 4), d.expand(2, 4), torch.zeros(2, 4, 3), torch.ones(2, 4), 16, 4, 4,
                                         n_cameras=2)
    with pytest.raises(NotImplementedError):
        G.isect_offset_encode(torch.zeros(3, dtype=torch.int64), 2, 4, 4)
    kw = dict(means2d=torch.zeros(4, 2), conics=torch.zeros(1, 4, 3), colors=torch.zeros(1, 4, 3), opacities=torch.zeros(1, 4), image_width=64,
              image_height=64, tile_size=16, isect_offsets=torch.zeros(1, 4, 4, dtype=torch.int32), flatten_ids=torch.zeros(0, dtype=torch.int32))
    with pytest.raises(ValueError):
        G.rasterize_to_pixels(**dict(kw, tile_size=8))
    with pytest.raises(NotImplementedError):
        G.rasterize_to_pixels(**dict(kw, colors=torch.zeros(2, 4, 3), isect_offsets=torch.zeros(2, 4, 4, dtype=torch.int32)))
    with pytest.raises(ValueError):
        G.rasterize_to_pixels(**dict(kw, image_width=80))
    with pytest.raises(ValueError):      # ids / offsets the kernels would dereference on the device must live there
        G.rasterize_to_pixels(**kw)
    from b200gs import ops
    with pytest.raises(ValueError):
        ops.spherical_harmonics_decomposed(0, torch.zeros(4, 3), torch.zeros(4, 1, 3), torch.zeros(4, 0, 3), torch.ones(4, dtype=torch.bool))
