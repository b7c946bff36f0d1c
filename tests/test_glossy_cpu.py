"""CPU checks of the Glossy-Gaussian opacity and colour: the float64 oracle against the recorded reference modules
(tests/golden/glossy.npz), the C ABI's argument validation (rejected before any CUDA call, so no GPU is needed), the shape and degree
refusals of ops.glossy_sh, and the renderer config."""
import ctypes
import dataclasses
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import glossy_oracle as O

Z = np.load(os.path.join(GOLDEN, "glossy.npz"))


def _t(key):
    return torch.from_numpy(Z[key]).double()


@pytest.mark.parametrize("degree", [0, 1, 2, 3])
@pytest.mark.parametrize("key", ["model", "renderer"])
def test_oracle_reproduces_the_recorded_modules(degree, key):
    dc, rest = _t("op_dc").requires_grad_(True), _t("op_rest").requires_grad_(True)
    out = O.glossy(degree, _t("means"), _t("campos"), dc, rest)
    want = _t(f"{key}_{degree}_opacity").reshape(-1)
    got = out["raw_opacity"] if key == "model" else out["opacity"]
    assert (got - want).abs().max() <= 2e-6 * (1 + want.abs().max())
    (got * _t("w")).sum().backward()
    for name, p in (("v_dc", dc), ("v_rest", rest)):
        ref = _t(f"{key}_{degree}_{name}")
        assert (p.grad - ref).abs().max() <= 2e-6 * (1 + ref.abs().max()), name
    if key == "renderer":
        dirs = O.directions(_t("means"), _t("campos"))
        assert (dirs - _t(f"renderer_{degree}_viewdirs")).abs().max() <= 1e-6
        assert bool((out["opacity"] == 0).any()) and bool((out["opacity"] == 1).any())
    assert not bool(O.directions(_t("means"), _t("campos"))[0].any())       # Gaussian 0 sits at the camera centre


def test_rows_beyond_the_degree_and_masked_colour_rows_get_no_gradient():
    g = torch.Generator().manual_seed(3)
    n = 40
    means, campos = torch.randn(n, 3, generator=g, dtype=torch.float64), torch.zeros(3, dtype=torch.float64)
    dc = torch.randn(n, 1, 1, generator=g, dtype=torch.float64).requires_grad_(True)
    rest = (0.3 * torch.randn(n, 24, 1, generator=g, dtype=torch.float64)).requires_grad_(True)
    feats = torch.randn(n, 16, 3, generator=g, dtype=torch.float64).requires_grad_(True)
    mask = torch.arange(n) % 3 != 0
    out = O.glossy(2, means, campos, dc, rest, colour=feats, mask=mask)
    assert bool((out["rgb"][~mask] == 0.5).all())
    (out["opacity"].sum() + out["rgb"].sum()).backward()
    assert not bool(rest.grad[:, 8:].any()) and not bool(feats.grad[:, 9:].any()) and not bool(feats.grad[~mask].any())


def _lib():
    from b200gs import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def test_abi_validation_without_gpu():
    L = _lib()
    d = ctypes.c_void_p(256)
    fwd = lambda deg, n, k_rest, stride, split, means=d, shs=d, rgb=d: L.b200gs_glossy_sh_fwd(  # noqa: E731
        deg, n, means, d, d, d, k_rest, shs, d, stride, split, None, d, rgb, d, None)
    bwd = lambda deg, n, k_rest, stride, split, v_rgb=d, v_shs=d: L.b200gs_glossy_sh_bwd(  # noqa: E731
        deg, n, d, d, k_rest, stride, split, d, d, v_rgb, d, d, v_shs, d, None)
    for call in (fwd, bwd):
        for args, msg in (((5, 4, 35, 36, 1), b"degree"), ((-1, 4, 15, 16, 1), b"degree"), ((3, -1, 15, 16, 1), b"n < 0"),
                          ((3, 4, 14, 16, 1), b"op_k_rest"), ((3, 4, 15, 15, 1), b"sh_stride"), ((3, 4, 15, 16, 2), b"sh_split")):
            assert call(*args) == -1, args
            assert msg in L.b200gs_last_error(), (args, L.b200gs_last_error())
        assert call(3, 0, 15, 16, 1) == 0                   # n = 0: a valid no-op
    assert fwd(3, 4, 15, 16, 1, means=None) == -1 and b"NULL" in L.b200gs_last_error()
    assert fwd(3, 4, 15, 16, 1, shs=None) == -1 and b"NULL" in L.b200gs_last_error()
    assert bwd(3, 4, 15, 16, 1, v_shs=None) == -1 and b"NULL" in L.b200gs_last_error()
    # without the colour its layout is not looked at
    assert fwd(3, 0, 15, 0, 7, rgb=None) == 0
    assert bwd(3, 0, 15, 0, 7, v_rgb=None) == 0


def test_glossy_sh_refusals():
    from b200gs import ops
    n = 4
    means, campos = torch.zeros(n, 3), torch.zeros(3)
    dc, rest = torch.zeros(n, 1, 1), torch.zeros(n, 15, 1)
    with pytest.raises(ValueError, match="degree"):
        ops.glossy_sh(5, means, campos, dc, rest)
    with pytest.raises(ValueError, match="needs 15"):
        ops.glossy_sh(3, means, campos, dc, rest[:, :14])
    with pytest.raises(ValueError, match="needs 24"):
        ops.glossy_sh(4, means, campos, dc, rest)
    with pytest.raises(ValueError, match="op_dc"):
        ops.glossy_sh(3, means, campos, dc[:, :, :0], rest)
    with pytest.raises(ValueError, match="needs 16"):
        ops.glossy_sh(3, means, campos, dc, rest, features=torch.zeros(n, 9, 3))
    with pytest.raises(ValueError, match="needs 15"):
        ops.glossy_sh(3, means, campos, dc, rest, shs_dc=torch.zeros(n, 1, 3), shs_rest=torch.zeros(n, 8, 3))
    with pytest.raises(ValueError, match="not both"):
        ops.glossy_sh(3, means, campos, dc, rest, features=torch.zeros(n, 16, 3), shs_dc=torch.zeros(n, 1, 3),
                      shs_rest=torch.zeros(n, 15, 3))
    with pytest.raises(ValueError, match="together"):
        ops.glossy_sh(3, means, campos, dc, rest, shs_dc=torch.zeros(n, 1, 3))
    with pytest.raises(ValueError, match="float32"):
        ops.glossy_sh(3, means.double(), campos, dc, rest)
    with pytest.raises(ValueError, match="CUDA"):       # no CPU path
        ops.glossy_sh(3, means, campos, dc, rest)


def test_renderer_config_fields():
    from b200gs.glossy import B200GlossyRenderer, B200GlossyRendererModule
    from b200gs.v1 import B200GSplatV1Renderer
    fields = {f.name: f.default for f in dataclasses.fields(B200GlossyRenderer)}
    assert fields == {f.name: f.default for f in dataclasses.fields(B200GSplatV1Renderer)}
    assert {"separate_sh", "tile_based_culling", "anti_aliased", "block_size", "filter_2d_kernel_size"} <= set(fields)
    m = B200GlossyRenderer(separate_sh=True, tile_based_culling=True).instantiate()
    assert isinstance(m, B200GlossyRendererModule) and m.config.separate_sh and m.config.tile_based_culling
