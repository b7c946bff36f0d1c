"""4DGS deformation without a GPU: the float64 oracle (oracle/gs4d_oracle.py) against the reference's own VanillaGS4DRenderer recorded
on the CPU (tests/golden/make_golden_gs4d.py), the renderer's parameter tree against the reference's state_dict, and the refusals of
every unsupported option by the renderer, the ops and the C ABI (before any CUDA call)."""
import ctypes
import json
import os
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import gs4d_oracle as O

sys.path.insert(0, GOLDEN)
import make_golden_gs4d as MG  # noqa: E402

ZS = np.load(os.path.join(GOLDEN, "gs4d.npz"))
META = json.load(open(os.path.join(GOLDEN, "gs4d.json")))
PLANES = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
HEAD_MODULES = {"dx": "pos_deform", "ds": "scales_deform", "dr": "rotations_deform", "dshs": "shs_deform"}


def load_case(name):
    """(cfg, state_dict, Gaussians, t) of a recorded case; the planes are the stored ones for the small grids, else rebuilt"""
    from b200gs.gs4d import B200GS4DDeformNetwork
    cfg = MG.case_cfg(name)
    sd = MG.state_dict_values(B200GS4DDeformNetwork(cfg).state_dict())
    if META["cases"][name]["stored_planes"]:
        for k in sd:
            if ".grids." in k:
                sd[k] = torch.from_numpy(ZS[f"{name}.{k}"])
    p = {k: torch.from_numpy(ZS[f"{name}.in.{k}"]) for k in ("means", "scales", "rotations", "opacities", "shs_dc", "shs_rest")}
    return cfg, sd, p, META["cases"][name]["t"]


def network(cfg, sd):
    """(grids, trunk, heads) of a deform_network state_dict, as the oracle takes them"""
    pre = "deformation_net."
    grids = [[sd[f"{pre}grid.grids.{l}.{k}"] for k in range(6)] for l in range(len(cfg.multires))]
    trunk = [(sd[f"{pre}feature_out.{i}.weight"], sd[f"{pre}feature_out.{i}.bias"]) for i in range(0, 2 * max(cfg.defor_depth, 1) - 1, 2)]
    heads = {}
    for name, mod in HEAD_MODULES.items():
        if not getattr(cfg, "no_" + name):
            heads[name] = tuple((sd[f"{pre}{mod}.{i}.weight"], sd[f"{pre}{mod}.{i}.bias"]) for i in (1, 3))
    return grids, trunk, heads


def oracle_case(name):
    cfg, sd, p, t = load_case(name)
    grids, trunk, heads = network(cfg, sd)
    shs = torch.cat([p["shs_dc"], p["shs_rest"]], 1)
    d = O.deform(p["means"], p["scales"], p["rotations"], t, sd["deformation_net.grid.aabb"], grids, trunk, heads, shs=shs,
                 apply_rotation=cfg.apply_rotation)
    return cfg, d, O.activate(d, p["opacities"])


def close(got, want, rel=1e-5):
    got, want = torch.as_tensor(got).double(), torch.as_tensor(want).double()
    assert got.shape == want.shape, (got.shape, want.shape)
    err = float((got - want).abs().max())
    assert err <= rel * max(1.0, float(want.abs().max())), err


@pytest.mark.parametrize("name", sorted(MG.CASES))
def test_oracle_matches_the_reference_recording(name):
    cfg, d, act = oracle_case(name)
    close(act["means"], ZS[f"{name}.out.means3D"])
    close(act["scales"], ZS[f"{name}.out.scales"])
    close(act["rotations"], ZS[f"{name}.out.rotations"])
    close(act["opacities"], ZS[f"{name}.out.opacity"])
    close(d["shs"], ZS[f"{name}.out.features"])
    assert META["cases"][name]["active_sh_degree"] == 3


def test_recordings_cover_what_the_kernel_must_match():
    cases = META["cases"]
    assert {c["t"] for c in cases.values()} >= {0.0, 1.0, 0.5} and any(0 < c["t"] < 1 and c["t"] != 0.5 for c in cases.values())
    assert {c["cfg"]["apply_rotation"] for c in cases.values()} == {True, False}
    assert {c["cfg"]["no_dshs"] for c in cases.values()} == {True, False}
    assert min(c["n"] for c in cases.values()) == 1
    hi, lo = torch.tensor(MG.AABB[0]), torch.tensor(MG.AABB[1])
    p = O.normalize_points(torch.from_numpy(ZS["default.in.means"]), torch.tensor(MG.AABB))
    assert bool((p < -1).any(0).all()) and bool((p > 1).any(0).all())          # beyond the aabb on every axis, both sides
    assert bool(((p + 1).abs() < 1e-6).all(1).any()) and bool(((p - 1).abs() < 1e-6).all(1).any())   # the corners
    q = torch.from_numpy(ZS["default.in.rotations"])
    assert float((q.norm(dim=1) - 1).abs().min()) > 1e-3
    assert bool((hi > lo).all())
    # the recorded features change with the deformation (dshs on) and stay put (dshs off)
    f_in = np.concatenate([ZS["small_d1.in.shs_dc"], ZS["small_d1.in.shs_rest"]], 1)
    assert np.abs(ZS["small_d1.out.features"] - f_in).max() > 1e-2
    f_in = np.concatenate([ZS["default.in.shs_dc"], ZS["default.in.shs_rest"]], 1)
    assert np.array_equal(ZS["default.out.features"], f_in)


def test_grid_sample_restatement_on_nodes_and_beyond_the_border():
    plane = torch.arange(2 * 3 * 4, dtype=torch.float64).reshape(2, 3, 4)
    u = torch.tensor([-1.0, 1.0, -1 + 2 / 3, -7.0, 9.0, 0.0], dtype=torch.float64)
    v = torch.tensor([-1.0, 1.0, 0.0, 5.0, -5.0, 0.0], dtype=torch.float64)
    got = O.sample_plane(plane, u, v)
    want = torch.nn.functional.grid_sample(plane[None], torch.stack([u, v], -1)[None, None], mode="bilinear", padding_mode="border",
                                           align_corners=True)[0, :, 0].T
    assert torch.allclose(got, want, atol=1e-12)
    assert got[0].tolist() == [0.0, 12.0] and got[1].tolist() == [11.0, 23.0] and got[2].tolist() == [5.0, 17.0]


def test_renderer_parameter_tree_is_the_references():
    from b200gs.gs4d import B200GS4DDeformNetwork
    sd = B200GS4DDeformNetwork(MG.case_cfg("small_d1")).state_dict()
    assert {k: list(v.shape) for k, v in sd.items()} == META["state_dict"]


# ---- refusals ----------------------------------------------------------------------------------------------------------------
REFUSED = [
    ("static_mlp", dict(static_mlp=True)),
    ("empty_voxel", dict(empty_voxel=True)),
    ("no_grid", dict(no_grid=True)),
    ("grid_pe", dict(grid_pe=2)),
    ("grid_dimensions", dict(kplanes_config={**MG.BASE_CFG["kplanes_config"], "grid_dimensions": 3})),
    ("input_coordinate_dim", dict(kplanes_config={**MG.BASE_CFG["kplanes_config"], "input_coordinate_dim": 3})),
    ("output_coordinate_dim", dict(kplanes_config={**MG.BASE_CFG["kplanes_config"], "output_coordinate_dim": 24})),
    ("multires", dict(multires=[1, 2, 4, 8, 16])),
    ("net_width", dict(net_width=256)),
    ("defor_depth", dict(defor_depth=3)),
    ("resolution", dict(kplanes_config={**MG.BASE_CFG["kplanes_config"], "resolution": [64, 64, 64, 20000]})),
]


@pytest.mark.parametrize("option,over", REFUSED, ids=[r[0] for r in REFUSED])
def test_renderer_refuses_unsupported_options(tmp_path, option, over):
    from b200gs.gs4d import B200VanillaGS4DRenderer
    cfg = Namespace(**{**MG.BASE_CFG, **over})
    MG.write_checkpoint(str(tmp_path), cfg, {}, 1)      # refused before the state dict is read
    with pytest.raises(NotImplementedError, match=option):
        B200VanillaGS4DRenderer(str(tmp_path), MG.ITERATION, "cpu")


def test_ops_accept_every_supported_shape_and_refuse_the_rest():
    from b200gs import ops
    for w in (64, 128):
        for d in (0, 1, 2):
            for c in (16, 32):
                for levels in (1, 2, 3, 4):
                    assert ops.gs4d_supported(levels, c, w, d, [(64 << l, 64 << l, 64 << l, 150) for l in range(levels)])
    assert not ops.gs4d_supported(5, 32, 64, 1)
    assert not ops.gs4d_supported(0, 32, 64, 1)
    assert not ops.gs4d_supported(4, 8, 64, 1) and not ops.gs4d_supported(4, 64, 64, 1)
    assert not ops.gs4d_supported(4, 32, 32, 1) and not ops.gs4d_supported(4, 32, 256, 1)
    assert not ops.gs4d_supported(4, 32, 64, 3) and not ops.gs4d_supported(4, 32, 64, -1)
    assert not ops.gs4d_supported(1, 32, 64, 1, [(0, 4, 4, 4)]) and not ops.gs4d_supported(1, 32, 64, 1, [(16385, 4, 4, 4)])
    assert not ops.gs4d_supported(1, 32, 64, 1, [(16384, 16384, 4, 4)])       # one plane of 2^33 floats
    assert ops.gs4d_supported(1, 16, 64, 1, [(1, 1, 1, 1)])


def test_plane_floats_is_the_sum_of_the_planes():
    from b200gs import _lib, ops
    res = [(6, 5, 4, 3), (12, 10, 8, 3)]
    g = ops._gs4d_struct(2, 16, 64, 1, 0, res)
    want = sum(r[b] * r[a] * 16 for r in res for a, b in PLANES)
    assert _lib.lib().b200gs_gs4d_plane_floats(ctypes.byref(g)) == want
    g.flags = 64
    assert _lib.lib().b200gs_gs4d_plane_floats(ctypes.byref(g)) == 0


def test_abi_refuses_before_any_cuda_call():
    from b200gs import _lib, ops
    L = _lib.lib()
    g = ops._gs4d_struct(1, 16, 64, 1, 0, [(4, 4, 4, 4)])
    assert L.b200gs_gs4d_deform_fwd(None, 1, *([None] * 13), None) == -1
    assert L.b200gs_gs4d_deform_fwd(ctypes.byref(g), 1, *([None] * 13), None) == -1      # trunk weight NULL
    assert b"NULL" in L.b200gs_last_error()
    g.weights[0] = g.biases[0] = 16
    assert L.b200gs_gs4d_deform_fwd(ctypes.byref(g), -1, *([None] * 13), None) == -1
    assert b"n out of range" in L.b200gs_last_error()
    assert L.b200gs_gs4d_deform_fwd(ctypes.byref(g), 5, *([None] * 13), None) == -1
    assert b"NULL planes" in L.b200gs_last_error()
    g.flags = 8                                                                         # dshs on, its layers NULL
    assert L.b200gs_gs4d_deform_fwd(ctypes.byref(g), 5, *([None] * 13), None) == -1
    assert b"NULL weight" in L.b200gs_last_error()
    g.flags, g.weights[0] = 0, 20                                                       # misaligned weights
    assert L.b200gs_gs4d_deform_fwd(ctypes.byref(g), 5, *([None] * 13), None) == -1
    assert b"aligned" in L.b200gs_last_error()
    g.channels = 24
    assert L.b200gs_gs4d_repack_planes(ctypes.byref(g), None, None, None) == -1
    g.channels = 16
    assert L.b200gs_gs4d_repack_planes(ctypes.byref(g), None, None, None) == -1
    assert b"NULL" in L.b200gs_last_error()
