"""The float64 bilateral-grid oracle (oracle/bilagrid_oracle.py) against the reference's lib_bilagrid and its unmodified
BilagridProcessorModule (tests/golden/bilagrid.npz, made by tests/golden/make_golden_bilagrid.py); the b200gs.bilagrid module's
state_dict against lib_bilagrid's; and the ``fused_bilagrid`` alias of ``b200gs.compat.install()``."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import bilagrid_oracle as O

Z = np.load(os.path.join(GOLDEN, "bilagrid.npz"))
META = json.load(open(os.path.join(GOLDEN, "bilagrid.json")))


def recorded(key, shape):
    """a recorded array at full shape, NaN at the entries the golden file does not keep (oracle.golden_index)"""
    size = int(np.prod(shape))
    full = np.full(size, np.nan)
    full[O.golden_index(size)] = Z[key]
    return full.reshape(shape)


def close(a, ref, atol):
    kept = ~np.isnan(ref)
    assert kept.any()
    return np.abs(a[kept] - ref[kept]).max() <= atol


def case_arrays(case):
    grids, xy, rgb, v_out = O.golden_inputs(META["n_grids"], case["grid"], case["image"], case["seed"])
    shape = rgb.shape
    return grids, xy, rgb, v_out, recorded(f"{case['key']}_out", shape), recorded(f"{case['key']}_v_rgb", shape), \
        recorded(f"{case['key']}_v_grids", grids.shape)


@pytest.mark.parametrize("case", META["cases"], ids=lambda c: c["key"])
def test_slice_matches_the_reference(case):
    grids, xy, rgb, v_out, ref_out, ref_vr, ref_vg = case_arrays(case)
    assert close(O.slice(grids, xy, rgb, case["grid_idx"]), ref_out, 1e-5)
    v_grids, v_rgb = O.slice_vjp(grids, xy, rgb, case["grid_idx"], v_out)
    assert close(v_grids, ref_vg, 1e-5 * max(np.nanmax(np.abs(ref_vg)), 1.0))
    unused = [i for i in range(grids.shape[0]) if i != case["grid_idx"]]
    assert not v_grids[unused].any() and not np.nan_to_num(ref_vg[unused]).any()
    amb = O.ambiguous(rgb, grids.shape[2])
    assert amb.sum() <= 4                         # the white pixels at most: gray = 1 within a float32 rounding of the bound
    assert close(v_rgb[~amb], ref_vr[~amb], 1e-5 * max(np.nanmax(np.abs(ref_vr)), 1.0))


def test_border_rule_black_pixels_pass_no_guidance_gradient():
    """gray = 0 exactly lands on iz = 0: the clip passes nothing, so v_rgb is the affine part alone (grid_sample's border rule; an
    autograd of clamp would pass gradient there)."""
    case = META["cases"][0]
    grids, xy, rgb, v_out, _, ref_vr, _ = case_arrays(case)
    black = (rgb == 0).all(-1)
    assert black.sum() >= 7
    d_int, d_bound = O.guidance_distances(rgb, grids.shape[2])
    assert (d_bound.reshape(black.shape)[black] == 0).all()
    _, v_rgb = O.slice_vjp(grids, xy, rgb, 1, v_out)
    # the affine part: v_rgb_j = sum_i v_out_i A[4i + j], with A at gray = 0
    A = O._affine(O._footprint(grids, xy, rgb, 1))[0].reshape(*rgb.shape[:3], 3, 4)
    affine = np.einsum("bhwi,bhwij->bhwj", v_out, A[..., :3])
    np.testing.assert_allclose(v_rgb[black], affine[black], rtol=0, atol=1e-12)
    assert not np.isnan(ref_vr[black]).any()      # every black pixel is recorded
    np.testing.assert_allclose(ref_vr[black], affine[black], rtol=0, atol=1e-5)


@pytest.mark.parametrize("tv", META["tv"], ids=lambda t: t["key"])
def test_total_variation_matches_the_reference(tv):
    grids = O.golden_inputs(META["n_grids"], tv["grid"], (1, 1), tv["seed"])[0]
    np.testing.assert_allclose(O.total_variation(grids), float(Z[f"{tv['key']}_value"]), rtol=1e-5, atol=1e-7)
    ref = recorded(f"{tv['key']}_grad", grids.shape)
    g = O.total_variation_grad(grids)
    assert close(g, ref, 1e-5 * max(np.nanmax(np.abs(ref)), 1e-30))
    if grids.shape[2:] == (1, 1, 1):
        assert O.total_variation(grids) == 0.0 and not g.any()


def test_processor_recording_matches_the_oracle():
    p = META["processor"]
    (call,) = p["calls"]
    H, W = p["image"]
    assert call["rgb"]["shape"] == [1, H, W, 3] and call["rgb"]["stride"][1:] == [W, 1, H * W]   # the permuted CHW render
    assert call["xy"]["shape"] == [1, H, W, 2] and not call["xy"]["requires_grad"]
    assert call["grid_idx"]["shape"] == [1, 1] and call["grid_idx"]["values"] == [p["appearance_id"]]
    grids, render = O.processor_inputs(p["seed"], META["n_grids"], (H, W))
    gy, gx = np.meshgrid(np.linspace(0, 1, H, dtype=np.float32), np.linspace(0, 1, W, dtype=np.float32), indexing="ij")
    xy = np.stack([gx, gy], -1)[None]
    out = O.slice(grids, xy, render.transpose(1, 2, 0)[None], p["appearance_id"])[0].transpose(2, 0, 1)
    assert close(out, recorded("proc_out", (3, H, W)), 1e-5)
    np.testing.assert_allclose(p["tv_loss_weight"] * O.total_variation(grids), float(Z["proc_tv"]), rtol=1e-5)


def test_state_dict_matches_lib_bilagrid():
    from b200gs.bilagrid import BilateralGrid
    sd = BilateralGrid(3).state_dict()
    assert list(sd) == list(META["state_dict"])
    for k, v in sd.items():
        assert list(v.shape) == META["state_dict"][k]["shape"] and str(v.dtype) == META["state_dict"][k]["dtype"]
        assert torch.equal(v, torch.from_numpy(Z[f"sd_{k}"]))
    # and a checkpoint of the reference's module loads
    m = BilateralGrid(3)
    m.load_state_dict({k: torch.from_numpy(Z[f"sd_{k}"]) for k in sd})


EARLIER_ALIASES = ["diff_gaussian_rasterization", "simple_knn", "simple_knn._C", "gsplat", "gsplat.v0_interfaces",
                   "gsplat.project_gaussians", "gsplat.rasterize", "gsplat.sh", "gsplat.cuda._wrapper",
                   "gsplat.cuda.isect_tiles_tile_based_culling", "gsplat.sh_decomposed", "gsplat.cuda", "gsplat.relocation"]


def test_compat_registers_fused_bilagrid_and_keeps_earlier_aliases(monkeypatch):
    from b200gs import bilagrid, compat, mcmc, ops
    from b200gs.compat import gsplat_v0, gsplat_v1
    for name in EARLIER_ALIASES + ["fused_bilagrid"]:
        monkeypatch.delitem(sys.modules, name, raising=False)
    before = set(sys.modules)
    compat.install()
    added = {m for m in set(sys.modules) - before if not m.startswith("b200gs.")}     # (install() imports its own submodules)
    assert added == set(EARLIER_ALIASES) | {"fused_bilagrid"}
    fb = sys.modules["fused_bilagrid"]
    assert (fb.BilateralGrid, fb.slice, fb.total_variation_loss) == (bilagrid.BilateralGrid, bilagrid.slice,
                                                                     bilagrid.total_variation_loss)
    assert sys.modules["gsplat.relocation"].compute_relocation is mcmc.compute_relocation
    assert sys.modules["simple_knn._C"].distCUDA2 is ops.knn_mean_dist2
    assert sys.modules["gsplat"].rasterize_gaussians is gsplat_v0.rasterize_gaussians
    assert sys.modules["gsplat.cuda._wrapper"].fully_fused_projection is gsplat_v1.fully_fused_projection
    # an existing module of that name is left alone unless forced
    sentinel = type(sys)("fused_bilagrid")
    monkeypatch.setitem(sys.modules, "fused_bilagrid", sentinel)
    compat.install()
    assert sys.modules["fused_bilagrid"] is sentinel
