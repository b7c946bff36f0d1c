"""The depth-normal oracle (oracle/normal_reg_oracle.py) against the reference's own VanillaWithNormalRegMetricsModule recorded in
tests/golden/normal_reg.npz, and against the closed form on planes; the plug-in's config, setup mutation and argument errors,
without a GPU."""
import dataclasses
import json
import os
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import normal_reg_oracle as O

Z = np.load(os.path.join(GOLDEN, "normal_reg.npz"))
META = json.load(open(os.path.join(GOLDEN, "normal_reg.json")))


def golden_inputs(c):
    from make_golden_normal_reg import inputs
    return inputs(c["kind"], *c["image"], c["seed"])


@pytest.fixture(scope="module", autouse=True)
def _golden_path():
    import sys
    sys.path.insert(0, GOLDEN)
    yield
    sys.path.remove(GOLDEN)


@pytest.mark.parametrize("c", META["cases"], ids=lambda c: c["key"])
def test_oracle_matches_the_reference_module(c):
    cfg = {**META["config"], **c["config"]}
    render, gt, depth, alpha, normal, w2c, K, scene = golden_inputs(c)
    k = c["key"]
    lam = cfg["normal_reg_lambda"]
    ref_loss = float(Z[f"{k}_normal_loss"])
    assert abs(float(O.loss(normal, depth[0], alpha[0], w2c, K, lam)) - ref_loss) <= 1e-6 * max(abs(ref_loss), lam)
    v = O.vjp(depth[0], alpha[0], w2c, K, lam).numpy()
    assert np.abs(v - Z[f"{k}_v_normal"]).max() <= 1e-5 * np.abs(v).max()
    # the flatten term on the mutated scales, and the total
    s = torch.from_numpy(Z[f"{k}_scales"]).double().requires_grad_(True)
    flat = torch.exp(s)[..., -1].mean() * cfg["flatten_reg"]
    flat.backward()
    flat = flat.detach()
    assert abs(float(flat) - float(Z[f"{k}_flatten_loss"])) <= 1e-6 * float(flat)
    assert np.abs(s.grad.numpy() - Z[f"{k}_v_scales"]).max() <= 1e-6 * np.abs(s.grad.numpy()).max()
    basic = (1 - cfg["lambda_dssim"]) * float(Z[f"{k}_rgb_diff"]) + cfg["lambda_dssim"] * (1 - float(Z[f"{k}_ssim"]))
    assert abs(float(Z[f"{k}_loss"]) - (basic + ref_loss + float(Z[f"{k}_flatten_loss"]))) <= 1e-6
    assert c["pbar"] == {"loss": True, "rgb_diff": True, "ssim": True, "normal_loss": False, "flatten_loss": False}


@pytest.mark.parametrize("kind", ["plane", "flat"])
@pytest.mark.parametrize("size", [(37, 50), (3, 3), (64, 48)])
def test_oracle_matches_the_closed_form_on_planes(kind, size):
    depth, alpha, normal, w2c, K = O.case(kind, *size, 5)
    n = O.normals_from_depth(depth, w2c, K, torch.ones_like(alpha))
    # the depth map is rounded to float32, which tilts each pixel's plane by ~eps * f
    assert float((n - O.plane_normals(kind, *size, 5)).abs().max()) <= 1e-5
    assert float((n - O.origin_free(depth.double(), w2c, K, torch.ones_like(alpha).double())).abs().max()) <= 1e-12


@pytest.mark.parametrize("size", [(1, 1), (2, 7), (7, 2), (3, 3)])
def test_border_and_tiny_images_are_zero(size):
    depth, alpha, normal, w2c, K = O.case("noise", *size, 2)
    n = O.normals_from_depth(depth, w2c, K, alpha)
    inner = torch.zeros_like(n, dtype=torch.bool)
    inner[:, 1:-1, 1:-1] = True
    assert float(n[~inner].abs().sum()) == 0.0
    if min(size) < 3:
        assert float(n.abs().max()) == 0.0


def test_config_fields_match_the_reference():
    from b200gs.metrics import B200VanillaWithNormalRegMetrics
    assert {f.name: f.default for f in dataclasses.fields(B200VanillaWithNormalRegMetrics)} == META["config"]


@pytest.mark.parametrize("c", META["cases"], ids=lambda c: c["key"])
def test_setup_mutation_matches_the_reference(c):
    """the same draws of torch's global generator: rotations uniform, last log-scale lowered by log 5"""
    from b200gs.metrics import B200VanillaWithNormalRegMetrics
    from b200gs.scene import SyntheticGaussians
    *_, scene = golden_inputs(c)
    model = SyntheticGaussians(scene)
    metric = B200VanillaWithNormalRegMetrics(**c["config"]).instantiate()
    torch.manual_seed(c["seed"])
    metric.setup("fit", types.SimpleNamespace(gaussian_model=model))
    assert np.array_equal(model.gaussians["rotations"].detach().numpy(), Z[f"{c['key']}_rotations"])
    assert np.array_equal(model.gaussians["scales"].detach().numpy(), Z[f"{c['key']}_scales"])
    # other stages leave the model alone
    before = {k: v.detach().clone() for k, v in model.gaussians.items()}
    metric.setup("validate", types.SimpleNamespace(gaussian_model=model))
    assert all(torch.equal(before[k], v) for k, v in model.gaussians.items())


@pytest.mark.parametrize("missing", ["exp_depth", "alpha", "normal", "preprocessed_camera"])
def test_missing_render_output_is_named(missing):
    from b200gs.metrics import B200VanillaWithNormalRegMetrics
    metric = B200VanillaWithNormalRegMetrics().instantiate()
    outputs = {"exp_depth": torch.ones(1, 4, 4), "alpha": torch.ones(1, 4, 4), "normal": torch.ones(3, 4, 4),
               "preprocessed_camera": (torch.eye(4)[None], torch.eye(3)[None], (4, 4))}
    outputs[missing] = None
    with pytest.raises(ValueError, match=missing):
        metric.get_normal_reg_metrics(None, outputs, None, {"loss": torch.tensor(0.)}, {})


def test_depth_to_normal_refuses_what_it_does_not_provide():
    from b200gs.metrics import depth_to_normal
    d = torch.ones(4, 4, 1)
    with pytest.raises(NotImplementedError, match="z_depth"):
        depth_to_normal(d, torch.eye(4), torch.eye(3), z_depth=False)
    with pytest.raises(NotImplementedError, match="backward"):
        depth_to_normal(d.requires_grad_(True), torch.eye(4), torch.eye(3))
