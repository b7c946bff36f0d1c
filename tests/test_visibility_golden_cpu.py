"""The float64 oracle and the plug-ins against recordings of the reference's own visibility-map renderer and metric
(tests/golden/visibility.npz / .json, made by make_golden_visibility.py from the unmodified modules, with the oracle's grid standing
in for tinycudann): the visibility map, the masked loss and its statistics, the gradients of the render, the visibility, the
transient embedding, the visibility network and the grid (through a probe), the appearance network, the encoder's inputs, and the
plug-in renderer's config defaults, state_dict keys and shapes, optimizers and warm-up branches."""
import dataclasses
import json
import os
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import visibility_oracle as V
from oracle.appearance_oracle import mlp as oracle_mlp

Z = np.load(os.path.join(GOLDEN, "visibility.npz"))
META = json.load(open(os.path.join(GOLDEN, "visibility.json")))
N_IMAGES = 3


def rel(a, ref):
    a, ref = np.asarray(a, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    return np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-30)


def golden_state(dtype=torch.float64):
    """the recorded Model's parameters, keyed as the reference's renderer state_dict (without the `model.` prefix)"""
    return {k[len("model."):]: V.golden_param(k[len("model."):], s).to(dtype) for k, s in META["state_dict"].items()}


def vnet(state):
    ws = [state[f"visibility_network.output_layers.{i}.weight"] for i in (0, 2, 4)]
    bs = [state[f"visibility_network.output_layers.{i}.bias"] for i in (0, 2, 4)]
    return ws, bs


@pytest.mark.parametrize("case", META["cases"], ids=[c["name"] for c in META["cases"]])
def test_oracle_matches_the_reference(case):
    W, H, aid, name = case["W"], case["H"], case["aid"], case["name"]
    state = {k: v.requires_grad_(True) for k, v in golden_state().items()}
    render, gt, mask = V.golden_inputs(W, H, len(name) + W)
    render = render.double().requires_grad_(True)
    ws, bs = vnet(state)
    vis = V.visibility(state[f"uv_encodings.{aid}.params"], state["transient_embedding.weight"][aid], ws, bs, W, H).unsqueeze(0)
    if not case["vis_grad"]:
        vis = vis.detach()
    else:
        vis.retain_grad()
    loss, l1, s, reg = V.masked_loss(render, gt.double(), vis, mask if case["masked"] else None)
    loss.backward()
    p = name + "."
    assert np.abs(vis.detach()[0].numpy() - Z[p + "visibility"]).max() <= 1e-6
    for k, v in (("loss", loss), ("rgb_diff", l1), ("ssim", s), ("vis_reg", reg)):
        assert abs(float(v) - float(Z[p + k])) <= 2e-6, k
    assert rel(render.grad, Z[p + "v_render"]) <= 1e-4
    assert case["pbar"] == {"loss": True, "rgb_diff": True, "ssim": True, "vis_reg": True}
    if case["vis_grad"]:
        assert rel(vis.grad[0], Z[p + "v_visibility"]) <= 1e-4
        assert rel(state["transient_embedding.weight"].grad[aid], Z[p + "v_transient"]) <= 1e-4
        for i in (0, 2, 4):
            for t in ("weight", "bias"):
                g = state[f"visibility_network.output_layers.{i}.{t}"].grad
                assert rel(g, Z[f"{p}v_vnet.output_layers.{i}.{t}"]) <= 1e-4
        g = state[f"uv_encodings.{aid}.params"].grad
        assert abs(float(g @ V.golden_probe(g.numel())) - case["grid_grad_probe"]) <= 1e-4 * abs(case["grid_grad_probe"])
        assert int((g != 0).sum()) == case["grid_grad_nonzero"] and case["grids_with_grad"] == [aid]


def test_encoder_inputs_are_the_oracle_pixel_grid():
    calls = [c for c in META["calls"] if c["call"] == "Encoding.forward"]
    assert len(calls) == len(META["cases"])
    for c, case in zip(calls, META["cases"]):
        u, v = V.pixel_uv(case["W"], case["H"])
        uv = np.stack([u, v], 1)
        assert c["shape"] == [case["W"] * case["H"], 2] and c["dtype"] == "float32"
        assert c["sum"] == float(uv.astype(np.float64).sum())
        assert np.array_equal(np.float32(c["first"]), uv[:2]) and np.array_equal(np.float32(c["last"]), uv[-2:])
    for e in META["encodings"]:
        assert e["n_input_dims"] == 2 and e["dtype"] == "torch.float32"
        assert e["encoding_config"] == {"otype": "DenseGrid", "n_levels": 8, "base_resolution": 16, "per_level_scale": 1.405}


def test_appearance_network_matches_the_reference():
    state = {k: v.requires_grad_(True) for k, v in golden_state().items()}
    feats = V.golden_param("features", (48, 64)).double().requires_grad_(True)
    cot = V.golden_param("cot", (48, 3)).double()
    ws = [state[f"appearance_network.output_layers.{i}.weight"] for i in (0, 2, 4)]
    bs = [state[f"appearance_network.output_layers.{i}.bias"] for i in (0, 2, 4)]
    out = oracle_mlp(feats, state["appearance_embedding.weight"][1], ws, bs)
    (out * cot).sum().backward()
    assert np.abs(out.detach().numpy() - Z["app.out"]).max() <= 1e-6
    assert rel(feats.grad, Z["app.v_features"]) <= 1e-4
    assert rel(state["appearance_embedding.weight"].grad[1], Z["app.v_embedding"]) <= 1e-4
    for i in (0, 2, 4):
        for t in ("weight", "bias"):
            assert rel(state[f"appearance_network.output_layers.{i}.{t}"].grad, Z[f"app.v_net.output_layers.{i}.{t}"]) <= 1e-4


class _Marker(torch.nn.Module):
    def forward(self, *args, **kwargs):
        return {"render": "plain"}


def test_plug_in_config_state_dict_optimizers_and_warm_ups_follow_the_reference():
    from b200gs import visibility as B
    from b200gs.metrics import B200VisibilityMapMetrics
    from b200gs.scene import make_ring_cameras
    assert dataclasses.asdict(B.ModelConfig()) == META["model_config"]
    assert dataclasses.asdict(B.OptimizationConfig()) == META["optimization_config"]
    m = B200VisibilityMapMetrics()
    assert (m.vis_reg_factor, m.lambda_dssim) == (META["metric"]["vis_reg_factor"], META["metric"]["lambda_dssim"])
    r = B.B200GSplatAppearanceEmbeddingVisibilityMapRenderer(B.ModelConfig(n_images=N_IMAGES), B.OptimizationConfig())
    r.setup("fit")
    assert {k: list(v.shape) for k, v in r.state_dict().items()} == META["state_dict"]
    r.load_state_dict({k: V.golden_param(k[len("model."):], s) for k, s in META["state_dict"].items()})
    opts, scheds = r.training_setup(None)
    got = [{"name": o.param_groups[0]["name"], "lr": o.param_groups[0]["lr"], "eps": o.defaults["eps"],
            "n_params": len(o.param_groups[0]["params"]),
            "lambda": {str(s): sc.lr_lambdas[0](s) for s in (0, 999, 1000, 2500, 31_000, 40_000)}} for o, sc in zip(opts, scheds)]
    assert got == META["optimizers"]
    cam = make_ring_cameras(5, 4)[0]
    r.renderer = _Marker()
    r.forward = lambda *a, **k: {"render": "full", "visibility": "map"}
    module = types.SimpleNamespace(device=torch.device("cpu"))
    for step, (render, vis) in META["warm_up"].items():
        o = r.training_forward(int(step), module, cam, None, None)
        v = o["visibility"]
        assert [o["render"], "ones" if torch.is_tensor(v) and bool((v == 1).all()) and tuple(v.shape) == (1, 4, 5) else v] == [render, vis]
