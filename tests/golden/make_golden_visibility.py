"""Record the reference's transient visibility map: the unmodified Model and GSplatAppearanceEmbeddingVisibilityMapRenderer of
internal/renderers/gsplat_appearance_embedding_visibility_map_renderer.py and VisibilityMapMetrics(Impl) of
internal/metrics/visibility_map_metrics.py, on the CPU in float32:
    python tests/golden/make_golden_visibility.py <reference checkout>   -> tests/golden/visibility.npz, visibility.json

tinycudann cannot be installed, so the renderer module imports a recording stand-in whose Encoding computes the oracle's grid
(oracle/visibility_oracle.py: the grid is parity unpinned) and stores every constructor and forward call it receives; the gsplat
names the module imports are inert stand-ins and torchmetrics' classes are inert too (VanillaMetricsImpl.setup builds PSNR and
LPIPS, which get_train_metrics never calls).  Parameters and inputs are not stored: they are rebuilt by visibility_oracle's
golden_param / golden_inputs.  Recorded per case (size, appearance id, dataset mask or none, the visibility's gradient on or off):
the visibility map, loss, rgb_diff, ssim, vis_reg, the progress-bar flags, and the gradients of the render, the visibility, the
image's transient embedding and the visibility network, plus the grid gradient's dot product with golden_probe and which grids got
one.  Once: the appearance network on 48 rows (outputs and gradients), the config defaults, the state_dict keys and shapes, the
five optimizers' groups, eps and LambdaLR values, and training_forward's warm-up branches."""
import dataclasses
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_v1_dropin as stubs  # noqa: E402  (puts the repository and the reference checkout on sys.path)
from oracle import visibility_oracle as V  # noqa: E402

N_IMAGES = 3
CASES = [  # name, W, H, appearance id, masked, visibility gradient (off: the map is a constant, as the warm-ups hand it)
    ("s0_plain", 23, 17, 1, False, True),
    ("s0_mask", 23, 17, 2, True, True),
    ("s1_mask", 13, 29, 0, True, True),
    ("s1_novisgrad", 13, 29, 2, False, False),
]
CALLS = []


class Encoding(torch.nn.Module):
    """tinycudann.Encoding stand-in: the oracle's DenseGrid, recording its calls"""

    def __init__(self, n_input_dims, encoding_config, seed=1337, dtype=None):
        super().__init__()
        self.config = dict(encoding_config)
        self.grid = {k: self.config[k] for k in ("n_levels", "base_resolution", "per_level_scale")}
        self.params = torch.nn.Parameter(torch.zeros(V.n_params(**self.grid)))
        self.n_output_dims = 2 * self.grid["n_levels"]
        CALLS.append({"call": "Encoding", "n_input_dims": n_input_dims, "encoding_config": self.config, "seed": seed, "dtype": str(dtype)})

    def forward(self, x):
        x = x.detach().numpy()
        CALLS.append({"call": "Encoding.forward", "shape": list(x.shape), "dtype": str(x.dtype), "sum": float(x.astype(np.float64).sum()),
                      "first": x[:2].tolist(), "last": x[-2:].tolist()})
        return V.encode(self.params, x[:, 0], x[:, 1], **self.grid).float()


class _Marker(torch.nn.Module):
    def forward(self, *args, **kwargs):
        return {"render": "plain"}


class _LambdaLR(torch.optim.lr_scheduler.LambdaLR):
    """the reference passes verbose=False, an argument later torch releases removed"""

    def __init__(self, *args, verbose=False, **kwargs):
        super().__init__(*args, **kwargs)


def install():
    stubs.install_stubs()
    torch.optim.lr_scheduler.LambdaLR = _LambdaLR
    noop = lambda *a, **k: None      # noqa: E731
    for name, attrs in (("gsplat.sh", {"spherical_harmonics": noop}), ("gsplat.v0_interfaces", {"project_gaussians": noop}),
                        ("gsplat.rasterize", {"rasterize_gaussians": noop}), ("tinycudann", {"Encoding": Encoding}),
                        ("torchmetrics", {}), ("torchmetrics.image", {"PeakSignalNoiseRatio": noop}),
                        ("torchmetrics.image.lpip", {"LearnedPerceptualImagePatchSimilarity": noop})):
        m = sys.modules.get(name) or types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m


def load_golden_state(model):
    model.load_state_dict({k: V.golden_param(k, v.shape) for k, v in model.state_dict().items()})


def main():
    install()
    import internal.renderers.gsplat_appearance_embedding_visibility_map_renderer as R
    from internal.metrics.visibility_map_metrics import VisibilityMapMetrics

    out, meta = {}, {"cases": [], "calls": None, "encodings": None}
    renderer = R.GSplatAppearanceEmbeddingVisibilityMapRenderer(R.ModelConfig(n_images=N_IMAGES), R.OptimizationConfig())
    renderer.setup("fit", None)
    model = renderer.model
    load_golden_state(model)
    meta["state_dict"] = {k: list(v.shape) for k, v in renderer.state_dict().items()}
    meta["model_config"] = dataclasses.asdict(R.ModelConfig())
    meta["optimization_config"] = dataclasses.asdict(R.OptimizationConfig())
    opts, scheds = renderer.training_setup(None)
    meta["optimizers"] = [{"name": o.param_groups[0]["name"], "lr": o.param_groups[0]["lr"], "eps": o.defaults["eps"],
                           "n_params": len(o.param_groups[0]["params"]),
                           "lambda": {str(s): sc.lr_lambdas[0](s) for s in (0, 999, 1000, 2500, 31_000, 40_000)}}
                          for o, sc in zip(opts, scheds)]
    metric_config = VisibilityMapMetrics()
    meta["metric"] = {"vis_reg_factor": metric_config.vis_reg_factor, "lambda_dssim": metric_config.lambda_dssim}
    metric = metric_config.instantiate()
    metric.setup("fit", None)

    # training_forward's warm-up branches, with the renders replaced by markers (the rasterizer is not what is recorded here)
    saved_forward, saved_renderer = renderer.forward, renderer.renderer
    renderer.renderer = _Marker()
    renderer.forward = lambda *a, **k: {"render": "full", "visibility": "map"}
    cam = types.SimpleNamespace(width=5, height=4)
    module = types.SimpleNamespace(device=torch.device("cpu"))
    meta["warm_up"] = {}
    for step in (0, 999, 1000, 1999, 2000, 5000):
        o = renderer.training_forward(step, module, cam, None, None)
        vis = o["visibility"]
        meta["warm_up"][str(step)] = [o["render"], "ones" if torch.is_tensor(vis) and bool((vis == 1).all()) and
                                      tuple(vis.shape) == (1, 4, 5) else vis]
    renderer.forward, renderer.renderer = saved_forward, saved_renderer

    meta["encodings"] = [c for c in CALLS if c["call"] == "Encoding"]
    CALLS.clear()
    for name, W, H, aid, masked, vis_grad in CASES:
        model.zero_grad(set_to_none=True)
        render, gt, mask = V.golden_inputs(W, H, len(name) + W)
        render.requires_grad_(True)
        appearance = torch.tensor([aid])
        vis = model.visibility_forward(W, H, appearance).unsqueeze(0)
        if not vis_grad:
            vis = vis.detach()
        else:
            vis.retain_grad()
        metrics, pbar = metric.get_train_metrics(None, None, 5000, (None, ("img", gt, mask if masked else None), None),
                                                 {"render": render, "visibility": vis})
        metrics["loss"].backward()
        p = f"{name}."
        out[p + "visibility"] = vis.detach()[0].numpy()
        out[p + "v_render"] = render.grad.numpy()
        for k in ("loss", "rgb_diff", "ssim", "vis_reg"):
            out[p + k] = np.float64(metrics[k].detach())
        case = {"name": name, "W": W, "H": H, "aid": aid, "masked": masked, "vis_grad": vis_grad, "pbar": pbar}
        if vis_grad:
            out[p + "v_visibility"] = vis.grad[0].numpy()
            out[p + "v_transient"] = model.transient_embedding.weight.grad[aid].numpy()
            for k, t in model.visibility_network.named_parameters():
                out[p + "v_vnet." + k] = t.grad.numpy()
            g = model.uv_encodings[aid].params.grad.double()
            case["grid_grad_probe"] = float(g @ V.golden_probe(g.numel()))
            case["grid_grad_nonzero"] = int((g != 0).sum())
            case["grids_with_grad"] = [i for i in range(N_IMAGES) if model.uv_encodings[i].params.grad is not None]
        meta["cases"].append(case)
    meta["calls"] = list(CALLS)

    # the appearance network (Model.appearance_forward), 48 rows, view-independent as the configs
    model.zero_grad(set_to_none=True)
    feats = V.golden_param("features", (48, 64)).requires_grad_(True)
    cot = V.golden_param("cot", (48, 3))
    rgb = model.appearance_forward(feats, torch.tensor([1]), None)
    (rgb * cot).sum().backward()
    out["app.out"] = rgb.detach().numpy()
    out["app.v_features"] = feats.grad.numpy()
    out["app.v_embedding"] = model.appearance_embedding.weight.grad[1].numpy()
    for k, t in model.appearance_network.named_parameters():
        out["app.v_net." + k] = t.grad.numpy()

    np.savez_compressed(os.path.join(HERE, "visibility.npz"), **{k: np.asarray(v, dtype=np.float32 if np.asarray(v).dtype != np.float64
                                                                                 or np.asarray(v).ndim else np.float64)
                                                                 for k, v in out.items()})
    with open(os.path.join(HERE, "visibility.json"), "w") as f:
        json.dump(meta, f, indent=1)


if __name__ == "__main__":
    main()
