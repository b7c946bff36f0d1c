"""Freeze the reference's Gaussian regularisers: the unmodified MCMCMetrics, ScaleRegularizationMetrics and
ScaleRegularizationWithDepthMetrics modules of internal/metrics/mcmc_metrics.py and scale_regularization_metrics.py, run on the CPU
in float32 on a stand-in Gaussian model with VanillaGaussianModel's activations (get_opacity = sigmoid, get_scaling =
get_scales() = exp of the raw parameters).  torchmetrics is replaced by stand-ins in sys.modules before the import, as in
make_golden_depth_metrics.py; validation's PSNR and LPIPS stand-ins return fixed numbers.
Two seeded scenes with oracle.gaussian_reg_oracle's crafted rows (isotropic, tied min / mid with a ratio > 10, underflowing
logits and log-scales, a scale equal to max_scale, ratios one ulp either side of 10).  Cases: steps either side of
mcmc_reg_until_iter and scale_reg_from, reg_weight_decay above 5, scale_reg = 0, scale_reg_lambda = 0, max_scale = -1 resolved in
setup, the validation path and the depth variant with an l1 depth map.
Recorded per case: every output key, the progress-bar flags, and the gradients of the raw opacities and scales.  Also recorded:
the three configs' fields and defaults.  Inputs are rebuilt by oracle.gaussian_reg_oracle.scene and rgb_inputs below.
Run:  python tests/golden/make_golden_gaussian_reg.py <reference checkout>     -> tests/golden/gaussian_reg.npz, gaussian_reg.json"""
import dataclasses
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, sys.argv[1])
from oracle.bilagrid_oracle import weyl  # noqa: E402
from oracle.gaussian_reg_oracle import MAX_SCALE, scene  # noqa: E402

PSNR, LPIPS = 23.5, 0.25


class _Inert:
    def __init__(self, *args, **kwargs):
        pass


class _Psnr(_Inert):
    def __call__(self, *args):
        return torch.tensor(PSNR)


class _Lpips(_Inert):
    def __call__(self, *args):
        return torch.tensor(LPIPS)


for name in ("torchmetrics", "torchmetrics.image", "torchmetrics.image.lpip"):
    sys.modules[name] = types.ModuleType(name)
sys.modules["torchmetrics.image"].PeakSignalNoiseRatio = _Psnr
sys.modules["torchmetrics.image"].StructuralSimilarityIndexMeasure = _Inert
sys.modules["torchmetrics.image.lpip"].LearnedPerceptualImagePatchSimilarity = _Lpips

from internal.metrics.mcmc_metrics import MCMCMetrics  # noqa: E402
from internal.metrics.scale_regularization_metrics import ScaleRegularizationMetrics, ScaleRegularizationWithDepthMetrics  # noqa: E402

SCENES = [(97, 5), (203, 6)]
H, W = 12, 16
CAMERA_EXTENT = 0.8           # max_scale = -1 resolves to 0.88


class Model(torch.nn.Module):
    """VanillaGaussianModel's parameters and getters (internal/models/vanilla_gaussian.py:345-358,422-440)"""

    def __init__(self, opac, scales):
        super().__init__()
        self.gaussians = torch.nn.ParameterDict({"opacities": torch.nn.Parameter(torch.from_numpy(opac)),
                                                 "scales": torch.nn.Parameter(torch.from_numpy(scales))})

    @property
    def get_opacity(self):
        return torch.sigmoid(self.gaussians["opacities"])

    @property
    def get_scaling(self):
        return torch.exp(self.gaussians["scales"])

    def get_scales(self):
        return self.get_scaling


def rgb_inputs(seed):
    """float32 render and gt image [3,H,W] in [0, 1), and the l1 depth maps [1,H,W] / [H,W]"""
    return (weyl((3, H, W), seed + 10).astype(np.float32), weyl((3, H, W), seed + 11).astype(np.float32),
            weyl((1, H, W), seed + 12).astype(np.float32), weyl((H, W), seed + 13).astype(np.float32))


CASES = [
    # (key, metric, config kwargs, stage, step, scene)
    ("mcmc_default", "mcmc", {}, "train", 100, 0),
    ("mcmc_before_until", "mcmc", {"mcmc_reg_until_iter": 500}, "train", 499, 1),
    ("mcmc_at_until", "mcmc", {"mcmc_reg_until_iter": 500}, "train", 500, 0),
    ("mcmc_decay_above_5", "mcmc", {"reg_weight_decay": 8.0, "opacity_reg": 0.05, "scale_reg": 0.02}, "train", 3, 1),
    ("mcmc_scale_reg_0", "mcmc", {"scale_reg": 0.0}, "train", 10, 0),
    ("mcmc_validate", "mcmc", {"mcmc_reg_until_iter": 10}, "validate", 0, 1),
    ("scale_default", "scale", {"max_scale": MAX_SCALE}, "train", 3100, 0),
    ("scale_before_from", "scale", {"max_scale": MAX_SCALE}, "train", 3099, 1),
    ("scale_from_0", "scale", {"max_scale": MAX_SCALE, "scale_reg_from": 0, "scale_reg_lambda": 0.1, "scale_ratio_reg_lambda": 0.2},
     "train", 0, 1),
    ("scale_lambda_0", "scale", {"max_scale": MAX_SCALE, "scale_reg_lambda": 0.0}, "train", 4000, 0),
    ("scale_max_resolved", "scale", {}, "train", 5000, 1),
    ("scale_validate", "scale", {"max_scale": MAX_SCALE}, "validate", 0, 0),
    ("depth_l1", "depth", {"max_scale": MAX_SCALE, "depth_loss_type": "l1"}, "train", 4000, 1),
    ("depth_before_from", "depth", {"max_scale": MAX_SCALE, "depth_loss_type": "l1"}, "train", 100, 0),
]
CONFIGS = {"mcmc": MCMCMetrics, "scale": ScaleRegularizationMetrics, "depth": ScaleRegularizationWithDepthMetrics}


class DepthStandIn:
    def __init__(self, gt):
        self.gt, self.median, self.mask, self.camera = gt, None, None, None

    def get(self, device):
        return self.gt.to(device)


def value(v):
    return float(v.detach()) if torch.is_tensor(v) else float(v)


arrays, meta = {"max_scale_threshold": np.float32(MAX_SCALE)}, {"scenes": SCENES, "image": [H, W], "camera_extent": CAMERA_EXTENT,
                                                                "psnr": PSNR, "lpips": LPIPS, "cases": []}
for si, (n, seed) in enumerate(SCENES):
    opac, scales = scene(n, seed)
    arrays[f"s{si}_opacities"], arrays[f"s{si}_scales"] = opac, scales
for key, kind, kwargs, stage, step, si in CASES:
    n, seed = SCENES[si]
    opac, scales = scene(n, seed)
    config = CONFIGS[kind](**kwargs)
    metric = config.instantiate()
    pl_module = types.SimpleNamespace(device=torch.device("cpu"), trainer=types.SimpleNamespace(datamodule=types.SimpleNamespace(
        dataparser_outputs=types.SimpleNamespace(camera_extent=CAMERA_EXTENT))))
    metric.setup("fit" if stage == "train" else "validate", pl_module)
    model = Model(opac, scales)
    render, gt_rgb, depth, gt_depth = rgb_inputs(seed)
    r = torch.from_numpy(render).requires_grad_(True)
    outputs = {"render": r}
    extra = None
    if kind == "depth":
        outputs["inverse_depth"] = torch.from_numpy(depth).requires_grad_(True)
        extra = DepthStandIn(torch.from_numpy(gt_depth))
    batch = (types.SimpleNamespace(device=torch.device("cpu")), ("img", torch.from_numpy(gt_rgb), None), extra)
    if stage == "train":
        metrics, pbar = metric.get_train_metrics(pl_module, model, step, batch, outputs)
    else:
        metrics, pbar = metric.get_validate_metrics(pl_module, model, batch, outputs)
    metrics["loss"].backward()
    for name, p in model.gaussians.items():
        arrays[f"{key}_v_{name}"] = (p.grad if p.grad is not None else torch.zeros_like(p)).numpy()
    arrays[f"{key}_v_render"] = r.grad.numpy()
    meta["cases"].append({"key": key, "metric": kind, "config": kwargs, "stage": stage, "step": step, "scene": si,
                          "resolved_max_scale": getattr(metric.config, "max_scale", None),
                          "metrics": {k: value(v) for k, v in metrics.items()}, "pbar": pbar,
                          "weights": [getattr(metric, "opacity_reg_weight", None), getattr(metric, "scale_reg_weight", None)]})

meta["config"] = {kind: {f.name: (dataclasses.asdict(f.default_factory()) if f.default_factory is not dataclasses.MISSING else f.default)
                         for f in dataclasses.fields(cls)} for kind, cls in CONFIGS.items()}
meta["mro"] = {kind: [c.__name__ for c in type(cls().instantiate()).__mro__]
               for kind, cls in CONFIGS.items()}
np.savez_compressed(os.path.join(HERE, "gaussian_reg.npz"), **arrays)
with open(os.path.join(HERE, "gaussian_reg.json"), "w") as f:
    json.dump(meta, f, indent=1)
print(len(meta["cases"]), "cases")
