"""Freeze the reference's depth-normal regulariser: the unmodified VanillaWithNormalRegMetrics / VanillaWithNormalRegMetricsModule of
internal/metrics/normal_reg.py (on VanillaMetricsImpl and the reference's own internal/utils/ssim.py), run on the CPU in float32.
gsplat is not installed: ``gsplat.utils.depth_to_normal`` is oracle.normal_reg_oracle.depth_to_normal, the torch restatement of
gsplat's published function.  torchmetrics' PSNR and LPIPS are inert stand-ins (training metrics do not call them).
Each case seeds torch's global generator, runs ``setup("fit")`` on a SyntheticGaussians model (the rotations and scales mutation),
then ``get_train_metrics`` on the render outputs of oracle.normal_reg_oracle.case and ``backward``.
Recorded per case: loss, rgb_diff, ssim, normal_loss, flatten_loss, the progress-bar flags and metric keys, the rotations and scales
after setup, and the gradients of the render, the normal map and the raw scales.  Also recorded: the config fields and defaults.
Inputs are rebuilt from the seeds (``inputs`` below).
Run:  python tests/golden/make_golden_normal_reg.py <reference checkout>     -> tests/golden/normal_reg.npz, normal_reg.json"""
import dataclasses
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import normal_reg_oracle as O  # noqa: E402
from oracle.bilagrid_oracle import weyl  # noqa: E402

N_GAUSSIANS = 64
# (key, kind, H, W, seed, config): small odd sizes, so the arrays stay small enough to keep in git
CASES = [("plane_23x31", "plane", 23, 31, 11, {}),
         ("sphere_23x31", "sphere", 23, 31, 12, {}),
         ("noise_13x41", "noise", 13, 41, 13, {"normal_reg_lambda": 0.2, "flatten_reg": 0.1}),
         ("flat_13x41", "flat", 13, 41, 14, {})]


def inputs(kind, H, W, seed):
    """(render [3,H,W], gt [3,H,W], depth [1,H,W], alpha [1,H,W], normal [3,H,W], w2c [4,4], K [3,3], scene dict) float32 CPU"""
    from b200gs.scene import make_scene
    depth, alpha, normal, w2c, K = O.case(kind, H, W, seed)
    render = torch.from_numpy(weyl((3, H, W), seed + 10).astype(np.float32))
    gt = torch.from_numpy(weyl((3, H, W), seed + 11).astype(np.float32))
    return render, gt, depth[None], alpha[None], normal, w2c, K, make_scene(N_GAUSSIANS, seed)


if __name__ == "__main__":
    sys.path.insert(0, sys.argv[1])

    class _Inert:
        def __init__(self, *args, **kwargs):
            pass

    for name in ("torchmetrics", "torchmetrics.image", "torchmetrics.image.lpip", "gsplat", "gsplat.utils"):
        sys.modules[name] = types.ModuleType(name)
    sys.modules["torchmetrics.image"].PeakSignalNoiseRatio = _Inert
    sys.modules["torchmetrics.image.lpip"].LearnedPerceptualImagePatchSimilarity = _Inert
    sys.modules["gsplat.utils"].depth_to_normal = O.depth_to_normal

    from internal.metrics.normal_reg import VanillaWithNormalRegMetrics  # noqa: E402
    from b200gs.scene import SyntheticGaussians  # noqa: E402

    arrays, meta = {}, {"n_gaussians": N_GAUSSIANS, "cases": []}
    for key, kind, H, W, seed, config in CASES:
        render, gt, depth, alpha, normal, w2c, K, scene = inputs(kind, H, W, seed)
        metric = VanillaWithNormalRegMetrics(**config).instantiate()
        model = SyntheticGaussians(scene)
        pl_module = types.SimpleNamespace(device=torch.device("cpu"), gaussian_model=model)
        torch.manual_seed(seed)
        metric.setup("fit", pl_module)
        arrays[f"{key}_rotations"] = model.gaussians["rotations"].detach().numpy().copy()
        arrays[f"{key}_scales"] = model.gaussians["scales"].detach().numpy().copy()
        r = render.clone().requires_grad_(True)
        n = normal.clone().requires_grad_(True)
        outputs = {"render": r, "alpha": alpha, "exp_depth": depth, "normal": n, "preprocessed_camera": (w2c[None], K[None], (W, H))}
        batch = (None, ("img", gt, None), None)
        metrics, pbar = metric.get_train_metrics(pl_module, model, 0, batch, outputs)
        metrics["loss"].backward()
        for name in ("loss", "rgb_diff", "ssim", "normal_loss", "flatten_loss"):
            arrays[f"{key}_{name}"] = metrics[name].detach().numpy()
        arrays[f"{key}_v_render"] = r.grad.numpy()
        arrays[f"{key}_v_normal"] = n.grad.numpy()
        arrays[f"{key}_v_scales"] = model.gaussians["scales"].grad.numpy()
        meta["cases"].append({"key": key, "kind": kind, "image": [H, W], "seed": seed, "config": config, "pbar": pbar,
                              "metric_keys": sorted(metrics)})

    meta["config"] = {f.name: f.default for f in dataclasses.fields(VanillaWithNormalRegMetrics)}
    np.savez_compressed(os.path.join(HERE, "normal_reg.npz"), **arrays)
    with open(os.path.join(HERE, "normal_reg.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print(json.dumps(meta["config"]), len(meta["cases"]), "cases")
