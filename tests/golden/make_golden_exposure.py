"""Freeze the reference's learned exposure correction: the unmodified ExposureProcessor / ExposureProcessorModule of
internal/output_processors/exposure.py, run on the CPU in float32, for with_bias x shade_correction at two odd image sizes.  The
inputs are rebuilt by oracle.exposure_oracle.inputs, so only the module's outputs are stored: the processed render and the
gradients of the render, the exposure parameters and the shade map for a seeded cotangent.  Also recorded: the config fields and
defaults, the state_dict keys and shapes, and the training_setup groups and learning-rate schedule.  The reference's LambdaLR call
passes ``verbose``, which current torch no longer takes; the recording drops that keyword and changes nothing else.
The reference checkout is the first argument.
Run:  python tests/golden/make_golden_exposure.py <reference checkout>     -> tests/golden/exposure.npz, exposure.json"""
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
from oracle.exposure_oracle import inputs  # noqa: E402
from internal.output_processors.exposure import ExposureProcessor  # noqa: E402

_LambdaLR = torch.optim.lr_scheduler.LambdaLR


def lambda_lr(*args, verbose=None, **kwargs):
    return _LambdaLR(*args, **kwargs)


torch.optim.lr_scheduler.LambdaLR = lambda_lr

N_APPEARANCES = 5
# (H, W, shade_correction_size): the default 128 map on an image smaller than it, and a 7x7 map on a wide strip
SIZES = [(37, 50, 128), (11, 200, 7)]
arrays, meta = {}, {"n_appearances": N_APPEARANCES, "cases": []}


def module(with_bias, shade, size):
    proc = ExposureProcessor(with_bias=with_bias, shade_correction=shade, shade_correction_size=size).instantiate()
    proc.init_exposures(N_APPEARANCES, "cpu")
    return proc


seed = 0
for si, (H, W, size) in enumerate(SIZES):
    for with_bias in (False, True):
        for shade in (False, True):
            seed += 10
            key = f"s{si}_b{int(with_bias)}_c{int(shade)}"
            app_id = [0, 2, N_APPEARANCES - 1, 3][(seed // 10) % 4]
            render, params, shade_map, v_out = inputs(H, W, with_bias, size if shade else 0, seed, N_APPEARANCES)
            proc = module(with_bias, shade, size)
            with torch.no_grad():
                proc.exposure_parameters.copy_(torch.from_numpy(params))
                if shade:
                    proc.shade_correction.copy_(torch.from_numpy(shade_map))
            r = torch.from_numpy(render).requires_grad_(True)
            outputs = {"render": r}
            proc(types.SimpleNamespace(appearance_id=torch.tensor(app_id)), outputs)
            outputs["render"].backward(torch.from_numpy(v_out))
            arrays[f"{key}_out"] = outputs["render"].detach().numpy()
            arrays[f"{key}_v_render"] = r.grad.numpy()
            arrays[f"{key}_v_params"] = proc.exposure_parameters.grad.numpy()
            if shade:
                arrays[f"{key}_v_shade"] = proc.shade_correction.grad.numpy()
            meta["cases"].append({"key": key, "image": [H, W], "shade_correction_size": size, "with_bias": with_bias,
                                  "shade_correction": shade, "appearance_id": app_id, "seed": seed})

# config fields and defaults, state_dict, optimizer groups and schedule
meta["config"] = {f.name: f.default for f in dataclasses.fields(ExposureProcessor)}
meta["state_dict"], meta["training_setup"] = {}, {}
for with_bias in (False, True):
    for shade in (False, True):
        proc = module(with_bias, shade, 16)
        k = f"b{int(with_bias)}_c{int(shade)}"
        sd = proc.state_dict()
        meta["state_dict"][k] = {n: {"shape": list(v.shape), "dtype": str(v.dtype)} for n, v in sd.items()}
        arrays.update({f"sd_{k}_{n}": v.numpy() for n, v in sd.items()})
        opt, sched = proc.training_setup(None)
        lrs = []
        for it in (0, 1, 15000, 29999, 30000, 45000):
            lrs.append([g["initial_lr"] * sched.lr_lambdas[0](it) for g in opt.param_groups])
        meta["training_setup"][k] = {"optimizer": type(opt).__name__, "scheduler": type(sched).__name__,
                                     "groups": [{"name": g["name"], "lr": g["lr"], "shapes": [list(p.shape) for p in g["params"]],
                                                 "betas": list(g["betas"]), "eps": g["eps"]} for g in opt.param_groups],
                                     "lr_at": {"iterations": [0, 1, 15000, 29999, 30000, 45000], "lr": lrs}}

np.savez_compressed(os.path.join(HERE, "exposure.npz"), **arrays)
with open(os.path.join(HERE, "exposure.json"), "w") as f:
    json.dump(meta, f, indent=1)
print(json.dumps(meta["config"]), len(meta["cases"]), "cases")
