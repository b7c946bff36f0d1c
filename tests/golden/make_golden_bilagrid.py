"""Freeze the reference's bilateral grid (internal/utils/lib_bilagrid.py: slice, total_variation_loss, BilateralGrid) and its
unmodified BilagridProcessorModule (internal/output_processors/bilagrid.py) with fused: true, run on the CPU in float32.  The inputs
are rebuilt by oracle.bilagrid_oracle.golden_inputs (grids perturbed away from the identity, black, white and out-of-range colours,
xy outside [0, 1]), so only the reference's outputs are stored, large ones at the flat entries golden_index(size) names.
``fused_bilagrid`` is a recording stand-in that delegates to lib_bilagrid; tensorly (imported by lib_bilagrid for the CP-decomposed
4-D grid only) is stubbed.  The reference checkout is the first argument.
Run:  python tests/golden/make_golden_bilagrid.py <reference checkout>     -> tests/golden/bilagrid.npz, bilagrid.json"""
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, sys.argv[1])
from oracle.bilagrid_oracle import golden_index, golden_inputs, processor_inputs  # noqa: E402

tl = types.ModuleType("tensorly")
tl.set_backend = lambda name: None
tl_dec = types.ModuleType("tensorly.decomposition")
tl_dec.parafac = None
tl.decomposition = tl_dec
sys.modules["tensorly"], sys.modules["tensorly.decomposition"] = tl, tl_dec
from internal.utils import lib_bilagrid as LB  # noqa: E402

calls = []
fb = types.ModuleType("fused_bilagrid")
fb.BilateralGrid = LB.BilateralGrid
fb.total_variation_loss = LB.total_variation_loss


def recording_slice(bil_grids, xy, rgb, grid_idx):
    calls.append({"xy": {"shape": list(xy.shape), "dtype": str(xy.dtype), "stride": list(xy.stride()),
                         "requires_grad": xy.requires_grad},
                  "rgb": {"shape": list(rgb.shape), "dtype": str(rgb.dtype), "stride": list(rgb.stride())},
                  "grid_idx": {"shape": list(grid_idx.shape), "dtype": str(grid_idx.dtype), "values": grid_idx.reshape(-1).tolist()}})
    return LB.slice(bil_grids, xy, rgb, grid_idx)


fb.slice = recording_slice
sys.modules["fused_bilagrid"] = fb
from internal.output_processors.bilagrid import BilagridProcessor  # noqa: E402

N_GRIDS = 3
GRID_SIZES = [(16, 16, 8), (5, 3, 2), (1, 1, 1)]      # (grid_X, grid_Y, grid_W)
IMAGES = {(16, 16, 8): [(37, 50), (1, 1)], (5, 3, 2): [(9, 13), (1, 1)], (1, 1, 1): [(9, 13), (1, 1)]}
arrays, meta = {}, {"n_grids": N_GRIDS, "cases": [], "tv": []}


def flat(a):
    a = np.ascontiguousarray(a).reshape(-1)
    return a[golden_index(a.size)]


def module(grids):
    bg = LB.BilateralGrid(grids.shape[0], grid_X=grids.shape[4], grid_Y=grids.shape[3], grid_W=grids.shape[2])
    with torch.no_grad():
        bg.grids.copy_(torch.from_numpy(grids))
    return bg


seed = 0
for gi, grid in enumerate(GRID_SIZES):
    for ii, image in enumerate(IMAGES[grid]):
        seed += 10
        key = f"g{gi}_i{ii}"
        grids, xy, rgb, v_out = golden_inputs(N_GRIDS, grid, image, seed)
        bg = module(grids)
        rgb_t = torch.from_numpy(rgb).requires_grad_(True)
        out = LB.slice(bg, torch.from_numpy(xy), rgb_t, torch.tensor([[1]]))["rgb"]
        (out * torch.from_numpy(v_out)).sum().backward()
        arrays.update({f"{key}_out": flat(out.detach().numpy()), f"{key}_v_rgb": flat(rgb_t.grad.numpy()),
                       f"{key}_v_grids": flat(bg.grids.grad.numpy())})
        meta["cases"].append({"key": key, "grid": list(grid), "image": list(image), "seed": seed, "grid_idx": 1})
    seed += 10
    grids = golden_inputs(N_GRIDS, grid, (1, 1), seed)[0]
    bg = module(grids)
    tv = LB.total_variation_loss(bg.grids)
    tv.backward()
    arrays.update({f"tv{gi}_value": np.float32(tv.item()), f"tv{gi}_grad": flat(bg.grids.grad.numpy())})
    meta["tv"].append({"key": f"tv{gi}", "grid": list(grid), "seed": seed})

# the unmodified processor with fused: true on a stub camera
H, W, SEED = 37, 50, 100
proc = BilagridProcessor().instantiate()
proc.init_bilagrid(N_GRIDS, "cpu")
proc_grids, proc_render = processor_inputs(SEED, N_GRIDS, (H, W))
with torch.no_grad():
    proc.bgrid.grids.copy_(torch.from_numpy(proc_grids))
camera = types.SimpleNamespace(device=torch.device("cpu"), height=torch.tensor(H), width=torch.tensor(W),
                               appearance_id=torch.tensor(2))
outputs = {"render": torch.from_numpy(proc_render)}
proc(camera, outputs)
metrics, pbar = {"loss": torch.tensor(0.0)}, {}
proc.tv_loss(outputs, None, None, 0, None, metrics, pbar)
arrays.update({"proc_out": flat(outputs["render"].detach().numpy()), "proc_tv": np.float32(metrics["tv"].item())})
meta["processor"] = {"calls": calls, "image": [H, W], "seed": SEED, "appearance_id": 2, "tv_loss_weight": proc.config.tv_loss_weight,
                     "out_shape": list(outputs["render"].shape), "out_stride": list(outputs["render"].stride())}

# state_dict of a fresh lib_bilagrid.BilateralGrid(3)
sd = LB.BilateralGrid(3).state_dict()
meta["state_dict"] = {k: {"shape": list(v.shape), "dtype": str(v.dtype)} for k, v in sd.items()}
arrays.update({f"sd_{k}": v.numpy() for k, v in sd.items()})

np.savez_compressed(os.path.join(HERE, "bilagrid.npz"), **arrays)
with open(os.path.join(HERE, "bilagrid.json"), "w") as f:
    json.dump(meta, f, indent=1)
print(json.dumps(meta["processor"]["calls"]), "tv", float(arrays["proc_tv"]))
