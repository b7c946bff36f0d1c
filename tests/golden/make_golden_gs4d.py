"""Record the reference's 4DGS deformation: the unmodified VanillaGS4DRenderer of internal/renderers/vanilla_gs4d_renderer.py (with
gs4d_deformation.deform_network and gs4d_hexplane.HexPlaneField) on the CPU in float32:
    python tests/golden/make_golden_gs4d.py <reference checkout>   -> tests/golden/gs4d.npz, gs4d.json

Per case a checkpoint directory in the reference's format is written (cfg_args as an argparse.Namespace repr, point_cloud/
iteration_<n>/deformation.pth and deformation_table.pth), the renderer is built on it, and VanillaRenderer.render is replaced by a stub
that captures what the renderer hands it: the deformed means, the activated deformed scales and rotations, the opacity and the SH
features.  Every parameter of the checkpoint is a function of its state_dict key and index (``state_dict_values``), so the tests
rebuild the large default-like grids instead of storing them; the small grids' planes are stored as well.  The Gaussians are seeded
and stored: points outside the aabb (border clamp), on grid nodes and at the aabb corners, unnormalised quaternions, t of 0, 1 and
interior values, and N = 1."""
import json
import os
import sys
import tempfile
import zlib
from argparse import Namespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))

BASE_CFG = dict(net_width=64, timebase_pe=4, defor_depth=1, posebase_pe=10, scale_rotation_pe=2, opacity_pe=2, timenet_width=64,
                timenet_output=32, bounds=1.6, grid_pe=0, no_grid=False, empty_voxel=False, static_mlp=False, no_dx=False, no_ds=False,
                no_dr=False, no_do=True, no_dshs=True, apply_rotation=False,
                kplanes_config={"grid_dimensions": 2, "input_coordinate_dim": 4, "output_coordinate_dim": 32, "resolution": [64, 64, 64, 25]},
                multires=[1, 2, 4, 8])
SMALL = {"grid_dimensions": 2, "input_coordinate_dim": 4, "output_coordinate_dim": 16, "resolution": [6, 5, 4, 3]}
# name: (cfg overrides, t, N, stored planes); the aabb is (xyz_max, xyz_min)
CASES = {
    "small_d1": (dict(kplanes_config=SMALL, multires=[1, 2], no_dshs=False), 0.0, 64, True),
    "small_rotation": (dict(kplanes_config=SMALL, multires=[1, 2], no_dshs=False, apply_rotation=True), 1.0, 64, True),
    "small_d2": (dict(kplanes_config=SMALL, multires=[1, 2, 3], defor_depth=2, no_ds=True, net_width=128), 0.37, 64, True),
    "small_d0_n1": (dict(kplanes_config={**SMALL, "output_coordinate_dim": 32}, multires=[2], defor_depth=0, no_dx=True,
                         apply_rotation=True), 0.5, 1, True),
    "default": (dict(), 0.6, 300, False),
    "hypernerf_like": (dict(kplanes_config={**BASE_CFG["kplanes_config"], "output_coordinate_dim": 16, "resolution": [64, 64, 64, 150]},
                            multires=[1, 2, 4], net_width=128, defor_depth=1, no_dshs=False, apply_rotation=True), 0.25, 300, False),
}
AABB = ((1.5, 1.2, 1.0), (-1.3, -1.1, -0.9))
ITERATION = 14000


def case_cfg(name) -> Namespace:
    over = CASES[name][0]
    return Namespace(**{**BASE_CFG, **over})


def resolutions(cfg):
    kp = cfg.kplanes_config
    return [[r * m for r in kp["resolution"][:3]] + list(kp["resolution"][3:]) for m in cfg.multires]


def golden_value(key: str, shape) -> torch.Tensor:
    """the checkpoint's value of state_dict entry ``key``: a smooth function of the index, salted by the key"""
    n = int(np.prod(shape)) if len(shape) else 1
    i = torch.arange(n, dtype=torch.float64)
    salt = (zlib.crc32(key.encode()) % 10007) / 1000.0
    if ".grids." in key:               # planes: in [0.3, 1.5], so the six-plane products keep their size
        v = 0.9 + 0.4 * torch.sin(i * 0.7071 + salt) + 0.2 * torch.cos(i * 0.0173 + salt)
    elif key.endswith("weight"):
        v = torch.sin(i * 0.61803 + salt) * (1.7 / np.sqrt(shape[-1]))
    else:
        v = 0.1 * torch.sin(i * 1.3 + salt)
    return v.float().reshape(shape)


def state_dict_values(state_dict):
    """the golden state dict for a deform_network state_dict (keys and shapes kept; the poc buffers and aabb as given)"""
    out = {}
    for k, v in state_dict.items():
        if k.endswith("_poc"):
            out[k] = v.clone()
        elif k.endswith("grid.aabb"):
            out[k] = torch.tensor(AABB, dtype=torch.float32)
        else:
            out[k] = golden_value(k, tuple(v.shape))
    return out


def write_checkpoint(path, cfg, state_dict, n):
    ckpt = os.path.join(path, "point_cloud", f"iteration_{ITERATION}")
    os.makedirs(ckpt, exist_ok=True)
    with open(os.path.join(path, "cfg_args"), "w") as f:
        f.write(repr(cfg))
    torch.save(state_dict, os.path.join(ckpt, "deformation.pth"))
    torch.save(torch.ones(n, dtype=torch.bool), os.path.join(ckpt, "deformation_table.pth"))


def gaussians(name, cfg):
    """seeded raw Gaussians: interior points, points beyond the aabb on every axis, the aabb's corners and points on grid nodes"""
    n = CASES[name][2]
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    hi, lo = torch.tensor(AABB[0]), torch.tensor(AABB[1])
    u = torch.rand(n, 3, generator=g) * 1.4 - 0.2                  # 20 % beyond either face
    special = [[0.0, 0.0, 0.0], [1.0, 1.0, 1.0], [-0.5, 0.5, 1.7], [1.3, -0.4, 0.5], [0.5, 2.0, -1.0]]
    res = resolutions(cfg)[0]
    for k in (1, 2):                                                # nodes of level 0: p = -1 + 2 j / (res - 1)
        special.append([min(k, r - 1) / max(r - 1, 1) for r in res[:3]])
    m = min(n, len(special)) if n > 1 else 0
    if m:
        u[:m] = torch.tensor(special[:m])
    means = hi + u * (lo - hi)                                      # u = 0: xyz_max (p = -1), u = 1: xyz_min (p = 1)
    scales = torch.randn(n, 3, generator=g) * 0.5 - 3.0
    quats = torch.randn(n, 4, generator=g) * 0.8                    # not normalised
    opacities = torch.randn(n, 1, generator=g)
    dc = torch.randn(n, 1, 3, generator=g) * 0.4
    rest = torch.randn(n, 15, 3, generator=g) * 0.2
    return {"means": means, "scales": scales, "rotations": quats, "opacities": opacities, "shs_dc": dc, "shs_rest": rest}


CAPTURED = {}


def capture_render(**kwargs):
    CAPTURED.update(kwargs)
    return {"render": None}


class Gaussians:
    """the attributes VanillaGS4DRenderer.forward reads of a (raw, not pre-activated) VanillaGaussianModel"""

    def __init__(self, p):
        self.p = p
        self.active_sh_degree = 3

    get_xyz = property(lambda self: self.p["means"])
    scales = property(lambda self: self.p["scales"])
    rotations = property(lambda self: self.p["rotations"])
    opacities = property(lambda self: self.p["opacities"])
    get_features = property(lambda self: torch.cat([self.p["shs_dc"], self.p["shs_rest"]], dim=1))

    def scale_activation(self, x):
        return torch.exp(x)

    def rotation_activation(self, x):
        return torch.nn.functional.normalize(x)

    def opacity_activation(self, x):
        return torch.sigmoid(x)


def main():
    sys.path.insert(0, HERE)
    import make_golden_v1_dropin as stubs  # noqa: E402  (puts the repository and the reference checkout on sys.path)
    stubs.install_stubs()
    import internal.renderers.vanilla_gs4d_renderer as R
    from internal.model_components.gs4d_deformation import deform_network
    R.VanillaRenderer.render = staticmethod(capture_render)

    out, meta = {}, {"cases": {}, "iteration": ITERATION, "aabb": AABB}
    for name, (over, t, n, stored) in CASES.items():
        cfg = case_cfg(name)
        torch.manual_seed(0)
        sd = state_dict_values(deform_network(cfg).state_dict())
        p = gaussians(name, cfg)
        with tempfile.TemporaryDirectory() as d:
            write_checkpoint(d, cfg, sd, n)
            renderer = R.VanillaGS4DRenderer(d, ITERATION, "cpu")
            if name == "small_d1":
                meta["state_dict"] = {k: list(v.shape) for k, v in renderer.deformation.state_dict().items()}
            CAPTURED.clear()
            with torch.no_grad():
                renderer(Namespace(time=torch.tensor([t])), Gaussians(p), torch.zeros(3))
        for k, v in p.items():
            out[f"{name}.in.{k}"] = v.numpy()
        for k in ("means3D", "scales", "rotations", "opacity", "features"):
            out[f"{name}.out.{k}"] = CAPTURED[k].detach().numpy()
        if stored:
            for k, v in sd.items():
                if ".grids." in k:
                    out[f"{name}.{k}"] = v.numpy()
        meta["cases"][name] = {"cfg": vars(cfg), "t": t, "n": n, "stored_planes": stored,
                               "active_sh_degree": int(CAPTURED["active_sh_degree"])}
    np.savez_compressed(os.path.join(HERE, "gs4d.npz"), **out)
    with open(os.path.join(HERE, "gs4d.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
