"""The reference's 4DGS dynamic-scene renderer (internal/renderers/vanilla_gs4d_renderer.py, which the viewer opens with
``--vanilla_gs4d``) on the b200gs kernels:

    renderer = B200VanillaGS4DRenderer(model_path, load_iteration, device)

Per frame the reference deforms every Gaussian with the HexPlane field and MLP of a 4DGaussians checkpoint in eager torch (24
``grid_sample`` calls, the plane products, the trunk and head ``Linear`` layers), then renders with ``VanillaRenderer.render``.  Here
the deformation is one kernel (``ops.gs4d_deform``, K51) and the render is ``ops.rasterize_vanilla_raw``, which applies exp, normalize
and sigmoid in its projection kernel.

The constructor reads what the reference reads: ``<model_path>/cfg_args`` (an ``argparse.Namespace(...)`` repr),
``point_cloud/iteration_<n>/deformation.pth`` (the reference's ``deform_network`` state_dict, loaded unchanged into a module with the
same parameter tree) and ``deformation_table.pth`` (loaded, never used, as in the reference).  ``timenet`` and the opacity head are
loaded and never run: the reference discards their results too.

The model must hold raw parameters (``simplified_model = False`` in the viewer, which is what it sets for ``--vanilla_gs4d``); a
pre-activated model is refused.  Options outside ``ops.GS4D_SUPPORTED`` raise NotImplementedError naming the option.

Declared differences: the MLP runs as 3xTF32 tensor-core GEMMs with fp32 accumulation, the plane samples and products in fp32; the
result agrees with the reference's fp32 torch to about 1e-6 relative, not bit for bit."""
import os
from argparse import Namespace

import torch
from torch import nn

from . import ops
from .renderers import MODE_VANILLA, Renderer, _raw_parameters, _view_with, camera_view

_PLANES = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
_HEAD_MODULES = {"dx": "pos_deform", "ds": "scales_deform", "dr": "rotations_deform", "dshs": "shs_deform"}
_HEAD_FLAGS = {"dx": "no_dx", "ds": "no_ds", "dr": "no_dr", "dshs": "no_dshs"}


def parse_cfg_args(path) -> Namespace:
    """the reference's parse_cfg_args: cfg_args holds the repr of an argparse.Namespace"""
    with open(path, "r") as f:
        return eval(f.read(), {"Namespace": Namespace})


def check_cfg(cfg) -> None:
    """NotImplementedError for a 4DGaussians configuration K51 does not run, naming the option"""
    for name in ("no_grid", "static_mlp", "empty_voxel"):
        if getattr(cfg, name, False):
            raise NotImplementedError(f"4DGS with {name}=True is not supported: b200gs 4DGS takes {ops.GS4D_SUPPORTED}")
    if getattr(cfg, "grid_pe", 0) != 0:
        raise NotImplementedError(f"4DGS with grid_pe={cfg.grid_pe} is not supported: b200gs 4DGS takes {ops.GS4D_SUPPORTED}")
    kp = cfg.kplanes_config
    if kp.get("grid_dimensions") != 2 or kp.get("input_coordinate_dim") != 4:
        raise NotImplementedError(f"4DGS with grid_dimensions={kp.get('grid_dimensions')} and input_coordinate_dim="
                                  f"{kp.get('input_coordinate_dim')} is not supported: b200gs 4DGS takes {ops.GS4D_SUPPORTED}")
    if kp.get("output_coordinate_dim") not in (16, 32):
        raise NotImplementedError(f"4DGS with output_coordinate_dim={kp.get('output_coordinate_dim')} is not supported: b200gs 4DGS "
                                  f"takes {ops.GS4D_SUPPORTED}")
    if not 1 <= len(cfg.multires) <= 4:
        raise NotImplementedError(f"4DGS with multires={list(cfg.multires)} ({len(cfg.multires)} levels) is not supported: b200gs 4DGS "
                                  f"takes {ops.GS4D_SUPPORTED}")
    if cfg.net_width not in (64, 128):
        raise NotImplementedError(f"4DGS with net_width={cfg.net_width} is not supported: b200gs 4DGS takes {ops.GS4D_SUPPORTED}")
    if not 0 <= cfg.defor_depth <= 2:
        raise NotImplementedError(f"4DGS with defor_depth={cfg.defor_depth} is not supported: b200gs 4DGS takes {ops.GS4D_SUPPORTED}")
    res = [[r * m for r in kp["resolution"][:3]] + list(kp["resolution"][3:]) for m in cfg.multires]
    if not ops.gs4d_supported(len(res), kp["output_coordinate_dim"], cfg.net_width, cfg.defor_depth, res):
        raise NotImplementedError(f"4DGS with resolution={kp['resolution']} and multires={list(cfg.multires)} is not supported: b200gs "
                                  f"4DGS takes {ops.GS4D_SUPPORTED}")


def _head(width, out):
    return nn.Sequential(nn.ReLU(), nn.Linear(width, width), nn.ReLU(), nn.Linear(width, out))


class _HexPlaneField(nn.Module):
    """HexPlaneField's parameter tree: aabb [2, 3] (xyz_max, xyz_min) and grids.<level>.<plane> [1, C, res_b, res_a]"""

    def __init__(self, bounds, kplanes_config, multires):
        super().__init__()
        self.aabb = nn.Parameter(torch.tensor([[bounds] * 3, [-bounds] * 3], dtype=torch.float32), requires_grad=False)
        self.grids = nn.ModuleList()
        c = kplanes_config["output_coordinate_dim"]
        for m in multires:
            reso = [r * m for r in kplanes_config["resolution"][:3]] + list(kplanes_config["resolution"][3:])
            self.grids.append(nn.ParameterList([nn.Parameter(torch.zeros(1, c, reso[b], reso[a])) for a, b in _PLANES]))


class _Deformation(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        W = cfg.net_width
        self.grid = _HexPlaneField(cfg.bounds, cfg.kplanes_config, cfg.multires)
        layers = [nn.Linear(cfg.kplanes_config["output_coordinate_dim"] * len(cfg.multires), W)]
        for _ in range(cfg.defor_depth - 1):
            layers += [nn.ReLU(), nn.Linear(W, W)]
        self.feature_out = nn.Sequential(*layers)
        self.pos_deform, self.scales_deform, self.rotations_deform = _head(W, 3), _head(W, 3), _head(W, 4)
        self.opacity_deform, self.shs_deform = _head(W, 1), _head(W, 16 * 3)


class B200GS4DDeformNetwork(nn.Module):
    """gs4d_deformation.deform_network's parameter tree and buffers, so its state_dict loads with the reference's keys"""

    def __init__(self, cfg):
        super().__init__()
        times_ch = 2 * cfg.timebase_pe + 1
        self.timenet = nn.Sequential(nn.Linear(times_ch, cfg.timenet_width), nn.ReLU(), nn.Linear(cfg.timenet_width, cfg.timenet_output))
        self.deformation_net = _Deformation(cfg)
        self.register_buffer("time_poc", torch.FloatTensor([2 ** i for i in range(cfg.timebase_pe)]))
        self.register_buffer("pos_poc", torch.FloatTensor([2 ** i for i in range(cfg.posebase_pe)]))
        self.register_buffer("rotation_scaling_poc", torch.FloatTensor([2 ** i for i in range(cfg.scale_rotation_pe)]))
        self.register_buffer("opacity_poc", torch.FloatTensor([2 ** i for i in range(cfg.opacity_pe)]))


class B200VanillaGS4DRenderer(Renderer):
    def __init__(self, model_path: str, load_iteration: int, device):
        super().__init__()
        self.model_path = model_path
        self.load_iteration = load_iteration
        self.device = device
        self.compute_cov3D_python = False
        self.convert_SHs_python = False
        self.cfg_args = parse_cfg_args(os.path.join(model_path, "cfg_args"))
        check_cfg(self.cfg_args)
        checkpoint_dir = os.path.join(model_path, "point_cloud", "iteration_{}".format(load_iteration))
        self.deformation = B200GS4DDeformNetwork(self.cfg_args).to(device)
        self.deformation.load_state_dict(torch.load(os.path.join(checkpoint_dir, "deformation.pth"), map_location=device))
        self.deformation_table = torch.load(os.path.join(checkpoint_dir, "deformation_table.pth"), map_location=device)
        self.deformation.requires_grad_(False)
        self.refresh()

    def refresh(self) -> None:
        """Repack the planes and gather the layers in use; call again after changing the deformation network's parameters."""
        cfg, net = self.cfg_args, self.deformation.deformation_net
        with torch.no_grad():
            self.planes = ops.gs4d_repack_planes([list(level) for level in net.grid.grids])
            self.trunk = [(m.weight, m.bias) for m in net.feature_out if isinstance(m, nn.Linear)]
            self.heads = {}
            for name, module in _HEAD_MODULES.items():
                if not getattr(cfg, _HEAD_FLAGS[name], False):
                    seq = getattr(net, module)
                    self.heads[name] = ((seq[1].weight, seq[1].bias), (seq[3].weight, seq[3].bias))
        self.apply_rotation = bool(getattr(cfg, "apply_rotation", False))

    def deform(self, viewpoint_camera, pc):
        """the deformed raw parameters (means, log_scales, quats, shs_dc, shs_rest) of pc at viewpoint_camera.time, and the raw
        parameter dict"""
        raw = _raw_parameters(pc)
        if raw is None or getattr(pc, "is_pre_activated", False):
            raise ValueError("B200VanillaGS4DRenderer needs a model with raw parameters (means, scales, rotations, opacities, shs_dc, "
                             "shs_rest); a pre-activated model is not supported (load it with simplified_model = False)")
        with torch.no_grad():
            out = ops.gs4d_deform(raw["means"], raw["scales"], raw["rotations"], viewpoint_camera.time, self.planes,
                                  self.deformation.deformation_net.grid.aabb, self.trunk, self.heads, shs_dc=raw["shs_dc"],
                                  shs_rest=raw["shs_rest"], apply_rotation=self.apply_rotation)
        return out, raw

    def forward(self, viewpoint_camera, pc, bg_color: torch.Tensor, scaling_modifier=1.0, **kwargs):
        (means, log_scales, quats, dc, rest), raw = self.deform(viewpoint_camera, pc)
        screenspace_points = torch.zeros_like(means, requires_grad=True)
        view = camera_view(viewpoint_camera, MODE_VANILLA)
        view = _view_with(view, sh_degree=int(pc.active_sh_degree), scale_modifier=float(scaling_modifier))
        image, radii = ops.rasterize_vanilla_raw(means, screenspace_points, dc, rest, raw["opacities"], log_scales, quats, bg_color, view)
        return {
            "render": image,
            "depth": None,
            "viewspace_points": screenspace_points,
            "visibility_filter": radii > 0,
            "radii": radii,
        }
