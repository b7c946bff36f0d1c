"""Freeze the reference's Glossy-Gaussian view-dependent opacity: the unmodified GlossyGaussianModel (internal/models/glossy_gaussian.py)
and GlossyRendererModule (internal/renderers/glossy_renderer.py), run on the CPU in float32 with a reference ``Cameras`` entry.
gsplat, lightning, viser and the other CUDA-only packages the reference imports are inert stand-ins: nothing recorded here calls
them (the colour needs gsplat, so it is checked against oracle/glossy_oracle.py only).

One seeded model of N = 96 Gaussians with opacity_sh_degree 3; Gaussian 0 sits exactly at the camera centre (zero direction) and
the opacity coefficients are wide enough that both clamps of get_opacities bite.  Per active degree d in 0..3:
  model_{d}:       get_view_dep_opacities(F.normalize(xyz - camera_center)) [N,1] and the gradients of sum(w * it) to the opacity dc
                   [N,1,1] and rest [N,15,1]
  renderer_{d}:    GlossyRendererModule.get_opacities(camera, model, ...) -> opacities [N] and viewdirs [N,3], and the gradients
                   of sum(w * opacities) to dc and rest (through the clamp)
Inputs (means, the opacity dc / rest, the camera centre, the cotangent w) are stored as well.
Run:  python tests/golden/make_golden_glossy.py <reference checkout>     -> tests/golden/glossy.npz"""
import importlib.abc
import importlib.machinery
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
N, SEED = 96, 11
DEGREES = (0, 1, 2, 3)
_STUBBED = {"gsplat", "viser", "lightning", "diff_gaussian_rasterization", "simple_knn", "tinycudann", "pytorch3d", "fused_ssim",
            "diff_surfel_rasterization", "torchmetrics", "lpips", "kornia"}


class _Stub(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)

        def inert(*args, **kwargs):
            raise RuntimeError(f"{self.__name__}.{name} is a stand-in")
        return inert


class _StubFinder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, name, path, target=None):
        return importlib.machinery.ModuleSpec(name, self, is_package=True) if name.split(".")[0] in _STUBBED else None

    def create_module(self, spec):
        m = _Stub(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        pass


def camera(cameras_cls):
    a = 0.4
    R = torch.tensor([[np.cos(a), 0.0, -np.sin(a)], [0.0, 1.0, 0.0], [np.sin(a), 0.0, np.cos(a)]], dtype=torch.float32)
    T = torch.tensor([0.3, -0.2, 2.5])
    return cameras_cls(R=R[None], T=T[None], fx=torch.tensor([500.0]), fy=torch.tensor([500.0]), cx=torch.tensor([320.0]),
                       cy=torch.tensor([240.0]), width=torch.tensor([640], dtype=torch.int32), height=torch.tensor([480], dtype=torch.int32),
                       appearance_id=torch.zeros(1, dtype=torch.int32), normalized_appearance_id=torch.zeros(1), distortion_params=None,
                       camera_type=torch.zeros(1, dtype=torch.int32))[0]


def inputs(campos):
    g = torch.Generator().manual_seed(SEED)
    means = torch.randn(N, 3, generator=g) * 2.0
    means[0] = campos
    dc = torch.randn(N, 1, 1, generator=g) * 1.5
    rest = torch.randn(N, 15, 1, generator=g) * 0.6
    w = torch.randn(N, generator=g)
    return means, dc, rest, w


if __name__ == "__main__":
    sys.meta_path.insert(0, _StubFinder())
    sys.path.insert(0, sys.argv[1])
    from internal.cameras.cameras import Cameras
    from internal.models.glossy_gaussian import GlossyGaussian
    from internal.renderers.glossy_renderer import GlossyRenderer

    cam = camera(Cameras)
    means, dc, rest, w = inputs(cam.camera_center)
    model = GlossyGaussian(sh_degree=3).instantiate()
    model.setup_from_number(N)
    with torch.no_grad():
        model.properties["means"].copy_(means)
        model.properties["opacities"].copy_(dc)
        model.properties["opacity_rest"].copy_(rest)
    renderer = GlossyRenderer(separate_sh=True, tile_based_culling=True).instantiate()
    out = {"means": means.numpy(), "op_dc": dc.numpy(), "op_rest": rest.numpy(), "campos": cam.camera_center.numpy(), "w": w.numpy()}
    for d in DEGREES:
        model.active_sh_degree = d
        dirs = torch.nn.functional.normalize(model.get_xyz.detach() - cam.camera_center, dim=-1)
        for key in ("model", "renderer"):
            for p in (model.properties["opacities"], model.properties["opacity_rest"]):
                p.grad = None
            if key == "model":
                o = model.get_view_dep_opacities(dirs=dirs)
                out[f"model_{d}_dirs"] = dirs.numpy()
            else:
                o, viewdirs = renderer.get_opacities(cam, model, None, torch.ones(N, dtype=torch.bool), None)
                out[f"renderer_{d}_viewdirs"] = viewdirs.numpy()
            (o.reshape(-1) * w).sum().backward()
            out[f"{key}_{d}_opacity"] = o.detach().numpy()
            for name, prop in (("v_dc", "opacities"), ("v_rest", "opacity_rest")):
                grad = model.properties[prop].grad           # None where nothing reached it (the rest at degree 0)
                out[f"{key}_{d}_{name}"] = (torch.zeros_like(model.properties[prop]) if grad is None else grad).detach().numpy().copy()
    clamped = out["renderer_3_opacity"]
    assert (clamped == 0).any() and (clamped == 1).any() and not (out["renderer_3_viewdirs"][0] != 0).any()
    np.savez(os.path.join(HERE, "glossy.npz"), **out)
    print("wrote glossy.npz", {k: v.shape for k, v in out.items()})
