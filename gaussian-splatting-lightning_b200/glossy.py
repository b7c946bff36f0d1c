"""The reference's Glossy-Gaussian renderer (internal/renderers/glossy_renderer.py, configs/glossy.yaml) on the b200gs kernels:

    model:
      gaussian: internal.models.glossy_gaussian.GlossyGaussian
      renderer:
        class_path: b200gs.glossy.B200GlossyRenderer
        init_args:
          separate_sh: true
          tile_based_culling: true

Opacity is a per-Gaussian SH function of the view direction (``GlossyGaussianModel.get_view_dep_opacities``).  The reference
evaluates it with a chain of torch ops and then sends the same directions to the SH colour op; here one kernel (K47) computes
the direction, the opacity and the colour, and one kernel (K48) their gradients.  The Gaussian model stays the reference's
unmodified ``GlossyGaussianModel``; ``outputs["opacities"]`` is what the v1 forward returns, so ``update_opacity_max`` and
``cull_by_max_opacity`` work as in the reference."""
from dataclasses import dataclass
from typing import Any, Tuple

import torch

from . import ops
from .v1 import B200GSplatV1Renderer, B200GSplatV1RendererModule


@dataclass
class B200GlossyRenderer(B200GSplatV1Renderer):
    def instantiate(self, *args, **kwargs) -> "B200GlossyRendererModule":
        return B200GlossyRendererModule(self)


class B200GlossyRendererModule(B200GSplatV1RendererModule):
    """``GlossyRendererModule``: ``get_opacities`` computes the opacities and the colours in one op and hands the colours to
    ``get_rgbs`` through ``status``.  The colour is skipped when the render types do not include ``rgb``."""

    _rgb_requested = True

    def forward(self, viewpoint_camera, pc, bg_color: torch.Tensor, scaling_modifier=1.0, render_types: list = None, **kwargs):
        # only the "rgb" type sets the RGB bit (RENDER_TYPE_BITS); parse_render_types itself is not called twice, it has state
        self._rgb_requested = render_types is None or "rgb" in render_types
        return super().forward(viewpoint_camera, pc, bg_color, scaling_modifier, render_types, **kwargs)

    def get_opacities(self, camera, gaussian_model, projections: Tuple, visibility_filter, status: Any, **kwargs) -> Tuple[torch.Tensor, Any]:
        colour = {}
        if self._rgb_requested:
            if getattr(gaussian_model, "is_pre_activated", False) or not self.config.separate_sh:
                colour = {"features": gaussian_model.get_features}
            else:
                colour = {"shs_dc": gaussian_model.get_shs_dc(), "shs_rest": gaussian_model.get_shs_rest()}
        rgbs, opacities = ops.glossy_sh(gaussian_model.active_sh_degree, gaussian_model.get_xyz.detach(), camera.camera_center,
                                        gaussian_model.gaussians["opacities"], gaussian_model.gaussians["opacity_rest"],
                                        mask=visibility_filter, **colour)
        return opacities, rgbs

    def get_rgbs(self, camera, gaussian_model, projections: Tuple, visibility_filter, status: Any, **kwargs) -> torch.Tensor:
        return status
