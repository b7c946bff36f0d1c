"""gsplat-v1 surface of the reference on the b200gs kernels: ``B200GSplatV1`` mirrors the static helper class ``GSplatV1``
(internal/renderers/gsplat_v1_renderer.py:370-612: preprocess_camera / project / isect_encode / isect_encode_tile_based_culling /
preprocess / rasterize) and ``B200GSplatV1RendererModule`` mirrors ``GSplatV1RendererModule`` (:56-368): overridable
``get_scales / get_opacities / get_rgbs`` hooks (:113-133), multi-channel rasterization (rgb + depth + normal in one call,
:226-287), optional exact tile-based culling (:476-522), the ``absgrad`` and ``has_hit_any_pixels`` side channels on
``viewspace_points`` (:287; vanilla_density_controller.py:112-113; optimizers.py:39), and the same output dict.

    model:
      renderer: b200gs.v1.B200GSplatV1Renderer
"""
import math
from dataclasses import dataclass
from typing import Any, Tuple

import torch

from . import ops
from ._lib import MODE_GSPLAT, TILE
from .renderers import Renderer, RendererConfig, RendererOutputInfo, RendererOutputTypes


class Isects(tuple):
    """(tiles_per_gauss [1,N], isect_ids, flatten_ids, isect_offsets [1,th,tw]) like gsplat's, plus the Binning the blend kernels read.
    isect_ids (gsplat's sorted 64-bit keys) are never materialised by the hierarchical binning: None."""
    binning: ops.Binning = None


def build_rotation(q: torch.Tensor) -> torch.Tensor:
    """Rotation matrices of unit quaternions (w, x, y, z) (internal/utils/general_utils.py build_rotation)."""
    q = q / q.norm(dim=-1, keepdim=True)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=-1)
    return R.reshape(-1, 3, 3)


def camera_views(viewmats: torch.Tensor, Ks: torch.Tensor, width: int, height: int):
    """Host-side gsplat-mode views of C cameras: viewmats [C,4,4] world-to-camera, Ks [C,3,3].  Both are read back in one copy
    (25 floats per camera)."""
    c = viewmats.shape[0]
    host = torch.cat((viewmats.detach().reshape(c, 16).float(), Ks.detach().reshape(c, 9).float()), dim=1).cpu()
    return [ops.make_view(MODE_GSPLAT, width, height, fx=float(h[16]), fy=float(h[20]), cx=float(h[18]), cy=float(h[21]),
                          viewmatrix=h[:16].reshape(4, 4).T.contiguous()) for h in host]


def tiles_per_gauss(means2d: torch.Tensor, radii: torch.Tensor, tile_width: int, tile_height: int, tile_size: int = TILE) -> torch.Tensor:
    """gsplat's tiles_per_gauss [1,N] int32: the tiles of each Gaussian's bounding rect (gaussian_projection.py:118-125)."""
    radii, means2d = radii.reshape(-1), means2d.reshape(-1, 2).detach()
    r = radii.to(means2d.dtype).unsqueeze(-1)
    grid = torch.tensor([tile_width, tile_height], device=means2d.device, dtype=torch.int32)
    rmin = torch.minimum(((means2d - r) / tile_size).to(torch.int32).clamp_min(0), grid)
    rmax = torch.minimum((((means2d + r) / tile_size).to(torch.int32) + 1).clamp_min(0), grid)
    return torch.where(radii > 0, (rmax - rmin).prod(dim=-1), torch.zeros_like(radii)).unsqueeze(0)


class B200GSplatV1:
    @classmethod
    def preprocess_camera(cls, viewpoint_camera):
        """-> (viewmats [1,4,4], Ks [1,3,3], (width, height)) like the reference; the host-side view struct the kernels take is cached
        on the camera (no per-step .item() syncs after the first call)."""
        from .renderers import camera_view
        view = camera_view(viewpoint_camera, MODE_GSPLAT)
        viewmats = viewpoint_camera.world_to_camera.T.unsqueeze(0)
        key = (view.fx, view.fy, view.cx, view.cy, str(viewmats.device))
        cached = getattr(viewpoint_camera, "_b200gs_Ks", None)      # a fresh torch.tensor(..., device=cuda) per step = a synchronising H2D copy
        if cached is None or cached[0] != key:
            Ks = torch.tensor([[[view.fx, 0., view.cx], [0., view.fy, view.cy], [0., 0., 1.]]], dtype=torch.float, device=viewmats.device)
            try:
                viewpoint_camera._b200gs_Ks = (key, Ks)
            except AttributeError:
                pass
        else:
            Ks = cached[1]
        pc = PreprocessedCamera((viewmats, Ks, (int(view.width), int(view.height))))
        pc.view = view
        return pc

    @classmethod
    def _view(cls, preprocessed_camera, eps2d, scale_modifier=1.0):
        view = getattr(preprocessed_camera, "view", None)
        if view is None:   # a plain (viewmats, Ks, (w, h)) tuple built by the caller
            viewmats, Ks, (w, h) = preprocessed_camera
            view = camera_views(viewmats[:1], Ks[:1], w, h)[0]
        return ops._copy_view(view, eps2d=float(eps2d), scale_modifier=float(scale_modifier))

    @classmethod
    def project(cls, preprocessed_camera: Tuple, means3d, scales, quats, eps2d: float = 0.3, anti_aliased: bool = True, radius_clip: float = 0.,
                camera_model: str = "pinhole", **kwargs):
        """-> radii [1,N] int32, means2d [1,N,2], depths [1,N], conics [1,N,3], compensations [1,N] (None unless anti_aliased)."""
        if camera_model != "pinhole":
            raise NotImplementedError("b200gs projects pinhole cameras only")
        if radius_clip != 0.:
            raise NotImplementedError("b200gs: radius_clip is unsupported")
        view = cls._view(preprocessed_camera, eps2d)
        xys, depths, radii, conics, comp, tiles, _ = ops.project_gaussians(means3d, scales, 1.0, quats, None, 0, 0, 0, 0, view.height, view.width, view=view)
        return radii.unsqueeze(0), xys.unsqueeze(0), depths.unsqueeze(0), conics.unsqueeze(0), (comp.unsqueeze(0) if anti_aliased else None)

    @classmethod
    def _isect(cls, preprocessed_camera, projection_results, tile_size, conics=None, opacities=None):
        if tile_size != TILE:
            raise ValueError(f"b200gs supports tile_size {TILE} only")
        img_width, img_height = preprocessed_camera[-1]
        radii, means2d, depths = projection_results[0], projection_results[1], projection_results[2]
        radii, depths = radii.reshape(-1), depths.reshape(-1).detach()
        means2d = means2d.reshape(-1, 2).detach()
        tw, th = math.ceil(img_width / float(tile_size)), math.ceil(img_height / float(tile_size))
        if conics is not None:
            binning = ops.bin_gaussians(MODE_GSPLAT, img_width, img_height, means2d.contiguous(), depths.contiguous(), radii.contiguous(),
                                        conics.reshape(-1, 3).detach().contiguous(), opacities.reshape(-1).detach().contiguous())
        else:   # no cull arrays: the reference's pair list (every tile of the 3-sigma rect)
            binning = ops.bin_gaussians(MODE_GSPLAT, img_width, img_height, means2d.contiguous(), depths.contiguous(), radii.contiguous())
        out = Isects((tiles_per_gauss(means2d, radii, tw, th, tile_size), None, binning.sorted_ids, binning.tile_ranges[:, 0].reshape(1, th, tw)))
        out.binning = binning
        return out

    @classmethod
    def isect_encode(cls, preprocessed_camera: Tuple, projection_results, tile_size: int = 16):
        return cls._isect(preprocessed_camera, projection_results, tile_size)

    @classmethod
    def isect_encode_with_unused_opacities(cls, preprocessed_camera: Tuple, projection_results, opacities, tile_size: int = 16):
        return cls._isect(preprocessed_camera, projection_results, tile_size)

    @classmethod
    def isect_encode_tile_based_culling(cls, preprocessed_camera: Tuple, projection_results, opacities, tile_size: int = 16):
        """Only (tile, Gaussian) pairs whose tile can see alpha >= 1/255 are listed (exact test, binning.cu); images and gradients are
        bit-identical to the unculled lists for these opacities.  A rasterize call with larger opacities over the same lists (the
        renderer's hard-depth passes) misses the pairs that only those opacities would have kept."""
        return cls._isect(preprocessed_camera, projection_results, tile_size, projection_results[3], opacities)

    @classmethod
    def preprocess(cls, preprocessed_camera: Tuple, means3d, scales, quats, eps2d: float = 0.3, anti_aliased: bool = True, tile_size: int = 16,
                   tile_based_culling: bool = False, opacities: torch.Tensor = None):
        projections = cls.project(preprocessed_camera, means3d=means3d, scales=scales, quats=quats, eps2d=eps2d, anti_aliased=anti_aliased)
        opacities = opacities.unsqueeze(0).squeeze(-1)  # [1, N]
        if anti_aliased:
            opacities = opacities * projections[-1]
        if tile_based_culling:
            isects = cls.isect_encode_tile_based_culling(preprocessed_camera, projections, opacities, tile_size=tile_size)
        else:
            isects = cls.isect_encode(preprocessed_camera, projections, tile_size=tile_size)
        radii, means2d, depths, conics, compensations = projections
        return (radii, means2d.squeeze(0), depths, conics, compensations), isects, opacities

    @classmethod
    def rasterize(cls, preprocessed_camera: Tuple, projections, isects, opacities, colors, background, tile_size: int = 16, absgrad: bool = True,
                  **kwargs):
        """colors [N, D] (any D), opacities [1, N], projections with means2d [N, 2] -> (image [H,W,D], alpha [H,W,1]).
        Side channels on `means2d`: .absgrad (after backward, when absgrad) and .has_hit_any_pixels (bool [N], now)."""
        if tile_size != TILE:
            raise ValueError(f"b200gs supports tile_size {TILE} only")
        img_width, img_height = preprocessed_camera[-1]
        _, means2d, _, conics, _ = projections
        binning = getattr(isects, "binning", None)
        if binning is None:
            raise ValueError("isects must come from B200GSplatV1.isect_encode*")
        image, alpha, hits = ops.rasterize_binned(means2d, conics.reshape(-1, 3), colors, opacities.reshape(-1), binning, img_height, img_width, background,
                                                  absgrad=absgrad, want_hits=True)
        means2d.has_hit_any_pixels = hits.bool()
        return image, alpha.unsqueeze(-1)

    @staticmethod
    def get_intrinsics_matrix(fx, fy, cx, cy, device):
        K = torch.eye(3, device=device)
        K[0, 0], K[1, 1], K[0, 2], K[1, 2] = fx, fy, cx, cy
        return K


class PreprocessedCamera(tuple):
    view = None


@dataclass
class B200GSplatV1Renderer(RendererConfig):
    block_size: int = 16
    anti_aliased: bool = True
    filter_2d_kernel_size: float = 0.3
    separate_sh: bool = False
    tile_based_culling: bool = False
    max_viewspace_grad_scale: float = 65535.

    def instantiate(self, *args, **kwargs) -> "B200GSplatV1RendererModule":
        return B200GSplatV1RendererModule(self)


@dataclass
class RuntimeOptions:
    radius_clip: float = 0.
    camera_model: str = "pinhole"


class B200GSplatV1RendererModule(Renderer):
    _RGB_REQUIRED = 1
    _ALPHA_REQUIRED = 1 << 1
    _ACC_DEPTH_REQUIRED = 1 << 2
    _ACC_DEPTH_INVERTED_REQUIRED = 1 << 3
    _EXP_DEPTH_REQUIRED = 1 << 4
    _EXP_DEPTH_INVERTED_REQUIRED = 1 << 5
    _INVERSE_DEPTH_REQUIRED = 1 << 6
    _HARD_DEPTH_REQUIRED = 1 << 7
    _HARD_INVERSE_DEPTH_REQUIRED = 1 << 8
    _DEPTH_ALTERNATIVE = 1 << 9
    _NORMAL_REQUIRED = 1 << 10

    RENDER_TYPE_BITS = {
        "rgb": _RGB_REQUIRED,
        "alpha": _ALPHA_REQUIRED | _ACC_DEPTH_REQUIRED,
        "acc_depth": _ACC_DEPTH_REQUIRED,
        "acc_depth_inverted": _ACC_DEPTH_REQUIRED | _ACC_DEPTH_INVERTED_REQUIRED,
        "exp_depth": _ACC_DEPTH_REQUIRED | _EXP_DEPTH_REQUIRED,
        "exp_depth_inverted": _ACC_DEPTH_REQUIRED | _EXP_DEPTH_REQUIRED | _EXP_DEPTH_INVERTED_REQUIRED,
        "inverse_depth": _INVERSE_DEPTH_REQUIRED,
        "hard_depth": _HARD_DEPTH_REQUIRED,
        "hard_inverse_depth": _HARD_INVERSE_DEPTH_REQUIRED,
        "inv_depth_alt": _DEPTH_ALTERNATIVE,
        "normal": _NORMAL_REQUIRED,
    }

    def __init__(self, config: B200GSplatV1Renderer = None):
        super().__init__()
        self.config = config if config is not None else B200GSplatV1Renderer()
        self.runtime_options = RuntimeOptions()
        self.isect_encode = B200GSplatV1.isect_encode_with_unused_opacities
        if self.config.tile_based_culling:
            self.isect_encode = B200GSplatV1.isect_encode_tile_based_culling
        self._inv_depth_alt_state = 0
        self._inv_depth_alt = [self.RENDER_TYPE_BITS["inverse_depth"], self.RENDER_TYPE_BITS["hard_inverse_depth"]]

    def parse_render_types(self, render_types: list) -> int:
        if render_types is None:
            return self._RGB_REQUIRED
        bits = 0
        for i in render_types:
            bits |= self.RENDER_TYPE_BITS[i]
        if self.is_type_required(bits, self._DEPTH_ALTERNATIVE):
            bits |= self._inv_depth_alt[self._inv_depth_alt_state]
            self._inv_depth_alt_state = int(not self._inv_depth_alt_state)
        return bits

    @staticmethod
    def is_type_required(bits: int, type: int) -> bool:
        return bits & type != 0

    # ---- the hooks derived renderers override (gsplat_v1_renderer.py:113-133) ---------------------------------------------------
    def get_scales(self, camera, gaussian_model, **kwargs) -> Tuple[torch.Tensor, Any]:
        return gaussian_model.get_scales(), None

    def get_opacities(self, camera, gaussian_model, projections: Tuple, visibility_filter, status: Any, **kwargs) -> Tuple[torch.Tensor, Any]:
        return gaussian_model.get_opacities().squeeze(-1), status

    def get_rgbs(self, camera, gaussian_model, projections: Tuple, visibility_filter, status: Any, **kwargs) -> torch.Tensor:
        viewdirs = gaussian_model.get_xyz.detach() - camera.camera_center  # (N, 3)
        if getattr(gaussian_model, "is_pre_activated", False) or not self.config.separate_sh:
            rgbs = ops.spherical_harmonics(gaussian_model.active_sh_degree, viewdirs, gaussian_model.get_features, visibility_filter)
        else:   # dc | rest kept apart by the model (Taming-3DGS style): read in place; invisible rows are in no tile list
            rgbs = ops.spherical_harmonics_decomposed(gaussian_model.active_sh_degree, viewdirs, gaussian_model.get_shs_dc(),
                                                      gaussian_model.get_shs_rest(), visibility_filter)
        return torch.clamp(rgbs + 0.5, min=0.0)

    def forward(self, viewpoint_camera, pc, bg_color: torch.Tensor, scaling_modifier=1.0, render_types: list = None, **kwargs):
        render_type_bits = self.parse_render_types(render_types)
        preprocessed_camera = B200GSplatV1.preprocess_camera(viewpoint_camera)

        # 1. scales, projection
        scales, status = self.get_scales(viewpoint_camera, pc, **kwargs)
        if scaling_modifier != 1.:
            scales = scales * scaling_modifier
        projections = B200GSplatV1.project(preprocessed_camera, pc.get_means(), scales, pc.get_rotations(), eps2d=self.config.filter_2d_kernel_size,
                                           anti_aliased=self.config.anti_aliased, radius_clip=self.runtime_options.radius_clip,
                                           camera_model=self.runtime_options.camera_model)
        radii, means2d, depths, conics, compensations = projections
        radii_squeezed = radii.squeeze(0)
        visibility_filter = radii_squeezed > 0

        # 2. opacities, tile intersection
        opacities, status = self.get_opacities(viewpoint_camera, pc, projections, visibility_filter, status, **kwargs)
        opacities = opacities.unsqueeze(0)  # [1, N]
        if self.config.anti_aliased:
            opacities = opacities * compensations
        isects = self.isect_encode(preprocessed_camera, projections, opacities, tile_size=self.config.block_size)

        # 3. rasterization
        means2d = means2d.squeeze(0)
        projection_for_rasterization = radii, means2d, depths, conics, compensations

        def rasterize(input_features, background, return_alpha: bool = False, opac=opacities, absgrad: bool = True):
            rendered_colors, rendered_alphas = B200GSplatV1.rasterize(preprocessed_camera, projection_for_rasterization, isects, opacities=opac,
                                                                      colors=input_features, background=background, tile_size=self.config.block_size,
                                                                      absgrad=absgrad)
            if return_alpha:
                return rendered_colors, rendered_alphas.squeeze(-1)
            return rendered_colors

        outputs = {
            "render": None, "alpha": None, "acc_depth": None, "acc_depth_inverted": None, "exp_depth": None, "exp_depth_inverted": None,
            "inverse_depth": None, "hard_depth": None, "hard_inverse_depth": None, "normal": None, "inv_depth_alt": None,
            "viewspace_points": means2d,
            "viewspace_points_grad_scale": 0.5 * torch.tensor([preprocessed_camera[-1]]).to(means2d).clamp_(max=self.config.max_viewspace_grad_scale),
            "visibility_filter": visibility_filter,
            "acc_vis": None,
            "radii": radii_squeezed,
            "scales": scales,
            "opacities": opacities[0],
            "projections": projections,
            "isects": isects,
            "camera": viewpoint_camera,
            "preprocessed_camera": preprocessed_camera,
        }

        input_feature_list, bg_color_list, out_slices, n_dims = [], [], {}, 0
        if self.is_type_required(render_type_bits, self._RGB_REQUIRED):
            input_feature_list.append(self.get_rgbs(viewpoint_camera, pc, projections, visibility_filter, status, **kwargs))
            bg_color_list.append(bg_color)
            out_slices["render"] = (n_dims, n_dims + 3)
            n_dims += 3
        if self.is_type_required(render_type_bits, self._ACC_DEPTH_REQUIRED):
            input_feature_list.append(depths[0].unsqueeze(-1))
            bg_color_list.append(torch.zeros((1,), device=bg_color.device))
            out_slices["acc_depth"] = (n_dims, n_dims + 1)
            n_dims += 1
        if self.is_type_required(render_type_bits, self._NORMAL_REQUIRED):
            normals = build_rotation(pc.get_rotations())[:, :3, -1]
            # normals point from primitives to camera centers
            dirs = pc.get_means() - viewpoint_camera.camera_center
            is_point_to_the_view = torch.einsum("ij,ij->i", normals, dirs) > 0
            normals = normals * torch.where(is_point_to_the_view, -1., 1.).unsqueeze(-1)
            input_feature_list.append(normals)
            bg_color_list.append(torch.zeros((3,), device=bg_color.device))
            out_slices["normal"] = (n_dims, n_dims + 3)
            n_dims += 3

        exp_depth_im = None
        if n_dims > 0:
            feats = input_feature_list[0] if len(input_feature_list) == 1 else torch.concat(input_feature_list, dim=-1)
            bgs = bg_color_list[0] if len(bg_color_list) == 1 else torch.concat(bg_color_list, dim=-1)
            render_features, render_alpha = rasterize(feats, background=bgs, return_alpha=True)
            render_features = render_features.permute(2, 0, 1)
            render_alpha = render_alpha.unsqueeze(0)
            for k, (a, b) in out_slices.items():
                outputs[k] = render_features[a:b]
            outputs["alpha"] = render_alpha
            outputs["acc_vis"] = means2d.has_hit_any_pixels    # avoid overriding by hard depth
            if self.is_type_required(render_type_bits, self._ACC_DEPTH_INVERTED_REQUIRED):
                acc = outputs["acc_depth"]
                outputs["acc_depth_inverted"] = torch.where(acc > 0, 1. / acc, acc.detach().max())
            if self.is_type_required(render_type_bits, self._EXP_DEPTH_REQUIRED):
                acc = outputs["acc_depth"]
                exp_depth_im = torch.where(render_alpha > 0, acc / render_alpha, acc.detach().max())
                outputs["exp_depth"] = exp_depth_im
            if self.is_type_required(render_type_bits, self._EXP_DEPTH_INVERTED_REQUIRED):
                outputs["exp_depth_inverted"] = torch.where(exp_depth_im > 0, 1. / exp_depth_im, exp_depth_im.detach().max())

        zero1 = torch.zeros((1,), dtype=torch.float, device=bg_color.device)
        if self.is_type_required(render_type_bits, self._INVERSE_DEPTH_REQUIRED):
            inverse_depth = 1. / (depths[0].clamp_min(0.) + 1e-8).unsqueeze(-1)
            outputs["inverse_depth"] = rasterize(inverse_depth, zero1).permute(2, 0, 1)
            outputs["inv_depth_alt"] = outputs["inverse_depth"]
        hard_opacities = opacities + (1 - opacities.detach())
        if self.is_type_required(render_type_bits, self._HARD_DEPTH_REQUIRED):
            outputs["hard_depth"] = rasterize(depths[0].unsqueeze(-1), zero1, opac=hard_opacities, absgrad=False).permute(2, 0, 1)
        if self.is_type_required(render_type_bits, self._HARD_INVERSE_DEPTH_REQUIRED):
            inverse_depth = 1. / (depths[0].clamp_min(0.) + 1e-8).unsqueeze(-1)
            outputs["hard_inverse_depth"] = rasterize(inverse_depth, zero1, opac=hard_opacities, absgrad=False).permute(2, 0, 1)
            outputs["inv_depth_alt"] = outputs["hard_inverse_depth"]
        return outputs

    def get_available_outputs(self):
        gray = RendererOutputTypes.GRAY
        return {
            "rgb": RendererOutputInfo("render"),
            "alpha": RendererOutputInfo("alpha", type=gray),
            "acc_depth": RendererOutputInfo("acc_depth", type=gray),
            "acc_depth_inverted": RendererOutputInfo("acc_depth_inverted", type=gray),
            "exp_depth": RendererOutputInfo("exp_depth", type=gray),
            "exp_depth_inverted": RendererOutputInfo("exp_depth_inverted", type=gray),
            "inverse_depth": RendererOutputInfo("inverse_depth", type=gray),
            "hard_depth": RendererOutputInfo("hard_depth", type=gray),
            "hard_inverse_depth": RendererOutputInfo("hard_inverse_depth", type=gray),
            "normal": RendererOutputInfo("normal", type=RendererOutputTypes.NORMAL_MAP),
        }
