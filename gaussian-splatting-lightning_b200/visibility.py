"""The reference's in-the-wild renderer with a transient visibility map
(internal/renderers/gsplat_appearance_embedding_visibility_map_renderer.py) on the b200gs kernels:

    model:
      renderer: b200gs.visibility.B200GSplatAppearanceEmbeddingVisibilityMapRenderer
      metric: b200gs.metrics.B200VisibilityMapMetrics

``B200VisibilityMapModel`` is the reference ``Model`` with the same parameter tree (``appearance_embedding``,
``appearance_network.output_layers.*``, ``transient_embedding``, ``uv_encodings.{i}.params`` in tiny-cuda-nn's flat layout,
``visibility_network.output_layers.*``), so checkpoints load both ways.  Per view, the appearance colours run on
``ops.appearance_mlp`` (K20-K22) and the visibility map on ``ops.uv_grid_encode`` (K32/K33) and ``ops.visibility_mlp`` (the
appearance kernels with one output): no [P, 128] repeat, no [P, 144] concat, and no host read of the appearance id or the image size
per step (both are read once per camera object and cached on it).

One declared difference: tiny-cuda-nn draws a grid's initial values from its own pcg32 stream; here they are
``uniform(-1e-4, 1e-4)`` from torch's generator.  ``skip_layers`` and tiny-cuda-nn networks are not provided."""
from dataclasses import dataclass, field
from typing import Any, List, Tuple

import torch
from torch import nn

from . import ops
from ._lib import MODE_GSPLAT
from .appearance import _Network
from .renderers import B200GSplatRenderer, DEFAULT_ANTI_ALIASED_STATUS, Renderer, camera_view


@dataclass
class UVEncodingConfig:
    n_levels: int = 8
    base_resolution: int = 16
    per_level_scale: float = 1.405


@dataclass
class NetworkConfig:
    n_neurons: int = 64
    n_layers: int = 3
    skip_layers: List[int] = field(default_factory=lambda: [])


@dataclass
class AppearanceNetworkConfig(NetworkConfig):
    pass


@dataclass
class VisibilityNetworkConfig(NetworkConfig):
    pass


@dataclass
class ModelConfig:
    n_images: int = -1

    # appearance
    n_gaussian_feature_dims: int = 64
    n_appearance_embedding_dims: int = 128
    appearance_network: AppearanceNetworkConfig = field(default_factory=lambda: AppearanceNetworkConfig())
    is_view_dependent: bool = False
    n_view_direction_frequencies: int = 4

    # transient
    n_transient_embedding_dims: int = 128
    uv_encoding: UVEncodingConfig = field(default_factory=lambda: UVEncodingConfig())
    visibility_network: VisibilityNetworkConfig = field(default_factory=lambda: VisibilityNetworkConfig())


@dataclass
class LRConfig:
    lr_init: float
    lr_final_factor: float = 0.1


@dataclass
class OptimizationConfig:
    gamma_eps: float = 1e-6

    appearance_embedding: LRConfig = field(default_factory=lambda: LRConfig(lr_init=2e-3))
    appearance_network: LRConfig = field(default_factory=lambda: LRConfig(lr_init=1e-3))

    transient_embedding: LRConfig = field(default_factory=lambda: LRConfig(lr_init=2e-3))
    uv_encoding: LRConfig = field(default_factory=lambda: LRConfig(lr_init=2e-3))
    visibility_network: LRConfig = field(default_factory=lambda: LRConfig(lr_init=1e-3))

    eps: float = 1e-15
    max_steps: int = 30_000
    appearance_warm_up: int = 1000
    transient_warm_up: int = 2000


class UVGridEncoding(nn.Module):
    """tiny-cuda-nn's ``Encoding(n_input_dims=2, {"otype": "DenseGrid", ...})`` with linear interpolation and 2 features per level:
    ``params`` is the flat grid in tcnn's layout.  ``forward(uv [n, 2])`` encodes given coordinates (K32, and K33 with float atomics);
    the renderer encodes its pixel grid through ``ops.uv_grid_encode`` instead, whose backward is deterministic."""

    def __init__(self, n_levels=8, base_resolution=16, per_level_scale=1.405):
        super().__init__()
        self.grid = dict(n_levels=int(n_levels), base_resolution=int(base_resolution), per_level_scale=float(per_level_scale))
        n = ops.uv_grid_params(**self.grid)
        if n == 0:
            raise NotImplementedError(f"b200gs DenseGrid: {self.grid} is not supported: it takes n_levels 1..16, base_resolution >= 1 "
                                      f"and per_level_scale >= 1, and a grid of at most 2^31 - 1 floats (this one would hold "
                                      f"{_dense_grid_floats(**self.grid)})")
        self.n_input_dims, self.n_output_dims = 2, 2 * self.grid["n_levels"]
        self.params = nn.Parameter(torch.empty(n, dtype=torch.float32).uniform_(-1e-4, 1e-4))

    def forward(self, x):
        return ops.uv_grid_encode([self.params], 0, uv=x.reshape(-1, 2).float(), **self.grid)


def _mlp(n_in, n_out, cfg: NetworkConfig) -> _Network:
    layers = []
    for _ in range(cfg.n_layers - 1):
        layers += [nn.Linear(n_in, cfg.n_neurons), nn.ReLU()]
        n_in = cfg.n_neurons
    return _Network(nn.Sequential(*layers, nn.Linear(n_in, n_out), nn.Sigmoid()))


def _linears(net: _Network):
    return [m for m in net.output_layers if isinstance(m, nn.Linear)]


def _dense_grid_floats(n_levels, base_resolution, per_level_scale):
    """floats of a DenseGrid by tcnn's rule, in Python integers (also for grids too large for the library; inf when a scale is
    not finite).  The scale is fp32, as tcnn and the library compute it: in float64, level 3 of (12, 16, 1.5) has the scale
    53.00000000000001 instead of 53, which would add a row and a column of vertices."""
    import math
    import numpy as np
    f32 = np.float32
    lg = f32(math.log2(float(f32(per_level_scale))))
    total = 0
    with np.errstate(over="ignore"):
        for l in range(int(n_levels)):
            scale = f32(f32(np.exp2(np.float64(f32(f32(l) * lg)))) * f32(base_resolution)) - f32(1.0)
            if not math.isfinite(scale):
                return math.inf
            res = math.ceil(float(scale)) + 1
            total += (res * res + 7) // 8 * 8
    return 2 * total


def host_appearance_id(camera) -> int:
    """The camera's appearance id on the host: it picks the grid that receives the gradient, while the kernels read the id on the
    device.  The two agree as long as this value is the id the tensor holds, so it is cached on the camera object together with
    the tensor it was read from (its storage address and version counter): replacing ``camera.appearance_id`` or writing it in
    place makes the next call read it again.  A CUDA id costs one device-to-host read per camera object and id, not per step."""
    aid = camera.appearance_id
    if not isinstance(aid, torch.Tensor):
        return int(aid)
    key = (aid.data_ptr(), aid._version, aid.device)
    cached = getattr(camera, "_b200gs_appearance_id", None)
    if cached is None or cached[0] != key:
        cached = (key, int(aid.reshape(-1)[0]))
        try:
            camera._b200gs_appearance_id = cached
        except Exception:
            pass
    return cached[1]


class B200VisibilityMapModel(nn.Module):
    def __init__(self, config: ModelConfig):
        super().__init__()
        self.config = c = config
        for name, net in (("appearance_network", c.appearance_network), ("visibility_network", c.visibility_network)):
            if len(net.skip_layers) > 0:
                raise NotImplementedError(f"b200gs: {name} with skip_layers is not provided")
        self.n_freq = c.n_view_direction_frequencies if c.is_view_dependent else -1
        if not ops.appearance_supported(c.n_gaussian_feature_dims, self.n_freq, c.appearance_network.n_neurons, c.appearance_network.n_layers, 3):
            raise NotImplementedError(f"b200gs appearance network: {c.appearance_network} on {c.n_gaussian_feature_dims} features is not supported")
        n_enc = 2 * c.uv_encoding.n_levels
        if not ops.visibility_supported(n_enc, c.visibility_network.n_neurons, c.visibility_network.n_layers):
            raise NotImplementedError(f"b200gs visibility network: {c.visibility_network} on {c.uv_encoding.n_levels} grid levels is not "
                                      "supported (n_levels 4, 8, 12 or 16; n_neurons 64 or 128; n_layers 2..4)")

        self.appearance_embedding = nn.Embedding(num_embeddings=c.n_images, embedding_dim=c.n_appearance_embedding_dims)
        n_in = c.n_gaussian_feature_dims + c.n_appearance_embedding_dims + (0 if self.n_freq < 0 else 3 * (2 * self.n_freq + 1))
        self.appearance_network = _mlp(n_in, 3, c.appearance_network)

        self.transient_embedding = nn.Embedding(num_embeddings=c.n_images, embedding_dim=c.n_transient_embedding_dims)
        u = c.uv_encoding
        self.uv_encodings = nn.ModuleList([UVGridEncoding(u.n_levels, u.base_resolution, u.per_level_scale) for _ in range(c.n_images)])
        self.visibility_network = _mlp(n_enc + c.n_transient_embedding_dims, 1, c.visibility_network)

    def appearance_colors(self, gaussian_features, appearance, xyz, camera_center, visible, base_rgb):
        """clamp(base_rgb + 0.5 + 2 network - 1, 0, 1) on the visible rows, zeros elsewhere [N, 3]."""
        lin = _linears(self.appearance_network)
        return ops.appearance_mlp(gaussian_features, self.appearance_embedding(appearance.reshape((-1,)))[0], [m.weight for m in lin],
                                  [m.bias for m in lin], dirs=xyz, cam=camera_center, n_freq=self.n_freq, normalize_dirs=True,
                                  mask=visible, base_rgb=base_rgb)

    def visibility_forward(self, width: int, height: int, appearance, selected: int):
        """The visibility map [H, W] of the image `appearance` (read on the device); `selected`, its host value, picks the grid
        that receives the gradient."""
        u = self.config.uv_encoding
        enc = ops.uv_grid_encode([e.params for e in self.uv_encodings], appearance, width=width, height=height, selected=selected,
                                 n_levels=u.n_levels, base_resolution=u.base_resolution, per_level_scale=u.per_level_scale)
        lin = _linears(self.visibility_network)
        embedding = self.transient_embedding(appearance.reshape((-1,)))[0]
        return ops.visibility_mlp(enc, embedding, [m.weight for m in lin], [m.bias for m in lin]).reshape(height, width)


class B200GSplatAppearanceEmbeddingVisibilityMapRenderer(Renderer):
    def __init__(self, model: ModelConfig, optimization: OptimizationConfig):
        super().__init__()
        self.anti_aliased = DEFAULT_ANTI_ALIASED_STATUS  # tell absgrad whether AA enabled
        self.model_config = model
        self.optimization_config = optimization

    def setup(self, stage: str, lightning_module=None, *args: Any, **kwargs: Any) -> Any:
        if self.model_config.n_images <= 0:
            max_input_id = 0
            appearance_group_ids = lightning_module.trainer.datamodule.dataparser_outputs.appearance_group_ids
            if appearance_group_ids is not None:
                for i in appearance_group_ids.values():
                    if i[0] > max_input_id:
                        max_input_id = i[0]
            self.model_config.n_images = max_input_id + 1
        self.model = B200VisibilityMapModel(self.model_config)
        self.renderer = B200GSplatRenderer()

    def load_state_dict(self, state_dict, strict: bool = True):
        if not hasattr(self, "model"):
            self.model_config.n_images = state_dict["model.appearance_embedding.weight"].shape[0]
            self.setup("fit")
            self.to(state_dict["model.appearance_embedding.weight"].device)
        return super().load_state_dict(state_dict, strict)

    def training_setup(self, module):
        o, m = self.optimization_config, self.model
        groups = (("appearance_embedding", m.appearance_embedding, o.appearance_embedding, o.appearance_warm_up),
                  ("appearance_network", m.appearance_network, o.appearance_network, o.appearance_warm_up),
                  ("transient_embedding", m.transient_embedding, o.transient_embedding, o.transient_warm_up),
                  ("uv_encoding", m.uv_encodings, o.uv_encoding, o.transient_warm_up),
                  ("visibility_network", m.visibility_network, o.visibility_network, o.transient_warm_up))
        made = [self._create_optimizer_and_scheduler(mod.parameters(), name, lr_init=lr.lr_init, lr_final_factor=lr.lr_final_factor,
                                                     max_steps=o.max_steps, eps=o.eps, warm_up=warm_up)
                for name, mod, lr, warm_up in groups]
        return [x[0] for x in made], [x[1] for x in made]

    def forward(self, viewpoint_camera, pc, bg_color: torch.Tensor, scaling_modifier=1.0, **kwargs):
        projection_results = B200GSplatRenderer.project(means3D=pc.get_xyz, scales=pc.get_scaling, rotations=pc.get_rotation,
                                                        viewpoint_camera=viewpoint_camera, scaling_modifier=scaling_modifier)
        is_gaussian_visible = projection_results[2] > 0
        xyz = pc.get_xyz.detach()
        base = ops.spherical_harmonics(pc.active_sh_degree, xyz - viewpoint_camera.camera_center, pc.get_features, is_gaussian_visible)
        rgbs = self.model.appearance_colors(pc.get_appearance_features(), viewpoint_camera.appearance_id, xyz,
                                            viewpoint_camera.camera_center, is_gaussian_visible, base)
        rasterize_outputs = B200GSplatRenderer.rasterize(opacities=pc.get_opacity, rgbs=rgbs, bg_color=bg_color,
                                                         project_results=projection_results, viewpoint_camera=viewpoint_camera)
        view = camera_view(viewpoint_camera, MODE_GSPLAT)
        visibility = self.model.visibility_forward(int(view.width), int(view.height), viewpoint_camera.appearance_id,
                                                   host_appearance_id(viewpoint_camera))
        rasterize_outputs["visibility"] = visibility.unsqueeze(0)
        rasterize_outputs["extra_image"] = rasterize_outputs["visibility"]  # for image saving
        return rasterize_outputs

    def training_forward(self, step: int, module, viewpoint_camera, pc, bg_color: torch.Tensor, scaling_modifier=1.0, **kwargs):
        view = camera_view(viewpoint_camera, MODE_GSPLAT)
        ones = (1, int(view.height), int(view.width))
        if step < self.optimization_config.appearance_warm_up:
            render_outputs = self.renderer(viewpoint_camera, pc, bg_color, scaling_modifier, **kwargs)
            render_outputs["visibility"] = torch.ones(ones, device=module.device)
            return render_outputs
        render_outputs = self.forward(viewpoint_camera, pc, bg_color, scaling_modifier, **kwargs)
        if step < self.optimization_config.transient_warm_up:
            render_outputs["visibility"] = torch.ones(ones, device=module.device)
        return render_outputs

    @staticmethod
    def _create_optimizer_and_scheduler(params, name, lr_init, lr_final_factor, max_steps, eps,
                                        warm_up) -> Tuple[torch.optim.Optimizer, torch.optim.lr_scheduler.LRScheduler]:
        optimizer = torch.optim.Adam(params=[{"params": list(params), "name": name}], lr=lr_init, eps=eps)
        scheduler = torch.optim.lr_scheduler.LambdaLR(
            optimizer=optimizer, lr_lambda=lambda iter: lr_final_factor ** min(max(iter - warm_up, 0) / max_steps, 1))
        return optimizer, scheduler
