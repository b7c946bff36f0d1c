"""The reference's in-the-wild pipeline (internal/renderers/gsplat_appearance_embedding_renderer.py) on the b200gs kernels:

    model:
      gaussian: internal.models.appearance_feature_gaussian.AppearanceFeatureGaussian
      renderer: b200gs.appearance.B200GSplatAppearanceEmbeddingRenderer

Past warm-up every visible Gaussian's colour is ``clamp(SH + 0.5 + 2 MLP(features | embedding [| PE(dir)]) - 1, 0, 1)``.
``B200AppearanceModel`` is the reference ``Model`` (:50-93) with the same parameter tree (``embedding.weight``,
``network.output_layers.{0,2,..}.{weight,bias}``), so checkpoints load both ways; its network runs on ``ops.appearance_mlp``.
``B200GSplatAppearanceEmbeddingRendererModule`` is ``GSplatAppearanceEmbeddingRendererModule`` (:115-323) on
``B200GSplatV1RendererModule``: one masked SH op and one fused colour op per view, no boolean-index gather, scatter or host
synchronisation.  ``skip_layers`` and ``tcnn`` are not provided."""
from dataclasses import dataclass, field
from typing import Any, List, Mapping, Tuple

import torch
from torch import nn

from . import ops
from .v1 import B200GSplatV1Renderer, B200GSplatV1RendererModule


@dataclass
class ModelConfig:
    n_gaussian_feature_dims: int = 64
    n_appearances: int = -1
    n_appearance_embedding_dims: int = 32
    is_view_dependent: bool = False
    n_view_direction_frequencies: int = 4
    n_neurons: int = 64
    n_layers: int = 3
    skip_layers: List[int] = field(default_factory=lambda: [])
    with_opacity: bool = False
    normalize: bool = False
    tcnn: bool = False


@dataclass
class OptimizationConfig:
    gamma_eps: float = 1e-6
    embedding_lr_init: float = 2e-3
    embedding_lr_final_factor: float = 0.1
    lr_init: float = 1e-3
    lr_final_factor: float = 0.1
    eps: float = 1e-15
    max_steps: int = 30_000
    warm_up: int = 4000


class _Network(nn.Module):
    """The parameter tree of the reference's NetworkWithSkipLayers without skips: ``output_layers`` is the whole network."""

    def __init__(self, output_layers: nn.Sequential):
        super().__init__()
        self.skip_layers = nn.ModuleList()
        self.output_layers = output_layers


class B200AppearanceModel(nn.Module):
    def __init__(self, config: ModelConfig):
        super().__init__()
        self.config = config
        c = config
        if c.tcnn:
            raise NotImplementedError("b200gs runs the appearance network on its own kernels: tcnn is not provided")
        if len(c.skip_layers) > 0:
            raise NotImplementedError("b200gs: appearance networks with skip_layers are not provided")
        self.n_output_dims = 4 if c.with_opacity else 3
        self.n_freq = c.n_view_direction_frequencies if c.is_view_dependent else -1
        if not ops.appearance_supported(c.n_gaussian_feature_dims, self.n_freq, c.n_neurons, c.n_layers, self.n_output_dims):
            raise NotImplementedError(
                f"b200gs appearance network: n_gaussian_feature_dims={c.n_gaussian_feature_dims} (a multiple of 8), n_neurons={c.n_neurons} "
                f"(64 or 128), n_layers={c.n_layers} (2..4) is not supported, or the first layer is too wide for shared memory")
        self.embedding = nn.Embedding(num_embeddings=c.n_appearances, embedding_dim=c.n_appearance_embedding_dims)
        n_in = c.n_gaussian_feature_dims + c.n_appearance_embedding_dims + (0 if self.n_freq < 0 else 3 * (2 * self.n_freq + 1))
        layers = []
        for _ in range(c.n_layers - 1):
            layers += [nn.Linear(n_in, c.n_neurons), nn.ReLU()]
            n_in = c.n_neurons
        layers += [nn.Linear(n_in, self.n_output_dims), nn.Sigmoid()]
        self.network = _Network(nn.Sequential(*layers))

    def linears(self):
        return [m for m in self.network.output_layers if isinstance(m, nn.Linear)]

    def embedding_row(self, appearance) -> torch.Tensor:
        """The image's embedding [E], normalised when the model normalises (looked up on the device)."""
        e = self.embedding(appearance.reshape((-1,)))[0]
        return torch.nn.functional.normalize(e, dim=-1) if self.config.normalize else e

    def forward(self, gaussian_features, appearance, view_dirs):
        """Compact rows in, sigmoid outputs [V, 3 | 4] out, as the reference Model.forward."""
        if gaussian_features.shape[0] == 0:
            return torch.zeros((0, self.n_output_dims), dtype=gaussian_features.dtype, device=gaussian_features.device)
        lin = self.linears()
        return ops.appearance_mlp(gaussian_features, self.embedding_row(appearance), [m.weight for m in lin], [m.bias for m in lin],
                                  dirs=view_dirs, n_freq=self.n_freq, normalize=self.config.normalize)


@dataclass
class B200GSplatAppearanceEmbeddingRenderer(B200GSplatV1Renderer):
    separate_sh: bool = True
    model: ModelConfig = field(default_factory=lambda: ModelConfig())
    optimization: OptimizationConfig = field(default_factory=lambda: OptimizationConfig())

    def instantiate(self, *args, **kwargs) -> "B200GSplatAppearanceEmbeddingRendererModule":
        assert self.separate_sh is True
        return B200GSplatAppearanceEmbeddingRendererModule(self)


class B200GSplatAppearanceEmbeddingRendererModule(B200GSplatV1RendererModule):
    """rgb = f(point_features, appearance_embedding, view_direction)"""

    opacity_offsets = None       # [N] of the last training view past warm-up (with_opacity), zeros outside _offset_rows
    _offset_rows = None

    def setup(self, stage: str, lightning_module=None, *args: Any, **kwargs: Any) -> Any:
        if lightning_module is not None:
            if self.config.model.n_appearances <= 0:
                max_input_id = 0
                appearance_group_ids = lightning_module.trainer.datamodule.dataparser_outputs.appearance_group_ids
                if appearance_group_ids is not None:
                    for i in appearance_group_ids.values():
                        max_input_id = max(max_input_id, i[0])
                self.config.model.n_appearances = max_input_id + 1
            self._setup_model()
            print(self.model)

    def _setup_model(self, device=None):
        self.model = B200AppearanceModel(self.config.model)
        if device is not None:
            self.model.to(device=device)

    def load_state_dict(self, state_dict: Mapping[str, Any], strict: bool = True):
        self.config.model.n_appearances = state_dict["model.embedding.weight"].shape[0]
        self._setup_model(device=state_dict["model.embedding.weight"].device)
        return super().load_state_dict(state_dict, strict)

    def training_setup(self, module):
        o = self.config.optimization
        embedding = self._create_optimizer_and_scheduler(self.model.embedding.parameters(), "embedding", lr_init=o.embedding_lr_init,
                                                         lr_final_factor=o.lr_final_factor, max_steps=o.max_steps, eps=o.eps, warm_up=o.warm_up)
        network = self._create_optimizer_and_scheduler(self.model.network.parameters(), "embedding_network", lr_init=o.lr_init,
                                                       lr_final_factor=o.lr_final_factor, max_steps=o.max_steps, eps=o.eps, warm_up=o.warm_up)
        if self.config.model.with_opacity:
            module.extra_train_metrics.append(self.opacity_offset_reg)
        return [embedding[0], network[0]], [embedding[1], network[1]]

    def opacity_offset_reg(self, outputs, batch, gaussian_model, global_step, pl_module):
        if self.opacity_offsets is None:
            return torch.tensor(0., dtype=torch.float, device=pl_module.device)
        # the mean over the visible rows; the offsets of the others are zero
        loss = self.opacity_offsets.sum() / self._offset_rows.sum()
        pl_module.log("train/opacity_offset_reg", loss, prog_bar=False, on_step=True, on_epoch=False, batch_size=pl_module.batch_size)
        return loss * 0.05

    def get_opacities(self, camera, gaussian_model, projections: Tuple, visibility_filter, status: Any, **kwargs) -> Tuple[torch.Tensor, Any]:
        rgbs, opacities, opacity_offsets = self._get_rgbs_and_opacities(camera, gaussian_model, projections, visibility_filter, status, **kwargs)
        if self.training:
            self.opacity_offsets, self._offset_rows = opacity_offsets, visibility_filter
        return opacities, rgbs

    def get_rgbs(self, camera, gaussian_model, projections: Tuple, visibility_filter, status: Any, **kwargs):
        return status

    def _get_rgbs_and_opacities(self, camera, pc, projections: Tuple, visibility_filter, status: Any, **kwargs):
        raw_opacities = pc.get_opacities().squeeze(-1)
        base = self.sh_colors(camera, pc, visibility_filter)
        if kwargs.get("warm_up", False):
            return torch.clamp(base + 0.5, min=0.), raw_opacities, None
        model, lin = self.model, self.model.linears()
        out = ops.appearance_mlp(pc.get_appearance_features(), model.embedding_row(camera.appearance_id), [m.weight for m in lin],
                                 [m.bias for m in lin], dirs=pc.get_xyz.detach(), cam=camera.camera_center, n_freq=model.n_freq,
                                 normalize=model.config.normalize, normalize_dirs=True, mask=visibility_filter, base_rgb=base,
                                 raw_opacity=raw_opacities if model.config.with_opacity else None)
        if model.config.with_opacity:
            return out
        return out, raw_opacities, None

    def training_forward(self, step: int, module, viewpoint_camera, pc, bg_color: torch.Tensor, scaling_modifier=1.0, **kwargs):
        return self.forward(viewpoint_camera, pc, bg_color, scaling_modifier, warm_up=step < self.config.optimization.warm_up, **kwargs)

    @staticmethod
    def _create_optimizer_and_scheduler(params, name, lr_init, lr_final_factor, max_steps, eps, warm_up):
        optimizer = torch.optim.Adam(params=[{"params": list(params), "name": name}], lr=lr_init, eps=eps)
        scheduler = torch.optim.lr_scheduler.LambdaLR(
            optimizer=optimizer, lr_lambda=lambda it: lr_final_factor ** min(max(it - warm_up, 0) / max_steps, 1))
        return optimizer, scheduler
