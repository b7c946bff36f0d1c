"""The reference's SWAG in-the-wild renderer (internal/renderers/swag_renderer.py with internal/models/swag_model.py,
configs/swag_baseline.yaml) on the b200gs kernels:

    model:
      renderer:
        class_path: b200gs.swag.B200SWAGRenderer
        init_args:
          embedding:
            num_embeddings: 1536

Per view and Gaussian the reference evaluates the SH colour, a 3-D hash-grid lookup of the Gaussian's normalised centre, a
[rgb | encoding | image embedding] -> 64 -> 64 -> 4 MLP and a Gumbel-sigmoid opacity, as a chain of tiny-cuda-nn and torch ops on
[N, 59] tensors, before rasterizing with ``VanillaRenderer.render``.  Here that is one autograd node (``ops.swag_colours_and_opacities``):
K49 builds the MLP's input rows, the appearance kernels K20/K21 run the network with SWAG's epilogue, and K50 returns the gradients
to the SH coefficients, the means and the grid.  The render is ``B200VanillaRenderer.render(colors_precomp=...)``.

The parameter tree is the reference's (``swag_model.grid_encoding.params`` in tiny-cuda-nn's flat layout,
``swag_model.image_embedding.weight``, ``swag_model.theta.{0,2,4}.weight / bias``), so checkpoints load both ways.  Like the
reference, ``GridEncodingConfig().n_levels`` is 8: the reference's ``n_levels = 12`` line has no annotation and does not change the
dataclass field.

Declared differences: the grid table is float32 (tiny-cuda-nn keeps it in half precision), and its initial values are
``uniform(-1e-4, 1e-4)`` from torch's generator, not tiny-cuda-nn's pcg32 stream.  The grid gradient is scattered with float
atomics, so it is not bit-reproducible.  ``densegrid`` and the other encoding types are not provided."""
from dataclasses import dataclass
from typing import Any, Literal, Optional, Tuple

import numpy as np
import torch
from torch import nn

from . import ops
from .renderers import B200VanillaRenderer, Renderer, _raw_parameters


@dataclass
class GridEncodingConfig:
    """internal/configs/tcnn_encoding_config.py TCNNEncodingConfig with SWAG's type; n_levels stays 8 (see the module docstring)"""
    type: Literal["frequency", "hashgrid", "densegrid", "identity", "SphericalHarmonics", "none"] = "hashgrid"
    n_frequencies: int = 4
    degree: int = 4
    n_features_per_level: int = 4
    log2_hashmap_size: int = 19
    max_resolution: int = 2048
    n_levels: int = 8
    base_resolution: int = 16
    per_level_scale: float = 1.405

    def get_encoder_config(self, n_input_channels: int):
        """the reference's hashgrid encoder config (per_level_scale grows from base_resolution to max_resolution); other types raise"""
        if self.type != "hashgrid":
            raise NotImplementedError(f"b200gs SWAG provides the hashgrid encoding only, got type={self.type!r}")
        num_levels = self.n_levels
        growth = np.exp((np.log(self.max_resolution) - np.log(self.base_resolution)) / (num_levels - 1)) if num_levels > 1 else 1
        return {"n_dims_to_encode": n_input_channels, "otype": "HashGrid", "n_levels": num_levels,
                "n_features_per_level": self.n_features_per_level, "log2_hashmap_size": self.log2_hashmap_size,
                "base_resolution": self.base_resolution, "per_level_scale": growth}


@dataclass
class NetworkConfig:
    n_neurons: int = 64
    n_layers: int = 3


@dataclass
class EmbeddingConfig:
    num_embeddings: int = 2048
    embedding_dim: int = 24


@dataclass
class GridEncodingOptimizationConfig:
    lr: float = 1e-3
    max_steps: int = 30_000
    lr_final_factor: float = 0.01
    eps: float = 1e-15


def grid_kwargs(encoding_config: dict) -> dict:
    """The ops' grid arguments of a tiny-cuda-nn HashGrid encoding config (3-D); NotImplementedError outside the supported set."""
    c = dict(encoding_config)
    if str(c.get("otype", "")).lower() not in ("hashgrid", "grid") or str(c.get("type", "Hash")).lower() != "hash" or \
            str(c.get("interpolation", "Linear")).lower() != "linear":
        raise NotImplementedError(f"b200gs provides the 3-D HashGrid encoding with linear interpolation only, got {c}")
    g = dict(n_levels=int(c.get("n_levels", 16)), n_features_per_level=int(c.get("n_features_per_level", 2)),
             log2_hashmap_size=int(c.get("log2_hashmap_size", 19)), base_resolution=int(c.get("base_resolution", 16)),
             per_level_scale=float(c.get("per_level_scale", 2.0)))
    if ops.hash_grid_params(**g) == 0:
        raise NotImplementedError(f"b200gs HashGrid: {g} is not supported: it takes {ops.HASH_GRID_SUPPORTED}")
    return g


class HashGridEncoding(nn.Module):
    """tiny-cuda-nn's ``Encoding(n_input_dims=3, {"otype": "HashGrid", ...})``: ``params`` is the flat float32 table in tcnn's layout
    (level-major, then vertex-major, the features of a vertex contiguous).  ``forward(x [n, 3])`` encodes on K49/K50."""

    def __init__(self, encoding_config: dict):
        super().__init__()
        self.grid = grid_kwargs(encoding_config)
        self.n_input_dims = 3
        self.n_output_dims = self.grid["n_levels"] * self.grid["n_features_per_level"]
        self.params = nn.Parameter(torch.empty(ops.hash_grid_params(**self.grid), dtype=torch.float32).uniform_(-1e-4, 1e-4))

    def forward(self, x):
        return ops.hash_grid_encode(self.params, x.reshape(-1, 3).float(), **self.grid)


class B200SWAGModel(nn.Module):
    """swag_model.SWAGModel's parameters: grid_encoding.params, image_embedding.weight, theta.{0,2,4}.*"""

    def __init__(self, network: NetworkConfig, grid_encoding: GridEncodingConfig, embedding: EmbeddingConfig):
        super().__init__()
        self.network_config, self.grid_encoding_config, self.embedding_config = network, grid_encoding, embedding
        self.grid_encoding = HashGridEncoding(grid_encoding.get_encoder_config(3))
        self.image_embedding = nn.Embedding(embedding.num_embeddings, embedding.embedding_dim)
        n_in = self.grid_encoding.n_output_dims + embedding.embedding_dim + 3
        if not ops.swag_supported(3 + self.grid_encoding.n_output_dims, network.n_neurons, network.n_layers):
            raise NotImplementedError(f"b200gs SWAG network: {network} on {n_in} inputs is not supported (n_neurons 64 or 128, "
                                      "n_layers 2..4)")
        layers = []
        for _ in range(network.n_layers - 1):
            layers += [nn.Linear(n_in, network.n_neurons), nn.ReLU()]
            n_in = network.n_neurons
        self.theta = nn.Sequential(*layers, nn.Linear(n_in, 4))

    def linears(self):
        return [m for m in self.theta if isinstance(m, nn.Linear)]


_HALF = {}


def _eval_u(device) -> torch.Tensor:
    """u = 0.5 on the device, made once per device (the reference builds it every call)"""
    t = _HALF.get(str(device))
    if t is None:
        t = _HALF[str(device)] = torch.full((1,), 0.5, dtype=torch.float32, device=device)
    return t


class B200SWAGRenderer(Renderer):
    def __init__(self, network: NetworkConfig = NetworkConfig(), grid_encoding: GridEncodingConfig = GridEncodingConfig(),
                 embedding: EmbeddingConfig = EmbeddingConfig(), optimization: GridEncodingOptimizationConfig = GridEncodingOptimizationConfig(),
                 temperature: float = 0.1, eps: float = 1e-8) -> None:
        super().__init__()
        self.network_config = network
        self.grid_encoding_config = grid_encoding
        self.embedding_config = embedding
        self.optimization_config = optimization
        self.temperature = temperature
        self.eps = eps

    def setup(self, stage: str, lightning_module=None, *args: Any, **kwargs: Any) -> Any:
        with torch.no_grad():
            xyz = torch.tensor(lightning_module.trainer.datamodule.dataparser_outputs.point_cloud.xyz)
            self.set_bbox(torch.min(xyz, dim=0).values, torch.max(xyz, dim=0).values)
        self.swag_model = B200SWAGModel(self.network_config, self.grid_encoding_config, self.embedding_config)

    def set_bbox(self, bbox_min: torch.Tensor, bbox_max: torch.Tensor):
        """The grid's box, as the reference's setup computes it: the minimum and 1.1 x the extent (kept on the host; a device copy is
        made once per device)."""
        self.bbox_min = bbox_min.float().cpu()
        self.bbox_max = bbox_max.float().cpu()
        self.bbox_size = (self.bbox_max - self.bbox_min) * 1.1
        self._bbox_dev = {}

    def _bbox(self, device) -> torch.Tensor:
        t = self._bbox_dev.get(str(device))
        if t is None:
            t = self._bbox_dev[str(device)] = torch.cat([self.bbox_min, self.bbox_size]).to(device)
        return t

    def training_setup(self, module) -> Tuple[Optional[torch.optim.Optimizer], Optional[torch.optim.lr_scheduler.LRScheduler]]:
        params = list(self.swag_model.parameters())
        self.uniform_sampler = torch.distributions.uniform.Uniform(torch.tensor(0, dtype=torch.float, device=params[0].device),
                                                                   torch.tensor(1, dtype=torch.float, device=params[0].device))
        o = self.optimization_config
        optimizer = torch.optim.Adam(params=[{"params": params, "name": "swag_model"}], lr=o.lr)
        return optimizer, torch.optim.lr_scheduler.LambdaLR(optimizer=optimizer,
                                                             lr_lambda=lambda iter: o.lr_final_factor ** min(iter / o.max_steps, 1))

    def colours_and_opacities(self, viewpoint_camera, pc, u: Optional[torch.Tensor] = None):
        """(colours [N, 3], opacities [N]) of SWAGModel and the Gumbel-sigmoid opacity; u None: 0.5 (evaluation)"""
        xyz = pc.get_xyz
        if u is None:
            u = _eval_u(xyz.device)
        raw = _raw_parameters(pc)
        colour = {"shs_dc": raw["shs_dc"], "shs_rest": raw["shs_rest"]} if raw is not None else {"features": pc.get_features}
        m = self.swag_model
        aid = viewpoint_camera.appearance_id
        aid = aid.reshape(-1)[:1].to(device=xyz.device, dtype=torch.long) if isinstance(aid, torch.Tensor) else \
            torch.tensor([int(aid)], device=xyz.device)
        embedding = m.image_embedding(aid)[0]
        lin = m.linears()
        return ops.swag_colours_and_opacities(pc.active_sh_degree, xyz, viewpoint_camera.camera_center, pc.get_opacity.reshape(-1), u,
                                              m.grid_encoding.params, embedding, [l.weight for l in lin], [l.bias for l in lin],
                                              bbox=self._bbox(xyz.device), temperature=self.temperature, eps=self.eps,
                                              **m.grid_encoding.grid, **colour)

    def forward(self, viewpoint_camera, pc, bg_color: torch.Tensor, scaling_modifier=1.0, u=None, **kwargs):
        colours, opacities = self.colours_and_opacities(viewpoint_camera, pc, u)
        return B200VanillaRenderer.render(means3D=pc.get_xyz, opacity=opacities.unsqueeze(-1), scales=pc.get_scaling,
                                          rotations=pc.get_rotation, features=None, active_sh_degree=pc.active_sh_degree,
                                          viewpoint_camera=viewpoint_camera, bg_color=bg_color, scaling_modifier=scaling_modifier,
                                          colors_precomp=colours)

    def training_forward(self, step: int, module, viewpoint_camera, pc, bg_color: torch.Tensor, scaling_modifier=1.0, **kwargs):
        return self(viewpoint_camera=viewpoint_camera, pc=pc, bg_color=bg_color, scaling_modifier=scaling_modifier,
                    u=self.uniform_sampler.sample((1,)))
