"""Record the reference's SWAG appearance: the unmodified SWAGRenderer of internal/renderers/swag_renderer.py with SWAGModel of
internal/models/swag_model.py, on the CPU in float32:
    python tests/golden/make_golden_swag.py <reference checkout>   -> tests/golden/swag.npz, swag.json

tinycudann cannot be installed, so swag_model imports a stand-in whose Encoding computes the oracle's grid (oracle/swag_oracle.py:
the grid is parity unpinned) and records its constructor calls; VanillaRenderer.render is replaced by a stub that captures the
opacities and colours the renderer hands it.  The grid table is golden_table (a function of the index, rebuilt by the tests);
the network, the embedding and the Gaussians are stored.  Recorded per case (degree, u or the evaluation branch): the colours,
the opacities and, for fixed cotangents, the gradients of the means, the SH features, the opacity logits, every theta weight and
bias, the embedding and the table (the touched entries: indices and values).  Once: the effective grid config (8 levels, not
the 12 swag_model.py appears to set), the state_dict keys and shapes, the optimizer group and LambdaLR values."""
import dataclasses
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_v1_dropin as stubs  # noqa: E402  (puts the repository and the reference checkout on sys.path)
from oracle import swag_oracle as S  # noqa: E402

N, N_EMB, AID = 96, 6, 4
CASES = [  # name, active degree, u (None: the evaluation branch, 0.5)
    ("d3_eval", 3, None),
    ("d3_u02", 3, 0.2),
    ("d1_u09", 1, 0.9),
    ("d0_eval", 0, None),
]
CALLS = []
CAPTURED = {}


def golden_table(n):
    """the recorded table: a smooth function of the index, so the tests rebuild it instead of storing 11.7 M floats"""
    i = torch.arange(n, dtype=torch.float64)
    return (0.6 * torch.sin(i * 0.7071) + 0.2 * torch.cos(i * 0.0173)).float()


class Encoding(torch.nn.Module):
    """tinycudann.Encoding stand-in: the oracle's HashGrid, recording its constructor calls"""

    def __init__(self, n_input_dims, encoding_config, seed=1337, dtype=None):
        super().__init__()
        self.config = dict(encoding_config)
        self.grid = {k: self.config[k] for k in ("n_levels", "n_features_per_level", "log2_hashmap_size", "base_resolution")}
        self.grid["per_level_scale"] = float(self.config["per_level_scale"])
        self.params = torch.nn.Parameter(torch.zeros(S.n_params(**self.grid)))
        self.n_output_dims = self.grid["n_levels"] * self.grid["n_features_per_level"]
        CALLS.append({"call": "Encoding", "n_input_dims": n_input_dims, "seed": seed, "dtype": str(dtype),
                      "encoding_config": {k: (float(v) if isinstance(v, (float, np.floating)) else v) for k, v in self.config.items()}})

    def forward(self, x):
        return S.encode(self.params, x.detach().numpy(), **self.grid).float()


class _LambdaLR(torch.optim.lr_scheduler.LambdaLR):
    """the reference passes verbose=False, an argument later torch releases removed"""

    def __init__(self, *args, verbose=False, **kwargs):
        super().__init__(*args, **kwargs)


def capture_render(**kwargs):
    CAPTURED.update(kwargs)
    return {"render": None}


class Gaussians:
    """the attributes SWAGRenderer.forward and eval_gaussian_model_sh read"""

    def __init__(self, means, features, opacity_logits, degree):
        self.means, self.features, self.logits = means, features, opacity_logits
        self.max_sh_degree, self.active_sh_degree = 3, degree
        self.get_scaling = torch.ones(means.shape[0], 3)
        self.get_rotation = torch.zeros(means.shape[0], 4)

    @property
    def get_xyz(self):
        return self.means

    @property
    def get_features(self):
        return self.features

    @property
    def get_opacity(self):
        return torch.sigmoid(self.logits)


def inputs(seed=0):
    g = torch.Generator().manual_seed(seed)
    campos = torch.tensor([0.3, -0.2, 2.5])
    means = torch.randn(N, 3, generator=g) * 1.2
    features = torch.randn(N, 16, 3, generator=g) * 0.4
    logits = torch.randn(N, 1, generator=g)
    point_cloud = torch.randn(200, 3, generator=g)            # the bbox source: some means fall outside the box
    cot_c, cot_o = torch.randn(N, 3, generator=g), torch.randn(N, generator=g)
    return campos, means, features, logits, point_cloud, cot_c, cot_o


def main():
    stubs.install_stubs()
    torch.optim.lr_scheduler.LambdaLR = _LambdaLR
    m = types.ModuleType("tinycudann")
    m.Encoding = Encoding
    sys.modules["tinycudann"] = m
    # swag_model.OptimizationConfig uses dataclass instances as field defaults, which Python >= 3.11 refuses for unhashable
    # (eq=True) dataclasses; the module is imported with hashable dataclasses, which changes nothing it computes
    plain = dataclasses.dataclass
    dataclasses.dataclass = lambda cls=None, **kw: plain(cls, unsafe_hash=True, **kw) if cls is not None else \
        (lambda c: plain(c, unsafe_hash=True, **kw))
    try:
        import internal.renderers.swag_renderer as R
        from internal.models import swag_model as SM
    finally:
        dataclasses.dataclass = plain
    R.VanillaRenderer.render = staticmethod(capture_render)

    campos, means0, features0, logits0, point_cloud, cot_c, cot_o = inputs()
    renderer = R.SWAGRenderer(embedding=SM.EmbeddingConfig(num_embeddings=N_EMB))
    module = types.SimpleNamespace(trainer=types.SimpleNamespace(datamodule=types.SimpleNamespace(
        dataparser_outputs=types.SimpleNamespace(point_cloud=types.SimpleNamespace(xyz=point_cloud.numpy())))))
    renderer.setup("fit", module)
    model = renderer.swag_model
    with torch.no_grad():
        model.grid_encoding.params.copy_(golden_table(model.grid_encoding.params.numel()))
    meta = {"calls": list(CALLS), "state_dict": {k: list(v.shape) for k, v in renderer.state_dict().items()},
            "grid_encoding_n_levels": SM.GridEncodingConfig().n_levels,
            "encoder_config": {k: (float(v) if isinstance(v, (float, np.floating)) else v)
                               for k, v in SM.GridEncodingConfig().get_encoder_config(3).items()},
            "defaults": {"network": dataclasses.asdict(SM.NetworkConfig()), "embedding": dataclasses.asdict(SM.EmbeddingConfig()),
                         "optimization": dataclasses.asdict(SM.GridEncodingOptimizationConfig()), "temperature": renderer.temperature,
                         "eps": renderer.eps},
            "bbox_min": renderer.bbox_min.tolist(), "bbox_size": renderer.bbox_size.tolist(), "cases": []}
    opt, sched = renderer.training_setup(None)
    meta["optimizer"] = {"names": [g["name"] for g in opt.param_groups], "lr": opt.param_groups[0]["lr"], "eps": opt.defaults["eps"],
                         "n_params": len(opt.param_groups[0]["params"]),
                         "lambda": {str(s): sched.lr_lambdas[0](s) for s in (0, 1, 15_000, 30_000, 45_000)}}
    u_sample = renderer.uniform_sampler.sample((1,))
    meta["uniform_sample_shape"] = list(u_sample.shape)

    out = {"campos": campos.numpy(), "means": means0.numpy(), "features": features0.numpy(), "logits": logits0.numpy(),
           "point_cloud": point_cloud.numpy(), "cot_c": cot_c.numpy(), "cot_o": cot_o.numpy(),
           "embedding": model.image_embedding.weight.detach().numpy()}
    for k, v in model.theta.state_dict().items():
        out[f"theta.{k}"] = v.numpy()
    for name, degree, u in CASES:
        means, features, logits = (t.clone().requires_grad_(True) for t in (means0, features0, logits0))
        pc = Gaussians(means, features, logits, degree)
        cam = types.SimpleNamespace(camera_center=campos, appearance_id=AID)
        model.zero_grad(set_to_none=True)
        CAPTURED.clear()
        renderer(cam, pc, torch.zeros(3), u=None if u is None else torch.tensor([u]))
        colours, opacity = CAPTURED["colors_precomp"], CAPTURED["opacity"]
        ((colours * cot_c).sum() + (opacity[:, 0] * cot_o).sum()).backward()
        p = f"{name}."
        out[p + "colours"], out[p + "opacities"] = colours.detach().numpy(), opacity.detach()[:, 0].numpy()
        grad = lambda t: (torch.zeros_like(t) if t.grad is None else t.grad).numpy()      # noqa: E731  (degree 0: none to the means)
        out[p + "v_means"], out[p + "v_features"], out[p + "v_logits"] = grad(means), grad(features), grad(logits)
        for k, v in model.theta.named_parameters():
            out[p + f"v_theta.{k}"] = v.grad.numpy()
        out[p + "v_embedding"] = model.image_embedding.weight.grad.numpy()
        gt = model.grid_encoding.params.grad
        nz = torch.nonzero(gt).reshape(-1)
        out[p + "v_table_idx"], out[p + "v_table_val"] = nz.numpy(), gt[nz].numpy()
        meta["cases"].append({"name": name, "degree": degree, "u": u})
    np.savez_compressed(os.path.join(HERE, "swag.npz"), **out)
    with open(os.path.join(HERE, "swag.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
