"""float64 restatement of the reference's appearance network and colour epilogue
(internal/renderers/gsplat_appearance_embedding_renderer.py: Model.forward :77-93, _get_rgbs_and_opacities :239-295,
internal/encodings/positional_encoding.py).  Plain torch, differentiable by autograd; the GPU tests compare the kernels against it
and tests/test_appearance_oracle_cpu.py compares it against recordings of the reference itself."""
import numpy as np
import torch
import torch.nn.functional as F

from .bilagrid_oracle import weyl


def positional_encoding(x: torch.Tensor, n_freq: int) -> torch.Tensor:
    """(x, sin(2^0 x), cos(2^0 x), sin(2^1 x), ..): 3 (2 n_freq + 1) channels."""
    out = [x]
    for k in range(n_freq):
        out += [torch.sin(2.0 ** k * x), torch.cos(2.0 ** k * x)]
    return torch.cat(out, dim=-1)


def mlp(features, embedding_row, weights, biases, view_dirs=None, n_freq=-1, normalize=False):
    """Sigmoid outputs [V, 3 | 4] of compact rows: features [V, F], embedding_row [E] (one image), view_dirs [V, 3] when n_freq >= 0;
    weights / biases are the Linear layers' (ReLU between them)."""
    e = embedding_row.reshape(1, -1).repeat(features.shape[0], 1)
    if normalize:
        features, e = F.normalize(features, dim=-1), F.normalize(e, dim=-1)
    x = [features, e]
    if n_freq >= 0:
        x.append(positional_encoding(view_dirs, n_freq))
    h = torch.cat(x, dim=-1)
    for l, (w, b) in enumerate(zip(weights, biases)):
        h = h @ w.T + b
        h = torch.relu(h) if l < len(weights) - 1 else torch.sigmoid(h)
    return h


def colors(features, mask, base_rgb, means, cam_center, raw_opacity, embedding_row, weights, biases, n_freq=-1, normalize=False,
           view_dirs=None):
    """The renderer's colours past warm-up on dense rows: features [N, F], mask bool [N], base_rgb [N, 3] (SH before the + 0.5).
    The view direction is normalize(means - cam_center), or ``view_dirs`` [N, 3] as given when that is passed.
    Returns (rgbs [N, 3], opacities [N], opacity_offsets [N] or None); rows outside the mask get rgb 0 and offset 0."""
    dirs = F.normalize(means.detach()[mask] - cam_center, dim=-1) if view_dirs is None else view_dirs[mask]
    s = mlp(features[mask], embedding_row, weights, biases, dirs, n_freq, normalize)
    rgbs = torch.zeros_like(base_rgb)
    rgbs[mask] = torch.clamp((base_rgb[mask] + 0.5) + (s[:, :3] * 2 - 1.), min=0., max=1.)
    if s.shape[1] == 3:
        return rgbs, raw_opacity, None
    offsets = torch.zeros_like(raw_opacity)
    offsets[mask] = s[:, 3]
    return rgbs, torch.clamp_max(offsets + raw_opacity, max=1.), offsets


class _Draws:
    """Consecutive stretches of one bilagrid_oracle.weyl sequence, uniform in [0, 1): tensors drawn one after another from it are
    not shifted copies of each other, as weyl sequences of different seeds would be."""

    def __init__(self, seed, size=1 << 20):
        self.u, self.at = weyl((size,), seed), 0

    def __call__(self, *shape):
        n = int(np.prod(shape))
        self.at += n
        return torch.from_numpy(self.u[self.at - n:self.at].reshape(shape).copy())


def shape_state(feat_dim=64, n_freq=-1, n_neurons=64, n_layers=3, n_out=3, embed_dims=32, n_appearances=4, seed=0):
    """A float32 state_dict of the reference Model's parameter tree for any network shape, rebuilt from weyl rather than stored: each
    weight uniform in +-2 / sqrt(fan_in) (nn.Linear's initialisation times 2, so the sigmoids leave 0.5), each bias in
    +-1 / sqrt(fan_in), the embedding with unit variance."""
    n_in = feat_dim + embed_dims + (0 if n_freq < 0 else 3 * (2 * n_freq + 1))
    u = _Draws(seed)
    st = {"embedding.weight": ((u(n_appearances, embed_dims) * 2 - 1) * 3 ** 0.5).float()}
    for l in range(n_layers):
        out = n_out if l == n_layers - 1 else n_neurons
        st[f"network.output_layers.{2 * l}.weight"] = ((u(out, n_in) * 2 - 1) * (2.0 / n_in ** 0.5)).float()
        st[f"network.output_layers.{2 * l}.bias"] = ((u(out) * 2 - 1) / n_in ** 0.5).float()
        n_in = n_neurons
    return st


def shape_inputs(n, feat_dim, seed):
    """float32 inputs of one recording of tests/golden/appearance_shapes.npz, rebuilt from weyl: features [n, F] with unit variance,
    a mask of about 2/3 of the rows, means [n, 3] in +-4 around a camera at (0.3, -4, 1.5), base colours in [-0.9, 0.9] (both
    colour clamps are active), raw opacities in [0, 1) (so is the opacity clamp) and cotangents in [-1, 1)."""
    u = _Draws(seed, n * (feat_dim + 17))
    x = {"features": ((u(n, feat_dim) * 2 - 1) * 3 ** 0.5).float(), "mask": u(n) < 0.66, "means": (u(n, 3) * 8 - 4).float(),
         "cam_center": torch.tensor([0.3, -4.0, 1.5]), "base": (u(n, 3) * 1.8 - 0.9).float(), "raw_opacity": u(n).float()}
    for k, c in (("cot_model", 4), ("cot_rgbs", 3), ("cot_opacities", 0), ("cot_offsets", 0)):
        x[k] = (u(n, c) * 2 - 1).float() if c else (u(n) * 2 - 1).float()
    return x


SHAPE_ROWS = 96          # rows of each recording of tests/golden/appearance_shapes.npz (make_golden_appearance_shapes.py)
SHAPES = {          # its configurations, name: (ModelConfig overrides, seed of shape_state / shape_inputs)
    "neurons128": ({"n_neurons": 128}, 21),
    "layers2": ({"n_layers": 2}, 22),
    "layers4_view": ({"n_layers": 4, "is_view_dependent": True}, 23),
    "neurons128_layers4_view_opacity": ({"n_neurons": 128, "n_layers": 4, "is_view_dependent": True, "with_opacity": True}, 24),
    "feat32_freq6_view": ({"n_gaussian_feature_dims": 32, "n_view_direction_frequencies": 6, "is_view_dependent": True}, 25),
    "view_freq0": ({"is_view_dependent": True, "n_view_direction_frequencies": 0}, 26),
    "feat8_normalize": ({"n_gaussian_feature_dims": 8, "normalize": True}, 27),
}


def sample_index(size):
    """Flat entries kept of a recorded v_features or parameter gradient: all of a small one; of a large one the first 64 and every
    73rd (73 divides no width used, so the kept entries run through every row and column)."""
    if size <= 384:
        return np.arange(size)
    return np.union1d(np.arange(64), np.arange(0, size, 73))


def network_shape(kw):
    """(feat_dim, n_freq, n_neurons, n_layers, n_out) of a ModelConfig's overrides"""
    n_freq = kw.get("n_view_direction_frequencies", 4) if kw.get("is_view_dependent") else -1
    return (kw.get("n_gaussian_feature_dims", 64), n_freq, kw.get("n_neurons", 64), kw.get("n_layers", 3), 4 if kw.get("with_opacity") else 3)
