"""float64 restatement of the reference's appearance network and colour epilogue
(internal/renderers/gsplat_appearance_embedding_renderer.py: Model.forward :77-93, _get_rgbs_and_opacities :239-295,
internal/encodings/positional_encoding.py).  Plain torch, differentiable by autograd; the GPU tests compare the kernels against it
and tests/test_appearance_oracle_cpu.py compares it against recordings of the reference itself."""
import torch
import torch.nn.functional as F


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


def colors(features, mask, base_rgb, means, cam_center, raw_opacity, embedding_row, weights, biases, n_freq=-1, normalize=False):
    """The renderer's colours past warm-up on dense rows: features [N, F], mask bool [N], base_rgb [N, 3] (SH before the + 0.5).
    Returns (rgbs [N, 3], opacities [N], opacity_offsets [N] or None); rows outside the mask get rgb 0 and offset 0."""
    dirs = F.normalize(means.detach()[mask] - cam_center, dim=-1)
    s = mlp(features[mask], embedding_row, weights, biases, dirs, n_freq, normalize)
    rgbs = torch.zeros_like(base_rgb)
    rgbs[mask] = torch.clamp((base_rgb[mask] + 0.5) + (s[:, :3] * 2 - 1.), min=0., max=1.)
    if s.shape[1] == 3:
        return rgbs, raw_opacity, None
    offsets = torch.zeros_like(raw_opacity)
    offsets[mask] = s[:, 3]
    return rgbs, torch.clamp_max(offsets + raw_opacity, max=1.), offsets
