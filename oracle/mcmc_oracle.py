"""float64 restatement of the two per-Gaussian updates of 3DGS-MCMC (Kheradmand et al., "3D Gaussian Splatting as Markov
Chain Monte Carlo", 2024), written from the paper and the density controller's formula:

  relocation (Eq. (9)): N Gaussians sharing one opacity o keep the rendered opacity and the summed contribution,
      o' = 1 - (1 - o)^(1/N),   scale' = scale * o / D,
      D  = sum_{i=1..N} sum_{k=0..i-1} C(i-1, k) (-1)^k o'^(k+1) / sqrt(k+1)           (double-sum form)
         = sum_{j=1..N} (-1)^(j-1) C(N, j) o'^j / sqrt(j)                              (hockey-stick form)
  position noise: Delta = c * w(o) * Sigma z with c = noise_lr * xyz_lr, Sigma = R diag(s)^2 R^T of the activated scales and
      unit quaternion, w(o) = 1 / (1 + exp(-100 ((1 - o) - 0.995))), z given.
"""
import math

import numpy as np


def relocated_opacity(o: float, N: int) -> float:
    return -math.expm1(math.log1p(-o) / N)


def denominator_double_sum(op: float, N: int) -> float:
    return sum(math.comb(i - 1, k) * (-1) ** k * op ** (k + 1) / math.sqrt(k + 1) for i in range(1, N + 1) for k in range(i))


def denominator_hockey_stick(op: float, N: int) -> float:
    return sum((-1) ** (j - 1) * math.comb(N, j) * op ** j / math.sqrt(j) for j in range(1, N + 1))


def relocation(opacities, scales, counts, n_max: int, form: str = "hockey_stick"):
    """(new opacities [n], new scales [n,3]) in float64; counts are clamped to [1, n_max]."""
    denominator = {"hockey_stick": denominator_hockey_stick, "double_sum": denominator_double_sum}[form]
    o = np.asarray(opacities, dtype=np.float64).reshape(-1)
    s = np.asarray(scales, dtype=np.float64).reshape(-1, 3)
    N = np.clip(np.asarray(counts, dtype=np.int64).reshape(-1), 1, n_max)
    new_o = np.empty_like(o)
    new_s = np.empty_like(s)
    for i in range(o.shape[0]):
        op = relocated_opacity(float(o[i]), int(N[i]))
        new_o[i] = op
        new_s[i] = s[i] * (o[i] / denominator(op, int(N[i])))
    return new_o, new_s


def rotation(quats):
    """Rotation matrices [n,3,3] of quaternions (w, x, y, z) normalised as F.normalize does (eps 1e-12)."""
    q = np.asarray(quats, dtype=np.float64)
    q = q / np.maximum(np.linalg.norm(q, axis=1, keepdims=True), 1e-12)
    w, x, y, z = q.T
    return np.stack([
        np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
        np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
        np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1),
    ], 1)


def covariance(log_scales, raw_quats):
    """Sigma = R diag(exp(log_scales))^2 R^T, [n,3,3]."""
    M = rotation(raw_quats) * np.exp(np.asarray(log_scales, dtype=np.float64))[:, None, :]
    return M @ np.transpose(M, (0, 2, 1))


def noise_weight(opacity_logits):
    o = 1.0 / (1.0 + np.exp(-np.asarray(opacity_logits, dtype=np.float64).reshape(-1)))
    return 1.0 / (1.0 + np.exp(-100.0 * ((1.0 - o) - 0.995)))


def noise_delta(log_scales, raw_quats, opacity_logits, c: float, z):
    """Delta [n,3] = c * w * Sigma z."""
    w = noise_weight(opacity_logits)
    return c * w[:, None] * np.einsum("nij,nj->ni", covariance(log_scales, raw_quats), np.asarray(z, dtype=np.float64))
