"""Float64 restatement of the per-Gaussian regularisers of MCMCMetricsModuleMixin.reg_loss (internal/metrics/mcmc_metrics.py:39-59)
and ScaleRegularizationMetricsModuleMixin.get_scale_regularization_metrics (internal/metrics/scale_regularization_metrics.py:51-115),
the formulation csrc/gauss_reg.cu (K36-K38) computes.  Parity: fully pinned, the reference code is pure torch.

Dtype- and device-generic torch with autograd: in float64 it is the oracle; in float32 on CUDA with ties=None it is the reference's
own formulation as it runs in production (torch.sort's routing of tied scales on the device included).
    ties=None      torch.sort(dim=-1), as the reference's metric sorts
    ties="stable"  a tied pair gives the higher rank to the later column (torch.sort on the CPU)
    ties="device"  ties routed as torch.sort's bitonic network routes them on the GPU (and the kernels): DEVICE_TIES, measured on an
                   H100 for every ordering of three values
"""
import numpy as np
import torch

# torch.sort(dim=-1) of a [N,3] row on an H100: dense ranks of the row -> the column of each sorted slot
DEVICE_TIES = {(0, 0, 0): (2, 1, 0), (0, 0, 1): (1, 0, 2), (0, 1, 0): (0, 2, 1), (0, 1, 1): (0, 2, 1), (0, 1, 2): (0, 1, 2),
               (0, 2, 1): (0, 2, 1), (1, 0, 0): (1, 2, 0), (1, 0, 1): (1, 2, 0), (1, 0, 2): (1, 0, 2), (1, 1, 0): (2, 1, 0),
               (1, 2, 0): (2, 0, 1), (2, 0, 1): (1, 2, 0), (2, 1, 0): (2, 1, 0)}
TERMS = ("o_reg", "s_reg", "scale_reg", "scale_ratio_reg")
STATS = ("n_over_scales", "n_over_ratios", "max_scale", "max_ratio", "mean_ratio")
MAX_SCALE = 1.0            # the scenes' threshold: exp(0) is exactly 1 in every fp32 exp


def activate(opacities, scales, raw):
    if not raw:
        return opacities, scales
    return (None if opacities is None else torch.sigmoid(opacities)), (None if scales is None else torch.exp(scales))


def sort_scales(s, ties=None):
    """(values, indices) of each row sorted ascending"""
    if ties is None:
        return torch.sort(s, dim=-1)
    if ties == "stable":
        return torch.sort(s, dim=-1, stable=True)
    # the dense ranks of each row (the number of distinct smaller values) pick the measured permutation
    lt = (s[:, None, :] < s[:, :, None])                        # lt[n, i, j]: s[n, j] < s[n, i]
    eq = (s[:, :, None] == s[:, None, :])
    both = lt[:, :, :, None] & lt[:, :, None, :] & eq[:, None, :, :] & ~torch.eye(3, dtype=torch.bool, device=s.device)
    dense = lt.sum(-1) - both.sum((-1, -2)) // 2
    key = dense[:, 0] * 9 + dense[:, 1] * 3 + dense[:, 2]
    perm = torch.tensor([DEVICE_TIES.get((k // 9, (k // 3) % 3, k % 3), (0, 1, 2)) for k in range(27)], device=s.device)[key]
    return torch.return_types.sort((torch.gather(s, 1, perm), perm))


def regularizers(opacities, scales, raw, opacity_weight=0.0, scale_weight=0.0, max_scale=-1.0, max_scale_ratio=10.0, scale_lambda=0.0,
                 ratio_lambda=0.0, ties=None, masks=None):
    """(terms [4], stats [5]) in the inputs' dtype, with the reference's order of operations (it decides the fp32 rounding):
        o_reg = w_o * mean|o|                     (any w_o != 0; the reference always adds it)
        s_reg = w_s * mean|s|                     (w_s > 0)
        scale_reg = (sum s [s > max_scale]) / (n_s + 1) * lambda                      (lambda > 0)
        scale_ratio_reg = (sum r [r > max_scale_ratio]) / (n_r + 1) * lambda_r       (lambda_r > 0), r = max / (mid + 1e-8)
        stats = [n_s, n_r, max of the largest scale, max r, mean r]
    A term that is off is 0, and so is its count.  masks: None, or the over-scale [N,3] and over-ratio [N] masks to use in place of
    the thresholds (the fp32 decisions, see threshold_distance)."""
    o, s = activate(opacities, scales, raw)
    zero = (opacities if opacities is not None else scales).new_zeros(())
    terms, counts = [zero] * 4, [zero, zero]
    if o is not None and opacity_weight != 0:
        terms[0] = opacity_weight * o.abs().mean()
    if s is not None and scale_weight > 0:
        terms[1] = scale_weight * s.abs().mean()
    if s is None:
        return torch.stack(terms), None
    ranked = sort_scales(s, ties).values
    largest = ranked[:, 2]
    ratio = largest / (ranked[:, 1] + 1e-8)
    for k, on, values, decide in ((0, scale_lambda, s, lambda: s.detach() > max_scale),
                                  (1, ratio_lambda, ratio, lambda: ratio.detach() > max_scale_ratio)):
        if on > 0.:
            sel = decide() if masks is None else masks[k]
            counts[k] = sel.sum().to(s.dtype)
            terms[2 + k] = (values * sel).sum() / (counts[k] + 1) * on
    with torch.no_grad():
        stats = torch.stack([counts[0], counts[1], largest.max(), ratio.max(), ratio.mean()])
    return torch.stack(terms), stats


def threshold_distance(scales, raw, max_scale, max_scale_ratio):
    """Each element's relative distance to its threshold, in float64: |s - max_scale| / |max_scale| [N,3] and
    |r - max_scale_ratio| / max_scale_ratio [N] (r from the stable sort: the ratio does not depend on the routing of ties).  A mask
    may flip between fp32 and float64 only where this is a few ulps (DESIGN §2's threshold-flip rule)."""
    with torch.no_grad():
        s = scales.detach().double()
        s = torch.exp(s) if raw else s
        v = torch.sort(s, dim=-1).values
        r = v[:, -1] / (v[:, -2] + 1e-8)
        return (s - max_scale).abs() / max(abs(max_scale), 1e-30), (r - max_scale_ratio).abs() / max(abs(max_scale_ratio), 1e-30)


def crafted_rows():
    """Raw (logit, log-scale) rows, float32, that sit on the edges:
    isotropic; a tied min / mid with a ratio > 10 in three column orders (rows 1, 2 and 11: every placement of the pair); a tied max / mid; logits and log-scales at and past
    torch's fp32 underflow (sigmoid is 0 from -88.72283935546875, exp from -103.97208404541016); a scale exactly MAX_SCALE (exp(0));
    a ratio of exactly 10 (mid exp(0), so mid + 1e-8 rounds to 1, and max 10 needs an exact fp32 exp, which none has: the three
    ratio rows are found by search: the fp32 ratios nearest 10 from below, at or nearest 10, and nearest 10 from above)."""
    f = np.float32
    rows = [
        (0.5, (-2.0, -2.0, -2.0)),                       # isotropic
        (1.0, (-5.0, -5.0, -1.0)),                       # tied min / mid, ratio e^4 > 10
        (-1.0, (-1.0, -5.0, -5.0)),                      # the same, other columns
        (2.0, (-3.0, -1.5, -1.5)),                       # tied max / mid
        (-90.0, (-105.0, -3.0, -2.0)),                   # sigmoid and exp exactly 0
        (-88.72283935546875, (-103.97208404541016, -104.5, -1.0)),   # the first inputs that give exactly 0
        (-88.72283172607422, (-103.97207641601562, -2.5, -2.0)),     # the last that give a (subnormal) nonzero value
        (3.0, (0.0, -4.0, -6.0)),                        # a scale exactly MAX_SCALE: not over (strict)
    ]
    for side in (-1, 0, 1):
        rows.append((0.0, (0.0, float(_log_for(f(10), side)), -3.0)))      # mid exp(0) = 1, ratio = exp(x)
    rows.append((0.25, (-5.0, -1.0, -5.0)))             # tied min / mid in the outer columns, ratio e^4 > 10
    opac = np.array([[r[0]] for r in rows], np.float32)
    scales = np.array([r[1] for r in rows], np.float32)
    return opac, scales


def _log_for(target, side):
    """a float32 x near log(target) whose fp32 exp (torch's CPU exp) is the closest to target below it (side -1), nearest to it
    (side 0) or the closest above it (side 1)"""
    x0 = np.float32(np.log(np.float64(target)))
    cands = [x0]
    for _ in range(8):
        cands.append(np.nextafter(cands[-1], np.float32(0)))
    x = x0
    for _ in range(8):
        x = np.nextafter(x, np.float32(10))
        cands.append(x)
    vals = torch.exp(torch.tensor(np.array(cands, np.float32))).numpy().astype(np.float64)
    dist = np.abs(vals - np.float64(target))
    if side:
        dist[np.sign(vals - np.float64(target)) != side] = np.inf
    return cands[int(np.argmin(dist))]


def scene(n, seed, crafted=True):
    """(logits [n,1], log-scales [n,3]) float32 numpy: seeded normal rows (log-scales around -2, so that some scales pass
    MAX_SCALE and many ratios pass 10), with the crafted rows placed at seeded positions when ``crafted``"""
    rng = np.random.default_rng(seed)
    opac = (rng.standard_normal((n, 1)) * 3.0).astype(np.float32)
    scales = (rng.standard_normal((n, 3)) * 1.5 - 2.0).astype(np.float32)
    if crafted:
        co, cs = crafted_rows()
        at = rng.choice(n, size=len(co), replace=False)
        opac[at], scales[at] = co, cs
    return opac, scales


def fp32_masks(scales, raw, max_scale, max_scale_ratio):
    """the over-scale [N,3] and over-ratio [N] masks as float32 arithmetic decides them (torch's fp32 exp, the fp32 ratio)"""
    with torch.no_grad():
        s = torch.as_tensor(scales).float()
        s = torch.exp(s) if raw else s
        v = torch.sort(s, dim=-1).values
        return s > max_scale, v[:, -1] / (v[:, -2] + 1e-8) > max_scale_ratio


def vjp(opacities, scales, raw, v_terms, ties="stable", **kw):
    """float64 (terms, stats, v_opacities, v_scales) of sum(v_terms * terms), from float32 numpy inputs"""
    o = torch.from_numpy(np.asarray(opacities, np.float64)).requires_grad_(True) if opacities is not None else None
    s = torch.from_numpy(np.asarray(scales, np.float64)).requires_grad_(True) if scales is not None else None
    terms, stats = regularizers(o, s, raw, ties=ties, **kw)
    (terms * torch.as_tensor(v_terms, dtype=torch.float64)).sum().backward()
    grad = lambda t: None if t is None else (t.grad.numpy() if t.grad is not None else np.zeros(t.shape))  # noqa: E731
    return terms.detach().numpy(), None if stats is None else stats.numpy(), grad(o), grad(s)


TIED_ROWS = (1, 2, 11)     # crafted rows with a tied min / mid and a ratio > 10: the routing of the tie decides the gradient


def crafted_at(n, seed):
    """the positions scene(n, seed) gives the crafted rows, in crafted_rows' order"""
    rng = np.random.default_rng(seed)
    rng.standard_normal((n, 1))
    rng.standard_normal((n, 3))
    return rng.choice(n, size=len(crafted_rows()[0]), replace=False)


def sigmoid_grad_slack(logits):
    """Relative error [N,1] that torch's fp32 sigmoid backward, v (1 - y) y from the fp32 output y, carries against float64: 1 - y
    cancels as y nears 1, so its relative error is up to 2^-24 / (1 - y) (y's half-ulp below 1), doubled for margin; where y
    rounds to 1 in fp32 the gradient is 0 and the slack exceeds 1."""
    x = np.asarray(logits, np.float64)
    one_minus_y = 1.0 / (1.0 + np.exp(np.clip(x, -700, 700)))
    return 2.0 ** -23 / np.maximum(one_minus_y, 1e-300)
