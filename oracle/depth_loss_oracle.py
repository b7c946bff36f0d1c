"""float64 restatement of the inverse-depth regularisation loss of internal/metrics/inverse_depth_metrics.py
(HasInverseDepthMetricsModule.get_inverse_depth_metric, :70-107), gradients by autograd, so its tie rules are the contract:

  pred' = (pred - min) / (max - min + 1e-8)  (depth_normalized; min, max of the whole pred under no_grad)
        | pred / median                     (elif median is not None)
        | pred / mean(gt), gt' = gt / mean(gt) (elif depth_mean_normalization)
  a = gt' k, b = pred' k                     (k the image mask, 1 without one)
  l1: mean|a - b|,  l2: mean (a - b)^2,  l1+ssim: (1 - w) l1 + w (1 - SSIM_tm(a, b))

The reference multiplies by the [C,H,W] image mask, which makes both maps [C,H,W] with identical channels; the mean over them equals
the mean over one channel, which is what this restatement takes (tests/test_depth_metrics_cpu.py checks it against the reference).

SSIM_tm is torchmetrics 1.x ``StructuralSimilarityIndexMeasure()`` as ``_ssim_update`` computes it: an 11-tap Gaussian (sigma 1.5,
built in float32 and normalised), the data range dr = max(range(preds), range(target)) taken from the maps themselves,
C1 = (0.01 dr)^2, C2 = (0.03 dr)^2, a reflect pad of 5, five depthwise convolutions, the SSIM map, a crop of 5 on every side and the
mean.  The range maximum is ``torch.maximum``, which gives half of the gradient to each side on a tie, and torch's max() / min()
split theirs evenly among tied pixels.  ``ssim_tm`` writes out the pad and crop; ``ssim_valid`` the mean over the full-window
positions, which it equals (``separable`` applies the window as a row and a column pass of shifted sums, the kernels' form, with
no convolution algorithm to choose).  ``TIE_SHARE`` is the share of the dr gradient that b gets on an exact tie of the two ranges.
PARITY UNPINNED: torchmetrics is not a dependency of this project, so SSIM_tm is restated from its
published source and has not been compared with torchmetrics' own output; the l1 and l2 losses are pinned to the unmodified
reference module by tests/golden/depth_metrics.npz.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.bilagrid_oracle import weyl

NORMS = ("none", "normalized", "median", "mean")
TIE_SHARE = 0.5         # torch.maximum's split of the dr gradient on an exact tie of range(a) and range(b)
MEDIAN = 2.5            # the median the tests pass in median mode
MEAN_SCALE = 3.0        # gt and pred are multiplied by it in mean mode, which the normalisation divides out


def gaussian_window(dtype=torch.float64):
    d = torch.arange(-5.0, 6.0, 1.0, dtype=torch.float32)
    g = torch.exp(-((d / 1.5) ** 2) / 2)
    return (g / g.sum()).to(dtype)


def _moments(a, b, pad, separable=False):
    g = gaussian_window(a.dtype).to(a.device)
    x = torch.stack([a, b, a * a, b * b, a * b])
    if separable:
        assert not pad
        H, W = a.shape
        x = sum(g[k] * x[:, :, k:k + W - 10] for k in range(11))
        return sum(g[k] * x[:, k:k + H - 10] for k in range(11))
    k = (g[:, None] * g[None, :])[None, None]
    x = x[:, None]
    if pad:
        x = F.pad(x, (5, 5, 5, 5), mode="reflect")
    return F.conv2d(x, k)[:, 0]


def _ssim_map(m, c1, c2):
    mu1, mu2, e11, e22, e12 = m
    s1, s2, s12 = e11 - mu1 * mu1, e22 - mu2 * mu2, e12 - mu1 * mu2
    return ((2 * mu1 * mu2 + c1) * (2 * s12 + c2)) / ((mu1 * mu1 + mu2 * mu2 + c1) * (s1 + s2 + c2))


def data_range(a, b, tie_share=TIE_SHARE):
    """max(range(a), range(b)); on an exact tie b's range gets ``tie_share`` of the gradient and a's the rest"""
    ra, rb = a.max() - a.min(), b.max() - b.min()
    if tie_share == 0.5:
        return torch.maximum(ra, rb)
    return torch.where(ra == rb, tie_share * rb + (1 - tie_share) * ra, torch.maximum(ra, rb))


def ssim_tm(a, b):
    """torchmetrics' SSIM of two [H,W] maps with the reflect pad and the crop written out"""
    dr = data_range(a, b)
    return _ssim_map(_moments(a, b, True), (0.01 * dr) ** 2, (0.03 * dr) ** 2)[5:-5, 5:-5].mean()


def ssim_valid(a, b, separable=False, tie_share=TIE_SHARE):
    """the same value as the mean over the windows that lie inside the image"""
    dr = data_range(a, b, tie_share)
    return _ssim_map(_moments(a, b, False, separable), (0.01 * dr) ** 2, (0.03 * dr) ** 2).mean()


def loss(gt, pred, loss_type="l1", ssim_weight=0.2, normalized=False, median=None, mean_normalization=False, mask=None,
         separable=False, tie_share=TIE_SHARE):
    """(loss, [l-term, SSIM or nan]) for [H,W] tensors (autograd through pred); mask None or [H,W] (nonzero keeps)"""
    if normalized:
        with torch.no_grad():
            mx, mn = pred.max(), pred.min()
        pred = (pred - mn) / (mx - mn + 1e-8)
    elif median is not None:
        pred = pred / median
    elif mean_normalization:
        m = torch.mean(gt)
        gt, pred = gt / m, pred / m
    if mask is not None:
        k = torch.as_tensor(mask).to(pred.device, torch.uint8).to(pred.dtype)
        gt, pred = gt * k, pred * k
    if loss_type == "l2":
        term = ((gt - pred) ** 2).mean()
        return term, (term.detach(), float("nan"))
    term = (gt - pred).abs().mean()
    if loss_type == "l1":
        return term, (term.detach(), float("nan"))
    s = ssim_valid(gt, pred, separable, tie_share)
    return (1 - ssim_weight) * term + ssim_weight * (1 - s), (term.detach(), s.detach())


def vjp(gt, pred, device="cpu", dtype=torch.float64, **cfg):
    """(loss, l-term, ssim, v_pred) for float arrays or tensors in, evaluated in ``dtype`` on ``device``: three floats and a float64
    numpy array.  On a GPU without cuDNN or TF32, so that the float32 error is the arithmetic's, not a convolution algorithm's."""
    p = torch.as_tensor(pred).detach().to(device, dtype, copy=True).requires_grad_(True)
    g = torch.as_tensor(gt).to(device, dtype)
    with torch.backends.cudnn.flags(enabled=False, allow_tf32=False):
        L, (term, s) = loss(g, p, **cfg)
        L.backward()
    return float(L.detach()), float(term), float(s), p.grad.double().cpu().numpy()


def normalize_pred(pred, norm, gt=None):
    """pred' in float64 as the loss computes it (mean mode divides by mean(gt))"""
    p = np.asarray(pred, np.float64)
    if norm == "normalized":
        return (p - p.min()) / (p.max() - p.min() + 1e-8)
    if norm == "median":
        return p / MEDIAN
    if norm == "mean":
        return p / np.asarray(gt, np.float64).mean()
    return p


def pred_map(H, W, seed, n_max=3, zeros=0.15):
    """float32 [H,W] inverse depth in [0, 1]: about ``zeros`` of the pixels exactly 0 (uncovered pixels, a tied minimum) and
    ``n_max`` pixels exactly at the maximum 1"""
    u = weyl((H, W), seed)
    p = 0.02 + 0.9 * weyl((H, W), seed + 1)
    p[u < zeros] = 0.0
    flat = p.reshape(-1)
    idx = (np.arange(n_max) * 7919 + 13) % flat.size
    flat[idx] = 1.0
    return p.astype(np.float32)


def gt_for(pred, norm, seed, k=0.6, equal=False):
    """float32 gt for a pred: a' = c + s m with c = b' scaled by k about its mid-range (k < 1: pred' has the larger range, k > 1:
    gt' has), s = sign(c - b') and m in [0.02, 0.05] of b's range, so |a' - b'| >= 0.02 of the range everywhere.  In mean mode
    the maps are both scaled by MEAN_SCALE, which the normalisation divides out.  ``equal``: every seventh pixel has a' = b'
    exactly (norm "none" only)."""
    b = normalize_pred(pred, "none" if norm == "mean" else norm)
    lo, hi = b.min(), b.max()
    mid = 0.5 * (lo + hi)
    c = k * (b - mid) + mid
    s = np.where(c >= b, 1.0, -1.0)
    a = c + s * (0.02 + 0.03 * weyl(b.shape, seed + 2)) * (hi - lo)
    if equal:
        assert norm == "none"
        a.reshape(-1)[::7] = b.reshape(-1)[::7]
    return a.astype(np.float32)


def noise_case(H, W, norm, seed, k=0.6, n_max=3, equal=False, masked=False):
    """(gt, pred, cfg) float32 inputs and the loss keywords of one test case; the mask (when ``masked``) drops about a quarter
    of the pixels, including some exact zeros and one of the tied maxima"""
    pred = pred_map(H, W, seed, n_max)
    gt = gt_for(pred, norm, seed, k, equal)
    if norm == "mean":
        pred, gt = (pred * MEAN_SCALE).astype(np.float32), (gt * MEAN_SCALE).astype(np.float32)
    cfg = {"normalized": norm == "normalized", "median": MEDIAN if norm == "median" else None, "mean_normalization": norm == "mean"}
    if masked:
        m = weyl((H, W), seed + 3) >= 0.25
        m.reshape(-1)[13] = False
        cfg["mask"] = m
    return gt, pred, cfg


# ---- seeded content of every kind ---------------------------------------------------------------------------------------------
# What a depth loss meets over training: noisy early maps; near-converged maps with exact equalities (l1 sign flips, E[x^2] - mu^2
# cancellation); flat plateaus, sky ramps and uncovered pixels at exactly 0; many pixels tied at pred's max and min over many tiles
# and statistics CTAs; a lone extremum in the last statistics CTA or on a tile seam; two data ranges that tie exactly; a constant
# pred; and near-camera inverse depths up to ~100.
KINDS = ("noise", "converged", "flat", "saturated", "lone", "tie", "flat_pred", "hdr")
STAT_PIXELS, STAT_MAX_BLOCKS = 2048, 1024       # the statistics grid of csrc/depth_loss.cu (K27): one CTA per 2048 pixels, at most 1024


def stat_blocks(n):
    return min(-(-n // STAT_PIXELS), STAT_MAX_BLOCKS)


def last_stat_pixel(n):
    """the last pixel that the statistics grid's last CTA reads (its threads stride by the grid's 256 * blocks pixels)"""
    sb = stat_blocks(n)
    i = np.arange(n)
    return int(i[(i // 256) % sb == sb - 1].max())


def pred32(pred, norm, gt=None):
    """pred' in float32, the way the reference computes it in float32 (correctly rounded; median as the product with the float32
    reciprocal); mean mode divides by the float32 mean of gt"""
    p = np.asarray(pred, np.float32)
    if norm == "normalized":
        return (p - p.min()) / ((p.max() - p.min()) + np.float32(1e-8))
    if norm == "median":
        return p * np.float32(1.0 / MEDIAN)
    if norm == "mean":
        return p / np.float32(np.asarray(gt, np.float64).mean())
    return p


def _edge(n, f):
    """a plateau edge near f * n that misses the 16-pixel tile grid"""
    k = int(n * f)
    return k + 1 if k % 16 in (0, 15) else k


def _plateaus(H, W, levels, ramp):
    """piecewise-constant map: four blocks whose edges miss the 16-pixel grid, a ramp in the last one and exact zeros in a band"""
    m = np.empty((H, W), np.float32)
    ya, yb, xa, xb = _edge(H, 0.4), _edge(H, 0.7), _edge(W, 0.35), _edge(W, 0.6)
    m[:ya, :xa], m[:ya, xa:], m[ya:, :xb], m[ya:yb, xb:] = levels[:4]
    m[yb:, xb:] = np.linspace(ramp[0], ramp[1], W, dtype=np.float32)[xb:]
    m[_edge(H, 0.15):_edge(H, 0.25), :_edge(W, 0.5)] = 0.0          # uncovered: nothing rendered
    return m


def case(*args, **kwargs):
    """(gt, pred, cfg) float32 [H,W] inputs and the loss keywords of one test case, in two call forms:
      case(kind, H, W, norm, seed, masked=False)                            one case of KINDS (kind_case)
      case(H, W, norm, seed, k=0.6, n_max=3, equal=False, masked=False)     the noise pair (noise_case), the inputs of the recorded
                                                                            goldens (tests/golden/depth_metrics.npz)"""
    return kind_case(*args, **kwargs) if isinstance(args[0], str) else noise_case(*args, **kwargs)


def kind_case(kind, H, W, norm, seed, masked=False):
    """(gt, pred, cfg) float32 [H,W] inputs and the loss keywords of one case of KINDS under normalisation ``norm``; ``masked`` adds
    a keep-mask that drops about a quarter of the pixels, the first and the last among them.  The properties each kind claims are
    checked by tests/test_depth_loss_oracle_cpu.py."""
    rng = np.random.default_rng(seed)
    n = H * W
    if kind == "noise":
        gt, pred, cfg = noise_case(H, W, norm, seed, k=0.6 if seed % 2 else 1.4, n_max=1 + 2 * (seed % 2))
    else:
        pred, gt = _pair(kind, H, W, norm, rng)
        if norm == "mean" and kind not in ("hdr", "tie"):
            pred, gt = pred * np.float32(MEAN_SCALE), gt * np.float32(MEAN_SCALE)
        cfg = {"normalized": norm == "normalized", "median": MEDIAN if norm == "median" else None, "mean_normalization": norm == "mean"}
    if masked:
        m = rng.random((H, W)) >= 0.25
        m.reshape(-1)[[0, n - 1]] = False
        cfg["mask"] = m
    return np.ascontiguousarray(gt, np.float32), np.ascontiguousarray(pred, np.float32), cfg


def _pair(kind, H, W, norm, rng):
    """(pred, gt) float32 of one kind before mean mode's scaling"""
    n = H * W
    space = "none" if norm == "mean" else norm            # mean mode divides both maps by one number: equalities hold in "none"
    if kind == "converged":
        # gt' = pred' + noise of 1e-4 of the range; every seventh pixel and the first exactly equal in float32
        # pred in [0.05, 0.88]: a range that is not a power of 2, so min-max normalisation really divides
        pred = (np.float32(0.05) + np.float32(0.83) * pred_map(H, W, int(rng.integers(1 << 30)))).astype(np.float32)
        b = pred32(pred, space)
        r = float(b.max() - b.min()) or 1.0
        a = (b + np.float32(1e-4 * r) * rng.standard_normal((H, W)).astype(np.float32)).astype(np.float32)
        a.reshape(-1)[::7] = b.reshape(-1)[::7]
        return pred, a
    if kind == "flat":
        pred = _plateaus(H, W, (0.3, 0.8, 0.55, 0.3), (0.2, 0.7))
        b = pred32(pred, space)
        a = b.copy()
        ya, xa = _edge(H, 0.4), _edge(W, 0.35)
        a[:ya, :xa] += np.float32(0.01)                     # one plateau off by a constant, the others equal
        a[_edge(H, 0.7):, _edge(W, 0.6):] *= np.float32(0.97)   # the ramp scaled
        return pred, a
    if kind == "saturated":
        # >= 5 % of pred exactly at its max 1 and >= 5 % exactly at its min 0, at random pixels; pixel 0 at the max, the last at the min
        pred = (0.02 + 0.9 * rng.random((H, W))).astype(np.float32)
        u = rng.random(n)
        flat = pred.reshape(-1)
        flat[u < 0.06] = 1.0
        flat[u > 0.94] = 0.0
        flat[0], flat[-1] = 1.0, 0.0
        return pred, _smaller_range(pred, space, rng)
    if kind == "lone":
        # one max 0.95, one min 0.05 (a range of 0.9): the min at pixel 0; the max at the last pixel of the last statistics CTA, or
        # (odd draws) on a tile seam
        pred = (0.1 + 0.8 * rng.random((H, W))).astype(np.float32)
        flat = pred.reshape(-1)
        if rng.integers(2) or H < 18 or W < 18:
            i = last_stat_pixel(n)
        else:
            i = min(16 * (H // 32) + 15, H - 1) * W + min(16 * (W // 32), W - 1)
        flat[0], flat[i] = 0.05, 0.95
        return pred, _smaller_range(pred, space, rng)
    if kind == "tie":
        # range(gt') == range(pred') exactly: pred and gt' in [0, 1] with exact 0 and 1 (median: pred in [0, 2.5], whose pred' =
        # pred x 0.4f rounds back to [0, 1] and pred / 2.5 is exact in float64; mean: both maps share the extremes, so dividing by
        # one mean keeps the tie; min-max: pred' has range exactly 1 in float32 only, float64 gives 1 - 1e-8 / range)
        pred = pred_map(H, W, int(rng.integers(1 << 30)), n_max=3)
        a = np.clip(pred + 0.1 * rng.standard_normal((H, W)), 0.0, 1.0).astype(np.float32)
        a.reshape(-1)[[1 % n, n // 2]] = [1.0, 0.0]
        if norm == "median":
            pred = (pred.astype(np.float64) * MEDIAN).astype(np.float32)
        return pred, a
    if kind == "flat_pred":
        pred = np.full((H, W), 0.37, np.float32)
        a = (0.05 + 0.9 * rng.random((H, W))).astype(np.float32)
        a.reshape(-1)[::11] = pred32(pred, space).reshape(-1)[::11]          # sgn(0) at pixels where gt' == pred'
        return pred, a
    if kind == "hdr":
        # inverse depths up to ~100 (near-camera surfaces), a far background near 0.01 and uncovered pixels at exactly 0
        pred = (0.01 + 2.0 * rng.random((H, W)) ** 4).astype(np.float32)
        pred[_plateaus(H, W, (1, 0, 1, 1), (1, 1)) == 0] = 0.0
        near = rng.random((H, W)) < 0.02
        pred[near] = (20 + 80 * rng.random(int(near.sum()))).astype(np.float32)
        b = pred32(pred, space)
        a = (b * (1 + 0.2 * rng.standard_normal((H, W)))).clip(0).astype(np.float32)
        return pred, a
    raise ValueError(f"unknown kind {kind!r}")


def _smaller_range(pred, space, rng):
    """a gt' correlated with pred' whose range is 0.8 of pred''s, so pred' sets the data range"""
    b = pred32(pred, space).astype(np.float64)
    lo, hi = b.min(), b.max()
    a = lo + 0.1 * (hi - lo) + 0.8 * (0.7 * (b - lo) + 0.3 * (hi - lo) * rng.random(b.shape))
    return a.astype(np.float32)
