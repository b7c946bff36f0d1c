"""CPU restatement of the training loss that follows the rasterizer every step — TEST INFRASTRUCTURE ONLY (SURVEY §8f row 2:
the fused L1 + SSIM kernel is the next row of the hot-path table; this oracle and its golden vectors come first).

Follows the reference:
  * `internal/utils/ssim.py:17-18`   l1_loss = mean |a - b|
  * `internal/utils/ssim.py:23-31`   11-tap Gaussian window, sigma 1.5, normalised; the 2-D window is its outer product
  * `internal/utils/ssim.py:43-63`   SSIM map from five zero-padded depthwise convolutions, C1 = 0.01^2, C2 = 0.03^2, mean
  * `internal/metrics/vanilla_metrics.py:57-74`  loss = (1 - lambda) * L1 + lambda * (1 - SSIM), lambda_dssim = 0.2

The window is applied SEPARABLY here (rows then columns) — the formulation a fused CUDA kernel uses — which equals the reference's
2-D convolution up to fp rounding; tests/test_loss_oracle_golden.py pins it against outputs of the reference's own functions.
dtype-generic: float32 to mimic the reference, float64 as the mathematical truth.  Differentiable through torch autograd.
"""
import math

import torch
import torch.nn.functional as F

WINDOW = 11
SIGMA = 1.5
C1 = 0.01 ** 2
C2 = 0.03 ** 2
LAMBDA_DSSIM = 0.2


def window_1d(dtype=torch.float32) -> torch.Tensor:
    g = torch.tensor([math.exp(-(x - WINDOW // 2) ** 2 / float(2 * SIGMA ** 2)) for x in range(WINDOW)], dtype=torch.float32)
    return (g / g.sum()).to(dtype)      # the reference builds it in float32 and casts (`ssim.py:23-25,39`)


def _blur(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """Zero-padded separable 11x11 Gaussian blur of x [C,H,W]."""
    c = x.shape[0]
    x = x.unsqueeze(0)
    kh = w.reshape(1, 1, 1, WINDOW).expand(c, 1, 1, WINDOW)
    kv = w.reshape(1, 1, WINDOW, 1).expand(c, 1, WINDOW, 1)
    x = F.conv2d(x, kh, padding=(0, WINDOW // 2), groups=c)
    x = F.conv2d(x, kv, padding=(WINDOW // 2, 0), groups=c)
    return x.squeeze(0)


def _blur_2d(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """The same blur as one 11x11 convolution with the outer-product window, the reference's form; fp32 rounds it differently"""
    c = x.shape[0]
    k = torch.outer(w, w).reshape(1, 1, WINDOW, WINDOW).expand(c, 1, WINDOW, WINDOW)
    return F.conv2d(x.unsqueeze(0), k, padding=WINDOW // 2, groups=c).squeeze(0)


def ssim_map(img1: torch.Tensor, img2: torch.Tensor, separable: bool = True) -> torch.Tensor:
    w = window_1d(img1.dtype).to(img1.device)
    blur = _blur if separable else _blur_2d
    mu1, mu2 = blur(img1, w), blur(img2, w)
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1 = blur(img1 * img1, w) - mu1_sq
    s2 = blur(img2 * img2, w) - mu2_sq
    s12 = blur(img1 * img2, w) - mu12
    return ((2 * mu12 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2))


def ssim(img1: torch.Tensor, img2: torch.Tensor, separable: bool = True) -> torch.Tensor:
    return ssim_map(img1, img2, separable).mean()


def l1(img1: torch.Tensor, img2: torch.Tensor) -> torch.Tensor:
    return (img1 - img2).abs().mean()


def training_loss(image: torch.Tensor, gt: torch.Tensor, lambda_dssim: float = LAMBDA_DSSIM, separable: bool = True):
    """Returns (loss, l1, ssim) exactly as `VanillaMetricsImpl._get_basic_metrics` combines them."""
    a, s = l1(image, gt), ssim(image, gt, separable)
    return (1.0 - lambda_dssim) * a + lambda_dssim * (1.0 - s), a, s


# ---- seeded test content ----------------------------------------------------------------------------------------------------
# The content of real renders: noise around the target early in training and nearly none late; flat backgrounds and sky, where
# s = E[x^2] - mu^2 cancels in fp32; pixels clamped to exactly 0 or 1 in both images; pixels the dataset mask zeroes in both; and
# values above 1 after exposure or bilateral-grid correction.
KINDS = ("noise", "converged", "flat", "saturated", "masked", "identical", "hdr")


def _edge(n: int, f: float) -> int:
    """a block edge near f * n that does not fall on a multiple of the 16-pixel tile"""
    k = int(n * f)
    return k + 1 if k % 16 == 0 else k


def blob_keep_mask(H: int, W: int, g: torch.Generator, fraction: float = 0.3) -> torch.Tensor:
    """bool [H,W] keep-mask whose False pixels (at least `fraction` of them) form round blobs, like a dataset's object masks"""
    y, x = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    drop = torch.zeros(H, W, dtype=torch.bool)
    while float(drop.float().mean()) < fraction:        # each disc has radius >= 1 and its centre in the image: it drops a pixel
        cy, cx, r = torch.rand(3, generator=g).tolist()
        r = 1.0 + (0.08 + 0.12 * r) * min(H, W)
        drop |= (y - cy * (H - 1)) ** 2 + (x - cx * (W - 1)) ** 2 <= r * r
    return ~drop


def case(kind: str, C: int, H: int, W: int, seed: int):
    """(img, gt) float32 [C,H,W] on the CPU, from torch's CPU generator (the same bits on every machine) for one of KINDS"""
    g = torch.Generator().manual_seed(seed)
    if kind == "flat":
        ya, yb, xa, xb = _edge(H, 0.4), _edge(H, 0.7), _edge(W, 0.35), _edge(W, 0.6)
        level = torch.tensor([0.3, 0.8, 0.55]) + 0.02 * torch.arange(C, dtype=torch.float32).reshape(C, 1)
        gt = torch.empty(C, H, W)
        gt[:, :ya, :xa] = level[:, 0, None, None]
        gt[:, :ya, xa:] = level[:, 1, None, None]
        gt[:, ya:, :xb] = level[:, 2, None, None]
        gt[:, ya:yb, xb:] = level[:, 0, None, None]
        gt[:, yb:, xb:] = torch.linspace(0.2, 0.7, W)[xb:]          # a smooth ramp, as in a sky gradient
        img = gt + 0.002 * torch.randn(C, H, W, generator=g)
        img[:, :ya, :xa] += 0.01                                     # one block off by a constant
        return img, gt
    scale = 4.0 if kind == "hdr" else 1.0
    gt = scale * torch.rand(C, H, W, generator=g)
    if kind == "identical":
        return gt.clone(), gt
    sigma = {"converged": 0.005, "hdr": 0.6}.get(kind, 0.15)
    img = (gt + sigma * torch.randn(C, H, W, generator=g)).clamp(0, scale)
    if kind == "saturated":
        ya, xa, yb, xb = _edge(H, 0.45), _edge(W, 0.4), _edge(H, 0.55), _edge(W, 0.5)
        for t in (img, gt):
            t[:, :ya, :xa] = 0.0
            t[:, yb:, xb:] = 1.0
    elif kind == "masked":
        keep = blob_keep_mask(H, W, g).to(torch.uint8)           # B200VanillaMetrics: image * mask, gt * mask
        img, gt = img * keep, gt * keep
    elif kind not in ("noise", "converged", "hdr"):
        raise ValueError(f"unknown kind {kind!r}")
    return img, gt
