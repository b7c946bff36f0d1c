"""Desk-check on CPU of K9/K10 (csrc/loss.cu) on the SSIM tile engine of csrc/ssim.cuh: the tiling and index expressions (16x16 tile,
5-pixel halo, LE = 26, horizontal pass over LE rows x LT columns, vertical pass over 11 rows, zero padding outside the image,
per-CTA partial sums, the derivative-map layout dmaps[3][C][H][W]) transcribed block by block into numpy and compared with
oracle/loss_oracle.py + autograd.  The CUDA kernels themselves are validated on the GPU by tests/test_gpu_loss.py; this pins the
indexing they were written with on the CPU."""
import numpy as np
import pytest
import torch

from oracle import loss_oracle as LO

LT, HALO, TAPS = 16, 5, 11
LE = LT + 2 * HALO
C1, C2 = 0.01 ** 2, 0.03 ** 2


def _load_halo(plane, x0, y0):
    H, W = plane.shape
    dst = np.zeros((LE, LE))
    for i in range(LE * LE):                      # the kernel's flat loop: ly = i / LE, lx = i - ly * LE
        ly, lx = divmod(i, LE)
        x, y = x0 + lx - HALO, y0 + ly - HALO
        if 0 <= x < W and 0 <= y < H:
            dst[ly, lx] = plane[y, x]
    return dst


def _emulate_fwd(img, gt, win):
    C, H, W = img.shape
    gx, gy = (W + LT - 1) // LT, (H + LT - 1) // LT
    dmaps = np.zeros((3, C, H, W))
    partials = np.zeros((C * gy * gx, 2))
    for c in range(C):
        for by in range(gy):
            for bx in range(gx):
                x0, y0 = bx * LT, by * LT
                s_a, s_b = _load_halo(img[c], x0, y0), _load_halo(gt[c], x0, y0)
                s_h = np.zeros((5, LE, LT))
                for i in range(LE * LT):          # ly = i / LT, lx = i - ly * LT
                    ly, lx = divmod(i, LT)
                    a, b = s_a[ly, lx:lx + TAPS], s_b[ly, lx:lx + TAPS]
                    s_h[:, ly, lx] = [win @ a, win @ b, win @ (a * a), win @ (b * b), win @ (a * b)]
                l1 = ss_sum = 0.0
                for t in range(LT * LT):          # lx = tid % LT, ly = tid / LT
                    lx, ly = t % LT, t // LT
                    x, y = x0 + lx, y0 + ly
                    mu1, mu2, e11, e22, e12 = (win @ s_h[m, ly:ly + TAPS, lx] for m in range(5))
                    if x < W and y < H:
                        a, b = s_a[ly + HALO, lx + HALO], s_b[ly + HALO, lx + HALO]
                        s1, s2, s12 = e11 - mu1 * mu1, e22 - mu2 * mu2, e12 - mu1 * mu2
                        A1, A2 = 2 * mu1 * mu2 + C1, 2 * s12 + C2
                        B1, B2 = mu1 * mu1 + mu2 * mu2 + C1, s1 + s2 + C2
                        ss = A1 * A2 / (B1 * B2)
                        dmaps[0, c, y, x] = (2 * mu2 * A2 - 2 * mu2 * A1) / (B1 * B2) - ss * (2 * mu1 / B1 - 2 * mu1 / B2)
                        dmaps[1, c, y, x] = -ss / B2
                        dmaps[2, c, y, x] = 2 * A1 / (B1 * B2)
                        l1 += abs(a - b)
                        ss_sum += ss
                partials[(c * gy + by) * gx + bx] = [l1, ss_sum]
    return dmaps, partials


def _emulate_bwd(img, gt, dmaps, win, lam, up):
    C, H, W = img.shape
    gx, gy = (W + LT - 1) // LT, (H + LT - 1) // LT
    v = np.zeros((C, H, W))
    for c in range(C):
        for by in range(gy):
            for bx in range(gx):
                x0, y0 = bx * LT, by * LT
                s_m = [_load_halo(dmaps[m, c], x0, y0) for m in range(3)]
                s_h = np.zeros((3, LE, LT))
                for i in range(LE * LT):
                    ly, lx = divmod(i, LT)
                    for m in range(3):
                        s_h[m, ly, lx] = win @ s_m[m][ly, lx:lx + TAPS]
                for t in range(LT * LT):
                    lx, ly = t % LT, t // LT
                    x, y = x0 + lx, y0 + ly
                    if x >= W or y >= H:
                        continue
                    g0, g1, g2 = (win @ s_h[m, ly:ly + TAPS, lx] for m in range(3))
                    a, b = img[c, y, x], gt[c, y, x]
                    v[c, y, x] = up / (C * H * W) * ((1 - lam) * np.sign(a - b) - lam * (g0 + 2 * a * g1 + b * g2))
    return v


@pytest.mark.parametrize("H,W", [(21, 37), (16, 16), (5, 40)])
def test_kernel_transcription_matches_oracle(H, W):
    g = torch.Generator().manual_seed(H + W)
    gt = torch.rand(3, H, W, generator=g, dtype=torch.float64)
    img = (gt + 0.15 * torch.randn(3, H, W, generator=g, dtype=torch.float64)).clamp(0, 1)
    win = LO.window_1d(torch.float64).numpy()
    dmaps, partials = _emulate_fwd(img.numpy(), gt.numpy(), win)
    n = img.numel()
    l1, ssim = partials[:, 0].sum() / n, partials[:, 1].sum() / n
    ar = img.clone().requires_grad_(True)
    loss, ref_l1, ref_ssim = LO.training_loss(ar, gt, 0.2)
    (2.5 * loss).backward()
    assert abs(l1 - float(ref_l1)) < 1e-12 and abs(ssim - float(ref_ssim)) < 1e-12
    v = _emulate_bwd(img.numpy(), gt.numpy(), dmaps, win, 0.2, 2.5)
    assert np.abs(v - ar.grad.numpy()).max() / np.abs(ar.grad.numpy()).max() < 1e-9
