"""oracle/loss_oracle.py (separable L1 + SSIM, the formulation of the planned fused kernel — SURVEY §8f row 2) against the
outputs of the reference's own `internal/utils/ssim.py` + the loss combination of `vanilla_metrics.py:57-74`, frozen by
tests/golden/make_golden_loss.py: values and the autograd gradient w.r.t. the rendered image."""
import glob
import os
import re

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import loss_oracle as L

FILES = sorted(f for f in glob.glob(os.path.join(GOLDEN, "loss_s*.npz")) if re.fullmatch(r"loss_s\d+_\d+x\d+\.npz", os.path.basename(f)))
CONTENT = sorted(set(glob.glob(os.path.join(GOLDEN, "loss_*.npz"))) - set(FILES))


def _pair(seed, H, W):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(3, H, W, generator=g)
    img = (gt + 0.15 * torch.randn(3, H, W, generator=g)).clamp(0, 1)
    return img, gt


def test_golden_files_present():
    assert len(FILES) >= 4 and len(CONTENT) >= 6


@pytest.mark.parametrize("path", FILES, ids=[os.path.basename(f) for f in FILES])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_loss_oracle_matches_reference(path, dtype):
    d = np.load(path)
    seed, H, W = (int(x) for x in d["meta"])
    img, gt = _pair(seed, H, W)
    img = img.to(dtype).requires_grad_(True)
    loss, l1, ssim = L.training_loss(img, gt.to(dtype))
    loss.backward()
    # the reference evaluates a 2-D 11x11 convolution in fp32; the separable form differs by rounding only
    assert abs(float(l1.detach()) - float(d["l1"])) < 2e-7
    assert abs(float(ssim.detach()) - float(d["ssim"])) < 5e-6
    assert abs(float(loss.detach()) - float(d["loss"])) < 2e-6
    g_ref = torch.tensor(d["grad"], dtype=torch.float64)
    err = (img.grad.double() - g_ref).abs().max() / g_ref.abs().max()
    assert float(err) < 2e-4, float(err)


def _within(err, e32, floor):
    """the bound of the fp32 content cases: 8x the fp32 oracle's own distance from float64 on the same input, or the floor"""
    return err <= max(8.0 * e32, floor)


@pytest.mark.parametrize("path", CONTENT, ids=[os.path.basename(f) for f in CONTENT])
def test_loss_oracle_matches_reference_on_content(path):
    """Flat, converged, masked and saturated content and 1 and 4 channels: there s = E[x^2] - mu^2 cancels in fp32 and both the
    reference's fp32 2-D convolution and the oracle's fp32 separable one carry errors well above the noise pair's.  e32 is the
    larger distance from float64 of the oracle in fp32 in its separable and in the reference's 2-D form, on this input; each bound
    is 8 e32, or the floor of the constant-tolerance test above.  (On the flat pair the 2-D form's SSIM is 3e-5 from float64, 20x
    the separable form's 1.4e-6: the 121-tap sums of a^2 round worse than two 11-tap passes.)"""
    d = np.load(path)
    seed, C, H, W = (int(x) for x in d["meta"])
    img, gt = L.case(str(d["kind"]), C, H, W, seed)
    assert tuple(d["grad"].shape[1:]) == (C, H, W)
    for k, lam in enumerate(d["lambdas"]):
        out = {}
        for dtype, separable in ((torch.float64, True), (torch.float32, True), (torch.float32, False)):
            x = img.to(dtype, copy=True).requires_grad_(True)
            loss, l1, ssim = L.training_loss(x, gt.to(dtype), float(lam), separable)
            loss.backward()
            out[dtype, separable] = [float(l1), float(ssim), float(loss), x.grad.double()]
        ref = [float(d["l1"]), float(d["ssim"]), float(d["loss"][k]), torch.tensor(d["grad"][k], dtype=torch.float64)]
        o64, o32, r32 = out[torch.float64, True], out[torch.float32, True], out[torch.float32, False]
        gmax = float(ref[3].abs().max())
        for o in (o64, o32):
            for q, floor in ((0, 2e-7), (1, 5e-6), (2, 2e-6)):
                e32 = max(abs(o32[q] - o64[q]), abs(r32[q] - o64[q]))
                assert _within(abs(o[q] - ref[q]), e32, floor), (float(lam), q, o[q], ref[q], e32)
            err = float((o[3] - ref[3]).abs().max())
            e32 = max(float((o32[3] - o64[3]).abs().max()), float((r32[3] - o64[3]).abs().max()))
            assert _within(err, e32, 2e-4 * gmax), (float(lam), err / gmax, e32 / gmax)


def test_noise_case_is_the_golden_pair():
    img, gt = _pair(0, 37, 50)
    c_img, c_gt = L.case("noise", 3, 37, 50, 0)
    assert torch.equal(img, c_img) and torch.equal(gt, c_gt)


@pytest.mark.parametrize("kind", L.KINDS)
def test_cases_have_their_content(kind):
    C, H, W = 3, 96, 128
    img, gt = L.case(kind, C, H, W, 1)
    assert img.dtype == gt.dtype == torch.float32 and img.shape == gt.shape == (C, H, W) and torch.isfinite(img).all()
    a, b = L.case(kind, C, H, W, 1)
    assert torch.equal(a, img) and torch.equal(b, gt)                  # seeded: the same bits every call
    eq = img == gt
    if kind == "identical":
        assert eq.all()
    elif kind == "saturated":
        assert float((eq & (gt == 0)).float().mean()) > 0.1 and float((eq & (gt == 1)).float().mean()) > 0.1
    elif kind == "masked":
        both0 = ((img == 0) & (gt == 0)).all(0)
        assert 0.3 <= float(both0.float().mean()) < 0.45
    elif kind == "flat":
        assert len(torch.unique(gt[0, :30, :40])) == 1 and float((img - gt).abs().max()) < 0.03
    elif kind == "hdr":
        assert float(gt.max()) > 3.5 and float(img.max()) <= 4.0 and float(img.min()) >= 0.0
    elif kind == "converged":
        assert float((img - gt).abs().mean()) < 0.005


def test_ssim_properties():
    img, gt = _pair(5, 40, 56)
    assert abs(float(L.ssim(gt, gt)) - 1.0) < 1e-6                       # identical images
    assert abs(float(L.ssim(img, gt)) - float(L.ssim(gt, img))) < 1e-7   # symmetric
    w = L.window_1d()
    assert abs(float(w.sum()) - 1.0) < 1e-6 and w.numel() == 11 and float(w[5]) == float(w.max())


def test_fused_kernel_formulas_match_autograd():
    """The closed-form pieces the fused kernels (csrc/loss.cu) evaluate — the three partial-derivative maps of the SSIM map
    w.r.t. the blurred moments mu1, E[a^2], E[ab], and  v_img = ((1-l) sign(a-b) - l (blur(d_mu1) + 2 a blur(d_e11) + b blur(d_e12))) / n
    — restated with torch ops and compared with autograd through the oracle loss.  Pins the math of K9/K10 on CPU."""
    g = torch.Generator().manual_seed(7)
    gt = torch.rand(3, 45, 61, generator=g, dtype=torch.float64)
    a = (gt + 0.15 * torch.randn(3, 45, 61, generator=g, dtype=torch.float64)).clamp(0, 1)
    lam = 0.2
    ar = a.clone().requires_grad_(True)
    loss, _, _ = L.training_loss(ar, gt, lam)
    loss.backward()

    w = L.window_1d(torch.float64)
    mu1, mu2 = L._blur(a, w), L._blur(gt, w)
    e11, e22, e12 = L._blur(a * a, w), L._blur(gt * gt, w), L._blur(a * gt, w)
    s1, s2, s12 = e11 - mu1 * mu1, e22 - mu2 * mu2, e12 - mu1 * mu2
    A1, A2 = 2 * mu1 * mu2 + L.C1, 2 * s12 + L.C2
    B1, B2 = mu1 * mu1 + mu2 * mu2 + L.C1, s1 + s2 + L.C2
    ss = A1 * A2 / (B1 * B2)
    d_mu1 = (2 * mu2 * A2 - 2 * mu2 * A1) / (B1 * B2) - ss * (2 * mu1 / B1 - 2 * mu1 / B2)
    d_e11 = -ss / B2
    d_e12 = 2 * A1 / (B1 * B2)
    n = a.numel()
    v_img = ((1 - lam) * torch.sign(a - gt) - lam * (L._blur(d_mu1, w) + 2 * a * L._blur(d_e11, w) + gt * L._blur(d_e12, w))) / n
    assert float((v_img - ar.grad).abs().max() / ar.grad.abs().max()) < 1e-9
