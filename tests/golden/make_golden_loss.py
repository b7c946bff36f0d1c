"""Freeze outputs of the reference's OWN loss functions (internal/utils/ssim.py, imported by file path from the
reference checkout given as the first argument) for seeded image pairs: SSIM, L1, the combined training loss of
vanilla_metrics.py:57-74 and its autograd gradient w.r.t. the rendered image.
  loss_s<seed>_<H>x<W>.npz:          the 3-channel noise pair, lambda_dssim 0.2
  loss_<kind>_c<C>_<H>x<W>.npz:      oracle/loss_oracle.case(kind, C, H, W, seed) at lambda_dssim 0, 0.2 and 1 (loss[k], grad[k])
Run:  python tests/golden/make_golden_loss.py <reference checkout>      -> tests/golden/loss_*.npz"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle.loss_oracle import case  # noqa: E402

spec = importlib.util.spec_from_file_location("ref_ssim", os.path.join(sys.argv[1], "internal", "utils", "ssim.py"))
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)

LAMBDAS = (0.0, 0.2, 1.0)
CASES = [("flat", 3, 48, 64, 10), ("converged", 3, 48, 64, 11), ("masked", 3, 48, 64, 12), ("saturated", 3, 48, 64, 13),
         ("noise", 1, 37, 50, 14), ("noise", 4, 37, 50, 15)]


def pair(seed, H, W):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(3, H, W, generator=g)
    img = (gt + 0.15 * torch.randn(3, H, W, generator=g)).clamp(0, 1)      # a plausible render: the target plus noise
    return img, gt


for seed, H, W in [(0, 37, 50), (1, 96, 128), (2, 11, 11), (3, 5, 200)]:
    img, gt = pair(seed, H, W)
    img.requires_grad_(True)
    l1 = ref.l1_loss(img, gt)
    ss = ref.ssim(img, gt)
    loss = 0.8 * l1 + 0.2 * (1.0 - ss)
    loss.backward()
    np.savez_compressed(os.path.join(HERE, f"loss_s{seed}_{H}x{W}.npz"), meta=np.array([seed, H, W]), l1=l1.detach().numpy(),
                        ssim=ss.detach().numpy(), loss=loss.detach().numpy(), grad=img.grad.numpy())
    print(seed, H, W, float(l1), float(ss), float(loss))

for kind, C, H, W, seed in CASES:
    img, gt = case(kind, C, H, W, seed)
    losses, grads = [], []
    for lam in LAMBDAS:
        x = img.clone().requires_grad_(True)
        l1 = ref.l1_loss(x, gt)
        ss = ref.ssim(x, gt)
        loss = (1.0 - lam) * l1 + lam * (1.0 - ss)          # vanilla_metrics.py:57-74
        loss.backward()
        losses.append(loss.detach().numpy())
        grads.append(x.grad.numpy())
    np.savez_compressed(os.path.join(HERE, f"loss_{kind}_c{C}_{H}x{W}.npz"), meta=np.array([seed, C, H, W]), kind=np.array(kind),
                        lambdas=np.array(LAMBDAS), l1=l1.detach().numpy(), ssim=ss.detach().numpy(), loss=np.stack(losses),
                        grad=np.stack(grads))
    print(kind, C, H, W, float(l1), float(ss), [float(v) for v in losses])
