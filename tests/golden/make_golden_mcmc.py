"""Freeze the position noise of the reference's own MCMCDensityControllerImpl._add_xyz_noise (mcmc_density_controller.py:93-120,
with compute_cov_3d of internal/utils/gaussian_projection.py), run on the CPU in float64 on a seeded model with a recorded z
(torch.randn_like is replaced by the recorded draw while the method runs).  The reference checkout is the first argument.
Run:  python tests/golden/make_golden_mcmc.py <reference checkout>      -> tests/golden/mcmc_noise.npz"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, sys.argv[1])
# the controller module imports lightning and gsplat.relocation at load time; neither is used by _add_xyz_noise
lightning = types.ModuleType("lightning")
lightning.LightningModule = type("LightningModule", (), {})
sys.modules["lightning"] = lightning
for name in ("gsplat", "gsplat.relocation"):
    sys.modules[name] = types.ModuleType(name)
sys.modules["gsplat"].__path__ = []
sys.modules["gsplat.relocation"].compute_relocation = None
from internal.density_controllers.mcmc_density_controller import MCMCDensityController  # noqa: E402

N, NOISE_LR, XYZ_LR = 512, 5e5, 1.6e-4
g = torch.Generator().manual_seed(20240607)
means = torch.zeros(N, 3, dtype=torch.float64)    # so the updated means are the noise itself, without cancellation
log_scales = -4.0 + 0.7 * torch.randn(N, 3, generator=g, dtype=torch.float64)
raw_quats = torch.randn(N, 4, generator=g, dtype=torch.float64) * (0.3 + 4.7 * torch.rand(N, 1, generator=g, dtype=torch.float64))
# opacities from 1e-3 (w ~ 0.6) to 0.99 (w ~ e^-98): the whole range of the noise weight
opacity_logits = torch.logit(10 ** (-3 + 3 * torch.rand(N, 1, generator=g, dtype=torch.float64)).clamp(max=0.99))
z = torch.randn(N, 3, generator=g, dtype=torch.float64)


class Model:
    def __init__(self):
        self.means = means.clone()

    def get_scales(self):
        return torch.exp(log_scales)

    def get_rotations(self):
        return torch.nn.functional.normalize(raw_quats)

    def get_opacities(self):
        return torch.sigmoid(opacity_logits)


class Module:
    def is_final_step(self):
        return False

    gaussian_optimizers = [types.SimpleNamespace(param_groups=[{"name": "opacities", "lr": 0.05}, {"name": "means", "lr": XYZ_LR}])]


impl = MCMCDensityController(cap_max=N, noise_lr=NOISE_LR).instantiate()
model = Model()
randn_like = torch.randn_like
torch.randn_like = lambda t: z.to(t.dtype)
try:
    impl._add_xyz_noise({}, None, model, 0, Module())
finally:
    torch.randn_like = randn_like
np.savez_compressed(os.path.join(HERE, "mcmc_noise.npz"), means=means.numpy(), log_scales=log_scales.numpy(), raw_quats=raw_quats.numpy(),
                    opacity_logits=opacity_logits.numpy(), z=z.numpy(), noise_lr=np.float64(NOISE_LR), xyz_lr=np.float64(XYZ_LR),
                    means_after=model.means.numpy())
print("max |delta| =", float((model.means - means).abs().max()))
