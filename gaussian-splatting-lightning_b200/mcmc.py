"""3DGS-MCMC training on the b200gs kernels (the reference's ``configs/mcmc.yaml`` / ``configs/gsplat-mcmc.yaml``).

    compute_relocation(...)          gsplat's ``gsplat.relocation.compute_relocation`` (mcmc_density_controller.py:13,121-128);
                                     ``b200gs.compat.install()`` registers it as ``gsplat.relocation``
    add_position_noise(...)          ``MCMCDensityControllerImpl._add_xyz_noise`` (mcmc_density_controller.py:93-120) as one
                                     in-place kernel over the model's raw parameters
    B200MCMCDensityController        drop-in for ``MCMCDensityController`` (select with
                                     ``model.density: b200gs.mcmc.B200MCMCDensityController``): the reference's controller with
                                     the position noise on the fused kernel
"""
from dataclasses import dataclass

import torch

from ._lib import check, lib, ptr
from .ops import _f32c, _stream


def compute_relocation(opacities: torch.Tensor, scales: torch.Tensor, ratios: torch.Tensor, binoms: torch.Tensor):
    """New opacities ``[n]`` and scales ``[n,3]`` of Gaussians that ``ratios[i]`` samples now share (3DGS-MCMC Eq. (9)):
    ``o' = 1 - (1 - o)^(1/N)``, ``scale' = scale * o / D`` with N = ``ratios`` clamped to ``[1, n_max]``, ``n_max =
    binoms.shape[0]``.  ``ratios`` may be int32 or int64 (the controller passes ``bincount(...) + 1``)."""
    opacities, scales, binoms = _f32c(opacities, "opacities"), _f32c(scales, "scales"), _f32c(binoms, "binoms")
    n = opacities.numel()
    if opacities.dim() != 1 or scales.shape != (n, 3) or ratios.shape != (n,):
        raise ValueError(f"expected opacities [n], scales [n, 3] and ratios [n], got {tuple(opacities.shape)}, "
                         f"{tuple(scales.shape)}, {tuple(ratios.shape)}")
    if binoms.dim() != 2 or binoms.shape[0] != binoms.shape[1] or binoms.shape[0] < 1:
        raise ValueError(f"binoms must be [n_max, n_max], got {tuple(binoms.shape)}")
    if ratios.dtype not in (torch.int32, torch.int64) or ratios.device != opacities.device:
        raise ValueError(f"ratios must be an int32 or int64 tensor on {opacities.device}, got {ratios.dtype} on {ratios.device}")
    n_max = binoms.shape[0]
    counts = ratios.contiguous() if ratios.dtype == torch.int32 else ratios.clamp(1, n_max).to(torch.int32)
    new_opacities = torch.empty_like(opacities)
    new_scales = torch.empty_like(scales)
    check(lib().b200gs_mcmc_relocation(n, ptr(opacities), ptr(scales), ptr(counts), ptr(binoms), n_max, ptr(new_opacities),
                                       ptr(new_scales), _stream()), "b200gs_mcmc_relocation")
    return new_opacities, new_scales


def add_position_noise(means: torch.Tensor, log_scales: torch.Tensor, raw_quats: torch.Tensor, opacity_logits: torch.Tensor,
                       noise_lr: float, xyz_lr: float, generator: torch.Generator = None) -> torch.Tensor:
    """``means += noise_lr * xyz_lr * op_sigmoid(1 - sigmoid(opacity_logits)) * Sigma z`` in place, Sigma the covariance of
    ``exp(log_scales)`` and ``normalize(raw_quats)``, z standard normal.  The Philox key is drawn on the host from
    ``generator`` (default: torch's default CPU generator), so the noise follows ``torch.manual_seed`` without a device sync
    and every call draws a fresh key.  Returns ``means``."""
    if means.dtype != torch.float32 or not means.is_cuda or not means.is_contiguous():
        raise ValueError("means must be a contiguous float32 CUDA tensor (it is updated in place)")
    log_scales, raw_quats = _f32c(log_scales, "log_scales"), _f32c(raw_quats, "raw_quats")
    opacity_logits = _f32c(opacity_logits, "opacity_logits")
    n = means.shape[0]
    if means.shape != (n, 3) or log_scales.shape != (n, 3) or raw_quats.shape != (n, 4) or opacity_logits.numel() != n:
        raise ValueError(f"expected means [n, 3], log_scales [n, 3], raw_quats [n, 4] and n opacity logits, got {tuple(means.shape)}, "
                         f"{tuple(log_scales.shape)}, {tuple(raw_quats.shape)}, {tuple(opacity_logits.shape)}")
    seed = int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64, generator=generator))
    with torch.no_grad():
        check(lib().b200gs_mcmc_position_noise(n, ptr(means), ptr(log_scales), ptr(raw_quats), ptr(opacity_logits),
                                               float(noise_lr) * float(xyz_lr), seed, 0, _stream()), "b200gs_mcmc_position_noise")
        torch.autograd.graph.increment_version(means)   # an in-place update, as the reference's means.add_(noise) is
    return means


@dataclass
class B200MCMCDensityController:
    """The fields and defaults of the reference's ``MCMCDensityController`` (mcmc_density_controller.py:20-42)."""
    cap_max: int
    noise_lr: float = 5e5
    densify_from_iter: int = 500
    densify_until_iter: int = 25_000
    densification_interval: int = 100
    min_opacity: float = 0.005
    N_max: int = 51

    def instantiate(self, *args, **kwargs):
        """The reference's ``MCMCDensityControllerImpl`` (relocation and growth unchanged; its ``compute_relocation`` import
        resolves to this module's through ``b200gs.compat``) with ``_add_xyz_noise`` on the fused kernel."""
        from . import compat
        compat.install()
        try:
            from internal.density_controllers.mcmc_density_controller import MCMCDensityControllerImpl
        except ImportError as e:
            raise ImportError("B200MCMCDensityController runs the reference's internal.density_controllers.mcmc_density_controller, "
                              f"which is not importable (run from a gaussian-splatting-lightning checkout): {e}") from e
        assert self.cap_max > 0, "cap_max must > 0"
        return _impl_class(MCMCDensityControllerImpl)(self)


_IMPL = {}


def _impl_class(base):
    if base not in _IMPL:
        class B200MCMCDensityControllerImpl(base):
            def _add_xyz_noise(self, outputs: dict, batch, gaussian_model, global_step: int, pl_module) -> None:
                from .renderers import _raw_parameters
                raw = _raw_parameters(gaussian_model)
                if raw is None:     # a model whose activations are not the vanilla ones: the reference's torch formula
                    return super()._add_xyz_noise(outputs, batch, gaussian_model, global_step, pl_module)
                # the reference's guard, kept as written: `is_final_step` is a method, so this never returns
                if pl_module.is_final_step is True:
                    return
                xyz_lr = -1
                for opt in pl_module.gaussian_optimizers:
                    for param_group in opt.param_groups:
                        if param_group["name"] == "means":
                            xyz_lr = param_group["lr"]
                    if xyz_lr >= 0:
                        break
                assert xyz_lr >= 0
                add_position_noise(raw["means"], raw["scales"], raw["rotations"], raw["opacities"], self.config.noise_lr, xyz_lr)

        _IMPL[base] = B200MCMCDensityControllerImpl
    return _IMPL[base]
