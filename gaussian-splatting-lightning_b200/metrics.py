"""Training metrics (the reference's ``internal/metrics/vanilla_metrics.py``, ``inverse_depth_metrics.py``, ``mcmc_metrics.py``,
``scale_regularization_metrics.py`` and ``normal_reg.py``) on the b200gs kernels.
Select them as the model's metric:

    model:
      metric:
        class_path: b200gs.metrics.B200InverseDepthMetrics
        init_args: {depth_loss_type: l1, depth_loss_weight: {init: 1.0, final_factor: 0.01, max_steps: 30000}}

``B200VanillaMetrics`` has ``VanillaMetrics``' config fields and defaults; its RGB loss is ``ops.l1_ssim_loss`` (K9/K10) for both
``fused_ssim`` settings.  ``B200InverseDepthMetrics`` has ``HasInverseDepthMetrics``' fields, defaults and ``WeightScheduler``, and its
module the same methods, output keys and progress-bar flags; the depth loss is ``inverse_depth_loss``: four kernel launches forward,
one backward, no host synchronisation.  PSNR and LPIPS for validation stay torchmetrics objects, created in ``setup`` when
torchmetrics imports.  ``B200MCMCMetrics``, ``B200ScaleRegularizationMetrics`` and ``B200ScaleRegularizationWithDepthMetrics`` have
``MCMCMetrics``', ``ScaleRegularizationMetrics``' and ``ScaleRegularizationWithDepthMetrics``' fields, defaults, output keys and
progress-bar flags; their per-Gaussian terms are ``gaussian_regularizers``: two kernel launches forward, one backward.
``B200VanillaWithNormalRegMetrics`` has ``VanillaWithNormalRegMetrics``' fields, defaults, ``setup`` mutation, output keys and
progress-bar flags; its depth-normal term is ``normal_consistency_loss``: two kernel launches forward, one backward.
``depth_to_normal`` is gsplat's ``utils.depth_to_normal`` for the reference's call, which ``compat.install()`` registers.
``B200VanillaMetricsWithSimilarityRegularization`` has ``VanillaMetricsWithSimilarityRegularization``' fields, defaults, backward
hook and logged key; its k-NN query is ``ops.knn_points`` and its term ``ops.similarity_regularization``.
"""
import time
from dataclasses import dataclass, field
from typing import Literal, Optional

import torch

from . import ops
from ._lib import check, lib, ptr
from .ops import _stream

try:  # inside the reference repo: subclass its config and module bases so the trainer's type checks hold
    from internal.metrics.metric import Metric, MetricModule  # type: ignore
except Exception:
    class Metric:
        def instantiate(self, *args, **kwargs):
            pass

    class MetricModule(torch.nn.Module):
        def __init__(self, config, *args, **kwargs) -> None:
            super().__init__()
            self.config = config

        def setup(self, stage: str, pl_module):
            pass

        def training_setup(self, pl_module):
            return [], []

        def on_parameter_move(self, *args, **kwargs):
            pass

DEPTH_LOSS_FWD_LAUNCHES = 4     # library launches of one inverse_depth_loss forward: statistics, prologue, tiles, loss
DEPTH_LOSS_BWD_LAUNCHES = 1     # and of its backward
_LOSS_TYPES = {"l1": 0, "l2": 1, "l1+ssim": 2}


class _InverseDepthLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, gt, mask, loss_type, norm, median, ssim_weight):
        H, W = pred.shape
        L = lib()
        nbytes = int(L.b200gs_depth_loss_workspace_bytes(H, W, loss_type))
        ws = torch.empty(nbytes // 4, dtype=torch.float32, device=pred.device)
        loss = torch.empty((), dtype=torch.float32, device=pred.device)
        stats = torch.empty(2, dtype=torch.float32, device=pred.device)
        msy, msx = mask.stride() if mask is not None else (0, 0)
        check(L.b200gs_depth_loss_fwd(H, W, ptr(pred), ptr(gt), ptr(mask), msy, msx, loss_type, norm, median, ssim_weight, ptr(ws), nbytes,
                                      ptr(loss), ptr(stats), _stream()), "b200gs_depth_loss_fwd")
        ctx.save_for_backward(pred, gt, mask, ws)
        ctx.args = (loss_type, norm, median, ssim_weight)
        ctx.mark_non_differentiable(stats)
        return loss, stats

    @staticmethod
    def backward(ctx, v_loss, _v_stats):
        pred, gt, mask, ws = ctx.saved_tensors
        loss_type, norm, median, ssim_weight = ctx.args
        H, W = pred.shape
        v = v_loss.reshape(1).to(torch.float32).contiguous()
        v_pred = torch.empty_like(pred)
        msy, msx = mask.stride() if mask is not None else (0, 0)
        check(lib().b200gs_depth_loss_bwd(H, W, ptr(pred), ptr(gt), ptr(mask), msy, msx, loss_type, norm, median, ssim_weight, ptr(ws),
                                          ws.numel() * 4, ptr(v), ptr(v_pred), _stream()), "b200gs_depth_loss_bwd")
        return v_pred, None, None, None, None, None, None


def inverse_depth_loss(gt, pred, *, loss_type="l1", ssim_weight=0.2, normalized=False, median=None, mean_normalization=False,
                       mask=None):
    """``HasInverseDepthMetricsModule.get_inverse_depth_metric``'s loss of one view: pred and gt float32 CUDA [H,W], the gradient to
    pred only.  The normalisation is the reference's if / elif chain: ``normalized`` (pred' = (pred - min) / (max - min + 1e-8),
    min / max detached), else ``median`` when not None (pred' = pred / median, a host number), else ``mean_normalization``
    (gt and pred divided by mean(gt)).  ``mask``: None, or the image mask [H,W] or [C,H,W] (bool or uint8, nonzero keeps; channel 0
    is read); masked pixels are 0 in both maps.  ``loss_type``: "l1", "l2" or "l1+ssim" = (1 - ssim_weight) l1 + ssim_weight
    (1 - SSIM) with torchmetrics' default SSIM (needs H, W >= 11; no mask).  Returns (loss, stats): a device scalar and
    [mean |a - b| or (a - b)^2, mean SSIM (NaN unless "l1+ssim")]."""
    if loss_type not in _LOSS_TYPES:
        raise NotImplementedError(f"depth_loss_type {loss_type!r}: only {sorted(_LOSS_TYPES)} are provided")
    if pred.shape != gt.shape or pred.dim() != 2:
        raise ValueError(f"pred and gt must both be [H, W], got {tuple(pred.shape)} and {tuple(gt.shape)}")
    if mask is not None and loss_type == "l1+ssim":
        raise NotImplementedError("l1+ssim with an image mask: the reference hands torchmetrics a [1,1,C,H,W] volume, whose "
                                  "3-D SSIM is not provided")
    if any(t.dtype != torch.float32 or not t.is_cuda for t in (pred, gt)):
        raise ValueError("pred and gt must be float32 CUDA tensors")
    H, W = pred.shape
    if mask is not None:
        if mask.dim() == 3:
            mask = mask[0]
        if tuple(mask.shape) != (H, W) or mask.dtype not in (torch.bool, torch.uint8) or mask.device != pred.device:
            raise ValueError(f"mask must be bool or uint8 [C,H,W] or [H,W] on the maps' device, got {mask.dtype} {tuple(mask.shape)}")
        mask = mask.view(torch.uint8)
    if loss_type == "l1+ssim" and (H < 11 or W < 11):
        raise ValueError(f"l1+ssim needs maps of at least 11x11, got {H}x{W}")
    norm = 1 if normalized else (2 if median is not None else (3 if mean_normalization else 0))
    return _InverseDepthLoss.apply(pred.contiguous(), gt.detach().contiguous(), mask, _LOSS_TYPES[loss_type], norm,
                                   float(median) if norm == 2 else 0.0, float(ssim_weight))


GAUSSIAN_REG_FWD_LAUNCHES = 2   # library launches of one gaussian_regularizers forward: per-CTA partials, reduce
GAUSSIAN_REG_BWD_LAUNCHES = 1   # and of its backward
_GREG_RAW, _GREG_OPACITY, _GREG_SCALE, _GREG_OVER_SCALE, _GREG_OVER_RATIO = 1, 2, 4, 8, 16


class _GaussianRegularizers(torch.autograd.Function):
    @staticmethod
    def forward(ctx, opacities, scales, flags, args, statistics):
        n = (opacities if opacities is not None else scales).shape[0]
        dev = (opacities if opacities is not None else scales).device
        L = lib()
        nbytes = int(L.b200gs_gaussian_reg_workspace_bytes(n))
        ws = torch.empty(nbytes // 4, dtype=torch.float32, device=dev)
        terms = torch.empty(4, dtype=torch.float32, device=dev)
        stats = torch.empty(5, dtype=torch.float32, device=dev) if statistics else None
        check(L.b200gs_gaussian_reg_fwd(n, ptr(opacities), ptr(scales), flags, *args, ptr(ws), nbytes, ptr(terms), ptr(stats), _stream()),
              "b200gs_gaussian_reg_fwd")
        ctx.save_for_backward(opacities, scales, ws)
        ctx.args = (flags, args)
        if stats is None:
            return terms
        ctx.mark_non_differentiable(stats)
        return terms, stats

    @staticmethod
    def backward(ctx, v_terms, *_v_stats):
        opacities, scales, ws = ctx.saved_tensors
        flags, args = ctx.args
        n = (opacities if opacities is not None else scales).shape[0]
        v = v_terms.to(torch.float32).contiguous()
        v_o = torch.empty_like(opacities) if opacities is not None else None
        v_s = torch.empty_like(scales) if scales is not None else None
        check(lib().b200gs_gaussian_reg_bwd(n, ptr(opacities), ptr(scales), flags, *args, ptr(ws), ws.numel() * 4, ptr(v), ptr(v_o),
                                            ptr(v_s), _stream()), "b200gs_gaussian_reg_bwd")
        return v_o, v_s, None, None, None


def gaussian_regularizers(opacities, scales, *, raw, opacity_weight=0.0, scale_weight=0.0, max_scale=-1.0, max_scale_ratio=10.0,
                          scale_lambda=0.0, ratio_lambda=0.0, statistics=True):
    """The per-Gaussian regularisers of ``MCMCMetrics`` and ``ScaleRegularizationMetrics`` in one fused pass (K36/K37, backward
    K38): opacities float32 CUDA [N,1] and scales [N,3], either None when no term reads it.  ``raw``: they are the logits and
    log-scales and the kernels apply torch's fp32 sigmoid / exp; otherwise they are the activated values (the getters' output).
    Returns (terms, stats), or terms alone with ``statistics=False``:
        terms [4] = [opacity_weight mean|o|, scale_weight mean|s|, scale_lambda sum(s [s > max_scale]) / (n_s + 1),
                     ratio_lambda sum(r [r > max_scale_ratio]) / (n_r + 1)],   r = max / (mid + 1e-8) of each sorted row
        stats [5] = [n_s, n_r, max of the largest scale, max r, mean r]        (not differentiable; needs scales)
    A term whose weight is 0 (or whose tensor is None) is an exact 0 and adds nothing to the gradient.  Gradients go to the
    tensors passed.  Tied scales are ranked as torch.sort ranks them on the GPU (csrc/gauss_reg.cu's table)."""
    t = opacities if opacities is not None else scales
    if t is None:
        raise ValueError("gaussian_regularizers needs opacities or scales")
    n = t.shape[0]
    if n == 0:
        raise ValueError("gaussian_regularizers needs at least one Gaussian")
    if opacities is not None and (opacities.dim() != 2 or opacities.shape[1] != 1):
        raise ValueError(f"opacities must be [N, 1], got {tuple(opacities.shape)}")
    if scales is not None and (scales.dim() != 2 or scales.shape[1] != 3):
        raise ValueError(f"scales must be [N, 3], got {tuple(scales.shape)}")
    if opacities is not None and scales is not None and opacities.shape[0] != scales.shape[0]:
        raise ValueError(f"opacities and scales hold {opacities.shape[0]} and {scales.shape[0]} Gaussians")
    if any(x is not None and (x.dtype != torch.float32 or not x.is_cuda) for x in (opacities, scales)):
        raise ValueError("opacities and scales must be float32 CUDA tensors")
    if statistics and scales is None:
        raise ValueError("the statistics need the scales")
    flags = _GREG_RAW if raw else 0
    if opacities is not None:
        flags |= _GREG_OPACITY
        opacities = opacities.contiguous()
    if scales is not None:
        flags |= _GREG_SCALE | _GREG_OVER_SCALE | _GREG_OVER_RATIO
        scales = scales.contiguous()
    args = tuple(float(a) for a in (opacity_weight, scale_weight, max_scale, max_scale_ratio, scale_lambda, ratio_lambda))
    return _GaussianRegularizers.apply(opacities, scales, flags, args, bool(statistics))


def _regularized_parameters(gaussian_model, opacities: bool, scales_getter):
    """(opacities or None, scales or None, raw): the raw parameters of a vanilla model that is not pre-activated
    (``renderers._raw_parameters``' rule), activated in the kernels; any other model's getters, which autograd chains.
    ``scales_getter`` None: no scales."""
    from .renderers import _raw_parameters
    params = None if getattr(gaussian_model, "is_pre_activated", False) else _raw_parameters(gaussian_model)
    if params is not None:
        return (params["opacities"] if opacities else None), (params["scales"] if scales_getter else None), True
    return ((gaussian_model.get_opacity if opacities else None), (scales_getter(gaussian_model) if scales_getter else None), False)


def _torchmetrics():
    try:
        from torchmetrics.image import PeakSignalNoiseRatio
        from torchmetrics.image.lpip import LearnedPerceptualImagePatchSimilarity
    except ImportError:
        return None
    return PeakSignalNoiseRatio, LearnedPerceptualImagePatchSimilarity


@dataclass
class B200VanillaMetrics(Metric):
    lambda_dssim: float = 0.2

    rgb_diff_loss: Literal["l1", "l2"] = "l1"

    lpips_net_type: Literal["vgg", "alex", "squeeze"] = "alex"

    fused_ssim: bool = False

    def instantiate(self, *args, **kwargs) -> "B200VanillaMetricsModule":
        self._check()
        return B200VanillaMetricsModule(self)

    def _check(self):
        if self.rgb_diff_loss != "l1":
            raise NotImplementedError(f"rgb_diff_loss {self.rgb_diff_loss!r}: the fused RGB loss is L1 + SSIM")


class B200VanillaMetricsModule(MetricModule):
    def __init__(self, config, *args, **kwargs) -> None:
        super().__init__(config, *args, **kwargs)
        self.no_state_dict_models = {}
        self.psnr = None

    def setup(self, stage: str, pl_module):
        # fused_ssim selects fused-ssim's "same" SSIM in the reference, the formula K9/K10 compute for both settings
        self.lambda_dssim = self.config.lambda_dssim
        tm = _torchmetrics()
        if tm is not None:
            self.psnr = tm[0](data_range=1.0)
            self.no_state_dict_models["lpips"] = tm[1](normalize=True, net_type=self.config.lpips_net_type)

    def _get_basic_metrics(self, pl_module, gaussian_model, batch, outputs):
        camera, image_info, _ = batch
        image_name, gt_image, masked_pixels = image_info
        image = outputs["render"]
        if masked_pixels is not None:
            masked_pixels = masked_pixels.to(torch.uint8)      # False represents masked pixels
            gt_image = gt_image * masked_pixels
            image = image * masked_pixels
        loss, stats = ops.l1_ssim_loss(image, gt_image, self.lambda_dssim)
        return {
            "loss": loss,
            "rgb_diff": stats[0],
            "ssim": stats[1],
        }, {
            "loss": True,
            "rgb_diff": True,
            "ssim": True,
        }

    def get_train_metrics(self, pl_module, gaussian_model, step: int, batch, outputs):
        return self._get_basic_metrics(pl_module=pl_module, gaussian_model=gaussian_model, batch=batch, outputs=outputs)

    def get_validate_metrics(self, pl_module, gaussian_model, batch, outputs):
        if self.psnr is None:
            raise ImportError("validation metrics need torchmetrics (PSNR and LPIPS), which is not installed")
        metrics, prog_bar = self._get_basic_metrics(pl_module, gaussian_model, batch, outputs)
        camera, image_info, _ = batch
        image_name, gt_image, _ = image_info
        metrics["psnr"] = self.psnr(outputs["render"], gt_image)
        prog_bar["psnr"] = True
        metrics["lpips"] = self.no_state_dict_models["lpips"](outputs["render"].clamp(0., 1.).unsqueeze(0), gt_image.unsqueeze(0))
        prog_bar["lpips"] = True
        prog_bar["ssim"] = True
        return metrics, prog_bar

    def on_parameter_move(self, *args, **kwargs):
        if "lpips" in self.no_state_dict_models:
            self.no_state_dict_models["lpips"] = self.no_state_dict_models["lpips"].to(*args, **kwargs)


try:
    from internal.metrics.inverse_depth_metrics import WeightScheduler  # type: ignore
except Exception:
    @dataclass
    class WeightScheduler:
        init: float = 1.0

        final_factor: float = 0.01

        max_steps: int = 30_000


@dataclass
class B200InverseDepthMetrics(B200VanillaMetrics):
    depth_loss_type: Literal["l1", "l1+ssim", "l2", "kl"] = "l1"

    depth_loss_ssim_weight: float = 0.2

    depth_loss_weight: WeightScheduler = field(default_factory=lambda: WeightScheduler())

    depth_normalized: bool = False

    depth_median_normalization: bool = False

    depth_mean_normalization: bool = False

    depth_output_key: str = "inverse_depth"

    def instantiate(self, *args, **kwargs) -> "B200InverseDepthMetricsModule":
        self._check()
        return B200InverseDepthMetricsModule(self)


class B200InverseDepthMetricsModule(B200VanillaMetricsModule):
    def setup(self, stage: str, pl_module):
        super().setup(stage, pl_module)
        if self.config.depth_loss_type not in _LOSS_TYPES:
            raise NotImplementedError()

    def get_inverse_depth_metric(self, batch, outputs):
        _, image_info, gt_inverse_depth_data = batch
        device = batch[0].device
        if gt_inverse_depth_data is None:
            return torch.tensor(0., device=device)
        if gt_inverse_depth_data.mask is not None:
            raise NotImplementedError("DepthMap.mask is not provided")
        c = self.config
        median = None
        if not c.depth_normalized and gt_inverse_depth_data.median is not None:
            assert c.depth_median_normalization
            median = gt_inverse_depth_data.median
        gt_inverse_depth = gt_inverse_depth_data.get(device=device)
        predicted_inverse_depth = outputs[c.depth_output_key].squeeze(0)
        loss, _ = inverse_depth_loss(gt_inverse_depth, predicted_inverse_depth, loss_type=c.depth_loss_type,
                                     ssim_weight=c.depth_loss_ssim_weight, normalized=c.depth_normalized, median=median,
                                     mean_normalization=c.depth_mean_normalization, mask=image_info[-1])
        return loss

    def get_weight(self, step: int):
        w = self.config.depth_loss_weight
        return w.init * (w.final_factor ** min(step / w.max_steps, 1))

    def get_predicted_depth(self, pl_module, gaussian_model, batch, outputs):
        predicted_depth = outputs
        if outputs.get(self.config.depth_output_key, None) is None and batch[-1] is not None:
            assert batch[-1].camera is not None
            depth_camera = batch[-1].camera.to_device(pl_module.device)
            predicted_depth = pl_module.renderer(
                depth_camera,
                gaussian_model,
                torch.zeros((3, ), dtype=torch.float32, device=pl_module.device),
                render_types=[self.config.depth_output_key],
            )
        return predicted_depth

    def get_train_metrics(self, pl_module, gaussian_model, step: int, batch, outputs):
        metrics, pbar = super().get_train_metrics(pl_module, gaussian_model, step, batch, outputs)
        d_reg_weight = self.get_weight(step)
        predicted_depth = self.get_predicted_depth(pl_module, gaussian_model, batch, outputs)
        d_reg = self.get_inverse_depth_metric(batch, predicted_depth) * d_reg_weight
        metrics["loss"] = metrics["loss"] + d_reg
        metrics["d_reg"] = d_reg
        metrics["d_w"] = d_reg_weight
        pbar["d_reg"] = True
        pbar["d_w"] = True
        return metrics, pbar

    def get_validate_metrics(self, pl_module, gaussian_model, batch, outputs):
        metrics, pbar = super().get_validate_metrics(pl_module, gaussian_model, batch, outputs)
        predicted_depth = self.get_predicted_depth(pl_module, gaussian_model, batch, outputs)
        d_reg = self.get_inverse_depth_metric(batch, predicted_depth)
        metrics["loss"] = metrics["loss"] + d_reg
        metrics["d_reg"] = d_reg
        pbar["d_reg"] = True
        return metrics, pbar


@dataclass
class B200VisibilityMapMetrics(B200VanillaMetrics):
    """``VisibilityMapMetrics``: the RGB loss on image * w and gt * w, w = outputs["visibility"] * the dataset mask, plus
    ``vis_reg_factor`` mean((1 - visibility)^2), on ``ops.visibility_l1_ssim_loss`` (K34/K35).  Validation metrics are
    ``B200VanillaMetrics``', as in the reference."""
    vis_reg_factor: float = 0.2

    def instantiate(self, *args, **kwargs) -> "B200VisibilityMapMetricsModule":
        self._check()
        return B200VisibilityMapMetricsModule(self)


class B200VisibilityMapMetricsModule(B200VanillaMetricsModule):
    def get_train_metrics(self, pl_module, gaussian_model, step: int, batch, outputs):
        camera, image_info, extra_data = batch
        image_name, gt_image, masked_pixels = image_info
        loss, stats = ops.visibility_l1_ssim_loss(outputs["render"], gt_image, outputs["visibility"], masked_pixels, self.lambda_dssim,
                                                  self.config.vis_reg_factor)
        metrics = {"loss": loss, "rgb_diff": stats[0], "ssim": stats[1], "vis_reg": stats[2]}
        return metrics, {k: True for k in metrics}


# ---- fused_ssim.fused_ssim (the name VanillaMetrics(fused_ssim=True) and the Taming density controller import) --------------
def fused_ssim(img1, img2, padding="same", train=True):
    """fused-ssim's ``fused_ssim``: the mean SSIM of img1 and img2 [1,C,H,W] (11-tap Gaussian, sigma 1.5, zero padding,
    C1 = 0.01^2, C2 = 0.03^2), the gradient to img1 only; on K9/K10.  Only padding="same" and a batch of one are provided.
    ``train`` is accepted and changes nothing: the gradient is computed in the backward, not the forward."""
    if padding != "same":
        raise NotImplementedError(f"fused_ssim padding={padding!r}: only 'same' is provided")
    if img1.dim() != 4 or img1.shape[0] != 1 or img1.shape != img2.shape:
        raise ValueError(f"fused_ssim takes two [1,C,H,W] images, got {tuple(img1.shape)} and {tuple(img2.shape)}")
    loss, stats = ops.l1_ssim_loss(img1[0], img2[0].detach(), 1.0)     # loss = 1 - SSIM, K10's gradient
    return stats[1] - (loss - loss.detach())


# ---- MCMCMetrics and ScaleRegularization*Metrics (internal/metrics/mcmc_metrics.py, scale_regularization_metrics.py) -------------
_SCALE_KEYS = ("scale_reg", "scale_ratio_reg", "n_over_scales", "n_over_ratios", "max_scale", "max_ratio", "mean_ratio")


@dataclass
class B200MCMCMetricsMixin:
    mcmc_reg_until_iter: int = -1

    opacity_reg: float = 0.01

    scale_reg: float = 0.01

    reg_weight_decay: float = 1.


class B200MCMCMetricsModuleMixin:
    """The MCMC regularisers: ``opacity_reg`` mean|get_opacity| and ``scale_reg`` mean|get_scaling|, both weights divided by
    ``reg_weight_decay`` capped at 5; the scale term is added only with a positive weight.  In training they stop at step
    ``mcmc_reg_until_iter`` when that is not negative; validation always reports them.  Keys ``o_reg`` and ``s_reg``, off the
    progress bar."""

    def setup(self, *args, **kwargs):
        super().setup(*args, **kwargs)
        divisor = min(self.config.reg_weight_decay, 5.)
        self.opacity_reg_weight, self.scale_reg_weight = self.config.opacity_reg / divisor, self.config.scale_reg / divisor

    def _mcmc_terms_apply(self, step: int) -> bool:
        until = self.config.mcmc_reg_until_iter
        return until < 0 or step < until

    def reg_loss(self, gaussian_model, basic_metrics):
        metrics, pbar = basic_metrics
        with_scale = self.scale_reg_weight > 0
        opacities, scales, raw = _regularized_parameters(gaussian_model, True, (lambda m: m.get_scaling) if with_scale else None)
        terms = gaussian_regularizers(opacities, scales, raw=raw, opacity_weight=self.opacity_reg_weight,
                                      scale_weight=self.scale_reg_weight if with_scale else 0.0, statistics=False)
        metrics["loss"] = metrics["loss"] + terms[0] + terms[1]
        metrics["o_reg"], metrics["s_reg"] = terms[0], terms[1]
        pbar["o_reg"] = pbar["s_reg"] = False
        return metrics, pbar

    def get_train_metrics(self, pl_module, gaussian_model, step: int, batch, outputs):
        result = super().get_train_metrics(pl_module, gaussian_model, step, batch, outputs)
        return self.reg_loss(gaussian_model, result) if self._mcmc_terms_apply(step) else result

    def get_validate_metrics(self, pl_module, gaussian_model, batch, outputs):
        return self.reg_loss(gaussian_model, super().get_validate_metrics(pl_module, gaussian_model, batch, outputs))


@dataclass
class B200MCMCMetrics(B200MCMCMetricsMixin, B200VanillaMetrics):
    def instantiate(self, *args, **kwargs) -> "B200MCMCMetricsModule":
        self._check()
        return B200MCMCMetricsModule(self)


class B200MCMCMetricsModule(B200MCMCMetricsModuleMixin, B200VanillaMetricsModule):
    pass


@dataclass
class B200ScaleRegularizationMetricsMixin:
    """Fields of the over-scale / over-ratio regularisers.  ``max_scale`` <= 0 is resolved in ``setup``; the configuration is
    rejected when ``scale_reg_from`` is negative, or when the ratio term is on (``scale_ratio_reg_lambda`` > 0) with a ratio
    threshold that is not positive."""

    scale_reg_from: int = 3100

    max_scale: float = -1

    max_scale_outside_partition: Optional[float] = None

    max_scale_ratio: float = 10

    scale_reg_lambda: float = 0.05

    scale_ratio_reg_lambda: float = 0.05

    def __post_init__(self):
        # no base of these configs defines __post_init__, so there is nothing to chain to
        assert self.scale_reg_from >= 0, f"scale_reg_from must not be negative, got {self.scale_reg_from}"
        assert self.scale_ratio_reg_lambda <= 0. or self.max_scale_ratio > 0, \
            f"max_scale_ratio must be positive when the ratio term is on, got {self.max_scale_ratio}"

    def _check(self):
        super()._check()
        if self.max_scale_outside_partition is not None:
            raise NotImplementedError("max_scale_outside_partition needs the partition store's distance_factors, which is not provided")


class B200ScaleRegularizationMetricsModuleMixin:
    """The over-scale and over-ratio regularisers of get_scales() with their statistics: added in training from step
    ``scale_reg_from`` on and always in validation.  A term whose lambda is not positive is a device 0, and so is its count; the
    ratio statistics are reported whatever ``scale_ratio_reg_lambda`` is.  The loss grows as (basic [+ d_reg]) + scale_reg +
    scale_ratio_reg.  Keys in _SCALE_KEYS, off the progress bar."""

    def setup(self, stage: str, pl_module):
        super().setup(stage, pl_module)
        c = self.config
        if stage == "fit" and c.max_scale <= 0:
            extent = pl_module.trainer.datamodule.dataparser_outputs.camera_extent
            c.max_scale = extent * 1.1
            assert c.max_scale > 0., f"the camera extent gives max_scale {c.max_scale}"

    def get_scale_regularization_metrics(self, gaussian_model, pl_module, metrics, pbar):
        c = self.config
        positive = lambda v: v if v > 0. else 0.0      # noqa: E731
        _, scales, raw = _regularized_parameters(gaussian_model, False, lambda m: m.get_scales())
        terms, stats = gaussian_regularizers(None, scales, raw=raw, max_scale=c.max_scale, max_scale_ratio=c.max_scale_ratio,
                                             scale_lambda=positive(c.scale_reg_lambda), ratio_lambda=positive(c.scale_ratio_reg_lambda))
        metrics["loss"] = metrics["loss"] + terms[2] + terms[3]
        for key, value in zip(_SCALE_KEYS, (terms[2], terms[3], *stats.unbind())):
            metrics[key] = value
            pbar[key] = False

    def get_train_metrics(self, pl_module, gaussian_model, step: int, batch, outputs):
        metrics, pbar = super().get_train_metrics(pl_module, gaussian_model, step, batch, outputs)
        if step >= self.config.scale_reg_from:
            self.get_scale_regularization_metrics(gaussian_model, pl_module, metrics, pbar)
        return metrics, pbar

    def get_validate_metrics(self, pl_module, gaussian_model, batch, outputs):
        metrics, pbar = super().get_validate_metrics(pl_module, gaussian_model, batch, outputs)
        self.get_scale_regularization_metrics(gaussian_model, pl_module, metrics, pbar)
        return metrics, pbar


@dataclass
class B200ScaleRegularizationMetrics(B200ScaleRegularizationMetricsMixin, B200VanillaMetrics):
    def instantiate(self, *args, **kwargs) -> "B200ScaleRegularizationMetricsModule":
        self._check()
        return B200ScaleRegularizationMetricsModule(self)


class B200ScaleRegularizationMetricsModule(B200ScaleRegularizationMetricsModuleMixin, B200VanillaMetricsModule):
    pass


@dataclass
class B200ScaleRegularizationWithDepthMetrics(B200ScaleRegularizationMetricsMixin, B200InverseDepthMetrics):
    def instantiate(self, *args, **kwargs) -> "B200ScaleRegularizationWithDepthMetricsModule":
        self._check()
        return B200ScaleRegularizationWithDepthMetricsModule(self)


class B200ScaleRegularizationWithDepthMetricsModule(B200ScaleRegularizationMetricsModuleMixin, B200InverseDepthMetricsModule):
    pass


# ---- VanillaWithNormalRegMetrics (internal/metrics/normal_reg.py) and gsplat.utils.depth_to_normal ------------------------------------
NORMAL_REG_FWD_LAUNCHES = 2     # library launches of one normal_consistency_loss forward: per-tile partials, reduce
NORMAL_REG_BWD_LAUNCHES = 1     # and of its backward


def _image_map(t, name):
    """[1,H,W] or [H,W] float32 CUDA -> detached contiguous [H,W] (a view when it already is one)"""
    if t.dim() == 3 and t.shape[0] == 1:
        t = t[0]
    if t.dim() != 2:
        raise ValueError(f"{name} must be [1, H, W] or [H, W], got {tuple(t.shape)}")
    if t.dtype != torch.float32 or not t.is_cuda:
        raise ValueError(f"{name} must be a float32 CUDA tensor")
    return t.detach().contiguous()


def _camera_matrix(t, rows, name, device):
    """[rows, rows] or [1, rows, rows] float32 on `device`, read in place through its strides"""
    if t.dim() == 3 and t.shape[0] == 1:
        t = t[0]
    if tuple(t.shape) != (rows, rows):
        raise ValueError(f"{name} must be [{rows}, {rows}] or [1, {rows}, {rows}], got {tuple(t.shape)}")
    if t.dtype != torch.float32 or t.device != device:
        raise ValueError(f"{name} must be float32 on {device}, got {t.dtype} on {t.device}")
    return t.detach()


class _NormalConsistencyLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, normal, depth, alpha, w2c, K, weight):
        H, W = depth.shape
        L = lib()
        nbytes = int(L.b200gs_normal_reg_workspace_bytes(H, W))
        ws = torch.empty(nbytes // 4, dtype=torch.float32, device=depth.device)
        loss = torch.empty((), dtype=torch.float32, device=depth.device)
        check(L.b200gs_normal_reg_fwd(H, W, ptr(normal), *normal.stride(), ptr(depth), ptr(alpha), ptr(w2c), *w2c.stride(), ptr(K), *K.stride(),
                                      weight, ptr(ws), nbytes, ptr(loss), _stream()), "b200gs_normal_reg_fwd")
        ctx.save_for_backward(depth, alpha, w2c, K, ws)
        return loss

    @staticmethod
    def backward(ctx, v_loss):
        depth, alpha, w2c, K, ws = ctx.saved_tensors
        H, W = depth.shape
        v = v_loss.reshape(1).to(torch.float32).contiguous()
        v_normal = torch.empty((3, H, W), dtype=torch.float32, device=depth.device)
        check(lib().b200gs_normal_reg_bwd(H, W, ptr(depth), ptr(alpha), ptr(w2c), w2c.stride(0), w2c.stride(1), ptr(K), K.stride(0),
                                          K.stride(1), ptr(ws), ws.numel() * 4, ptr(v), ptr(v_normal), _stream()), "b200gs_normal_reg_bwd")
        return v_normal, None, None, None, None, None


def normal_consistency_loss(normal, exp_depth, alpha, w2c, K, weight):
    """``NormalRegModuleMixin.get_normal_reg_metrics``' normal term of one view on K39/K40 (backward K41):
        weight mean(1 - sum_c normal[c] n_d[c]),   n_d = depth_to_normal(exp_depth, inv(w2c), K) * alpha
    normal float32 CUDA [3,H,W], read in place through its strides (the render's channel slice needs no copy); exp_depth and alpha
    [1,H,W] or [H,W], detached as the reference detaches them; w2c the world-to-camera matrix [4,4] or [1,4,4] and K [3,3] or
    [1,3,3], float32 on the same device, read there (the 3x3 block of w2c is inverted in the kernels: no torch.linalg.inv, no host
    synchronisation).  Returns a device scalar; the gradient goes to normal only, -weight / (H W) n_d."""
    if normal.dim() != 3 or normal.shape[0] != 3:
        raise ValueError(f"normal must be [3, H, W], got {tuple(normal.shape)}")
    if normal.dtype != torch.float32 or not normal.is_cuda:
        raise ValueError("normal must be a float32 CUDA tensor")
    depth, alpha = _image_map(exp_depth, "exp_depth"), _image_map(alpha, "alpha")
    if depth.shape != normal.shape[1:] or alpha.shape != depth.shape or depth.device != normal.device or alpha.device != normal.device:
        raise ValueError(f"normal {tuple(normal.shape)}, exp_depth {tuple(exp_depth.shape)} and alpha {tuple(alpha.shape)} must be one "
                         "image size on one device")
    w2c, K = _camera_matrix(w2c, 4, "w2c", normal.device), _camera_matrix(K, 3, "K", normal.device)
    return _NormalConsistencyLoss.apply(normal, depth, alpha, w2c, K, float(weight))


def depth_to_normal(depths, camtoworlds, Ks, z_depth: bool = True):
    """gsplat's ``utils.depth_to_normal`` for the call ``NormalRegModuleMixin`` makes, on K42: depths [H,W,1] (or [1,H,W,1]) of z
    depth, camtoworlds [4,4] and Ks [3,3] (or with a leading 1), float32 CUDA.  Returns the [H,W,3] (or [1,H,W,3]) map of
    normalize(cross(p[y+1,x] - p[y-1,x], p[y,x+1] - p[y,x-1])), 0 on the one-pixel border.  Not differentiable: depths that require
    grad raise NotImplementedError, and so does z_depth=False (ray distance)."""
    if not z_depth:
        raise NotImplementedError("depth_to_normal with z_depth=False is not provided")
    if depths.requires_grad:
        raise NotImplementedError("depth_to_normal has no backward: pass depths.detach()")
    batched = depths.dim() == 4
    d = depths[0] if batched and depths.shape[0] == 1 else depths
    if d.dim() != 3 or d.shape[-1] != 1:
        raise ValueError(f"depths must be [H, W, 1] or [1, H, W, 1], got {tuple(depths.shape)}")
    d = _image_map(d[..., 0], "depths")
    H, W = d.shape
    c2w, K = _camera_matrix(camtoworlds, 4, "camtoworlds", d.device), _camera_matrix(Ks, 3, "Ks", d.device)
    out = torch.empty((H, W, 3), dtype=torch.float32, device=d.device)
    check(lib().b200gs_depth_to_normal(H, W, ptr(d), ptr(c2w), c2w.stride(0), c2w.stride(1), ptr(K), K.stride(0), K.stride(1), ptr(out),
                                       _stream()), "b200gs_depth_to_normal")
    return out[None] if batched else out


_NORMAL_REG_OUTPUTS = ("exp_depth", "alpha", "normal", "preprocessed_camera")


@dataclass
class B200NormalRegMixin:
    normal_reg_lambda: float = 0.05

    flatten_reg: float = 0.02

    def instantiate(self, *args, **kwargs):
        raise NotImplementedError()


class B200NormalRegModuleMixin:
    """The depth-normal consistency and flatten terms, in training only: ``normal_loss`` = ``normal_consistency_loss`` of the render's
    ``normal``, ``exp_depth``, ``alpha`` and ``preprocessed_camera`` times ``normal_reg_lambda``, and ``flatten_loss`` =
    ``flatten_reg`` mean(get_scales()[..., -1]) (the last scale column, in torch).  Both are added to the loss; keys off the progress
    bar.  ``setup("fit")`` changes the model as the reference does: uniform random rotations and the last log-scale lowered by log 5,
    both from torch's global generator."""

    def setup(self, stage: str, pl_module):
        super().setup(stage, pl_module)
        if stage == "fit":
            with torch.no_grad():
                gaussians = pl_module.gaussian_model.gaussians
                gaussians["rotations"].copy_(torch.rand_like(gaussians["rotations"]))
                gaussians["scales"][..., -1] -= torch.log(torch.tensor(5., dtype=torch.float, device=gaussians["scales"].device))

    def get_normal_reg_metrics(self, gaussian_model, outputs, pl_module, metrics, pbar):
        missing = [k for k in _NORMAL_REG_OUTPUTS if outputs.get(k) is None]
        if missing:
            raise ValueError(f"the normal regulariser needs the render outputs {missing}: render with renderer_output_types "
                             "[rgb, alpha, exp_depth, normal] on a gsplat v1 renderer")
        w2c, K, _ = outputs["preprocessed_camera"]
        normal_loss = normal_consistency_loss(outputs["normal"], outputs["exp_depth"], outputs["alpha"], w2c[0], K[0],
                                              self.config.normal_reg_lambda)
        flatten_loss = gaussian_model.get_scales()[..., -1].mean() * self.config.flatten_reg

        metrics["loss"] = metrics["loss"] + normal_loss + flatten_loss
        metrics["normal_loss"] = normal_loss
        metrics["flatten_loss"] = flatten_loss
        pbar["normal_loss"] = False
        pbar["flatten_loss"] = False

    def get_train_metrics(self, pl_module, gaussian_model, step: int, batch, outputs):
        metrics, pbar = super().get_train_metrics(pl_module, gaussian_model, step, batch, outputs)
        self.get_normal_reg_metrics(gaussian_model, outputs, pl_module, metrics, pbar)
        return metrics, pbar


@dataclass
class B200VanillaWithNormalRegMetrics(B200NormalRegMixin, B200VanillaMetrics):
    def instantiate(self, *args, **kwargs) -> "B200VanillaWithNormalRegMetricsModule":
        self._check()
        return B200VanillaWithNormalRegMetricsModule(self)


class B200VanillaWithNormalRegMetricsModule(B200NormalRegModuleMixin, B200VanillaMetricsModule):
    pass


# ---- VanillaMetricsWithSimilarityRegularization (internal/metrics/appearance_feature_similarity_regularization_metrics.py) ------------
class Similarity:
    """The similarity of ``SimilarityRegularizationConfigMixin.similarity_type``; the term runs on ``ops.similarity_regularization``."""


@dataclass
class Cosine(Similarity):
    pass


@dataclass
class Euclidean(Similarity):
    pass


def _similarity_kind(similarity_type) -> str:
    """"cosine" or "euclidean" from the reference's Cosine() / Euclidean() objects, these classes, or {"class_path": "Cosine"}"""
    if isinstance(similarity_type, dict):
        name = str(similarity_type.get("class_path", "")).rsplit(".", 1)[-1]
    else:
        name = type(similarity_type).__name__
    if name not in ("Cosine", "Euclidean"):
        raise NotImplementedError(f"similarity_type {similarity_type!r}: only Cosine and Euclidean are provided")
    return name.lower()


@dataclass
class B200SimilarityRegularizationConfigMixin:
    n_appearance_samples: int = 20_480

    n_appearance_nn: int = 16

    distance_weight_decay: float = 200.
    """
    Used to decrease the weights with increasing distance.
    The value should be higher for smaller scenes.
    """

    similarity_reg_from: int = 0

    similarity_reg_lambda: float = 0.2

    similarity_reg_interval: int = 50

    similarity_type: Similarity = field(default_factory=lambda: {"class_path": "Cosine"})


class B200SimilarityRegularizationMixin:
    """Every ``similarity_reg_interval`` steps from ``similarity_reg_from`` on, after the main backward: ``n_appearance_samples``
    Gaussians drawn by ``torch.randperm``, their ``n_appearance_nn`` nearest Gaussians by ``ops.knn_points`` and the weighted
    similarity term by ``ops.similarity_regularization``, back-propagated into the appearance features with ``manual_backward``
    and logged as ``train/as_r``.  No host synchronisation on the way."""

    def get_similarity_metric(self, gaussian_model):
        """(loss, meta, knn_time) as the reference returns them.  meta has the reference's nine slots in its order: sample_indices,
        the KNN result ([1,S,K] dists and idx), None, distance_based_weight [S,K], None, None, triu_mask [K,K], None and the unscaled
        mean; the [S,K,K] intermediates are never formed.  knn_time is the host time of the k-NN call (the reference's time.time()
        difference, which does not wait for the device either)."""
        from .compat import KNN
        kind = _similarity_kind(self.config.similarity_type)
        started_at = time.time()
        with torch.no_grad():
            means = gaussian_model.get_means()
            sample_indices = torch.randperm(means.shape[0], device=means.device)[:self.config.n_appearance_samples]
            dists, idx = ops.knn_points(means[sample_indices], means, self.config.n_appearance_nn)
            knn_consumed_time = time.time() - started_at
        loss, mean, weights = ops.similarity_regularization(gaussian_model.get_appearance_features(), idx, dists,
                                                            decay=self.config.distance_weight_decay,
                                                            weight=self.config.similarity_reg_lambda, kind=kind)
        k = idx.shape[1]
        triu_mask = torch.triu(torch.ones((k, k), dtype=torch.bool, device=means.device), diagonal=1)
        return loss, (sample_indices, KNN(dists[None], idx[None], None), None, weights, None, None, triu_mask, None, mean), \
            knn_consumed_time

    def similarity_metric_backward_hook(self, outputs, batch, gaussian_model, step, pl_module):
        if step < self.config.similarity_reg_from:
            return
        if step % self.config.similarity_reg_interval != 0:
            return

        similarities_reg, meta, _ = self.get_similarity_metric(gaussian_model)
        pl_module.manual_backward(similarities_reg)
        pl_module.log("train/as_r", meta[-1], prog_bar=True, on_step=False, on_epoch=True, batch_size=pl_module.batch_size)

    def training_setup(self, pl_module):
        pl_module.on_after_backward_hooks.append(self.similarity_metric_backward_hook)
        return super().training_setup(pl_module)


@dataclass
class B200VanillaMetricsWithSimilarityRegularization(B200SimilarityRegularizationConfigMixin, B200VanillaMetrics):
    def instantiate(self, *args, **kwargs) -> "B200VanillaMetricsWithSimilarityRegularizationModule":
        self._check()
        _similarity_kind(self.similarity_type)
        return B200VanillaMetricsWithSimilarityRegularizationModule(self)


class B200VanillaMetricsWithSimilarityRegularizationModule(B200SimilarityRegularizationMixin, B200VanillaMetricsModule):
    pass
