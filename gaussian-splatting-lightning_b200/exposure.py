"""Learned exposure correction (the reference's ``configs/learn_exposure*.yaml``, internal/output_processors/exposure.py) on the
b200gs kernels.  Select it as the model's output processor:

    model:
      output_processor:
        class_path: b200gs.exposure.B200ExposureProcessor
        init_args: {with_bias: true, shade_correction: true}

``B200ExposureProcessor`` has ``ExposureProcessor``'s config fields, defaults and ``instantiate()`` checks;
``B200ExposureProcessorModule`` has ``ExposureProcessorModule``'s methods, initial values, optimizer groups and ``state_dict`` keys
(``exposure_parameters``, ``shade_correction``), so checkpoints load both ways.  Its ``forward`` runs ``exposure_correct``: two
kernel launches forward and three backward, the appearance id read on the device, no host synchronisation.  The exposure
parameters' Adam step stays torch.
"""
from dataclasses import dataclass

import torch

from ._lib import check, lib, ptr
from .bilagrid import _same_layout
from .ops import _stream

try:  # inside the reference repo: subclass its config base so the trainer's type checks hold
    from internal.output_processors.output_processors import OutputProcessor  # type: ignore
except Exception:
    @dataclass
    class OutputProcessor:
        pass

EXPOSURE_FWD_LAUNCHES = 2       # library launches of one exposure_correct forward: the prologue and the pixel pass
EXPOSURE_BWD_LAUNCHES = 3       # and of its backward: the prologue, the pixel pass and the reduction


def _appearance_id(appearance_id, device):
    """(int64 [1] device tensor or None, host id): a CUDA tensor is read by the kernels, a CPU tensor or int on the host."""
    if isinstance(appearance_id, torch.Tensor):
        if appearance_id.numel() != 1 or appearance_id.is_floating_point() or appearance_id.is_complex():
            raise ValueError(f"appearance_id must be one integer, got {appearance_id.dtype} of shape {tuple(appearance_id.shape)}")
        if appearance_id.is_cuda:
            return appearance_id.reshape(1).to(device=device, dtype=torch.int64), 0
        return None, int(appearance_id.reshape(()))
    return None, int(appearance_id)


class _ExposureCorrect(torch.autograd.Function):
    @staticmethod
    def forward(ctx, render, params, shade, id_dev, host_id, max_gray, max_gamma):
        C, H, W = render.shape
        s = 0 if shade is None else shade.shape[-1]
        out = torch.empty_like(render)
        if not _same_layout(out, render):       # not a dense layout: the kernels read and write one set of strides
            render = render.contiguous()
            out = torch.empty_like(render)
        L = lib()
        nbytes = int(L.b200gs_exposure_workspace_bytes(H, W, s, 0))
        ws = torch.empty(nbytes // 4, dtype=torch.float32, device=render.device)
        check(L.b200gs_exposure_fwd(C, H, W, ptr(render), *render.stride(), params.shape[0], params.shape[1], ptr(params), ptr(id_dev),
                                    host_id, s, ptr(shade), max_gray, max_gamma, ptr(ws), nbytes, ptr(out), _stream()),
              "b200gs_exposure_fwd")
        ctx.save_for_backward(render, params, shade, id_dev)
        ctx.host_id, ctx.max_gray, ctx.max_gamma = host_id, max_gray, max_gamma
        return out

    @staticmethod
    def backward(ctx, v_out):
        render, params, shade, id_dev = ctx.saved_tensors
        C, H, W = render.shape
        s = 0 if shade is None else shade.shape[-1]
        if v_out.dtype != torch.float32 or not _same_layout(v_out, render):
            v_out = torch.empty_like(render).copy_(v_out)
        v_render = torch.empty_like(render)
        v_params = torch.empty_like(params)
        # the kernels write the gradient of shade[0], the only map the reference uses
        v_shade = None if shade is None else (torch.empty_like(shade) if shade.shape[0] == 1 else torch.zeros_like(shade))
        L = lib()
        nbytes = int(L.b200gs_exposure_workspace_bytes(H, W, s, 1))
        ws = torch.empty(nbytes // 4, dtype=torch.float32, device=render.device)
        check(L.b200gs_exposure_bwd(C, H, W, ptr(render), *render.stride(), params.shape[0], params.shape[1], ptr(params), ptr(id_dev),
                                    ctx.host_id, s, ptr(shade), ctx.max_gray, ctx.max_gamma, ptr(ws), nbytes, ptr(v_out), ptr(v_render),
                                    ptr(v_params), ptr(v_shade), _stream()), "b200gs_exposure_bwd")
        return v_render, v_params, v_shade, None, None, None, None


def exposure_correct(render, exposure_parameters, appearance_id, shade, *, max_gray_scale, max_gamma, with_bias):
    """``ExposureProcessorModule.forward``'s transform of one render [3,H,W]: with a = sigmoid(exposure_parameters[appearance_id]),
    out = (clamp((a[:3] max_gray_scale) (render m) [+ 2 a[3:6] - 1], 0, 1) + 1e-5) ^ (a[-1] max_gamma), the clamp straight
    through, m the bilinear (align_corners) upsampling of sigmoid(shade[0]) / max(max(sigmoid(shade[0])), 1e-4) (shade None: 1).
    ``appearance_id`` is an int, a CPU tensor or a one-element CUDA tensor (read on the device); an id outside the parameter rows
    gives a NaN image.  The output is laid out like ``render`` (a permuted view of an [H,W,3] image gives the same permuted view)."""
    if render.dim() != 3 or render.shape[0] != 3:
        raise ValueError(f"exposure_correct takes a [3, H, W] render, got {tuple(render.shape)}")
    n_params = 7 if with_bias else 4
    if exposure_parameters.dim() != 2 or exposure_parameters.shape[1] != n_params:
        raise ValueError(f"exposure_parameters must be [n_appearances, {n_params}] with with_bias={with_bias}, "
                         f"got {tuple(exposure_parameters.shape)}")
    tensors = [render, exposure_parameters] + ([] if shade is None else [shade])
    if any(t.dtype != torch.float32 or not t.is_cuda for t in tensors):
        raise ValueError("render, exposure_parameters and shade must be float32 CUDA tensors")
    if shade is not None and (shade.dim() != 3 or shade.shape[1] != shade.shape[2]):
        raise ValueError(f"shade must be [n_cameras, s, s], got {tuple(shade.shape)}")
    id_dev, host_id = _appearance_id(appearance_id, render.device)
    return _ExposureCorrect.apply(render, exposure_parameters.contiguous(), None if shade is None else shade.contiguous(), id_dev,
                                  host_id, float(max_gray_scale), float(max_gamma))


def _inverse_sigmoid(x):
    return torch.log(x / (1 - x))


@dataclass
class B200ExposureProcessor(OutputProcessor):
    lr_init: float = 1e-2

    lr_final_factor: float = 0.1

    max_steps: int = 30_000

    max_gray_scale: float = 5.

    with_bias: bool = False

    max_gamma: float = 5.

    shade_correction: bool = False

    shade_correction_size: int = 128

    def instantiate(self, *args, **kwargs):
        # configs saved before these fields existed
        if not hasattr(self, "with_bias"):
            self.with_bias = False
        if not hasattr(self, "shade_correction"):
            self.shade_correction = False

        # must be > 1 or the optimisation does not work
        assert self.max_gray_scale > 1.
        assert self.max_gamma > 1.
        return B200ExposureProcessorModule(self)


class B200ExposureProcessorModule(torch.nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config

    def init_exposures(self, n_appearances: int, device, n_cameras: int = 1):
        c = self.config
        n_parameters = 7 if c.with_bias else 4
        exposures = torch.full((n_appearances, n_parameters),
                               _inverse_sigmoid(torch.tensor(1. / c.max_gray_scale, dtype=torch.float32, device=device)),
                               dtype=torch.float32, device=device)
        exposures[:, -1] = _inverse_sigmoid(torch.tensor(1. / c.max_gamma, dtype=torch.float32, device=device))
        if c.with_bias:
            # bias = sigmoid(x) * 2 - 1 = 0
            exposures[:, 3:6].fill_(_inverse_sigmoid(torch.tensor(0.5, dtype=torch.float32, device=device)))
            assert torch.allclose(torch.sigmoid(exposures[:, 3:6]) * 2. - 1., torch.tensor(0., device=device))
        assert torch.allclose(torch.sigmoid(exposures[:, :3]) * c.max_gray_scale, torch.tensor(1., device=device))
        assert torch.allclose(torch.sigmoid(exposures[:, -1]) * c.max_gamma, torch.tensor(1., device=device))
        self.exposure_parameters = torch.nn.Parameter(exposures, requires_grad=True)

        if c.shade_correction:
            # one map, shade_correction[0], is used for every camera, as in the reference
            self.shade_correction = torch.nn.Parameter(
                torch.full(size=(n_cameras, c.shade_correction_size, c.shade_correction_size),
                           fill_value=_inverse_sigmoid(torch.tensor(0.95, device=device)), device=device),
                requires_grad=True)

    def setup(self, stage: str, pl_module=None, *args, **kwargs):
        if pl_module is not None:
            max_input_id = 0
            appearance_group_ids = pl_module.trainer.datamodule.dataparser_outputs.appearance_group_ids
            if appearance_group_ids is not None:
                for i in appearance_group_ids.values():
                    if i[0] > max_input_id:
                        max_input_id = i[0]
            n_appearances = max_input_id + 1
            assert n_appearances > 1

            self.init_exposures(n_appearances, pl_module.device)

            print("{} exposure groups".format(n_appearances))

    def load_state_dict(self, state_dict, strict=True):
        n_appearances = state_dict["exposure_parameters"].shape[0]
        self.init_exposures(n_appearances, state_dict["exposure_parameters"].device)
        return super().load_state_dict(state_dict, strict)

    def training_setup(self, pl_module):
        params = [{"params": [self.exposure_parameters], "name": "exposure"}]
        if self.config.shade_correction:
            params.append({"params": [self.shade_correction], "name": "shade"})
        optimizer = torch.optim.Adam(params=params, lr=self.config.lr_init)
        return optimizer, torch.optim.lr_scheduler.LambdaLR(
            optimizer=optimizer, lr_lambda=lambda it: self.config.lr_final_factor ** min(it / self.config.max_steps, 1))

    def forward(self, camera, outputs) -> None:
        if "render" not in outputs:
            return
        c = self.config
        outputs["render"] = exposure_correct(outputs["render"], self.exposure_parameters, camera.appearance_id,
                                             self.shade_correction if c.shade_correction else None, max_gray_scale=c.max_gray_scale,
                                             max_gamma=c.max_gamma, with_bias=c.with_bias)

    def training_forward(self, batch, outputs):
        return self(batch[0], outputs)
