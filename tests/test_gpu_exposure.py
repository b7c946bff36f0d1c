"""Exposure kernels (csrc/exposure.cu) on the GPU against the float64 oracle (oracle/exposure_oracle.py) and the reference's own
module (tests/golden/exposure.npz): output and all three gradients at 1080p, 800x800, the golden sizes and one-pixel-tall and
-wide images, in the contiguous [3,H,W] layout and as a permuted [H,W,3] view, for every with_bias x shade_correction
combination, with the appearance id on the device, on the host and as a Python int; the recorded module replayed through the
plug-in; state_dict round trips; bit-identical gradients; no host synchronisation; launch counts; out-of-range ids; and one
renderer -> processor -> loss chain against the same chain with the oracle's processor in fp32 torch."""
import json
import os
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import exposure_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
Z = np.load(os.path.join(GOLDEN, "exposure.npz"))
META = json.load(open(os.path.join(GOLDEN, "exposure.json")))
N_APP = 5
OPTIONS = [(False, False), (True, False), (False, True), (True, True)]       # (with_bias, shade_correction)


def layout(a, kind):
    """a float32 [3,H,W] array as a contiguous CUDA tensor ("chw") or as the permuted view of a contiguous [H,W,3] one ("hwc")"""
    t = torch.from_numpy(np.ascontiguousarray(a))
    if kind == "chw":
        return t.to(DEV)
    return t.permute(1, 2, 0).contiguous().to(DEV).permute(2, 0, 1)


def device_id(app_id, kind):
    if kind == "device":
        return torch.tensor(app_id, dtype=torch.int32, device=DEV)
    if kind == "host":
        return torch.tensor([app_id])
    return int(app_id)


def run(render, params, shade, app_id, v_out, with_bias):
    """(out, v_render, v_params, v_shade) of b200gs.exposure.exposure_correct as float64 numpy"""
    from b200gs.exposure import exposure_correct
    render = render.detach().requires_grad_(True)
    P = params.detach().clone().requires_grad_(True)
    S = None if shade is None else shade.detach().clone().requires_grad_(True)
    out = exposure_correct(render, P, app_id, S, max_gray_scale=5.0, max_gamma=5.0, with_bias=with_bias)
    assert out.stride() == render.stride()
    out.backward(v_out)
    torch.cuda.synchronize()
    f = lambda t: None if t is None else t.detach().cpu().double().numpy()      # noqa: E731
    return f(out), f(render.grad), f(P.grad), None if S is None else f(S.grad)


def rel(a, ref):
    return np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-30)


def check_against_oracle(H, W, with_bias, shade_size, kind, id_kind, app_id, seed):
    render, params, shade, v_out = O.inputs(H, W, with_bias, shade_size, seed, N_APP)
    out, v_render, v_params, v_shade = run(layout(render, kind), torch.from_numpy(params).to(DEV),
                                           None if shade is None else torch.from_numpy(shade).to(DEV), device_id(app_id, id_kind),
                                           layout(v_out, kind), with_bias)
    ref_out, ref_vr, ref_vp, ref_vs = O.vjp(render, params, app_id, shade, v_out, with_bias=with_bias)
    assert np.abs(out - ref_out).max() <= 1e-5
    # pixels scaled to within 1e-3 of 0 have a render gradient that float32 inputs fix only to about 1e-2 of itself
    # (O.near_zero); they are held to that, the others to 1e-4 of the largest magnitude
    near = O.near_zero(render, params, app_id, shade, with_bias=with_bias)
    assert near.mean() <= 0.01
    assert rel(v_render[~near], ref_vr[~near]) <= 1e-4
    assert (np.abs(v_render - ref_vr)[near] <= 2e-2 * np.abs(ref_vr[near]) + 1e-4 * np.abs(ref_vr[~near]).max()).all()
    assert rel(v_params[app_id], ref_vp[app_id]) <= 1e-4
    assert not v_params[[i for i in range(N_APP) if i != app_id]].any()
    if shade is not None:
        assert rel(v_shade, ref_vs) <= 1e-4


SIZES = [(1080, 1920), (800, 800), (37, 50), (11, 200), (1, 64), (48, 1)]
CASES = [(size, kind, opt) for size in SIZES for kind in ("chw", "hwc") for opt in OPTIONS]


@pytest.mark.parametrize("size,kind,opt", CASES, ids=[f"{h}x{w}-{k}-b{int(b)}c{int(c)}" for (h, w), k, (b, c) in CASES])
def test_matches_the_oracle(size, kind, opt):
    i = CASES.index((size, kind, opt))
    H, W = size
    with_bias, shade = opt
    check_against_oracle(H, W, with_bias, 128 if shade else 0, kind, ("device", "host", "int")[i % 3], (0, 2, 4, 3)[i % 4], seed=i)


@pytest.mark.parametrize("id_kind", ["device", "host", "int"])
@pytest.mark.parametrize("app_id", [0, 1, N_APP - 1])
def test_appearance_id_on_the_device_on_the_host_and_as_an_int(id_kind, app_id):
    check_against_oracle(37, 50, True, 24, "hwc", id_kind, app_id, seed=100 + app_id)


@pytest.mark.parametrize("case", META["cases"], ids=lambda c: c["key"])
def test_reference_module_replayed_through_the_plug_in(case):
    """The recorded ExposureProcessorModule outputs and gradients (float32 on the CPU) from B200ExposureProcessorModule with the
    same config, parameters, camera and cotangent."""
    from b200gs.exposure import B200ExposureProcessor
    H, W = case["image"]
    size = case["shade_correction_size"]
    render, params, shade, v_out = O.inputs(H, W, case["with_bias"], size if case["shade_correction"] else 0, case["seed"],
                                            META["n_appearances"])
    proc = B200ExposureProcessor(with_bias=case["with_bias"], shade_correction=case["shade_correction"],
                                 shade_correction_size=size).instantiate()
    proc.init_exposures(META["n_appearances"], DEV)
    with torch.no_grad():
        proc.exposure_parameters.copy_(torch.from_numpy(params))
        if shade is not None:
            proc.shade_correction.copy_(torch.from_numpy(shade))
    r = torch.from_numpy(render).to(DEV).requires_grad_(True)
    outputs = {"render": r}
    proc.training_forward((types.SimpleNamespace(appearance_id=torch.tensor(case["appearance_id"], device=DEV)),), outputs)
    outputs["render"].backward(torch.from_numpy(v_out).to(DEV))
    k = case["key"]
    assert np.abs(outputs["render"].detach().cpu().double().numpy() - Z[f"{k}_out"]).max() <= 1e-5
    assert rel(r.grad.cpu().double().numpy(), Z[f"{k}_v_render"]) <= 1e-4
    vp, ref_vp = proc.exposure_parameters.grad.cpu().double().numpy(), Z[f"{k}_v_params"]
    assert rel(vp, ref_vp) <= 1e-4
    assert not vp[[i for i in range(params.shape[0]) if i != case["appearance_id"]]].any()
    if shade is not None:
        assert rel(proc.shade_correction.grad.cpu().double().numpy(), Z[f"{k}_v_shade"]) <= 1e-4
    assert proc(types.SimpleNamespace(appearance_id=0), {}) is None          # no render: nothing to do


@pytest.mark.parametrize("with_bias", [False, True])
def test_reference_keyed_state_dict_round_trips(with_bias):
    from b200gs.exposure import B200ExposureProcessor
    k = f"b{int(with_bias)}_c1"
    sd = {n: torch.from_numpy(Z[f"sd_{k}_{n}"]).to(DEV) for n in META["state_dict"][k]}
    sd["exposure_parameters"] = sd["exposure_parameters"] + 0.25
    proc = B200ExposureProcessor(with_bias=with_bias, shade_correction=True, shade_correction_size=16).instantiate()
    proc.load_state_dict(sd)
    back = proc.state_dict()
    assert list(back) == list(META["state_dict"][k])
    assert all(torch.equal(back[n], sd[n]) for n in sd)
    assert back["exposure_parameters"].device.type == "cuda"


def test_two_backwards_give_bit_identical_gradients():
    render, params, shade, v_out = O.inputs(1080, 1920, True, 128, 7, N_APP)
    args = (layout(render, "hwc"), torch.from_numpy(params).to(DEV), torch.from_numpy(shade).to(DEV), device_id(3, "device"),
            layout(v_out, "hwc"), True)
    first, second = run(*args), run(*args)
    for a, b in zip(first, second):
        assert np.array_equal(a, b)


def test_no_host_synchronisation_and_launch_counts():
    from b200gs import _lib
    from b200gs.exposure import EXPOSURE_BWD_LAUNCHES, EXPOSURE_FWD_LAUNCHES, exposure_correct
    L = _lib.lib()
    render, params, shade, v_out = O.inputs(96, 128, True, 128, 3, N_APP)
    r = layout(render, "hwc").requires_grad_(True)
    P = torch.from_numpy(params).to(DEV).requires_grad_(True)
    S = torch.from_numpy(shade).to(DEV).requires_grad_(True)
    cot = layout(v_out, "hwc")
    app_id = torch.tensor(2, dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        n0 = L.b200gs_launch_count()
        out = exposure_correct(r, P, app_id, S, max_gray_scale=5.0, max_gamma=5.0, with_bias=True)
        n1 = L.b200gs_launch_count()
        out.backward(cot)
        n2 = L.b200gs_launch_count()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert (n1 - n0, n2 - n1) == (EXPOSURE_FWD_LAUNCHES, EXPOSURE_BWD_LAUNCHES) == (2, 3)
    assert torch.isfinite(r.grad).all() and torch.isfinite(P.grad).all() and torch.isfinite(S.grad).all()


@pytest.mark.parametrize("app_id", [N_APP, -1, 1 << 40])
@pytest.mark.parametrize("id_kind", ["device", "int"])
def test_out_of_range_id_gives_nan(app_id, id_kind):
    from b200gs.exposure import exposure_correct
    render, params, shade, v_out = O.inputs(37, 50, True, 16, 4, N_APP)
    r = layout(render, "chw").requires_grad_(True)
    P = torch.from_numpy(params).to(DEV).requires_grad_(True)
    S = torch.from_numpy(shade).to(DEV).requires_grad_(True)
    idx = torch.tensor(app_id, device=DEV) if id_kind == "device" else app_id
    out = exposure_correct(r, P, idx, S, max_gray_scale=5.0, max_gamma=5.0, with_bias=True)
    out.backward(layout(v_out, "chw"))
    assert torch.isnan(out).all() and torch.isnan(r.grad).all()
    assert not P.grad.any() and not S.grad.any()


def test_rejects_other_channel_counts():
    from b200gs.exposure import exposure_correct
    P = torch.zeros(2, 4, device=DEV)
    for C in (1, 4):
        with pytest.raises(ValueError):
            exposure_correct(torch.rand(C, 8, 8, device=DEV), P, 0, None, max_gray_scale=5.0, max_gamma=5.0, with_bias=False)
    with pytest.raises(ValueError):
        exposure_correct(torch.rand(3, 8, 8, device=DEV), P, 0, None, max_gray_scale=5.0, max_gamma=5.0, with_bias=True)


def test_renderer_processor_loss_chain_matches_the_torch_chain():
    """B200GSplatV1Renderer (permuted [H,W,3] render) -> processor -> ops.l1_ssim_loss -> backward: the Gaussian-parameter
    gradients match the same chain with the oracle's processor in fp32 torch within 1e-3 of each tensor's largest entry."""
    from b200gs import ops
    from b200gs.exposure import B200ExposureProcessor
    from b200gs.scene import SyntheticGaussians, make_ring_cameras, make_scene
    from b200gs.v1 import B200GSplatV1Renderer
    H, W = 192, 256
    cam = make_ring_cameras(W, H)[3].to_device(DEV)
    cam.appearance_id = torch.tensor(2, dtype=torch.int32, device=DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    renderer = B200GSplatV1Renderer().instantiate().to(DEV)
    _, params, shade, _ = O.inputs(H, W, True, 128, 11, N_APP)
    target = torch.rand(3, H, W, generator=torch.Generator().manual_seed(2)).to(DEV)
    proc = B200ExposureProcessor(with_bias=True, shade_correction=True).instantiate()
    proc.init_exposures(N_APP, DEV)
    with torch.no_grad():
        proc.exposure_parameters.copy_(torch.from_numpy(params))
        proc.shade_correction.copy_(torch.from_numpy(shade))

    def chain(processor):
        pc = SyntheticGaussians(make_scene(4096, 5, mean_scale=0.05)).to(DEV)
        outputs = renderer(cam, pc, bg)
        assert not outputs["render"].is_contiguous()            # the v1 renderer's permuted [H,W,3] image
        processor(outputs)
        loss, _ = ops.l1_ssim_loss(outputs["render"], target, 0.2)
        loss.backward()
        return {k: v.grad.detach().clone() for k, v in pc.gaussians.items()}

    fused = chain(lambda outputs: proc(cam, outputs))
    P, S = proc.exposure_parameters.detach(), proc.shade_correction.detach()
    torch_chain = chain(lambda outputs: outputs.update(render=O.forward(outputs["render"], P, 2, S, with_bias=True)))
    assert set(fused) == set(torch_chain)
    for k in fused:
        scale = float(torch_chain[k].abs().max())
        assert scale > 0, k
        assert float((fused[k] - torch_chain[k]).abs().max()) <= 1e-3 * scale, k
