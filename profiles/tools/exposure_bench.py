"""Per-view cost of the learned exposure correction: the fused kernels (b200gs.exposure.exposure_correct) against the reference's
torch formulation (ExposureProcessorModule.forward of internal/output_processors/exposure.py, restated below), alternated in one
process.  Forward and forward + backward at 1920x1080 and 800x800, for every with_bias x shade_correction combination (default
128x128 shade map), on the contiguous [3,H,W] render of the vanilla renderers and the permuted [H,W,3] view of the v1 renderers.
CUDA events around blocks of calls, each block queued behind a device-side sleep so the times are device times (the torch
formulation's indexing by a device tensor synchronises the host once per call, which is part of its cost); medians and min-max
over the blocks.  A separate torch.profiler run times each kernel of the fused path and sets it against the kernel's
algorithmic bytes and the 3.35 TB/s HBM3 data-sheet bound.  Prints one JSON line with the card's name and power limit.

    python profiles/tools/exposure_bench.py [--calls 200] [--block 10] [--warmup 20]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from b200gs.exposure import exposure_correct  # noqa: E402

HBM_PEAK = 3.35e12
# device-side sleep ahead of each block (cycles at ~2 GHz): longer than the host takes to enqueue the block, so the block runs
# back to back on the device.  The host side of a fused forward + backward (autograd, allocations, ctypes) costs more than its
# ~0.1 ms of kernels, so that block needs the longer one.
SLEEP_FWD, SLEEP_FWD_BWD = 10_000_000, 80_000_000
MAX_GRAY, MAX_GAMMA, SHADE = 5.0, 5.0, 128
N_APP = 16
OPTIONS = [(False, False), (True, False), (False, True), (True, True)]       # (with_bias, shade_correction)


def torch_exposure(render, params, appearance_id, shade, with_bias):
    """ExposureProcessorModule.forward on one render, as the reference evaluates it"""
    adjustment = torch.sigmoid(params[appearance_id])
    rendered_image = render
    if shade is not None:
        m = torch.sigmoid(shade[0][None, None, :, :])
        m = m / m.detach().max().clamp_min_(1e-4)
        m = F.interpolate(m, size=(render.shape[1], render.shape[2]), mode="bilinear", align_corners=True)[0]
        rendered_image = rendered_image * m
    rendered_image = adjustment[:3, None, None] * MAX_GRAY * rendered_image
    if with_bias:
        rendered_image = rendered_image + (adjustment[3:6, None, None] * 2. - 1.)
    with torch.no_grad():
        diff = rendered_image - torch.clamp(rendered_image, min=0., max=1.)
    rendered_image = rendered_image - diff
    return torch.pow(rendered_image + 1e-5, adjustment[-1] * MAX_GAMMA)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": name, "power_limit_w": float(out[0]), "sm_max_mhz": float(out[1])}
    except Exception as e:      # the number is then reported without it, and says so
        return {"gpu": name, "power_limit_w": "not measured", "sm_max_mhz": "not measured", "nvidia_smi": str(e)}


def time_paths(paths, args, sleep):
    for fn in paths.values():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in paths}
    for _ in range(args.calls // args.block):
        for k, fn in paths.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(sleep)
            a.record()
            for _ in range(args.block):
                fn()
            b.record()
            ms[k].append((a, b))
    torch.cuda.synchronize()
    per_call = {k: sorted(a.elapsed_time(b) / args.block for a, b in v) for k, v in ms.items()}
    return {k: v[len(v) // 2] for k, v in per_call.items()}, {k: [v[0], v[-1]] for k, v in per_call.items()}


def kernel_bytes(H, W, shade):
    """algorithmic bytes of each fused kernel (b200gs.h): the render and its gradients once, v_m once each way, the shade map"""
    P, s2 = H * W, (SHADE * SHADE if shade else 0)
    blocks = -(-W // 32) * -(-H // 8)
    return {"exposure_prep": 8 * s2, "exposure_fwd": 24 * P,
            "exposure_bwd": 36 * P + (4 * P if shade else 0) + 32 * blocks,
            "exposure_reduce": (4 * P + 8 * s2 if shade else 0) + 28 * blocks}


def kernel_times(fn, n):
    """mean device time (us) per call of each exposure kernel over n calls of fn, from a torch.profiler trace"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in ("exposure_prep", "exposure_fwd", "exposure_bwd", "exposure_reduce"):
            if k + "_kernel" in e.key:
                out[k] = out.get(k, 0.0) + e.device_time_total / n
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--block", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--profile-calls", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("exposure_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    gen = torch.Generator().manual_seed(0)
    results, kernels = [], []
    app_id = torch.tensor(5, dtype=torch.int32, device=dev)          # camera.appearance_id: a 0-d tensor on the device
    for H, W in ((1080, 1920), (800, 800)):
        for lay in ("chw", "hwc"):
            base = torch.rand(3, H, W, generator=gen).to(dev)
            render = (base if lay == "chw" else base.permute(1, 2, 0).contiguous().permute(2, 0, 1)).requires_grad_(True)
            cot = torch.rand(3, H, W, generator=gen).to(dev)
            for with_bias, shade_on in OPTIONS:
                params = (torch.randn(N_APP, 7 if with_bias else 4, generator=gen) * 0.3 - 1.0).to(dev).requires_grad_(True)
                shade = (torch.randn(1, SHADE, SHADE, generator=gen) * 0.3 + 2.9).to(dev).requires_grad_(True) if shade_on else None

                def fused():
                    return exposure_correct(render, params, app_id, shade, max_gray_scale=MAX_GRAY, max_gamma=MAX_GAMMA, with_bias=with_bias)

                def reference():
                    return torch_exposure(render, params, app_id, shade, with_bias)

                size = {"height": H, "width": W, "layout": lay, "with_bias": with_bias, "shade_correction": shade_on}
                with torch.no_grad():
                    med, spread = time_paths({"fused": fused, "torch": reference}, args, SLEEP_FWD)
                results.append({"what": "fwd", **size, **row(med, spread)})
                med, spread = time_paths({"fused": lambda: torch.autograd.backward(fused(), cot),
                                          "torch": lambda: torch.autograd.backward(reference(), cot)}, args, SLEEP_FWD_BWD)
                results.append({"what": "fwd_bwd", **size, **row(med, spread)})
                if lay == "chw":
                    us = kernel_times(lambda: torch.autograd.backward(fused(), cot), args.profile_calls)
                    nbytes = kernel_bytes(H, W, shade_on)
                    kernels.append({**size, "kernels": {k: {"us": round(t, 2), "algorithmic_MB": round(nbytes[k] / 1e6, 2),
                                                            "GB_per_s": round(nbytes[k] / (t * 1e-6) / 1e9, 1),
                                                            "share_of_hbm_bound": round(nbytes[k] / HBM_PEAK / (t * 1e-6), 3)}
                                                        for k, t in us.items()}})
                render.grad, params.grad = None, None
            del render, cot, base
    print(json.dumps({"metric": "exposure", "shade_size": SHADE, "hbm_peak_GBps": HBM_PEAK / 1e9, **card(), "results": results,
                      "fused_kernels_fwd_bwd": kernels}))


def row(med, spread):
    return {"fused_us": round(med["fused"] * 1e3, 2), "torch_us": round(med["torch"] * 1e3, 2),
            "speedup": round(med["torch"] / med["fused"], 2),
            "fused_us_min_max": [round(x * 1e3, 2) for x in spread["fused"]],
            "torch_us_min_max": [round(x * 1e3, 2) for x in spread["torch"]]}


if __name__ == "__main__":
    main()
