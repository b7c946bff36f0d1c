"""Per-step cost of the 3DGS-MCMC position noise: the fused kernel (b200gs.mcmc.add_position_noise) against the reference's torch
formula (mcmc_density_controller.py:93-120 with compute_cov_3d of gaussian_projection.py:211-254, restated below), on the
benchmark's scene law make_scene(N, 0) at N = 1 M and 3 M.  CUDA events around blocks of calls, the two paths alternated in one
process; each block is queued behind a device-side sleep, so the times are device times, not the
host's launch rate.  Prints one JSON line with both times, the fused kernel's achieved bandwidth on its 56 algorithmic bytes per Gaussian
against the 3.35 TB/s HBM3 data-sheet peak, and the card's name and power limit read in the same run.

    python profiles/tools/mcmc_noise_bench.py [--sizes 1000000,3000000] [--calls 200] [--block 10] [--warmup 20]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

from b200gs.mcmc import add_position_noise  # noqa: E402
from b200gs.scene import make_scene  # noqa: E402

NOISE_LR, XYZ_LR = 5e5, 1.6e-4        # the controller's default noise_lr; the reference's initial position lr
BYTES_PER_GAUSSIAN = 12 + 12 + 16 + 4 + 12     # means, log-scales, quaternion, opacity logit in; means out
HBM_PEAK = 3.35e12
SLEEP_CYCLES = 10_000_000          # ~5 ms at 2 GHz, longer than the host takes to enqueue one block of either path


def torch_noise(means, log_scales, raw_quats, opacity_logits):
    """The reference's _add_xyz_noise on the model getters' activations, op for op."""
    scales = torch.exp(log_scales)
    q = torch.nn.functional.normalize(raw_quats)
    opacities = torch.sigmoid(opacity_logits)
    n = scales.shape[0]
    S = torch.zeros((n, 3, 3), dtype=scales.dtype, device=scales.device)
    for i in range(3):
        S[:, i, i] = scales[:, i] * 1.0
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.zeros((n, 3, 3), dtype=q.dtype, device=q.device)
    R[:, 0, 0] = 1 - 2 * (y * y + z * z)
    R[:, 0, 1] = 2 * (x * y - r * z)
    R[:, 0, 2] = 2 * (x * z + r * y)
    R[:, 1, 0] = 2 * (x * y + r * z)
    R[:, 1, 1] = 1 - 2 * (x * x + z * z)
    R[:, 1, 2] = 2 * (y * z - r * x)
    R[:, 2, 0] = 2 * (x * z - r * y)
    R[:, 2, 1] = 2 * (y * z + r * x)
    R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    m = torch.bmm(R, S)
    cov = torch.matmul(m, m.transpose(1, 2))
    w = 1 / (1 + torch.exp(-100 * ((1 - opacities) - 0.995)))
    noise = torch.randn_like(means) * w * NOISE_LR * XYZ_LR
    noise = torch.bmm(cov, noise.unsqueeze(-1)).squeeze(-1)
    means.add_(noise)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": name, "power_limit_w": float(out[0]), "sm_max_mhz": float(out[1])}
    except Exception as e:      # the number is then reported without it, and says so
        return {"gpu": name, "power_limit_w": "not measured", "sm_max_mhz": "not measured", "nvidia_smi": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,3000000")
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--block", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mcmc_noise_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    results = []
    for n in (int(s) for s in args.sizes.split(",")):
        raw = {k: v.to(dev) for k, v in make_scene(n, 0).items()}
        operands = (raw["means"], raw["scales"], raw["rotations"], raw["opacities"])
        paths = {"fused": lambda: add_position_noise(*operands, NOISE_LR, XYZ_LR), "torch": lambda: torch_noise(*operands)}
        for fn in paths.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in paths}
        for _ in range(args.calls // args.block):
            for k, fn in paths.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda._sleep(SLEEP_CYCLES)   # the host enqueues the whole block meanwhile: the events time the device work
                a.record()
                for _ in range(args.block):
                    fn()
                b.record()
                ms[k].append((a, b))
        torch.cuda.synchronize()
        per_call = {k: sorted(a.elapsed_time(b) / args.block for a, b in v) for k, v in ms.items()}
        med = {k: v[len(v) // 2] for k, v in per_call.items()}
        gbps = n * BYTES_PER_GAUSSIAN / (med["fused"] * 1e-3) / 1e9
        results.append({"n": n, "calls_each": len(ms["fused"]) * args.block, "fused_us": round(med["fused"] * 1e3, 2),
                        "torch_us": round(med["torch"] * 1e3, 2), "speedup": round(med["torch"] / med["fused"], 1),
                        "fused_algorithmic_GBps": round(gbps, 1), "fused_share_of_hbm_peak": round(gbps * 1e9 / HBM_PEAK, 3),
                        "fused_us_min_max": [round(per_call["fused"][0] * 1e3, 2), round(per_call["fused"][-1] * 1e3, 2)],
                        "torch_us_min_max": [round(per_call["torch"][0] * 1e3, 2), round(per_call["torch"][-1] * 1e3, 2)]})
        del raw, operands, paths
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "mcmc_position_noise", "bytes_per_gaussian": BYTES_PER_GAUSSIAN, "hbm_peak_GBps": HBM_PEAK / 1e9,
                      **card(), "results": results}))


if __name__ == "__main__":
    main()
