"""Per-step cost of the bilateral-grid colour correction: the fused kernels (b200gs.bilagrid) against a torch formulation on
F.grid_sample (restated below from the contract of internal/utils/lib_bilagrid.py, including its torch.unique of the grid index),
alternated in one process.  Slice forward and forward + backward at 1920x1080 and 800x800 with the default 16x16x8 grid (the
processor's permuted CHW render); total variation forward + backward at N = 1, 64 and 512 grids.  CUDA events around blocks of
calls, each block queued behind a device-side sleep, so the times are device times.  Prints one JSON line with both times, the
fused path's algorithmic bytes and its share of the 3.35 TB/s HBM3 data-sheet bound, and the card's name and power limit read in
the same run.

    python profiles/tools/bilagrid_bench.py [--calls 200] [--block 10] [--warmup 20]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from b200gs import bilagrid  # noqa: E402

HBM_PEAK = 3.35e12
SLEEP_CYCLES = 10_000_000          # ~5 ms at 2 GHz, longer than the host takes to enqueue one block of either path
GRID = (16, 16, 8)                 # grid_X, grid_Y, grid_W: the processor's defaults
N_GRIDS = 8


def torch_slice(grids, xy, rgb, grid_idx):
    """slice(...)["rgb"] on grid_sample(align_corners=True, padding_mode='border') for one image, as lib_bilagrid evaluates it"""
    idx = torch.unique(grid_idx)                                            # the reference's host sync
    w = torch.tensor([[0.299, 0.587, 0.114]], device=rgb.device)
    z = (rgb @ w.T) * 2.0 - 1.0
    coords = torch.cat([(xy - 0.5) * 2, z], dim=-1).unsqueeze(0)             # [1, 1, H, W, 3]
    A = F.grid_sample(grids[idx], coords, mode="bilinear", align_corners=True, padding_mode="border")
    A = A.permute(0, 2, 3, 4, 1).reshape(*rgb.shape[:-1], 3, 4)
    return torch.matmul(A[..., :3], rgb.unsqueeze(-1)).squeeze(-1) + A[..., 3]


def torch_tv(x):
    tv = 0
    for i in range(2, x.dim()):
        n = x.shape[i]
        d = x.index_select(i, torch.arange(1, n, device=x.device)) - x.index_select(i, torch.arange(0, n - 1, device=x.device))
        tv = tv + d.pow(2).sum() / max(float(torch.tensor(d.shape[1:]).prod()), 1.0)
    return tv / x.shape[0]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": name, "power_limit_w": float(out[0]), "sm_max_mhz": float(out[1])}
    except Exception as e:      # the number is then reported without it, and says so
        return {"gpu": name, "power_limit_w": "not measured", "sm_max_mhz": "not measured", "nvidia_smi": str(e)}


def time_paths(paths, args):
    for fn in paths.values():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in paths}
    for _ in range(args.calls // args.block):
        for k, fn in paths.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(SLEEP_CYCLES)
            a.record()
            for _ in range(args.block):
                fn()
            b.record()
            ms[k].append((a, b))
    torch.cuda.synchronize()
    per_call = {k: sorted(a.elapsed_time(b) / args.block for a, b in v) for k, v in ms.items()}
    return {k: v[len(v) // 2] for k, v in per_call.items()}, {k: [v[0], v[-1]] for k, v in per_call.items()}


def entry(what, size, med, spread, nbytes):
    share = nbytes / HBM_PEAK / (med["fused"] * 1e-3)
    return {"what": what, **size, "fused_us": round(med["fused"] * 1e3, 2), "torch_us": round(med["torch"] * 1e3, 2),
            "speedup": round(med["torch"] / med["fused"], 2), "fused_algorithmic_MB": round(nbytes / 1e6, 2),
            "fused_share_of_hbm_bound": round(share, 3),
            "fused_us_min_max": [round(x * 1e3, 2) for x in spread["fused"]],
            "torch_us_min_max": [round(x * 1e3, 2) for x in spread["torch"]]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--block", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bilagrid_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    gen = torch.Generator().manual_seed(0)
    results = []
    bg = bilagrid.BilateralGrid(N_GRIDS, *GRID)
    with torch.no_grad():
        bg.grids.add_(0.1 * torch.randn(bg.grids.shape, generator=gen))
    bg = bg.to(dev)
    grid_bytes = bg.grids[0].numel() * 4
    for H, W in ((1080, 1920), (800, 800)):
        gy, gx = torch.meshgrid(torch.linspace(0, 1., H, device=dev), torch.linspace(0, 1., W, device=dev), indexing="ij")
        xy = torch.stack([gx, gy], dim=-1).unsqueeze(0)
        render = torch.rand(3, H, W, generator=gen).to(dev).requires_grad_(True)
        cot = torch.rand(3, H, W, generator=gen).to(dev)
        idx = torch.tensor(3, device=dev)[None, None]
        P = H * W

        def fused():
            return bilagrid.slice(bg, xy, render.permute(1, 2, 0).unsqueeze(0), idx)["rgb"].squeeze(0).permute(2, 0, 1)

        def reference():
            return torch_slice(bg.grids, xy, render.permute(1, 2, 0).unsqueeze(0), idx).squeeze(0).permute(2, 0, 1)

        with torch.no_grad():
            med, spread = time_paths({"fused": fused, "torch": reference}, args)
        results.append(entry("slice_fwd", {"height": H, "width": W}, med, spread, P * (8 + 12 + 12) + grid_bytes))
        med, spread = time_paths({"fused": lambda: torch.autograd.backward(fused(), cot),
                                  "torch": lambda: torch.autograd.backward(reference(), cot)}, args)
        results.append(entry("slice_fwd_bwd", {"height": H, "width": W}, med, spread,
                             P * (8 + 12 + 12) + P * (8 + 12 + 12 + 12) + 3 * grid_bytes))
        bg.grids.grad = None
        del render, cot, xy
    for n in (1, 64, 512):
        grids = (torch.randn(n, 12, GRID[2], GRID[1], GRID[0], generator=gen) * 0.1).to(dev).requires_grad_(True)
        med, spread = time_paths({"fused": lambda: bilagrid.total_variation_loss(grids).backward(),
                                  "torch": lambda: torch_tv(grids).backward()}, args)
        results.append(entry("tv_fwd_bwd", {"n_grids": n}, med, spread, grids.numel() * 4 * 3))
    print(json.dumps({"metric": "bilagrid", "grid": list(GRID), "hbm_peak_GBps": HBM_PEAK / 1e9, **card(), "results": results}))


if __name__ == "__main__":
    main()
