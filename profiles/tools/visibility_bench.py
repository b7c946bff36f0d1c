"""Per-view cost of the transient visibility map and its masked loss: the fused path (ops.uv_grid_encode, ops.visibility_mlp,
ops.visibility_l1_ssim_loss: K32, K20, K34 forward; K35, K21 + K22, K33 backward) against the reference's torch formulation
(Model.visibility_forward and VisibilityMapMetricsImpl.get_train_metrics: the [P,128] repeat, the meshgrid, the [P,144] concat, a
torch MLP, image and gt times the map, the reference's ssim.py SSIM), alternated in one process at 1920x1080 and 800x600, forward +
backward.  A third arm is the fused path with the visibility network in torch (cuBLAS) on the same folded [P,16] input, which
says whether K20/K21 pay off at this network shape.  tiny-cuda-nn is not installed, so the torch arm's grid is a STAND-IN: the oracle's corner indices and weights are
computed once on the host and each call gathers and weights the grid on the device; its time is not tiny-cuda-nn's.  CUDA
events around blocks of calls; medians and min-max over the blocks.  A separate torch.profiler run lists the fused path's kernel
times.  Prints one JSON line with the card's name and power limit.

    python profiles/tools/visibility_bench.py [--blocks 15] [--block 5] [--warmup 5] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

from b200gs import ops  # noqa: E402
from oracle import loss_oracle, visibility_oracle as V  # noqa: E402

SIZES = [(1920, 1080), (800, 600)]
N_IMAGES = 8
DEV = "cuda"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": name, "power_limit_w": float(out[0]), "sm_max_mhz": float(out[1])}
    except Exception as e:
        return {"gpu": name, "power_limit_w": "not measured", "sm_max_mhz": "not measured", "nvidia_smi": str(e)}


def state(W, H):
    g = torch.Generator().manual_seed(0)
    grids = [(torch.rand(V.n_params(), generator=g) * 2e-4 - 1e-4).to(DEV).requires_grad_(True) for _ in range(N_IMAGES)]
    emb = torch.nn.Embedding(N_IMAGES, 128).to(DEV)
    net = torch.nn.Sequential(torch.nn.Linear(144, 64), torch.nn.ReLU(), torch.nn.Linear(64, 64), torch.nn.ReLU(),
                              torch.nn.Linear(64, 1), torch.nn.Sigmoid()).to(DEV)
    image = torch.rand(3, H, W, generator=g).to(DEV).requires_grad_(True)
    gt = torch.rand(3, H, W, generator=g).to(DEV)
    u, v = V.pixel_uv(W, H)
    corners = [(i.to(DEV), w.float().to(DEV)) for i, w in V.corners(u, v, V.levels())]
    return grids, emb, net, image, gt, corners


def fused(W, H, st, app_id):
    grids, emb, net, image, gt, _ = st
    lin = [m for m in net if isinstance(m, torch.nn.Linear)]
    enc = ops.uv_grid_encode(grids, app_id, width=W, height=H, selected=3)
    vis = ops.visibility_mlp(enc, emb(app_id.reshape(-1))[0], [m.weight for m in lin], [m.bias for m in lin]).reshape(1, H, W)
    loss, _ = ops.visibility_l1_ssim_loss(image, gt, vis)
    loss.backward()


def folded_torch_mlp(W, H, st, app_id):
    """the fused path with the visibility network in torch (cuBLAS) on the same folded [P,16] input instead of K20/K21"""
    grids, emb, net, image, gt, _ = st
    lin = [m for m in net if isinstance(m, torch.nn.Linear)]
    enc = ops.uv_grid_encode(grids, app_id, width=W, height=H, selected=3)
    e = emb(app_id.reshape(-1))[0]
    h = torch.relu(enc @ lin[0].weight[:, :16].T + torch.addmv(lin[0].bias, lin[0].weight[:, 16:], e))
    h = torch.relu(lin[1](h))
    vis = torch.sigmoid(lin[2](h)).reshape(1, H, W)
    loss, _ = ops.visibility_l1_ssim_loss(image, gt, vis)
    loss.backward()


def reference(W, H, st, app_id):
    """Model.visibility_forward + VisibilityMapMetricsImpl.get_train_metrics as the reference evaluates them (grid: stand-in)"""
    grids, emb, net, image, gt, corners = st
    n = W * H
    transient = emb(app_id.reshape((-1,))).repeat(n, 1)
    gx, gy = torch.meshgrid(torch.arange(W, dtype=torch.float, device=DEV), torch.arange(H, dtype=torch.float, device=DEV), indexing="xy")
    _ = torch.concat([gx.unsqueeze(-1) / (W - 1), gy.unsqueeze(-1) / (H - 1)], dim=-1).reshape((-1, 2))
    table = grids[app_id.item()].reshape(-1, 2)
    enc = torch.cat([(table[i] * w.unsqueeze(-1)).sum(1) for i, w in corners], dim=1)
    vis = net(torch.concat([enc, transient], dim=-1)).reshape(H, W).unsqueeze(0)
    a, b = image * vis, gt * vis
    loss = 0.8 * (a - b).abs().mean() + 0.2 * (1. - torch_ssim(a, b))
    loss = loss + ((1. - vis) ** 2).mean() * 0.2
    loss.backward()


def torch_ssim(img1, img2):
    """the reference's internal/utils/ssim.py on a [3,H,W] pair: 11x11 Gaussian window (outer product), zero padding"""
    w1 = loss_oracle.window_1d().to(img1.device)
    win = (w1[:, None] @ w1[None, :]).expand(3, 1, 11, 11).contiguous()
    conv = lambda x: torch.nn.functional.conv2d(x, win, padding=5, groups=3)      # noqa: E731
    mu1, mu2 = conv(img1), conv(img2)
    mu1_sq, mu2_sq, mu1_mu2 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1, s2, s12 = conv(img1 * img1) - mu1_sq, conv(img2 * img2) - mu2_sq, conv(img1 * img2) - mu1_mu2
    c1, c2 = loss_oracle.C1, loss_oracle.C2
    return (((2 * mu1_mu2 + c1) * (2 * s12 + c2)) / ((mu1_sq + mu2_sq + c1) * (s1 + s2 + c2))).mean()


def timed(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=15)
    ap.add_argument("--block", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    app_id = torch.tensor([3], device=DEV)
    result = {"card": card(), "note": "reference arm: torch formulation with the oracle's grid standing in for tiny-cuda-nn "
                                      "(not tiny-cuda-nn's timing); forward + backward per call, ms", "sizes": {}}
    for W, H in SIZES:
        st = state(W, H)
        arms = {"fused": lambda: fused(W, H, st, app_id), "torch_reference": lambda: reference(W, H, st, app_id),
                "fused_with_torch_mlp": lambda: folded_torch_mlp(W, H, st, app_id)}
        for fn in arms.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for _ in range(args.blocks):
            for k, fn in arms.items():
                times[k].append(timed(fn, args.block))
        res = {}
        for k, t in times.items():
            t = sorted(t)
            res[k] = {"median_ms": t[len(t) // 2], "min_ms": t[0], "max_ms": t[-1]}
        res["speedup"] = res["torch_reference"]["median_ms"] / res["fused"]["median_ms"]
        res["speedup_vs_torch_mlp"] = res["fused_with_torch_mlp"]["median_ms"] / res["fused"]["median_ms"]
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fused(W, H, st, app_id)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            if e.device_type == torch.autograd.DeviceType.CUDA and e.count > 0:
                kern[e.key[:60]] = round(e.device_time_total / e.count / 1000.0, 4)        # ms per launch
        res["fused_kernels_ms"] = dict(sorted(kern.items(), key=lambda kv: -kv[1])[:12])
        result["sizes"][f"{W}x{H}"] = res
        del st
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "visibility_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
