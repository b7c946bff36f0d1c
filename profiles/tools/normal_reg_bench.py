"""Per-step cost of the depth-normal consistency term: the fused kernels (b200gs.metrics.normal_consistency_loss, K39-K41) against
the reference's torch chain (NormalRegModuleMixin.get_normal_reg_metrics of internal/metrics/normal_reg.py with gsplat's
depth_to_normal, restated below: torch.linalg.inv of the camera, the ray grid, points, differences, cross product, normalisation,
padding, the alpha multiply, the dot product and the mean), alternated in one process, at 1920x1080 and 800x800, forward and
forward + backward.  The normal map is a channel slice of a permuted [H,W,7] render, as the gsplat v1 renderer produces it.  Also
timed: the flatten term (mean of the last scale column, torch in both arms) at 1 M Gaussians, forward + backward.
Timing as profiles/tools/exposure_bench.py: CUDA events around blocks of calls behind a device-side sleep, medians and min-max over
the blocks; kernel times from a separate torch.profiler run against each kernel's algorithmic bytes; the card's name and power
limit read in the same call.  Prints one JSON line.

    python profiles/tools/normal_reg_bench.py [--calls 200] [--block 10] [--warmup 20]
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from b200gs.metrics import normal_consistency_loss  # noqa: E402
from exposure_bench import HBM_PEAK, SLEEP_FWD, SLEEP_FWD_BWD, card, row, time_paths  # noqa: E402

KERNELS = ("normal_reg_partials", "normal_reg_reduce", "normal_reg_bwd")
LAMBDA, FLATTEN = 0.05, 0.02


def torch_depth_to_normal(depths, camtoworlds, Ks):
    """gsplat utils.depth_to_normal (z_depth) as the reference calls it: [H,W,1] depths -> [H,W,3]"""
    height, width = depths.shape[-3:-1]
    x, y = torch.meshgrid(torch.arange(width, device=depths.device), torch.arange(height, device=depths.device), indexing="xy")
    fx, fy, cx, cy = Ks[..., 0, 0], Ks[..., 1, 1], Ks[..., 0, 2], Ks[..., 1, 2]
    camera_dirs = F.pad(torch.stack([(x - cx + 0.5) / fx, (y - cy + 0.5) / fy], dim=-1), (0, 1), value=1.0)
    directions = torch.einsum("...ij,...hwj->...hwi", camtoworlds[..., :3, :3], camera_dirs)
    points = camtoworlds[..., :3, -1] + depths * directions
    dx = torch.cat([points[..., 2:, 1:-1, :] - points[..., :-2, 1:-1, :]], dim=-3)
    dy = torch.cat([points[..., 1:-1, 2:, :] - points[..., 1:-1, :-2, :]], dim=-2)
    normals = F.normalize(torch.cross(dx, dy, dim=-1), dim=-1)
    return F.pad(normals, (0, 0, 1, 1, 1, 1), value=0.0)


def torch_normal_loss(normal, exp_depth, alpha, w2c, K):
    n_d = torch_depth_to_normal(exp_depth.detach().permute(1, 2, 0), torch.linalg.inv(w2c[0]), K[0]).permute(2, 0, 1) * alpha.squeeze(0).detach()
    return (1 - (normal * n_d).sum(dim=0)).mean() * LAMBDA


def kernel_bytes(H, W):
    """algorithmic bytes (b200gs.h): depth, alpha and the three normal channels in; the backward writes v_normal; partials"""
    P, tiles = H * W, -(-H // 16) * -(-W // 16)
    return {"normal_reg_partials": 20 * P + 4 * tiles, "normal_reg_reduce": 4 * tiles, "normal_reg_bwd": 20 * P}


def kernel_times(fn, n):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in KERNELS:
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
        sys.exit("normal_reg_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    gen = torch.Generator().manual_seed(0)
    results, kernels = [], []
    for H, W in ((1080, 1920), (800, 800)):
        feats = torch.rand(H, W, 7, generator=gen).to(dev).requires_grad_(True)
        normal = feats.permute(2, 0, 1)[4:7]
        exp_depth = (1 + 4 * torch.rand(1, H, W, generator=gen)).to(dev)
        alpha = torch.rand(1, H, W, generator=gen).to(dev)
        w2c = torch.eye(4)
        w2c[:3, 3] = torch.tensor([0.3, -0.2, 2.0])
        w2c = w2c.T.contiguous().to(dev).T.unsqueeze(0)        # the renderer's viewmats: world_to_camera.T, a strided view
        K = torch.tensor([[[0.9 * W, 0., W / 2], [0., 0.9 * W, H / 2], [0., 0., 1.]]]).to(dev)
        fused = lambda: normal_consistency_loss(normal, exp_depth, alpha, w2c[0], K[0], LAMBDA)      # noqa: E731
        reference = lambda: torch_normal_loss(normal, exp_depth, alpha, w2c, K)                     # noqa: E731
        with torch.no_grad():
            med, spread = time_paths({"fused": fused, "torch": reference}, args, SLEEP_FWD)
        results.append({"what": "fwd", "image": [H, W], **row(med, spread)})
        med, spread = time_paths({"fused": lambda: fused().backward(), "torch": lambda: reference().backward()}, args, SLEEP_FWD_BWD)
        results.append({"what": "fwd_bwd", "image": [H, W], **row(med, spread)})
        us = kernel_times(lambda: fused().backward(), args.profile_calls)
        nbytes = kernel_bytes(H, W)
        kernels.append({"image": [H, W],
                        "kernels": {k: {"us": round(t, 2), "algorithmic_MB": round(nbytes[k] / 1e6, 2),
                                        "GB_per_s": round(nbytes[k] / (t * 1e-6) / 1e9, 1),
                                        "share_of_hbm_bound": round(nbytes[k] / HBM_PEAK / (t * 1e-6), 3)} for k, t in us.items()}})
        del feats, normal
    # the flatten term stays torch in both arms: its cost at 1 M Gaussians (exp of the raw scales, as get_scales() does)
    scales = (torch.randn(1_000_000, 3, generator=gen) - 4).to(dev).requires_grad_(True)
    flat = lambda: (torch.exp(scales)[..., -1].mean() * FLATTEN).backward()       # noqa: E731
    med, spread = time_paths({"fused": flat, "torch": flat}, args, SLEEP_FWD_BWD)
    flatten = {"what": "flatten_fwd_bwd", "n": 1_000_000, "torch_us": round(med["torch"] * 1e3, 2),
               "torch_us_min_max": [round(x * 1e3, 2) for x in spread["torch"]]}
    print(json.dumps({"metric": "normal_consistency_loss", "hbm_peak_GBps": HBM_PEAK / 1e9, **card(), "results": results,
                      "flatten": flatten, "fused_kernels_fwd_bwd": kernels}))


if __name__ == "__main__":
    main()
