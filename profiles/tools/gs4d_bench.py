"""Cost of the 4DGS deformation (B200VanillaGS4DRenderer: K51) against the same math as fp32 torch ops on the GPU, the way the
reference runs it every frame (grid_sample on the channel-first planes, the plane products and concatenation, the trunk and head
Linear layers, the additions and the quaternion product).  Both arms alternate in one process.
    op:     the deformation alone at N = 300 K and 1 M for two networks: the 4DGaussians defaults (C 32, 4 levels multires 1/2/4/8,
            resolution 64/64/64/25, net_width 64, defor_depth 1, dx/ds/dr) and a HyperNeRF-like one (C 16, 3 levels, time resolution
            150, net_width 128, every head including dshs, apply_rotation); K51's device time from a separate torch.profiler run and
            its gathered bytes (24 L corner rows of 4 C bytes per Gaussian, plus the parameters in and out) over that time
    render: deformation + render at 1920x1080, N = 1 M, through B200VanillaGS4DRenderer's path (K51, then the fused-activation
            rasterizer) and through the torch deformation followed by the same rasterizer
Timing as profiles/tools/exposure_bench.py: CUDA events around blocks of calls behind a device-side sleep, medians and min-max over
the blocks; the card's name and power limit read in the same call.  Writes one JSON line to stdout and to --out.

    python profiles/tools/gs4d_bench.py [--calls 40] [--block 4] [--warmup 4] [--out profiles/gs4d_bench_h100.json]
"""
import argparse
import json
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from b200gs import ops  # noqa: E402
from exposure_bench import HBM_PEAK, card, time_paths  # noqa: E402
from glossy_bench import profiled  # noqa: E402

PLANES = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
NETS = {
    "default_c32_l4_w64": dict(C=32, multires=[1, 2, 4, 8], res=[64, 64, 64, 25], W=64, D=1, heads=("dx", "ds", "dr"), rot=False),
    "hypernerf_c16_l3_w128": dict(C=16, multires=[1, 2, 4], res=[64, 64, 64, 150], W=128, D=1, heads=("dx", "ds", "dr", "dshs"), rot=True),
}
AABB = [[1.6, 1.6, 1.6], [-1.6, -1.6, -1.6]]
SLEEP = 20_000_000


def make_net(cfg, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    grids = []
    for m in cfg["multires"]:
        r = [x * m for x in cfg["res"][:3]] + cfg["res"][3:]
        grids.append([torch.rand(1, cfg["C"], r[b], r[a], generator=g, device=dev) + 0.5 for a, b in PLANES])
    lin = lambda o, i: (torch.randn(o, i, generator=g, device=dev) / math.sqrt(i), torch.randn(o, generator=g, device=dev) * 0.1)  # noqa
    W = cfg["W"]
    trunk = [lin(W, cfg["C"] * len(grids))] + [lin(W, W) for _ in range(cfg["D"] - 1)]
    heads = {h: (lin(W, W), lin({"dx": 3, "ds": 3, "dr": 4, "dshs": 48}[h], W)) for h in cfg["heads"]}
    return grids, trunk, heads


def torch_deform(means, scales, quats, dc, rest, t, grids, aabb, trunk, heads, rot):
    """the reference's deformation in fp32 torch ops (the work it throws away left out)"""
    p = (means - aabb[0]) * (2.0 / (aabb[1] - aabb[0])) - 1.0
    pts = torch.cat([p, t.expand(p.shape[0], 1)], -1)
    feats = []
    for level in grids:
        prod = 1.0
        for (a, b), plane in zip(PLANES, level):
            s = F.grid_sample(plane, pts[:, [a, b]].view(1, 1, -1, 2), align_corners=True, mode="bilinear", padding_mode="border")
            prod = prod * s.view(plane.shape[1], -1).T
        feats.append(prod)
    h = F.linear(torch.cat(feats, -1), *trunk[0])
    for wb in trunk[1:]:
        h = F.linear(F.relu(h), *wb)

    def head(name):
        (w1, b1), (w2, b2) = heads[name]
        return F.linear(F.relu(F.linear(F.relu(h), w1, b1)), w2, b2)

    m = means + head("dx") if "dx" in heads else means
    s = scales + head("ds") if "ds" in heads else scales
    q = quats
    if "dr" in heads:
        dr = head("dr")
        if rot:
            q1, q2 = quats, dr
            w = q1[:, 0] * q2[:, 0] - q1[:, 1] * q2[:, 1] - q1[:, 2] * q2[:, 2] - q1[:, 3] * q2[:, 3]
            x = q1[:, 0] * q2[:, 1] + q1[:, 1] * q2[:, 0] + q1[:, 2] * q2[:, 3] - q1[:, 3] * q2[:, 2]
            y = q1[:, 0] * q2[:, 2] - q1[:, 1] * q2[:, 3] + q1[:, 2] * q2[:, 0] + q1[:, 3] * q2[:, 1]
            z = q1[:, 0] * q2[:, 3] + q1[:, 1] * q2[:, 2] - q1[:, 2] * q2[:, 1] + q1[:, 3] * q2[:, 0]
            q = torch.stack((w, x, y, z), 1)
            q = q / q.norm(dim=1, keepdim=True)
        else:
            q = quats + dr
    if "dshs" in heads:
        shs = torch.cat([dc, rest], 1) + head("dshs").reshape(-1, 16, 3)
        dc, rest = shs[:, :1], shs[:, 1:]
    return m, s, q, dc, rest


def gaussians(n, dev, seed=1):
    g = torch.Generator(device=dev).manual_seed(seed)
    return dict(means=(torch.rand(n, 3, generator=g, device=dev) * 2 - 1) * 1.5, scales=torch.randn(n, 3, generator=g, device=dev) * 0.3 - 4.5,
                rotations=torch.randn(n, 4, generator=g, device=dev), opacities=torch.randn(n, 1, generator=g, device=dev),
                shs_dc=torch.randn(n, 1, 3, generator=g, device=dev) * 0.4, shs_rest=torch.randn(n, 15, 3, generator=g, device=dev) * 0.1)


def gathered_bytes(cfg, n):
    L, C = len(cfg["multires"]), cfg["C"]
    per = 24 * L * 4 * C + 40 + 40 + (384 if "dshs" in cfg["heads"] else 0)
    return per * n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--block", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gs4d_bench needs a CUDA device: there is no CPU measurement")
    dev = "cuda:0"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    aabb = torch.tensor(AABB, device=dev)
    t = torch.tensor([0.4], device=dev)
    res = {"metric": "gs4d_deform", "hbm_peak_TBps": HBM_PEAK / 1e12, **card(), "results": {}}
    torch.set_grad_enabled(False)
    for net_name, cfg in NETS.items():
        grids, trunk, heads = make_net(cfg, dev)
        planes = ops.gs4d_repack_planes(grids)
        for n in (300_000, 1_000_000):
            p = gaussians(n, dev)
            args5 = (p["means"], p["scales"], p["rotations"], p["shs_dc"], p["shs_rest"])

            def fused():
                return ops.gs4d_deform(p["means"], p["scales"], p["rotations"], t, planes, aabb, trunk, heads, shs_dc=p["shs_dc"],
                                       shs_rest=p["shs_rest"], apply_rotation=cfg["rot"])

            def eager():
                return torch_deform(*args5, t, grids, aabb, trunk, heads, cfg["rot"])

            a, b = fused(), eager()
            diff = max(float((x - y).abs().max()) for x, y in zip(a, b))
            med, spread = time_paths({"fused": fused, "torch": eager}, args, SLEEP)
            kern = {k: v for k, v in profiled(fused, 10).items() if "gs4d" in k}
            k_us = sum(v[0] for v in kern.values())
            nbytes = gathered_bytes(cfg, n)
            res["results"][f"{net_name}_n{n}"] = {
                "n": n, "net": cfg, "ms": {k: round(v, 4) for k, v in med.items()}, "ms_min_max": spread,
                "speedup": round(med["torch"] / med["fused"], 2), "max_abs_diff_vs_torch_fp32": diff,
                "k51_us": round(k_us, 1), "k51_launches": sum(v[1] for v in kern.values()),
                "gathered_bytes": nbytes, "gathered_TBps_over_k51": round(nbytes / (k_us * 1e-6) / 1e12, 3) if k_us else None}
            del p, a, b
            torch.cuda.empty_cache()
    # deformation + render at 1920x1080, N = 1 M, default network
    from b200gs.renderers import MODE_VANILLA, _view_with, camera_view
    from b200gs.scene import make_ring_cameras
    cfg = NETS["default_c32_l4_w64"]
    grids, trunk, heads = make_net(cfg, dev)
    planes = ops.gs4d_repack_planes(grids)
    n = 1_000_000
    p = gaussians(n, dev, seed=3)
    cam = make_ring_cameras(1920, 1080)[0].to_device(dev)
    view = _view_with(camera_view(cam, MODE_VANILLA), sh_degree=3)
    bg = torch.zeros(3, device=dev)
    m2d = torch.zeros(n, 3, device=dev)

    def render(d):
        m, s, q, dc, rest = d
        return ops.rasterize_vanilla_raw(m, m2d, dc, rest, p["opacities"], s, q, bg, view)

    def fused_render():
        return render(ops.gs4d_deform(p["means"], p["scales"], p["rotations"], t, planes, aabb, trunk, heads, shs_dc=p["shs_dc"],
                                      shs_rest=p["shs_rest"]))

    def eager_render():
        return render(torch_deform(p["means"], p["scales"], p["rotations"], p["shs_dc"], p["shs_rest"], t, grids, aabb, trunk, heads, False))

    img_a, img_b = fused_render()[0], eager_render()[0]
    med, spread = time_paths({"fused": fused_render, "torch": eager_render}, args, SLEEP)
    res["results"]["deform_render_1920x1080_n1000000"] = {
        "n": n, "visible": int((fused_render()[1] > 0).sum()), "ms": {k: round(v, 4) for k, v in med.items()}, "ms_min_max": spread,
        "speedup": round(med["torch"] / med["fused"], 2), "max_abs_image_diff": float((img_a - img_b).abs().max())}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
