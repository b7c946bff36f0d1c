"""Cost of the appearance colour pass per view: the fused op (ops.appearance_mlp: one kernel forward, two backward) against a torch
restatement of the reference's path (boolean-mask gathers, embedding repeat, concat, nn.Linear layers, masked scatter) in FP32 and,
for context, with allow_tf32 on; and the appearance renderer end to end (forward + backward) with the fused op and with the torch
colour path plugged into the same renderer.  The benchmark's synthetic scene (1 M Gaussians, 1920x1080) plus seeded appearance
features; the default network (64 features, 32-dim embedding, 64 neurons, 3 layers).  Arms alternate within the one process; CUDA
events around blocks of calls.  Prints one JSON line with the times, the shape-derived FLOPs and bytes of the fused pass, what they
come to per second, which data-sheet bound (67 TFLOP/s FP32 is not used: the kernels run on the TF32 tensor cores, 495 TFLOP/s dense
for single-pass TF32, three passes per product; 3.35 TB/s HBM3) is the tighter one, and the card's name and power limit.

    python profiles/tools/appearance_bench.py [--n 1000000] [--calls 60] [--block 5] [--warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

from b200gs import ops  # noqa: E402
from b200gs.appearance import B200GSplatAppearanceEmbeddingRenderer, ModelConfig  # noqa: E402
from b200gs.scene import SyntheticGaussians, make_ring_cameras, make_scene  # noqa: E402

HBM_PEAK, TF32_PEAK = 3.35e12, 495e12
F_DIM, E_DIM, HID = 64, 32, 64


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": name, "power_limit_w": float(out[0]), "sm_max_mhz": float(out[1])}
    except Exception as e:      # the number is then reported without it, and says so
        return {"gpu": name, "power_limit_w": "not measured", "sm_max_mhz": "not measured", "nvidia_smi": str(e)}


def torch_colors(model, features, vis, base, appearance_id):
    """The reference's colour path restated: gathers by boolean mask (a host synchronisation each), the embedding repeated per row"""
    f = features[vis]
    e = model.embedding(appearance_id.reshape(-1)).repeat(f.shape[0], 1)
    s = model.network.output_layers(torch.cat([f, e], dim=-1))
    rgbs = torch.zeros_like(base)
    rgbs[vis] = torch.clamp(base[vis] + 0.5 + (s[:, :3] * 2 - 1.), min=0., max=1.)
    return rgbs


def time_paths(paths, args):
    for fn in paths.values():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in paths}
    for _ in range(args.calls // args.block):
        for k, fn in paths.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.block):
                fn()
            b.record()
            ms[k].append((a, b))
    torch.cuda.synchronize()
    per_call = {k: sorted(a.elapsed_time(b) / args.block for a, b in v) for k, v in ms.items()}
    return {k: {"median_ms": round(v[len(v) // 2], 4), "min_ms": round(v[0], 4), "max_ms": round(v[-1], 4)} for k, v in per_call.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--calls", type=int, default=60)
    ap.add_argument("--block", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("appearance_bench needs a CUDA device")
    dev = torch.device("cuda", 0)

    class AppearanceGaussians(SyntheticGaussians):
        def __init__(self, raw):
            super().__init__(raw)
            self.appearance_features = torch.nn.Parameter(torch.randn(raw["means"].shape[0], F_DIM, generator=torch.Generator().manual_seed(1)))

        def get_appearance_features(self):
            return self.appearance_features

    pc = AppearanceGaussians(make_scene(args.n, 0)).to(dev)
    cam = make_ring_cameras(1920, 1080)[0].to_device(dev)
    cam.appearance_id = torch.tensor([1], dtype=torch.int32, device=dev)
    bg = torch.zeros(3, device=dev)
    torch.manual_seed(0)
    renderer = B200GSplatAppearanceEmbeddingRenderer(model=ModelConfig(n_appearances=4)).instantiate()
    renderer._setup_model(device=dev)
    model = renderer.model
    with torch.no_grad():
        vis = renderer(cam, pc, bg, warm_up=True)["visibility_filter"]
    V = int(vis.sum())
    base = renderer.sh_colors(cam, pc, vis).detach().requires_grad_(True)
    cot = torch.randn(args.n, 3, device=dev)
    feats = pc.appearance_features
    lin = model.linears()

    def fused():
        out = ops.appearance_mlp(feats, model.embedding_row(cam.appearance_id), [m.weight for m in lin], [m.bias for m in lin], mask=vis, base_rgb=base)
        torch.autograd.backward(out, cot)

    def torch_fp32():
        torch.autograd.backward(torch_colors(model, feats, vis, base, cam.appearance_id), cot)

    def torch_tf32():
        torch.backends.cuda.matmul.allow_tf32 = True
        try:
            torch_fp32()
        finally:
            torch.backends.cuda.matmul.allow_tf32 = False

    colour = time_paths({"fused": fused, "torch_fp32": torch_fp32, "torch_tf32": torch_tf32}, args)

    # end to end: the same renderer, the colour hook swapped for the torch restatement
    def torch_hook(camera, gm, projections, visibility, status, **kw):
        b = renderer.sh_colors(camera, gm, visibility)
        return torch_colors(model, gm.get_appearance_features(), visibility, b, camera.appearance_id), gm.get_opacities().squeeze(-1), None

    def e2e():
        renderer(cam, pc, bg, warm_up=False)["render"].sum().backward()

    def e2e_torch():
        renderer._get_rgbs_and_opacities = torch_hook
        try:
            e2e()
        finally:
            del renderer._get_rgbs_and_opacities

    def e2e_warm_up():
        renderer(cam, pc, bg, warm_up=True)["render"].sum().backward()

    render = time_paths({"fused": e2e, "torch_fp32": e2e_torch, "sh_only": e2e_warm_up}, args)

    mac_fwd = F_DIM * HID + HID * HID + 8 * HID                    # per row, the output layer padded to 8
    flops = V * 2 * mac_fwd * (1 + 3)                               # forward; backward = recompute + input and weight gradients
    nbytes = V * (256 + 12 + 12) + V * (256 + 12 + 12 + 256 + 12) + 2 * args.n * (1 + 12) + (args.n - V) * 256
    t = colour["fused"]["median_ms"] * 1e-3
    bound_flop, bound_byte = 3 * flops / TF32_PEAK, nbytes / HBM_PEAK
    print(json.dumps({
        "metric": "appearance_colour_pass", **card(), "n": args.n, "visible": V, "width": 1920, "height": 1080,
        "colour_pass_fwd_bwd": colour, "renderer_fwd_bwd": render,
        "fused_useful_GFLOP": round(flops / 1e9, 2), "fused_algorithmic_MB": round(nbytes / 1e6, 1),
        "fused_useful_TFLOPs_per_s": round(flops / t / 1e12, 2), "fused_GB_per_s": round(nbytes / t / 1e9, 1),
        "tighter_bound": "tensor cores (3 TF32 passes per product at 495 TFLOP/s)" if bound_flop > bound_byte else "HBM (3.35 TB/s)",
        "share_of_tighter_bound": round(max(bound_flop, bound_byte) / t, 3),
    }))


if __name__ == "__main__":
    main()
