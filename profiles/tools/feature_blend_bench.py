"""Cost of a 32-channel feature render on the benchmark scene (make_scene(1 M, 0), pose 0 of the ring): (a) the channel groups of
ops.rasterize_binned — 8 x K6 forward and 8 x K7 backward of 4 channels each — against (b) the D-channel kernels: the forward, the
features-only backward (geometry frozen, as in the feature renderers) and the backward with geometry gradients.  Seeded random
features, one binning per resolution, 1920x1080 and 800x800.  Before timing it asserts that (a) and (b) composite bit-identical
images (without the background term) and alpha.  CUDA events around blocks of calls, each queued behind a device-side sleep (the events time device work, not the host's
launch rate); the paths alternate in one process; medians over the blocks.  Prints one JSON line with the card's name and power
limit read in the same run.

    python profiles/tools/feature_blend_bench.py [--n 1000000] [--D 32] [--blocks 20] [--block 5] [--warmup 5]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch  # noqa: E402

from b200gs import ops  # noqa: E402
from b200gs._lib import MODE_GSPLAT  # noqa: E402
from b200gs.renderers import camera_view  # noqa: E402
from b200gs.scene import activate, make_ring_cameras, make_scene  # noqa: E402
from mcmc_noise_bench import SLEEP_CYCLES, card  # noqa: E402


def projected(n, W, H, dev):
    sc = {k: v.to(dev) for k, v in activate(make_scene(n, 0)).items()}
    view = camera_view(make_ring_cameras(W, H)[0], MODE_GSPLAT, cache=False)
    xy, depth, radii, conic, comp, _, _, _, _ = ops.project_forward(view, sc["means"], sc["scales"], sc["rotations"], None, True)
    return xy, depth, radii, conic, (sc["opacities"].reshape(-1) * comp).contiguous()


def time_paths(paths, blocks, block, warmup):
    for fn in paths.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    ev = {k: [] for k in paths}
    for _ in range(blocks):
        for k, fn in paths.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(SLEEP_CYCLES)
            a.record()
            for _ in range(block):
                fn()
            b.record()
            ev[k].append((a, b))
    torch.cuda.synchronize()
    out = {}
    for k, v in ev.items():
        t = sorted(a.elapsed_time(b) / block for a, b in v)
        out[k] = {"median_ms": round(t[len(t) // 2], 4), "min_ms": round(t[0], 4), "max_ms": round(t[-1], 4)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--D", type=int, default=32)
    ap.add_argument("--sizes", default="1920x1080,800x800")
    ap.add_argument("--blocks", type=int, default=20)
    ap.add_argument("--block", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("feature_blend_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    D = args.D
    g = torch.Generator(device=dev).manual_seed(0)
    results = []
    for size in args.sizes.split(","):
        W, H = (int(s) for s in size.split("x"))
        xy, depth, radii, conic, op = projected(args.n, W, H, dev)
        feats = torch.rand(args.n, D, generator=g, device=dev) * 2 - 1
        bg = torch.rand(D, generator=g, device=dev)
        v_img = torch.rand(H, W, D, generator=g, device=dev) * 2 - 1
        v_alpha = torch.rand(H, W, generator=g, device=dev) * 2 - 1
        binning = ops.bin_gaussians(MODE_GSPLAT, W, H, xy, depth, radii, conic, op)
        groups = [(c0, min(D, c0 + 4)) for c0 in range(0, D, 4)]
        g_feats = [feats[:, a:b].contiguous() for a, b in groups]
        g_bg = [bg[a:b].contiguous() for a, b in groups]
        g_vimg = [v_img[..., a:b].contiguous() for a, b in groups]

        def a_fwd():
            return [ops.blend_forward(MODE_GSPLAT, W, H, binning, xy, conic, op, f, b, False, True) for f, b in zip(g_feats, g_bg)]

        # bit-identical composites (the + T bg term is left out: K6 rounds it differently from channel to channel, see
        # tests/test_gpu_feature_blend.py)
        image_a = torch.cat([ops.blend_forward(MODE_GSPLAT, W, H, binning, xy, conic, op, f, None, False, True)[0] for f in g_feats], dim=-1)
        image_b, _, _, alpha_b = ops.blend_features_forward(W, H, binning, xy, conic, op, feats, None)
        assert torch.equal(image_a, image_b), "the D-channel forward differs from the 4-channel groups"
        fwd_a = a_fwd()
        image_b, final_T, n_contrib, alpha_b = ops.blend_features_forward(W, H, binning, xy, conic, op, feats, bg)
        assert torch.equal(fwd_a[0][3], alpha_b), "alpha differs from the 4-channel groups"
        fT, nc = fwd_a[0][1], fwd_a[0][2]

        def a_bwd():
            for i, (f, b, v) in enumerate(zip(g_feats, g_bg, g_vimg)):
                ops.blend_backward(MODE_GSPLAT, W, H, binning, xy, conic, op, f, b, fT, nc, v, v_alpha if i == 0 else None, False)

        def b_bwd(geometry):
            return ops.blend_features_backward(W, H, binning, xy, conic, op, feats, bg, final_T, n_contrib, v_img, v_alpha, geometry, False)

        t = time_paths({"a_fwd_groups": a_fwd, "b_fwd": lambda: ops.blend_features_forward(W, H, binning, xy, conic, op, feats, bg),
                        "a_bwd_groups": a_bwd, "b_bwd_features_only": lambda: b_bwd(False), "b_bwd_geom": lambda: b_bwd(True)},
                       args.blocks, args.block, args.warmup)
        results.append({"size": f"{W}x{H}", "pairs": int(binning.total), **t,
                        "fwd_speedup": round(t["a_fwd_groups"]["median_ms"] / t["b_fwd"]["median_ms"], 2),
                        "bwd_features_only_speedup": round(t["a_bwd_groups"]["median_ms"] / t["b_bwd_features_only"]["median_ms"], 2),
                        "bwd_geom_speedup": round(t["a_bwd_groups"]["median_ms"] / t["b_bwd_geom"]["median_ms"], 2)})
        del xy, depth, radii, conic, op, feats, v_img, binning, g_feats, g_vimg, fwd_a
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "feature_blend", "n": args.n, "D": D, "composite_bit_identical": True, **card(), "results": results}))


if __name__ == "__main__":
    main()
