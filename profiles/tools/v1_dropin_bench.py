"""Cost of the gsplat-v1 drop-in (b200gs.compat.gsplat_v1) against the plug-in B200GSplatV1Renderer on the benchmark scene
(make_scene(N, 0), pose 0 of the ring), and of the three kernels the drop-in adds on their own.

The drop-in path is the reference's GSplatV1Renderer rgb render (gsplat_v1_renderer.py:137-287 with GSplatV1's helpers) written
out below, since the reference is not importable here: fully_fused_projection, isect_tiles + isect_offset_encode (or the
tile-based-culling pair), spherical_harmonics(_decomposed), rasterize_to_pixels.  Forward + backward of both paths, alternating
in one process, one call per CUDA-event pair (both paths wait on the host once per view for the exact pair count, so a call is
timed as a whole); medians over the blocks.  Before timing it asserts that the two renders are bit-identical.  The keys, offsets and
split-SH kernels are timed in blocks of calls queued behind a device-side sleep, and so is the SH step of
B200GSplatV1Renderer(separate_sh=True) before (torch.cat + the concatenated kernel) and after (the split kernel), forward +
backward.  Prints one JSON line with the card's name and power limit read in the same run.

    python profiles/tools/v1_dropin_bench.py [--cases 1000000:1920x1080,3000000:1600x1063] [--blocks 20] [--warmup 3]
"""
import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch  # noqa: E402

from b200gs import ops  # noqa: E402
from b200gs.compat import gsplat_v1 as G  # noqa: E402
from b200gs.scene import SyntheticGaussians, make_ring_cameras, make_scene  # noqa: E402
from b200gs.v1 import B200GSplatV1Renderer  # noqa: E402
from feature_blend_bench import time_paths  # noqa: E402
from mcmc_noise_bench import card  # noqa: E402


def dropin_render(cam, pc, bg, separate_sh, culling):
    """The reference's GSplatV1Renderer forward for render_types=["rgb"], through the drop-in."""
    viewmats = cam.world_to_camera.T.unsqueeze(0)
    Ks = torch.tensor([[[float(cam.fx), 0., float(cam.cx)], [0., float(cam.fy), float(cam.cy)], [0., 0., 1.]]], dtype=torch.float,
                      device=viewmats.device)
    w, h = int(cam.width), int(cam.height)
    radii, means2d, depths, conics, comp = G.fully_fused_projection(pc.get_means(), None, pc.get_rotations(), pc.get_scales(), viewmats=viewmats,
                                                                    Ks=Ks, width=w, height=h, eps2d=0.3, calc_compensations=True, packed=False,
                                                                    radius_clip=0.0, camera_model="pinhole")
    vis = radii.squeeze(0) > 0
    opacities = pc.get_opacities().squeeze(-1).unsqueeze(0) * comp
    tw, th = math.ceil(w / 16.), math.ceil(h / 16.)
    if culling:
        _, isect_ids, flatten_ids = G.isect_tiles_tile_based_culling(means2d, radii, depths, conics, opacities.detach(), 16, tw, th, packed=False,
                                                                     n_cameras=1, camera_ids=None, gaussian_ids=None)
        offsets, flatten_ids = G.isect_offset_encode_tile_based_culling(isect_ids, flatten_ids, 1, tw, th)
    else:
        _, isect_ids, flatten_ids = G.isect_tiles(means2d, radii, depths, 16, tw, th, packed=False, n_cameras=1, camera_ids=None, gaussian_ids=None)
        offsets = G.isect_offset_encode(isect_ids, 1, tw, th)
    means2d = means2d.squeeze(0)
    dirs = pc.get_xyz.detach() - cam.camera_center
    if separate_sh:
        rgbs = G.spherical_harmonics_decomposed(pc.active_sh_degree, dirs, pc.get_shs_dc(), pc.get_shs_rest(), vis)
    else:
        rgbs = G.spherical_harmonics(pc.active_sh_degree, dirs, pc.get_features, vis)
    colors, _ = G.rasterize_to_pixels(means2d=means2d, conics=conics, colors=torch.clamp(rgbs + 0.5, min=0.0).unsqueeze(0), opacities=opacities,
                                      image_width=w, image_height=h, tile_size=16, isect_offsets=offsets, flatten_ids=flatten_ids,
                                      backgrounds=bg.unsqueeze(0), absgrad=True)
    return colors.squeeze(0).permute(2, 0, 1), (isect_ids, flatten_ids, depths)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="1000000:1920x1080,3000000:1600x1063")
    ap.add_argument("--blocks", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("v1_dropin_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    results = []
    for case in args.cases.split(","):
        n, size = case.split(":")
        n = int(n)
        W, H = (int(s) for s in size.split("x"))
        model = SyntheticGaussians(make_scene(n, 0)).to(dev)
        cam = make_ring_cameras(W, H)[0].to_device(dev)
        cot = torch.rand(3, H, W, generator=torch.Generator().manual_seed(1)).to(dev)
        row = {"n": n, "size": f"{W}x{H}"}
        for separate_sh, culling in ((False, False), (True, True)):
            plugin = B200GSplatV1Renderer(separate_sh=separate_sh, tile_based_culling=culling).instantiate().to(dev)
            with torch.no_grad():
                a = dropin_render(cam, model, bg, separate_sh, culling)[0]
                b = plugin(cam, model, bg)["render"]
            assert torch.equal(a, b), "drop-in and plug-in renders differ"

            def run(fn):
                def step():
                    for p in model.parameters():
                        p.grad = None
                    (fn() * cot).sum().backward()
                return step

            t = time_paths({"dropin_fwd_bwd": run(lambda: dropin_render(cam, model, bg, separate_sh, culling)[0]),
                            "plugin_fwd_bwd": run(lambda: plugin(cam, model, bg)["render"])}, args.blocks, 1, args.warmup)
            row[f"sh{int(separate_sh)}_cull{int(culling)}"] = {**t, "dropin_over_plugin_ms": round(
                t["dropin_fwd_bwd"]["median_ms"] - t["plugin_fwd_bwd"]["median_ms"], 4)}
        # the new kernels on their own, on this view's culled lists
        with torch.no_grad():
            _, (keys, flat, depths) = dropin_render(cam, model, bg, True, True)
        tw, th = math.ceil(W / 16.), math.ceil(H / 16.)
        vis = torch.ones(n, dtype=torch.bool, device=dev)
        vis[::3] = False
        dirs = torch.randn(n, 3, device=dev)
        dc, rest = model.get_shs_dc().detach(), model.get_shs_rest().detach()
        v_rgb = torch.rand(n, 3, device=dev)
        starts = G.isect_offset_encode(keys, 1, tw, th).reshape(-1)
        ends = torch.cat((starts[1:], torch.tensor([keys.numel()], dtype=torch.int32, device=dev)))
        binning = ops.Binning(flat, torch.stack((starts, ends), -1).contiguous(), keys.numel())
        d = depths.reshape(-1).contiguous()
        L = ops.lib()
        v_dc, v_rest = torch.empty_like(dc), torch.empty_like(rest)
        mask = vis.view(torch.uint8)
        rgb = torch.empty(n, 3, device=dev)
        dc_p, rest_p = dc.clone().requires_grad_(True), rest.clone().requires_grad_(True)

        def sh_cat():        # what B200GSplatV1Renderer(separate_sh=True) ran before: concatenation, the concatenated kernel, autograd's split
            ops.spherical_harmonics(3, dirs, torch.cat((dc_p, rest_p), dim=1), vis).backward(v_rgb)

        def sh_split():      # what it runs now
            ops.spherical_harmonics_decomposed(3, dirs, dc_p, rest_p, vis).backward(v_rgb)

        t = time_paths({
            "sh_cat_fwd_bwd": sh_cat,
            "sh_split_fwd_bwd": sh_split,
            "isect_keys": lambda: ops.isect_keys(binning, d),
            "isect_offsets": lambda: ops.isect_offsets(keys, tw * th),
            "sh_split_fwd": lambda: L.b200gs_sh_split_fwd(3, 15, n, ops.ptr(dirs), ops.ptr(dc), ops.ptr(rest), ops.ptr(mask), ops.ptr(rgb),
                                                          ops._stream()),
            "sh_split_bwd": lambda: L.b200gs_sh_split_bwd(3, 15, n, ops.ptr(dirs), ops.ptr(dc), ops.ptr(rest), ops.ptr(mask), ops.ptr(v_rgb),
                                                          ops.ptr(v_dc), ops.ptr(v_rest), None, ops._stream()),
        }, args.blocks, 20, args.warmup)
        pairs, visible = int(keys.numel()), int(vis.sum())
        row["kernels"] = t
        row["pairs_culled"] = pairs
        # algorithmic bytes (include/b200gs.h): keys 4 B id + 4 B depth + 8 B key per pair; split SH 12 B dirs + 192 B coefficients
        # + 12 B rgb per visible row at degree 3, + n B of mask
        row["isect_keys_GBps"] = round(16 * pairs / (t["isect_keys"]["median_ms"] * 1e-3) / 1e9, 1)
        row["sh_split_fwd_GBps"] = round((216 * visible + n) / (t["sh_split_fwd"]["median_ms"] * 1e-3) / 1e9, 1)
        results.append(row)
        del model, binning, keys, flat, dc, rest, v_dc, v_rest
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "v1_dropin", **card(), "results": results}))


if __name__ == "__main__":
    main()
