"""Cost of the Glossy-Gaussian view-dependent opacity and colour (B200GlossyRenderer, K47 / K48) against the chain the reference
runs every step, restated below in torch: F.normalize of the detached means minus the camera centre, eval_sh_decomposed of
internal/utils/sh_utils.py:115-171 on the opacity SH, the [0, 1] clamp, then the SH colour through ops.spherical_harmonics_decomposed
(the v1 drop-in's gsplat call, K15) and its clamp, with autograd for the backward.  Both arms alternate in one process.
    op:    ops.glossy_sh forward and forward + backward at N = 1 M and 3 M, degree 3, split colour, every row visible; launches of
           one forward + backward counted with torch.profiler; K47 / K48 kernel times from a separate torch.profiler run, with
           their algorithmic bytes (b200gs.h) over the 3.35 TB/s HBM3 data-sheet bound
    step:  one training step (render forward and backward at 1920x1080, degree 3, tile-based culling) through B200GlossyRenderer
           and through the same v1 renderer with the reference-style hooks, at N = 1 M
Timing as profiles/tools/exposure_bench.py: CUDA events around blocks of calls behind a device-side sleep, medians and min-max over
the blocks; the card's name and power limit read in the same call.  Writes one JSON line to stdout and to --out.

    python profiles/tools/glossy_bench.py [--calls 40] [--block 4] [--warmup 4] [--out profiles/glossy_bench_h100.json]
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

from b200gs import ops  # noqa: E402
from exposure_bench import HBM_PEAK, SLEEP_FWD, SLEEP_FWD_BWD, card, time_paths  # noqa: E402

DEG = 3
C0, C1 = 0.28209479177387814, 0.4886025119029199
C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658, 1.445305721320277,
      -0.5900435899266435]


def eval_sh_decomposed(deg, shs_dc, shs_rest, dirs):
    """sh_utils.eval_sh_decomposed for degrees 0..3, as the reference evaluates it"""
    result = C0 * shs_dc[..., 0, :]
    if deg > 0:
        x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
        result = result - C1 * y * shs_rest[..., 0, :] + C1 * z * shs_rest[..., 1, :] - C1 * x * shs_rest[..., 2, :]
        if deg > 1:
            xx, yy, zz = x * x, y * y, z * z
            xy, yz, xz = x * y, y * z, x * z
            result = (result + C2[0] * xy * shs_rest[..., 3, :] + C2[1] * yz * shs_rest[..., 4, :]
                      + C2[2] * (2.0 * zz - xx - yy) * shs_rest[..., 5, :] + C2[3] * xz * shs_rest[..., 6, :]
                      + C2[4] * (xx - yy) * shs_rest[..., 7, :])
            if deg > 2:
                result = (result + C3[0] * y * (3 * xx - yy) * shs_rest[..., 8, :] + C3[1] * xy * z * shs_rest[..., 9, :]
                          + C3[2] * y * (4 * zz - xx - yy) * shs_rest[..., 10, :]
                          + C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * shs_rest[..., 11, :]
                          + C3[4] * x * (4 * zz - xx - yy) * shs_rest[..., 12, :] + C3[5] * z * (xx - yy) * shs_rest[..., 13, :]
                          + C3[6] * x * (xx - 3 * yy) * shs_rest[..., 14, :])
    return result


def torch_chain(deg, means, campos, op_dc, op_rest, shs_dc, shs_rest, mask):
    """GlossyRendererModule.get_opacities then get_rgbs on the v1 drop-in: returns (rgb, opacity)"""
    viewdirs = F.normalize(means.detach() - campos, dim=-1)
    opacity = torch.clamp(eval_sh_decomposed(deg, op_dc, op_rest, viewdirs).squeeze(-1) + 0.5, min=0., max=1.)
    rgb = torch.clamp(ops.spherical_harmonics_decomposed(deg, viewdirs, shs_dc, shs_rest, mask) + 0.5, min=0.0)
    return rgb, opacity


def glossy_bytes(n, k_rest=15, stride=16):
    """algorithmic bytes of K47 and K48 (include/b200gs.h), every row visible"""
    fwd = n * (12 + 4 + 4 * k_rest + 12 + 12 * (stride - 1) + 1) + n * (4 + 12 + 1)
    bwd = n * (12 + 1 + 4 + 12) + n * (4 + 4 * k_rest + 12 + 12 * (stride - 1))
    return fwd, bwd


def inputs(n, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, device="cuda")     # noqa: E731
    p = {"means": r(n, 3) * 2, "op_dc": r(n, 1, 1), "op_rest": r(n, 15, 1) * 0.3, "shs_dc": r(n, 1, 3), "shs_rest": r(n, 15, 3) * 0.3}
    for k in ("op_dc", "op_rest", "shs_dc", "shs_rest"):
        p[k].requires_grad_(True)
    return p, r(3), torch.ones(n, dtype=torch.bool, device="cuda"), r(n, 3), r(n)


def arms(p, campos, mask, v_rgb, v_op):
    def fused():
        return ops.glossy_sh(DEG, p["means"], campos, p["op_dc"], p["op_rest"], shs_dc=p["shs_dc"], shs_rest=p["shs_rest"], mask=mask)

    def chain():
        return torch_chain(DEG, p["means"], campos, p["op_dc"], p["op_rest"], p["shs_dc"], p["shs_rest"], mask)

    params = [p[k] for k in ("op_dc", "op_rest", "shs_dc", "shs_rest")]

    def with_bwd(fn):
        def run():
            rgb, op = fn()
            torch.autograd.backward([rgb, op], [v_rgb, v_op], inputs=params)
        return run
    return fused, chain, with_bwd(fused), with_bwd(chain)


def profiled(fn, calls=10):
    """kernel names -> (total µs per call, launches per call) of `fn` from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.count > 0 and not e.key.startswith("Memcpy"):
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            out[e.key] = (t / calls, e.count / calls)
    return out


def step_renderers():
    from b200gs.glossy import B200GlossyRenderer
    from b200gs.v1 import B200GSplatV1RendererModule

    class ReferenceHooks(B200GSplatV1RendererModule):
        """GlossyRendererModule's get_opacities / get_rgbs, as the reference runs them on the v1 drop-in"""

        def get_opacities(self, camera, gm, projections, visibility_filter, status, **kwargs):
            viewdirs = F.normalize(gm.get_xyz.detach() - camera.camera_center, dim=-1)
            op = eval_sh_decomposed(gm.active_sh_degree, gm.gaussians["opacities"], gm.gaussians["opacity_rest"], viewdirs)
            return torch.clamp(op.squeeze(-1) + 0.5, min=0., max=1.), viewdirs

        def get_rgbs(self, camera, gm, projections, visibility_filter, status, **kwargs):
            rgbs = ops.spherical_harmonics_decomposed(gm.active_sh_degree, status, gm.get_shs_dc(), gm.get_shs_rest(), visibility_filter)
            return torch.clamp(rgbs + 0.5, min=0.0)

    cfg = B200GlossyRenderer(separate_sh=True, tile_based_culling=True)
    return cfg.instantiate().cuda(), ReferenceHooks(cfg).cuda()


def glossy_scene(n):
    from b200gs.scene import SyntheticGaussians, make_scene
    raw = make_scene(n, 5, mean_scale=0.01)
    g = torch.Generator().manual_seed(21)
    raw["opacities"] = torch.randn(n, 1, 1, generator=g) * 1.2 + 0.4
    raw["opacity_rest"] = torch.randn(n, 15, 1, generator=g) * 0.4
    return SyntheticGaussians(raw).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--block", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    results = {}
    for n in (1 << 20, 3 << 20):
        p, campos, mask, v_rgb, v_op = inputs(n)
        fused, chain, fused_bwd, chain_bwd = arms(p, campos, mask, v_rgb, v_op)
        fwd_med, fwd_rng = time_paths({"fused": fused, "torch": chain}, args, SLEEP_FWD)
        fb_med, fb_rng = time_paths({"fused": fused_bwd, "torch": chain_bwd}, args, SLEEP_FWD_BWD)
        kf, kc = profiled(fused_bwd), profiled(chain_bwd)
        k47 = sum(t for k, (t, _) in kf.items() if "glossy_fwd_kernel" in k)
        k48 = sum(t for k, (t, _) in kf.items() if "glossy_bwd_kernel" in k)
        bf, bb = glossy_bytes(n)
        results[f"n{n}"] = {
            "n": n, "forward_ms": {k: fwd_med[k] for k in fwd_med}, "forward_range_ms": fwd_rng,
            "forward_backward_ms": {k: fb_med[k] for k in fb_med}, "forward_backward_range_ms": fb_rng,
            "launches_fwd_bwd": {"fused": sum(c for _, c in kf.values()), "torch": sum(c for _, c in kc.values())},
            "fused_kernels_us": {k: t for k, (t, _) in kf.items()},
            "K47_us": k47, "K48_us": k48, "K47_bytes": bf, "K48_bytes": bb,
            "K47_TBps": bf / (k47 * 1e-6) / 1e12, "K48_TBps": bb / (k48 * 1e-6) / 1e12,
            "K47_share_of_hbm": bf / (k47 * 1e-6) / HBM_PEAK, "K48_share_of_hbm": bb / (k48 * 1e-6) / HBM_PEAK,
        }
        del p, fused, chain, fused_bwd, chain_bwd
        torch.cuda.empty_cache()

    from b200gs.scene import make_ring_cameras
    fused_r, ref_r = step_renderers()
    cam = make_ring_cameras(1920, 1080)[3].to_device("cuda")
    bg = torch.tensor([0.1, 0.2, 0.3], device="cuda")
    pcs = {"fused": glossy_scene(1 << 20), "torch": glossy_scene(1 << 20)}

    def step(r, pc):
        def run():
            out = r(cam, pc, bg)
            out["render"].sum().backward()
        return run
    step_med, step_rng = time_paths({"fused": step(fused_r, pcs["fused"]), "torch": step(ref_r, pcs["torch"])}, args, SLEEP_FWD_BWD)
    results["step_1080p_n1048576"] = {"ms": step_med, "range_ms": step_rng}
    line = json.dumps({"metric": "glossy", "degree": DEG, "hbm_peak_TBps": HBM_PEAK / 1e12, **card(), "results": results})
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
