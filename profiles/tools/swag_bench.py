"""Cost of SWAG's image-conditioned colours and opacities (B200SWAGRenderer: K49 -> K20 forward, K21 -> K22 -> K50 backward) against
the same math as fp32 torch ops on the GPU (tiny-cuda-nn cannot be installed): the SH colour of eval_gaussian_model_sh, the 3-D
hash grid as gathers over the 8 corners of every level (int64 index arithmetic masked to uint32, as tcnn's grid_index), the
59 -> 64 -> 64 -> 4 network, the sigmoid and the Gumbel-sigmoid opacity, with autograd for the backward.  Both arms alternate in
one process.
    op:    forward and forward + backward at N = 1 M, degree 3, the default grid (8 levels x 4 features, 2^19 table); the fused
           kernels' times from a separate torch.profiler run, with their algorithmic bytes (include/b200gs.h) over the 3.35 TB/s HBM3
           data-sheet bound, and the launches of one forward + backward
    step:  one training step (render forward and backward at 1920x1080) through B200SWAGRenderer and through a plain
           B200VanillaRenderer at N = 1 M
Timing as profiles/tools/exposure_bench.py: CUDA events around blocks of calls behind a device-side sleep, medians and min-max over
the blocks; the card's name and power limit read in the same call.  Writes one JSON line to stdout and to --out.

    python profiles/tools/swag_bench.py [--calls 40] [--block 4] [--warmup 4] [--out profiles/swag_bench_h100.json]
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

from b200gs import ops  # noqa: E402
from exposure_bench import HBM_PEAK, SLEEP_FWD, SLEEP_FWD_BWD, card, time_paths  # noqa: E402
from glossy_bench import profiled  # noqa: E402
from oracle import swag_oracle as S  # noqa: E402
from oracle.gs_oracle import sh_basis  # noqa: E402

DEG = 3
GRID = dict(S.DEFAULT_GRID)
M32 = 0xFFFFFFFF


def torch_hash_encode(table, x, F=4):
    """the grid in fp32 torch ops on the device: per level and corner one gather"""
    tab = table.view(-1, F)
    cols = []
    for scale, res, size, offset in S.levels(**GRID):
        pos = x * float(scale) + 0.5
        fl = torch.floor(pos)
        c, f = fl.long() & M32, pos - fl
        acc = 0
        for k in range(8):
            cc = [(c[:, d] + ((k >> d) & 1)) & M32 for d in range(3)]
            if res ** 3 <= size:
                idx = (cc[0] + cc[1] * res + cc[2] * res * res) & M32
            else:
                idx = cc[0] ^ ((cc[1] * S.PRIMES[1]) & M32) ^ ((cc[2] * S.PRIMES[2]) & M32)
            w = 1
            for d in range(3):
                w = w * (f[:, d] if (k >> d) & 1 else 1 - f[:, d])
            acc = acc + w.unsqueeze(-1) * tab[idx % size + offset]
        cols.append(acc)
    return torch.cat(cols, 1)


def torch_chain(p, campos, bbox_min, bbox_size, u):
    """SWAGRenderer.forward's colours and opacities, as the reference evaluates them, in torch"""
    feats = torch.cat([p["shs_dc"], p["shs_rest"]], 1)
    d = p["means"] - campos
    d = d / d.norm(dim=1, keepdim=True)
    rgb = torch.clamp_min((sh_basis(DEG, d).unsqueeze(-1) * feats).sum(1) + 0.5, 0.0)
    x = (p["means"].detach() - bbox_min) / bbox_size
    enc = torch_hash_encode(p["table"], x)
    h = torch.cat([rgb, enc, p["embedding"].expand(rgb.shape[0], -1)], 1)
    for l, (w, b) in enumerate(zip(p["ws"], p["bs"])):
        h = torch.nn.functional.linear(h, w, b)
        if l < len(p["ws"]) - 1:
            h = torch.relu(h)
    z = 1 / 0.1 * (torch.log(torch.abs(h[:, 3]) + 1e-8) + torch.log(u + 1e-8) - torch.log(1 - u + 1e-8))
    return torch.sigmoid(h[:, :3]), torch.clamp_min(p["base"] - torch.sigmoid(z), 0)


def inputs(n, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, device="cuda")     # noqa: E731
    means = r(n, 3) * 2
    p = {"means": means, "shs_dc": r(n, 1, 3), "shs_rest": r(n, 15, 3) * 0.3,
         "table": (torch.rand(S.n_params(**GRID), generator=g, device="cuda") * 2 - 1) * 1e-2,
         "ws": [r(64, 59) / math.sqrt(59), r(64, 64) / 8, r(4, 64) / 8], "bs": [r(64) * 0.1, r(64) * 0.1, r(4) * 0.1],
         "embedding": r(24), "base": torch.rand(n, generator=g, device="cuda")}
    for k, v in p.items():
        for t in (v if isinstance(v, list) else [v]):
            t.requires_grad_(True)
    lo, hi = means.detach().min(0).values, means.detach().max(0).values
    return p, r(3), lo, (hi - lo) * 1.1, torch.full((1,), 0.37, device="cuda"), r(n, 3), r(n)


def leaves(p):
    return [t for v in p.values() for t in (v if isinstance(v, list) else [v])]


def swag_bytes(n, row=40, gathers=64):
    """algorithmic bytes of each fused kernel (include/b200gs.h), degree 3, the default grid; a gathered or atomically added corner
    row counts 16 B"""
    return {"swag_inputs_fwd": n * (12 + 192 + 4 * row + 1 + 16 * gathers), "appearance_mlp_fwd": n * (4 * row + 4 + 16),
            "appearance_mlp_bwd": n * (4 * row + 20 + 4 * row + 4), "swag_inputs_bwd": n * (12 + 192 + 1 + 4 * row + 192 + 12 + 16 * gathers)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--block", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    n = args.n
    p, campos, bmin, bsize, u, v_col, v_op = inputs(n)
    bbox = torch.cat([bmin, bsize])

    def fused():
        return ops.swag_colours_and_opacities(DEG, p["means"], campos, p["base"], u, p["table"], p["embedding"], p["ws"], p["bs"],
                                              bbox=bbox, shs_dc=p["shs_dc"], shs_rest=p["shs_rest"], **GRID)

    def chain():
        return torch_chain(p, campos, bmin, bsize, u)

    def with_bwd(fn):
        def run():
            c, o = fn()
            torch.autograd.backward([c, o], [v_col, v_op], inputs=leaves(p))
        return run

    with torch.no_grad():
        cf, of = fused()
        ct, ot = chain()
        agree = {"colour_max_abs_diff": float((cf - ct).abs().max()), "opacity_max_abs_diff": float((of - ot).abs().max())}
    fwd_med, fwd_rng = time_paths({"fused": fused, "torch": chain}, args, SLEEP_FWD)
    fb_med, fb_rng = time_paths({"fused": with_bwd(fused), "torch": with_bwd(chain)}, args, SLEEP_FWD_BWD)
    kf, kc = profiled(with_bwd(fused)), profiled(with_bwd(chain))
    kb = swag_bytes(n)
    kernels = {}
    for name, b in kb.items():
        t = sum(us for k, (us, _) in kf.items() if name + "_kernel" in k)
        kernels[name] = {"us": t, "bytes": b, "TBps": b / (t * 1e-6) / 1e12 if t else None,
                         "share_of_hbm": b / (t * 1e-6) / HBM_PEAK if t else None}
    results = {"op_n%d" % n: {
        "n": n, "forward_ms": fwd_med, "forward_range_ms": fwd_rng, "forward_backward_ms": fb_med, "forward_backward_range_ms": fb_rng,
        "launches_fwd_bwd": {"fused": sum(c for _, c in kf.values()), "torch": sum(c for _, c in kc.values())},
        "fused_kernels_us": {k: t for k, (t, _) in kf.items()}, "kernels": kernels, "agreement": agree}}
    del p, fused, chain
    torch.cuda.empty_cache()

    from b200gs.renderers import B200VanillaRenderer
    from b200gs.scene import SyntheticGaussians, make_ring_cameras, make_scene
    from b200gs.swag import B200SWAGModel, B200SWAGRenderer
    cam = make_ring_cameras(1920, 1080)[3].to_device("cuda")
    cam.appearance_id = torch.tensor(3, device="cuda")
    bg = torch.tensor([0.1, 0.2, 0.3], device="cuda")
    pcs = {k: SyntheticGaussians(make_scene(n, 5, mean_scale=0.01)).cuda() for k in ("swag", "vanilla")}
    sw = B200SWAGRenderer()
    xyz = pcs["swag"].get_xyz.detach().cpu()
    sw.set_bbox(xyz.min(0).values, xyz.max(0).values)
    sw.swag_model = B200SWAGModel(sw.network_config, sw.grid_encoding_config, sw.embedding_config)
    sw = sw.cuda()
    sw.uniform_sampler = torch.distributions.uniform.Uniform(torch.tensor(0., device="cuda"), torch.tensor(1., device="cuda"))
    van = B200VanillaRenderer().cuda()

    def step(fn, pc):
        def run():
            out = fn(pc)
            out["render"].sum().backward()
        return run
    step_med, step_rng = time_paths({"swag": step(lambda pc: sw.training_forward(0, None, cam, pc, bg), pcs["swag"]),
                                     "vanilla": step(lambda pc: van(cam, pc, bg), pcs["vanilla"])}, args, SLEEP_FWD_BWD)
    results["step_1080p_n%d" % n] = {"ms": step_med, "range_ms": step_rng}
    line = json.dumps({"metric": "swag", "degree": DEG, "grid": GRID, "hbm_peak_TBps": HBM_PEAK / 1e12, **card(), "results": results})
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
