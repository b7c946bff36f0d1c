"""Cost of the appearance-feature similarity regulariser (VanillaMetricsWithSimilarityRegularization, every
similarity_reg_interval steps): the k-NN query (b200gs.ops.knn_points) and the fused term (b200gs.ops.similarity_regularization,
K43-K46) against the reference's torch formula (SimilarityRegularizationMixin.get_similarity_metric after knn_points, restated
below: the gather, F.normalize, the [S,K,K,D] broadcast product, the column weights, the triangular mask and the mean) fed with the
same idx, alternated in one process.  The scene is clustered synthetic: 1 M or 3 M Gaussians around 2 000 centres, optionally with 1 % of them spread over a
box 1000x wider (the grid is uniform over the bounding box, so far-flung points crowd the rest into fewer cells).
    knn:    S = 20 480 sampled queries, K = 16, at N = 1 M and 3 M, and at 1 M with outliers; and SegAny's call, all N queries at 1 M
    term:   the defaults (S = 20 480, K = 16, D = 64, Cosine, decay 200, lambda 0.2) at N = 1 M, forward and forward + backward
Timing as profiles/tools/exposure_bench.py: CUDA events around blocks of calls behind a device-side sleep, medians and min-max over
the blocks; kernel times of forward + backward from a separate torch.profiler run; the card's name and power limit read in
the same call.  pytorch3d's own knn_points is not installed here, so its time
is not measured.  Writes one JSON line to stdout and to --out.

    python profiles/tools/similarity_reg_bench.py [--calls 40] [--block 4] [--warmup 4] [--out profiles/similarity_reg_bench_h100.json]
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
import torch  # noqa: E402

from b200gs import ops  # noqa: E402
from exposure_bench import HBM_PEAK, card, time_paths  # noqa: E402

S, K, D, DECAY, LAMBDA = 20_480, 16, 64, 200.0, 0.2


def scene(n, seed, outliers=0.0):
    """clustered points; `outliers` of them spread over a box 1000x wider, as sky and background Gaussians of an unbounded capture"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    centers = torch.rand(2000, 3, generator=g, device="cuda") * 20
    p = centers[torch.randint(0, 2000, (n,), generator=g, device="cuda")] + 0.2 * torch.randn(n, 3, generator=g, device="cuda")
    far = torch.rand(n, generator=g, device="cuda") < outliers
    p[far] = (torch.rand(int(far.sum()), 3, generator=g, device="cuda") - 0.5) * 20_000
    return p


KERNELS = ("similarity_fwd", "similarity_reduce", "similarity_bwd_entry", "hist4", "onesweep_pass", "similarity_runs",
           "similarity_bwd_gather")


def kernel_times(fn, n):
    """mean device time (us) per call of each library kernel over n calls of fn, from a torch.profiler trace"""
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
                out[k] = round(out.get(k, 0.0) + e.device_time_total / n, 1)
    return out


def torch_term(features, idx, dists):
    """the reference's formula (Cosine) on the same idx / dists"""
    w = torch.exp(-DECAY * dists)
    g = features[idx]
    n = torch.nn.functional.normalize(g, dim=-1)
    raw = -(n[:, :, None, :] * n[:, None, :, :]).sum(dim=-1)
    weighted = raw * w[:, None, :]
    triu = torch.triu(torch.ones(raw.shape[1:3], dtype=torch.bool, device=raw.device), diagonal=1)
    return weighted[:, triu].mean() * LAMBDA


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--block", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("similarity_reg_bench needs a CUDA device")
    results = {}
    few = argparse.Namespace(calls=4, block=2, warmup=1)      # the outlier scene runs near brute force: fewer calls
    for n, outliers in ((1_000_000, 0.0), (3_000_000, 0.0), (1_000_000, 0.01)):
        pts = scene(n, n, outliers)
        q = pts[torch.randperm(n, device="cuda")[:S]]
        med, spread = time_paths({"fused": lambda: ops.knn_points(q, pts, K)}, few if outliers else args, 10_000_000)
        results[f"knn_S{S}_K{K}_N{n}" + (f"_outliers{outliers}" if outliers else "")] = {"us": round(med["fused"] * 1e3, 1), "us_min_max": [round(x * 1e3, 1) for x in spread["fused"]],
                                          "speedup_vs_pytorch3d": "not measured"}
    pts = scene(1_000_000, 5)
    med, spread = time_paths({"fused": lambda: ops.knn_points(pts, pts, K)}, few, 10_000_000)
    results["knn_segany_all_N1000000_K16"] = {"ms": round(med["fused"], 3), "ms_min_max": [round(x, 3) for x in spread["fused"]],
                                              "speedup_vs_pytorch3d": "not measured"}

    n = 1_000_000
    q = pts[torch.randperm(n, device="cuda")[:S]]
    dists, idx = ops.knn_points(q, pts, K)
    feats = torch.randn(n, D, device="cuda", requires_grad=True)

    def fused_fwd():
        with torch.no_grad():
            ops.similarity_regularization(feats, idx, dists, decay=DECAY, weight=LAMBDA)

    def torch_fwd():
        with torch.no_grad():
            torch_term(feats, idx, dists)

    def fused_fb():
        ops.similarity_regularization(feats, idx, dists, decay=DECAY, weight=LAMBDA)[0].backward()

    def torch_fb():
        torch_term(feats, idx, dists).backward()

    torch.cuda.reset_peak_memory_stats()
    for name, paths, sleep in (("term_fwd", {"fused": fused_fwd, "torch": torch_fwd}, 10_000_000),
                               ("term_fwd_bwd", {"fused": fused_fb, "torch": torch_fb}, 80_000_000)):
        med, spread = time_paths(paths, args, sleep)
        results[name] = {"fused_us": round(med["fused"] * 1e3, 1), "torch_us": round(med["torch"] * 1e3, 1),
                         "speedup": round(med["torch"] / med["fused"], 2),
                         "fused_us_min_max": [round(x * 1e3, 1) for x in spread["fused"]],
                         "torch_us_min_max": [round(x * 1e3, 1) for x in spread["torch"]]}
    # algorithmic bytes: the gathered rows and idx / dists in the forward; the backward also writes and reads back the per-entry
    # rows, sorts 8-byte records (histogram + 3 passes, each reading and writing them) and writes the dense [N,D] gradient
    e = S * K
    fwd_bytes = e * (D * 4 + 12)
    bwd_bytes = e * (D * 4 + 12) + 2 * e * D * 4 + e * 8 * (1 + 2 * 3 + 1) + n * D * 4
    results["term_fwd"]["fused_GBps"] = round(fwd_bytes / (results["term_fwd"]["fused_us"] * 1e-6) / 1e9, 1)
    results["term_fwd_bwd"]["fused_GBps"] = round((fwd_bytes + bwd_bytes) / (results["term_fwd_bwd"]["fused_us"] * 1e-6) / 1e9, 1)
    results["term_bytes"] = {"fwd": fwd_bytes, "bwd": bwd_bytes, "torch_SKKD_intermediate": S * K * K * D * 4}
    results["kernels_us_fwd_bwd"] = kernel_times(fused_fb, 20)
    results["peak_memory_MB"] = round(torch.cuda.max_memory_allocated() / 2 ** 20, 1)
    line = json.dumps({"metric": "similarity_regularization", "hbm_peak_GBps": HBM_PEAK / 1e9, **card(), "results": results})
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
