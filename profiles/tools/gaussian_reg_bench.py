"""Per-step cost of the Gaussian regularisers: the fused kernels (b200gs.metrics.gaussian_regularizers, K36-K38) against the
reference's torch formulation (MCMCMetricsModuleMixin.reg_loss of internal/metrics/mcmc_metrics.py and
ScaleRegularizationMetricsModuleMixin.get_scale_regularization_metrics of scale_regularization_metrics.py, restated below),
alternated in one process.  N = 1 M and 3 M raw Gaussians; the MCMC terms, the scale terms with their statistics, and the whole
training metric (RGB L1 + SSIM at 1080p and the MCMC or scale terms) through B200MCMCMetricsModule /
B200ScaleRegularizationMetricsModule against the reference's formulation of it; forward and forward + backward.
Timing as profiles/tools/exposure_bench.py: CUDA events around blocks of calls behind a device-side sleep, medians and min-max over
the blocks; kernel times from a separate torch.profiler run against each kernel's algorithmic bytes; the card's name and power
limit read in the same call.  Prints one JSON line.

    python profiles/tools/gaussian_reg_bench.py [--calls 200] [--block 10] [--warmup 20]
"""
import argparse
import json
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
import torch  # noqa: E402

from b200gs.metrics import B200MCMCMetrics, B200ScaleRegularizationMetrics, gaussian_regularizers  # noqa: E402
from b200gs.scene import SyntheticGaussians  # noqa: E402
from depth_loss_bench import torch_rgb_ssim  # noqa: E402
from exposure_bench import HBM_PEAK, SLEEP_FWD, SLEEP_FWD_BWD, card, row, time_paths  # noqa: E402

KERNELS = ("reg_partials", "reg_reduce", "reg_bwd")
MAX_SCALE, W_O, W_S, LAM, LAM_R = 0.5, 0.01, 0.01, 0.05, 0.05


def torch_mcmc(opacities, scales):
    """reg_loss's two terms as the reference evaluates them on the raw parameters"""
    return W_O * torch.abs(torch.sigmoid(opacities)).mean() + W_S * torch.abs(torch.exp(scales)).mean()


def torch_scale(scales):
    """the over-scale and over-ratio terms with their statistics, in the reference's order of operations (a sort of [N,3], two
    masks, masked sums over count + 1, and the statistics without autograd)"""
    s = torch.exp(scales)
    ranked = torch.sort(s, dim=-1).values
    ratio = ranked[:, 2] / (ranked[:, 1] + 1e-8)
    total = 0.0
    for values, sel, lam in ((s, s.detach() > MAX_SCALE, LAM), (ratio, ratio.detach() > 10., LAM_R)):
        count = sel.sum().float()
        total = total + (values * sel).sum() / (count + 1) * lam
    with torch.no_grad():
        stats = (ranked[:, 2].max(), ratio.max(), ratio.mean())
    return total, stats


def kernel_bytes(n, which):
    """algorithmic bytes (b200gs.h): 4 B opacity and 12 B scales per Gaussian in, the same out in the backward, plus the partials"""
    blocks = min(-(-n // 1024), 2048)
    per = {"mcmc": 16, "scale": 12}[which]
    return {"reg_partials": per * n + 36 * blocks, "reg_reduce": 36 * blocks, "reg_bwd": 2 * per * n}


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
        sys.exit("gaussian_reg_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    gen = torch.Generator().manual_seed(0)
    results, kernels, metric_rows = [], [], []
    H, W = 1080, 1920
    render = torch.rand(3, H, W, generator=gen).to(dev).requires_grad_(True)
    gt_rgb = torch.rand(3, H, W, generator=gen).to(dev)
    for n in (1_000_000, 3_000_000):
        o = (torch.randn(n, 1, generator=gen) * 3).to(dev).requires_grad_(True)
        s = (torch.randn(n, 3, generator=gen) * 1.5 - 3).to(dev).requires_grad_(True)
        arms = {
            "mcmc": (lambda: gaussian_regularizers(o, s, raw=True, opacity_weight=W_O, scale_weight=W_S, statistics=False).sum(),
                     lambda: torch_mcmc(o, s)),
            "scale": (lambda: gaussian_regularizers(None, s, raw=True, max_scale=MAX_SCALE, scale_lambda=LAM, ratio_lambda=LAM_R)[0].sum(),
                      lambda: torch_scale(s)[0]),
        }
        for which, (fused, reference) in arms.items():
            with torch.no_grad():
                med, spread = time_paths({"fused": fused, "torch": reference}, args, SLEEP_FWD)
            results.append({"what": "fwd", "n": n, "terms": which, **row(med, spread)})
            med, spread = time_paths({"fused": lambda: fused().backward(), "torch": lambda: reference().backward()}, args, SLEEP_FWD_BWD)
            results.append({"what": "fwd_bwd", "n": n, "terms": which, **row(med, spread)})
            us = kernel_times(lambda: fused().backward(), args.profile_calls)
            nbytes = kernel_bytes(n, which)
            kernels.append({"n": n, "terms": which,
                            "kernels": {k: {"us": round(t, 2), "algorithmic_MB": round(nbytes[k] / 1e6, 2),
                                            "GB_per_s": round(nbytes[k] / (t * 1e-6) / 1e9, 1),
                                            "share_of_hbm_bound": round(nbytes[k] / HBM_PEAK / (t * 1e-6), 3)} for k, t in us.items()}})
            o.grad, s.grad = None, None
        # the whole training metric: RGB L1 + SSIM at 1080p and the regularisers, forward + backward
        model = SyntheticGaussians({"means": torch.zeros(n, 3), "scales": torch.zeros(n, 3), "rotations": torch.zeros(n, 4),
                                    "opacities": torch.zeros(n, 1), "shs_dc": torch.zeros(n, 1, 3), "shs_rest": torch.zeros(n, 15, 3)}).to(dev)
        with torch.no_grad():
            model.gaussians["opacities"].copy_(o)
            model.gaussians["scales"].copy_(s)
        cam = types.SimpleNamespace(device=dev)
        for which, cls, kw in (("mcmc", B200MCMCMetrics, {}), ("scale", B200ScaleRegularizationMetrics, {"max_scale": MAX_SCALE})):
            metric = cls(**kw).instantiate()
            metric.setup("fit", None)

            def fused_metric():
                metrics, _ = metric.get_train_metrics(None, model, 5000, (cam, ("img", gt_rgb, None), None), {"render": render})
                metrics["loss"].backward()

            def reference_metric():
                rgb = 0.8 * torch.abs(render - gt_rgb).mean() + 0.2 * (1 - torch_rgb_ssim(render, gt_rgb))
                p = model.gaussians
                extra = torch_mcmc(p["opacities"], p["scales"]) if which == "mcmc" else torch_scale(p["scales"])[0]
                (rgb + extra).backward()

            med, spread = time_paths({"fused": fused_metric, "torch": reference_metric}, args, SLEEP_FWD_BWD)
            metric_rows.append({"what": "metric_fwd_bwd", "n": n, "terms": which, "image": [H, W], **row(med, spread)})
            render.grad = None
            model.zero_grad(set_to_none=True)
        del o, s, model
    print(json.dumps({"metric": "gaussian_regularizers", "hbm_peak_GBps": HBM_PEAK / 1e9, **card(), "results": results,
                      "whole_metric": metric_rows, "fused_kernels_fwd_bwd": kernels}))


if __name__ == "__main__":
    main()
