"""Freeze the reference's appearance-feature similarity regulariser: the unmodified VanillaMetricsWithSimilarityRegularization /
VanillaMetricsWithSimilarityRegularizationModule of internal/metrics/appearance_feature_similarity_regularization_metrics.py, run on the
CPU in float32.  pytorch3d is not installed: ``pytorch3d.ops.knn_points`` is oracle.similarity_reg_oracle.knn (float64 brute force,
ties to the lower index), its distances rounded to float32.  torchmetrics' PSNR and LPIPS are inert stand-ins.
Each case seeds torch's global generator and calls the module's ``similarity_metric_backward_hook`` through ``training_setup`` at the
steps in STEPS with a stand-in LightningModule (``manual_backward`` = ``backward``, ``log`` recorded).
Recorded per case (the means and features are rebuilt from the seeds by ``inputs``): the sample indices, knn idx and dists, loss, as_r and the appearance-feature gradient of the
first call (step 0 or the first step the hook runs), and which steps ran the hook.  Also recorded: the config fields and defaults
and the log call's keyword arguments.
Run:  python tests/golden/make_golden_similarity_reg.py <reference checkout>     -> tests/golden/similarity_reg.npz, .json"""
import dataclasses
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import similarity_reg_oracle as O  # noqa: E402

STEPS = [0, 1, 20, 49, 50, 60, 80, 100]
# (key, kind, N, points, features, seed, config)
CASES = [("cos_k16_d64", "cosine", 300, "uniform", "randn", 1, {"n_appearance_samples": 64, "n_appearance_nn": 16}),
         ("euc_k16_d64", "euclidean", 300, "uniform", "randn", 2, {"n_appearance_samples": 64, "n_appearance_nn": 16}),
         ("cos_k2_d1", "cosine", 200, "uniform", "randn1", 3, {"n_appearance_samples": 48, "n_appearance_nn": 2}),
         ("euc_k32_d33", "euclidean", 200, "uniform", "randn33", 4, {"n_appearance_samples": 40, "n_appearance_nn": 32,
                                                                     "similarity_reg_from": 60, "similarity_reg_interval": 20}),
         ("cos_s_gt_n", "cosine", 40, "uniform", "randn33", 5, {"n_appearance_samples": 64, "n_appearance_nn": 16}),
         ("euc_duplicated", "euclidean", 200, "duplicated", "randn", 6, {"n_appearance_samples": 48, "n_appearance_nn": 16}),
         ("cos_zero", "cosine", 120, "uniform", "zero", 7, {"n_appearance_samples": 32, "n_appearance_nn": 16}),
         ("euc_zero", "euclidean", 120, "uniform", "zero", 8, {"n_appearance_samples": 32, "n_appearance_nn": 16}),
         ("cos_zero_row", "cosine", 120, "uniform", "zero_row", 9, {"n_appearance_samples": 32, "n_appearance_nn": 16}),
         ("euc_underflow", "euclidean", 120, "uniform", "randn", 10, {"n_appearance_samples": 32, "n_appearance_nn": 16,
                                                                      "distance_weight_decay": 1e9}),
         ("cos_lambda", "cosine", 150, "uniform", "randn", 11, {"n_appearance_samples": 50, "n_appearance_nn": 16,
                                                                "distance_weight_decay": 20.0, "similarity_reg_lambda": 0.7})]


def inputs(n, points, features, seed):
    """(means [n,3], features [n,D]) float32 CPU"""
    g = torch.Generator().manual_seed(seed)
    means = torch.rand(n, 3, generator=g) * 0.1
    if points == "duplicated":
        means[n // 2:] = means[torch.randint(0, n // 2, (n - n // 2,), generator=g)]
    d = 64 if features in ("randn", "zero", "zero_row") else int(features[5:])
    f = torch.randn(n, d, generator=g)
    if features == "zero":
        f.zero_()
    elif features == "zero_row":
        f[:: 7] = 0.0
    return means, f


if __name__ == "__main__":
    sys.path.insert(0, sys.argv[1])

    class _Inert:
        def __init__(self, *args, **kwargs):
            pass

    KNN = __import__("collections").namedtuple("KNN", ["dists", "idx", "knn"])

    def knn_points(p1, p2, K=1, **kwargs):
        d, i, _ = O.knn(p1[0], p2[0], K)
        return KNN(d.float()[None], i[None], None)

    for name in ("torchmetrics", "torchmetrics.image", "torchmetrics.image.lpip", "pytorch3d", "pytorch3d.ops"):
        sys.modules[name] = types.ModuleType(name)
    sys.modules["torchmetrics.image"].PeakSignalNoiseRatio = _Inert
    sys.modules["torchmetrics.image.lpip"].LearnedPerceptualImagePatchSimilarity = _Inert
    sys.modules["pytorch3d.ops"].knn_points = knn_points

    from internal.metrics.appearance_feature_similarity_regularization_metrics import (  # noqa: E402
        Cosine, Euclidean, VanillaMetricsWithSimilarityRegularization)

    class Model:
        def __init__(self, means, features):
            self.means, self.features = means, features

        def get_means(self):
            return self.means

        def get_appearance_features(self):
            return self.features

    class Module:
        batch_size = 1

        def __init__(self):
            self.on_after_backward_hooks, self.logged = [], []

        def manual_backward(self, loss):
            loss.backward()

        def log(self, name, value, **kwargs):
            self.logged.append((name, float(value), kwargs))

    arrays, meta = {}, {"steps": STEPS, "cases": []}
    cfg0 = VanillaMetricsWithSimilarityRegularization()
    meta["config"] = {f.name: getattr(cfg0, f.name) for f in dataclasses.fields(cfg0)}
    for key, kind, n, points, features, seed, config in CASES:
        means, f = inputs(n, points, features, seed)
        sim = Cosine() if kind == "cosine" else Euclidean()
        metric = VanillaMetricsWithSimilarityRegularization(similarity_type=sim, **config).instantiate()
        pl = Module()
        metric.training_setup(pl) if hasattr(metric, "training_setup") else None
        hook = pl.on_after_backward_hooks[0]
        called, first = [], None
        for step in STEPS:
            x = f.clone().requires_grad_(True)
            torch.manual_seed(seed * 1000 + step)
            n_logged = len(pl.logged)
            hook(None, None, Model(means, x), step, pl)
            ran = len(pl.logged) > n_logged
            called.append(ran)
            if ran and first is None:
                torch.manual_seed(seed * 1000 + step)
                loss, m, _ = metric.get_similarity_metric(Model(means, f))
                first = step
                arrays[f"{key}_samples"] = m[0].numpy().astype(np.int32)
                arrays[f"{key}_idx"] = m[1].idx[0].numpy().astype(np.int32)
                arrays[f"{key}_dists"] = m[1].dists[0].numpy()
                arrays[f"{key}_loss"] = np.float32(loss.item())
                arrays[f"{key}_as_r"] = np.float32(pl.logged[-1][1])
                arrays[f"{key}_grad"] = x.grad.numpy()
                meta["log_kwargs"] = pl.logged[-1][2]
        full = {**{k: v for k, v in meta["config"].items() if k != "similarity_type"}, **config}
        meta["cases"].append({"key": key, "kind": kind, "seed": seed, "points": points, "features": features, "n": n,
                              "config": {k: full[k] for k in ("n_appearance_samples", "n_appearance_nn", "distance_weight_decay",
                                                              "similarity_reg_from", "similarity_reg_lambda",
                                                              "similarity_reg_interval")},
                              "hook_called": called, "first_step": first})
    np.savez_compressed(os.path.join(HERE, "similarity_reg.npz"), **arrays)
    json.dump(meta, open(os.path.join(HERE, "similarity_reg.json"), "w"), indent=1, default=str)
