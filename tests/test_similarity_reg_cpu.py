"""CPU checks of the similarity regulariser: the float64 oracle against the recorded reference module (tests/golden/similarity_reg.*),
the config fields and defaults, the pytorch3d drop-in's import hook and refusals, and the C ABI's argument validation (rejected
before any CUDA call, so no GPU is needed)."""
import ctypes
import dataclasses
import json
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle import similarity_reg_oracle as O

META = json.load(open(os.path.join(GOLDEN, "similarity_reg.json")))
Z = np.load(os.path.join(GOLDEN, "similarity_reg.npz"))


def golden_inputs(c):
    sys.path.insert(0, GOLDEN)
    try:
        from make_golden_similarity_reg import inputs
    finally:
        sys.path.remove(GOLDEN)
    return inputs(c["n"], c["points"], c["features"], c["seed"])


@pytest.mark.parametrize("c", META["cases"], ids=lambda c: c["key"])
def test_oracle_reproduces_the_recorded_module(c):
    k, cfg = c["key"], c["config"]
    means, features = golden_inputs(c)
    samples = torch.from_numpy(Z[f"{k}_samples"]).long()
    assert samples.shape[0] == min(cfg["n_appearance_samples"], c["n"])
    d, i, _ = O.knn(means[samples], means, cfg["n_appearance_nn"])
    assert torch.equal(i, torch.from_numpy(Z[f"{k}_idx"]).long())
    assert torch.equal(d.float(), torch.from_numpy(Z[f"{k}_dists"]))
    loss, mean, grad = O.similarity_grad(features, i, d.float(), cfg["distance_weight_decay"], cfg["similarity_reg_lambda"], c["kind"])
    ref_loss, ref_grad = float(Z[f"{k}_loss"]), Z[f"{k}_grad"]
    assert abs(float(loss) - ref_loss) <= 1e-5 * abs(ref_loss) + 1e-12
    assert abs(float(mean) - float(Z[f"{k}_as_r"])) <= 1e-5 * abs(float(Z[f"{k}_as_r"])) + 1e-12
    assert np.abs(grad.numpy() - ref_grad).max() <= 1e-4 * np.abs(ref_grad).max() + 1e-8
    l32, _, g32 = O.similarity_grad(features, i, d.float(), cfg["distance_weight_decay"], cfg["similarity_reg_lambda"], c["kind"],
                                    torch.float32)
    assert abs(float(l32) - ref_loss) <= 1e-6 * abs(ref_loss) + 1e-12           # the fp32 restatement is the reference's arithmetic


def test_recorded_edge_cases():
    cases = {c["key"]: c for c in META["cases"]}
    assert float(Z["cos_zero_loss"]) == 0.0 and float(Z["euc_zero_loss"]) == 0.0 and float(Z["euc_underflow_loss"]) == 0.0
    assert not np.any(Z["euc_zero_grad"]) and not np.any(Z["euc_underflow_grad"])
    assert np.abs(Z["cos_zero_row_grad"]).max() > 1e6                               # F.normalize's 1/eps branch
    assert cases["euc_k32_d33"]["hook_called"] == [s >= 60 and s % 20 == 0 for s in META["steps"]]
    assert cases["cos_k16_d64"]["hook_called"] == [s % 50 == 0 for s in META["steps"]]


def test_config_fields_and_defaults_match_the_reference():
    from b200gs.metrics import B200VanillaMetricsWithSimilarityRegularization
    cfg = B200VanillaMetricsWithSimilarityRegularization()
    assert {f.name: getattr(cfg, f.name) for f in dataclasses.fields(cfg)} == META["config"]


def test_similarity_type_forms():
    from b200gs.metrics import B200VanillaMetricsWithSimilarityRegularization, Cosine, Euclidean, _similarity_kind

    class ReferenceCosine:            # the reference's classes are matched by name
        pass
    ReferenceCosine.__name__ = "Cosine"
    assert _similarity_kind({"class_path": "Cosine"}) == "cosine"
    assert _similarity_kind({"class_path": "internal.metrics.appearance_feature_similarity_regularization_metrics.Euclidean"}) == "euclidean"
    assert _similarity_kind(Cosine()) == "cosine" and _similarity_kind(Euclidean()) == "euclidean"
    assert _similarity_kind(ReferenceCosine()) == "cosine"
    with pytest.raises(NotImplementedError):
        B200VanillaMetricsWithSimilarityRegularization(similarity_type={"class_path": "Manhattan"}).instantiate()


def test_pytorch3d_appears_only_on_import_and_refuses():
    import subprocess
    code = ("import sys, b200gs.compat as c; c.install(); assert not any(m.startswith('pytorch3d') for m in sys.modules); "
            "from pytorch3d.ops import knn_points, KNN; assert knn_points is c.knn_points and 'pytorch3d.ops' in sys.modules\n"
            "try:\n    import pytorch3d.ops.iou_box3d\nexcept ImportError as e:\n    assert 'knn_points' in str(e)\n"
            "else:\n    raise SystemExit('iou_box3d imported')\n"
            "import torch\np = torch.zeros(1, 4, 3)\n"
            "for kw in ({'norm': 1}, {'return_nn': True}, {'return_sorted': False}, {'lengths2': torch.tensor([4])}):\n"
            "    try:\n        knn_points(p, p, K=2, **kw)\n    except NotImplementedError as e:\n        assert 'norm=2' in str(e)\n"
            "    else:\n        raise SystemExit(kw)\n"
            "try:\n    knn_points(p.requires_grad_(True), p, K=2)\nexcept NotImplementedError:\n    pass\n"
            "else:\n    raise SystemExit('grad')\n")
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_abi_validation_without_gpu():
    from b200gs import _lib
    from b200gs import ops
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    L = _lib.lib()
    d = ctypes.c_void_p(256)
    # knn_points: K range, K > N, NULL pointers
    for s, n, k, msg in ((4, 10, 0, b"1..32"), (4, 10, 33, b"1..32"), (4, 10, 11, b"K exceeds"), (-1, 10, 2, b"negative")):
        assert L.b200gs_knn_points(s, d, n, d, k, d, d, d, 1 << 30, None) == -1
        assert msg in L.b200gs_last_error()
    assert L.b200gs_knn_points(4, None, 10, d, 2, d, d, d, 1 << 30, None) == -1 and b"NULL" in L.b200gs_last_error()
    assert L.b200gs_knn_points(4, d, 10, d, 2, d, d, d, 16, None) == -3 and b"workspace" in L.b200gs_last_error()
    assert L.b200gs_knn_points(4, d, 1 << 30, d, 2, d, d, d, 1 << 62, None) == -3 and b"2^30" in L.b200gs_last_error()
    # similarity: D, K, kind, sizes, NULL pointers, workspace
    assert int(L.b200gs_similarity_reg_workspace_bytes(100, 8, 16, 64, 0)) == 256             # the forward's 8 per-sample sums
    ws = int(L.b200gs_similarity_reg_workspace_bytes(100, 8, 16, 64, 1))
    assert ws >= 8 * 16 * (64 * 4 + 16) + 100 * 8
    for args, msg in (((100, 0, 8, 16, 0), b"dimension"), ((100, 257, 8, 16, 0), b"dimension"), ((100, 64, 8, 1, 0), b"2..32"),
                      ((100, 64, 8, 33, 0), b"2..32"), ((100, 64, 8, 16, 2), b"kind"), ((100, 64, 0, 16, 0), b">= 1"),
                      ((0, 64, 8, 16, 0), b">= 1"), ((1 << 30, 64, 8, 16, 0), b"2^30")):
        n, dd, s, k, kind = args
        assert L.b200gs_similarity_reg_fwd(n, dd, d, s, k, d, d, kind, 200.0, 0.2, d, 1 << 40, d, None, None) == -1, args
        assert L.b200gs_similarity_reg_workspace_bytes(n, s, k, dd, 1) == 0 or kind == 2, args
        assert msg in L.b200gs_last_error(), (args, L.b200gs_last_error())
        assert L.b200gs_similarity_reg_bwd(n, dd, d, s, k, d, d, kind, 200.0, 0.2, d, 1 << 40, d, d, None) == -1, args
    assert L.b200gs_similarity_reg_fwd(100, 64, None, 8, 16, d, d, 0, 200.0, 0.2, d, ws, d, None, None) == -1
    assert b"NULL" in L.b200gs_last_error()
    assert L.b200gs_similarity_reg_fwd(100, 64, d, 8, 16, d, d, 0, 200.0, 0.2, d, ws, None, None, None) == -1
    assert L.b200gs_similarity_reg_bwd(100, 64, d, 8, 16, d, d, 0, 200.0, 0.2, d, ws, None, d, None) == -1
    assert L.b200gs_similarity_reg_fwd(100, 64, d, 8, 16, d, d, 0, 200.0, 0.2, d, 255, d, None, None) == -3
    assert b"workspace" in L.b200gs_last_error()
    assert L.b200gs_similarity_reg_bwd(100, 64, d, 8, 16, d, d, 0, 200.0, 0.2, d, ws - 1, d, d, None) == -3
    assert b"workspace" in L.b200gs_last_error()
    for args in ((100, 0, 16, 64), (100, 8, 1, 64), (100, 8, 33, 64), (100, 8, 16, 0), (100, 8, 16, 257), (0, 8, 16, 64)):
        assert L.b200gs_similarity_reg_workspace_bytes(*args, 1) == 0
    # the Python layer refuses before the library
    with pytest.raises(NotImplementedError):
        ops.similarity_regularization(torch.zeros(4, 2), torch.zeros(1, 2, dtype=torch.int64), torch.zeros(1, 2), decay=1.0,
                                      weight=1.0, kind="manhattan")
    with pytest.raises(ValueError):
        ops.similarity_regularization(torch.zeros(4, 300), torch.zeros(1, 2, dtype=torch.int64), torch.zeros(1, 2), decay=1.0,
                                      weight=1.0)
    assert ops.knn_launches(300_000) == 9 and ops.similarity_bwd_launches(300_000) == 7 and ops.similarity_bwd_launches(2) == 5


SIZING_HARNESS = r"""
#include <cstdio>
#include <cstdlib>
#include "knn_grid.h"
int main(int argc, char** argv) {
    float lo[3], hi[3];
    for (int a = 0; a < 3; ++a) { lo[a] = strtof(argv[1 + a], nullptr); hi[a] = strtof(argv[4 + a], nullptr); }
    const long long n = atoll(argv[7]);
    const b200gs::KnnGrid g = b200gs::size_knn_grid(lo, hi, n, 4 * n + 64);
    printf("%d %d %d %.9g %.9g %.9g %.9g %.9g\n", g.gx, g.gy, g.gz, g.cs, g.inv_cs, g.lox, g.loy, g.loz);
    return 0;
}
"""


def test_grid_sizing_terminates_on_any_box(tmp_path):
    """knn_grid.h's size_knn_grid, the code knn_grid_kernel runs in one device thread, compiled for the host: every box, including
    infinite, NaN, empty (no finite point) and overflowing ones, gives a grid within the caps, with a finite cell size, in bounded time"""
    import shutil
    import subprocess
    cxx = shutil.which("g++") or shutil.which("c++") or shutil.which("clang++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    src, exe = tmp_path / "sizing.cpp", tmp_path / "sizing"
    src.write_text(SIZING_HARNESS)
    subprocess.run([cxx, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "gaussian-splatting-lightning_b200", "csrc"), str(src), "-o", str(exe)],
                   check=True, timeout=120)
    inf, nan = "inf", "nan"
    boxes = [
        ((0, 0, 0), (1, 1, 1), 1_000_000),                  # an ordinary box
        ((0, 0, 0), (0, 0, 0), 10),                         # one point, repeated
        ((-1, 0, 0), (1, 0, 0), 1000),                      # collinear
        ((-3e38, -3e38, -3e38), (3e38, 3e38, 3e38), 1000),  # the float width overflows
        (("-" + inf, 0, 0), (inf, 1, 1), 1000),             # infinite bounds
        ((nan, nan, nan), (nan, nan, nan), 1000),           # no finite point: the zeroed bounds decode to NaN
        ((1, 1, 1), (0, 0, 0), 1000),                       # empty box (lo > hi)
        ((0, 0, 0), (1e-40, 1e-40, 1e-40), 100),            # denormal extents
        ((0, 0, 0), (3.4e38, 1e-30, 1), 1 << 29),           # extreme aspect ratio at the largest n
    ]
    for lo, hi, n in boxes:
        r = subprocess.run([str(exe), *map(str, lo), *map(str, hi), str(n)], capture_output=True, text=True, timeout=10)
        assert r.returncode == 0, (lo, hi, r.stderr)
        gx, gy, gz = map(int, r.stdout.split()[:3])
        cs, inv_cs, lox, loy, loz = map(float, r.stdout.split()[3:])
        assert all(1 <= g <= 1024 for g in (gx, gy, gz)) and gx * gy * gz <= 4 * n + 64, (lo, hi, r.stdout)
        assert all(np.isfinite(v) for v in (cs, inv_cs, lox, loy, loz)) and cs > 0 and inv_cs > 0, (lo, hi, r.stdout)
    r = subprocess.run([str(exe), "0", "0", "0", "1", "1", "1", "1000000"], capture_output=True, text=True, timeout=10)
    gx, gy, gz = map(int, r.stdout.split()[:3])
    assert 2e5 <= gx * gy * gz <= 4e6        # about two points per cell in an ordinary box
