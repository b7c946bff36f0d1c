"""Gaussian regularisers without a GPU: the float64 oracle (oracle/gaussian_reg_oracle.py) against the reference's own
MCMCMetrics, ScaleRegularizationMetrics and ScaleRegularizationWithDepthMetrics modules (tests/golden/gaussian_reg.npz), the
plug-in configs' fields, defaults, asserts and class order against the reference's, and the argument validation of the C ABI
(every bad argument rejected before any CUDA call, nothing launched) with its workspace formula."""
import ctypes
import dataclasses
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import gaussian_reg_oracle as O

Z = np.load(os.path.join(GOLDEN, "gaussian_reg.npz"))
META = json.load(open(os.path.join(GOLDEN, "gaussian_reg.json")))
DEFAULTS = {"mcmc": {"mcmc_reg_until_iter": -1, "opacity_reg": 0.01, "scale_reg": 0.01, "reg_weight_decay": 1.0},
            "scale": {"scale_reg_from": 3100, "max_scale": -1, "max_scale_outside_partition": None, "max_scale_ratio": 10,
                      "scale_reg_lambda": 0.05, "scale_ratio_reg_lambda": 0.05}}


def expected(c):
    """the oracle's (terms, stats, v_opacities, v_scales) for a recorded case, or None when the case adds no regulariser"""
    cfg = {**META["config"][c["metric"]], **c["config"]}
    si = c["scene"]
    opac, scales = Z[f"s{si}_opacities"], Z[f"s{si}_scales"]
    if c["metric"] == "mcmc":
        if c["stage"] == "train" and cfg["mcmc_reg_until_iter"] >= 0 and c["step"] >= cfg["mcmc_reg_until_iter"]:
            return None
        decay = min(cfg["reg_weight_decay"], 5.)
        return O.vjp(opac, scales, True, [1, 1, 0, 0], opacity_weight=cfg["opacity_reg"] / decay,
                     scale_weight=cfg["scale_reg"] / decay)
    if c["stage"] == "train" and c["step"] < cfg["scale_reg_from"]:
        return None
    return O.vjp(None, scales, True, [0, 0, 1, 1], max_scale=c["resolved_max_scale"], max_scale_ratio=cfg["max_scale_ratio"],
                 scale_lambda=cfg["scale_reg_lambda"], ratio_lambda=cfg["scale_ratio_reg_lambda"],
                 masks=flip_checked_masks(scales, c["resolved_max_scale"], cfg["max_scale_ratio"]))


def flip_checked_masks(scales, max_scale, max_ratio, raw=True, ulps=8):
    """The fp32 decisions of the two masks, after checking that they differ from float64's only on elements the oracle marks as
    within a few ulps of their threshold, and that such elements are rare"""
    m32 = tuple(m.cpu() for m in O.fp32_masks(scales, raw, max_scale, max_ratio))     # on the scales' device: its fp32 exp
    s64 = torch.as_tensor(scales).cpu().double()
    s64 = torch.exp(s64) if raw else s64
    v = torch.sort(s64, dim=-1).values
    m64 = (s64 > max_scale, v[:, -1] / (v[:, -2] + 1e-8) > max_ratio)
    d = O.threshold_distance(torch.as_tensor(scales).cpu(), raw, max_scale, max_ratio)
    for a, b, dist in zip(m32, m64, d):
        flips = a != b
        assert bool((dist[flips] <= ulps * 2.0 ** -23).all()), dist[flips]
        assert int(flips.sum()) <= 8 + 1e-4 * flips.numel()
    return m32


@pytest.mark.parametrize("c", META["cases"], ids=lambda c: c["key"])
def test_oracle_matches_the_reference_modules(c):
    k, m = c["key"], c["metrics"]
    r = expected(c)
    if r is None:
        assert not ({"o_reg", "scale_reg"} & set(m)), k
        assert not Z[f"{k}_v_opacities"].any() and not Z[f"{k}_v_scales"].any()
        return
    terms, stats, v_o, v_s = r
    names = ("o_reg", "s_reg") if c["metric"] == "mcmc" else ("scale_reg", "scale_ratio_reg")
    for name in names:
        t = terms[O.TERMS.index(name)]
        assert abs(m[name] - t) <= 1e-5 * max(abs(t), 1e-6), (k, name, m[name], t)
    if c["metric"] != "mcmc":
        assert m["n_over_scales"] == stats[0] and m["n_over_ratios"] == stats[1], k
        for i, name in ((2, "max_scale"), (3, "max_ratio"), (4, "mean_ratio")):
            assert abs(m[name] - stats[i]) <= 1e-5 * abs(stats[i]), (k, name)
    slack = O.sigmoid_grad_slack(Z[f"s{c['scene']}_opacities"])
    for got, ref, name, extra in ((Z[f"{k}_v_opacities"], v_o, "v_opacities", slack), (Z[f"{k}_v_scales"], v_s, "v_scales", 0.0)):
        ref = np.zeros(got.shape) if ref is None else ref
        assert np.abs(got - ref).max() <= 1e-5 * max(np.abs(ref).max(), 1e-30), (k, name)
        # and row by row: the ratio term's rows with a tiny mid set the largest entry, which would hide the ordinary rows; raw
        # opacity rows also carry the conditioning of fp32's y (1 - y) near y = 1
        g2, r2 = got.reshape(len(got), -1), ref.reshape(len(ref), -1)
        assert (np.abs(g2 - r2) <= 1e-5 * np.abs(r2).max(1, keepdims=True) + extra * np.abs(r2) + 1e-30).all(), (k, name, "rows")


def test_loss_is_the_sum_in_the_reference_order():
    for c in META["cases"]:
        m = c["metrics"]
        base = m["rgb_diff"] * 0.8 + 0.2 * (1 - m["ssim"]) + m.get("d_reg", 0.0)
        extra = m.get("o_reg", 0.0) + m.get("s_reg", 0.0) + m.get("scale_reg", 0.0) + m.get("scale_ratio_reg", 0.0)
        assert abs(m["loss"] - (base + extra)) <= 1e-5 * abs(m["loss"]), c["key"]


def test_crafted_rows_hit_their_edges():
    o, s = O.crafted_rows()
    y = torch.sigmoid(torch.from_numpy(o)).numpy()
    e = torch.exp(torch.from_numpy(s)).numpy()
    assert y[4, 0] == 0 and y[5, 0] == 0 and y[6, 0] != 0
    assert e[4, 0] == 0 and e[5, 0] == 0 and e[6, 0] != 0
    assert e[7, 0] == O.MAX_SCALE
    ratios = [float(e[i, 1] / (e[i, 0] + np.float32(1e-8))) for i in (8, 9, 10)]
    assert ratios[0] < 10 < ratios[2] and ratios == sorted(ratios)
    d_s, d_r = O.threshold_distance(torch.from_numpy(s), True, O.MAX_SCALE, 10.0)
    assert float(d_s[7, 0]) == 0 and all(float(d_r[i]) < 1e-6 for i in (8, 9, 10))
    for i in O.TIED_ROWS:
        assert sorted(e[i])[0] == sorted(e[i])[1] and sorted(e[i])[2] / sorted(e[i])[1] > 10


def test_oracle_tie_rules():
    s = torch.tensor([[1., 1., 2.], [2., 1., 1.], [3., 3., 1.], [2., 2., 2.]])
    assert O.sort_scales(s, "stable").indices.tolist() == [[0, 1, 2], [1, 2, 0], [2, 0, 1], [0, 1, 2]]
    # torch.sort on the GPU (measured): its bitonic network routes ties by the pattern of the row, not by column order
    assert O.sort_scales(s, "device").indices.tolist() == [[1, 0, 2], [1, 2, 0], [2, 1, 0], [2, 1, 0]]
    x = torch.randn(1000, 3, dtype=torch.float64)
    assert torch.equal(O.sort_scales(x, "device").values, torch.sort(x, dim=-1).values)


def test_configs_match_the_reference():
    from b200gs import metrics as M
    for cls, kind, extra in ((M.B200MCMCMetrics, "mcmc", DEFAULTS["mcmc"]), (M.B200ScaleRegularizationMetrics, "scale", DEFAULTS["scale"]),
                             (M.B200ScaleRegularizationWithDepthMetrics, "depth", DEFAULTS["scale"])):
        ref = META["config"][kind]
        ours = {f.name: (dataclasses.asdict(f.default_factory()) if f.default_factory is not dataclasses.MISSING else f.default)
                for f in dataclasses.fields(cls)}
        assert list(ours) == list(ref) and ours == ref, kind
        assert {k: ref[k] for k in extra} == extra
    # the module classes keep the reference's order of mixins and bases
    for cls, kind in ((M.B200MCMCMetrics, "mcmc"), (M.B200ScaleRegularizationMetrics, "scale"),
                      (M.B200ScaleRegularizationWithDepthMetrics, "depth")):
        ours = [c.__name__ for c in type(cls().instantiate()).__mro__]
        ref = META["mro"][kind]
        strip = lambda names: [n.replace("B200", "").replace("Impl", "Module").replace("HasInverse", "Inverse")  # noqa: E731
                               for n in names if n not in ("MetricImpl", "MetricModule", "Module", "object")]
        assert strip(ours) == strip(ref), (ours, ref)
    with pytest.raises(AssertionError):
        M.B200ScaleRegularizationMetrics(scale_reg_from=-1)
    with pytest.raises(AssertionError):
        M.B200ScaleRegularizationWithDepthMetrics(max_scale_ratio=0)
    M.B200ScaleRegularizationMetrics(max_scale_ratio=0, scale_ratio_reg_lambda=0)
    with pytest.raises(NotImplementedError):
        M.B200ScaleRegularizationMetrics(max_scale_outside_partition=2.0).instantiate()


def test_setup_resolves_max_scale_and_the_weights():
    import types
    from b200gs import metrics as M
    pl = types.SimpleNamespace(trainer=types.SimpleNamespace(datamodule=types.SimpleNamespace(
        dataparser_outputs=types.SimpleNamespace(camera_extent=META["camera_extent"]))))
    for c in META["cases"]:
        if c["metric"] == "mcmc":
            m = M.B200MCMCMetrics(**c["config"]).instantiate()
            m.setup("fit", pl)
            assert [m.opacity_reg_weight, m.scale_reg_weight] == c["weights"], c["key"]
        else:
            cls = M.B200ScaleRegularizationMetrics if c["metric"] == "scale" else M.B200ScaleRegularizationWithDepthMetrics
            m = cls(**c["config"]).instantiate()
            m.setup("fit" if c["stage"] == "train" else "validate", pl)
            assert m.config.max_scale == c["resolved_max_scale"], c["key"]
    m = M.B200ScaleRegularizationMetrics().instantiate()
    m.setup("validate", pl)
    assert m.config.max_scale == -1


def test_op_rejects_bad_inputs_before_any_launch():
    from b200gs.metrics import gaussian_regularizers
    with pytest.raises(ValueError, match="at least one"):
        gaussian_regularizers(torch.zeros(0, 1), torch.zeros(0, 3), raw=True)
    with pytest.raises(ValueError, match=r"\[N, 3\]"):
        gaussian_regularizers(None, torch.zeros(4, 2), raw=True)
    with pytest.raises(ValueError, match="CUDA"):
        gaussian_regularizers(torch.zeros(4, 1), torch.zeros(4, 3), raw=True)


# ---- C ABI ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    from b200gs import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


D = ctypes.c_void_p(16)    # non-NULL dummy; never dereferenced here
N = 1000
ALL = 1 | 2 | 4 | 8 | 16
SCALARS = (0.01, 0.01, 1.0, 10.0, 0.05, 0.05)


def fwd(L, n=N, flags=ALL, ptrs=(D, D), ws=None, outs=(D, D)):
    ws = L.b200gs_gaussian_reg_workspace_bytes(n) if ws is None else ws
    return L.b200gs_gaussian_reg_fwd(n, ptrs[0], ptrs[1], flags, *SCALARS, D, ws, outs[0], outs[1], None)


def bwd(L, n=N, flags=ALL, ptrs=(D, D), ws=None, outs=(D, D)):
    ws = L.b200gs_gaussian_reg_workspace_bytes(n) if ws is None else ws
    return L.b200gs_gaussian_reg_bwd(n, ptrs[0], ptrs[1], flags, *SCALARS, D, ws, D, outs[0], outs[1], None)


@pytest.mark.parametrize("call", [fwd, bwd], ids=["fwd", "bwd"])
def test_gaussian_reg_rejects_bad_arguments(L, call):
    before = L.b200gs_launch_count()
    for n in (0, -1, -(1 << 40)):
        assert call(L, n=n, ws=1 << 20) == -1 and b"n must be >= 1" in L.b200gs_last_error()
    assert call(L, n=(1 << 31), ws=1 << 30) == -1 and b"too large" in L.b200gs_last_error()
    for flags in (32, 64, -1, ALL | 128):
        assert call(L, flags=flags) == -1 and b"unknown flags" in L.b200gs_last_error()
    assert call(L, ptrs=(None, D)) == -1 and b"opacities" in L.b200gs_last_error()
    for flags in (4, 8, 16):
        assert call(L, ptrs=(D, None), flags=flags | 2) == -1 and b"scales" in L.b200gs_last_error()
    assert L.b200gs_gaussian_reg_fwd(N, D, D, ALL, *SCALARS, None, 1 << 20, D, D, None) == -1 and b"workspace" in L.b200gs_last_error()
    assert call(L, ws=L.b200gs_gaussian_reg_workspace_bytes(N) - 4) == -3 and b"workspace too small" in L.b200gs_last_error()
    assert L.b200gs_launch_count() == before


def test_forward_and_backward_reject_null_outputs(L):
    before = L.b200gs_launch_count()
    assert fwd(L, outs=(None, D)) == -1 and b"terms" in L.b200gs_last_error()
    # the statistics read the scales: with stats requested, scales may not be NULL even with no scale term
    assert fwd(L, flags=2, ptrs=(D, None), outs=(D, D)) == -1 and b"scales" in L.b200gs_last_error()
    assert L.b200gs_gaussian_reg_bwd(N, D, D, ALL, *SCALARS, D, 1 << 20, None, D, D, None) == -1 and b"v_terms" in L.b200gs_last_error()
    assert bwd(L, outs=(None, D)) == -1 and b"v_opacities" in L.b200gs_last_error()
    assert bwd(L, outs=(D, None)) == -1 and b"v_scales" in L.b200gs_last_error()
    assert L.b200gs_launch_count() == before


def test_workspace_size_follows_the_layout(L):
    def expect(n):
        return 4 * (8 + 9 * min((n + 1023) // 1024, 2048))
    for n in (1, 2, 1023, 1024, 1025, 2048 * 1024, 2048 * 1024 + 1, 3_000_000, (1 << 31) - 1):
        assert L.b200gs_gaussian_reg_workspace_bytes(n) == expect(n), n
    for n in (0, -1, 1 << 31):
        assert L.b200gs_gaussian_reg_workspace_bytes(n) == 0
