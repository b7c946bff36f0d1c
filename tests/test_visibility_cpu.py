"""The transient visibility map without a GPU: the DenseGrid layout and parameter count of the library and the oracle, a known
answer for the wrapped corner pixels, argument validation of the new entry points (every bad argument rejected before any CUDA
call), and the plug-ins' config fields, defaults, state_dict keys and optimizer groups, which follow the reference's
gsplat_appearance_embedding_visibility_map_renderer.py and visibility_map_metrics.py."""
import ctypes
import dataclasses
import os

import numpy as np
import pytest
import torch

from oracle import visibility_oracle as V


@pytest.fixture(scope="module")
def L():
    from b200gs import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


D = ctypes.c_void_p(16)    # non-NULL dummy; never dereferenced here


def test_grid_layout_and_parameter_count(L):
    from b200gs import _lib
    lv = V.levels()
    assert [r for _, r, _, _ in lv] == [16, 23, 32, 45, 63, 88, 124, 173]
    assert sum(s for _, _, s, _ in lv) == 60880 and V.n_params() == 121760
    assert all(s % 8 == 0 and s >= r * r for _, r, s, _ in lv)
    assert L.b200gs_uv_grid_params(ctypes.byref(_lib.B200gsUvGrid(8, 16, 1.405))) == 121760
    for n, base, s in [(4, 16, 1.405), (16, 16, 1.5), (1, 2, 1.0), (12, 8, 1.3)]:
        assert L.b200gs_uv_grid_params(ctypes.byref(_lib.B200gsUvGrid(n, base, s))) == V.n_params(n, base, s)
    for bad in [(0, 16, 1.405), (17, 16, 1.405), (8, 0, 1.405), (8, 16, 0.5), (8, 16, float("nan"))]:
        assert L.b200gs_uv_grid_params(ctypes.byref(_lib.B200gsUvGrid(*bad))) == 0


def test_wrapped_corners_known_answer():
    """The last pixel column reaches corner res_l exactly on the levels whose scale has a fractional part >= 0.5 (or none), and the %
    sends that corner to the first vertex of the next row; the last pixel of all wraps past the level's res^2 vertices."""
    W, H = 64, 48
    lv = V.levels()
    wraps = [l for l, (scale, res, _, _) in enumerate(lv) if int(np.floor(np.float32(scale) + np.float32(0.5))) + 1 == res]
    assert wraps == [0, 2, 5, 7]
    u, v = V.pixel_uv(W, H)
    last_col = np.arange(H) * W + W - 1
    per_level = V.corners(u, v, lv)
    for l in wraps:
        scale, res, size, offset = lv[l]
        idx, w = per_level[l]
        cy = np.floor((np.float64(scale) * v[last_col] + 0.5).astype(np.float32)).astype(np.int64)
        # corner k = 1 (x + 1) of the last column: cell_x = res - 1, so (res + cy res) % size = the start of row cy + 1
        assert np.array_equal(idx[last_col, 1].numpy() - offset, ((cy + 1) * res) % size)
        assert np.allclose(w[last_col].sum(1).numpy(), 1.0)
        # the very last pixel: corner 3 is (res, res) -> (res + res^2) % size
        assert int(idx[-1, 3]) - offset == (res + res * res) % size
    # the encoding of a grid whose vertex values are their own index: the last pixel of level 0 (u = v = 1, pos = 15.5, frac 0.5)
    # averages vertices (15, 15), (16 -> row 16 start, 15 + 1 wraps), ...
    params = torch.arange(V.n_params() // 2, dtype=torch.float64).repeat_interleave(2)
    enc = V.encode(params, u[-1:], v[-1:])
    scale, res, size, offset = lv[0]
    expect = 0.25 * sum(((15 + kx) + (15 + ky) * res) % size for kx in (0, 1) for ky in (0, 1))
    assert float(enc[0, 0]) == expect == float(enc[0, 1])


def test_uv_grid_entry_points_validate_before_any_cuda_call(L):
    from b200gs import _lib
    g = ctypes.byref(_lib.B200gsUvGrid(8, 16, 1.405))
    bad = ctypes.byref(_lib.B200gsUvGrid(0, 16, 1.405))
    assert L.b200gs_uv_grid_fwd(bad, 8, 8, None, 0, D, 1, None, 0, D, None) != 0
    assert L.b200gs_uv_grid_fwd(g, 1, 8, None, 0, D, 1, None, 0, D, None) != 0         # the pixel grid divides by W - 1
    assert L.b200gs_uv_grid_fwd(g, 8, 1, None, 0, D, 1, None, 0, D, None) != 0
    assert L.b200gs_uv_grid_fwd(g, 8, 8, None, 0, D, 0, None, 0, D, None) != 0         # no grid
    assert L.b200gs_uv_grid_fwd(g, 8, 8, None, 0, None, 1, None, 0, D, None) != 0
    assert L.b200gs_uv_grid_fwd(g, 8, 8, None, 0, D, 1, None, 0, ctypes.c_void_p(20), None) != 0   # misaligned enc
    assert L.b200gs_uv_grid_fwd(g, 0, 0, D, -1, D, 1, None, 0, D, None) != 0           # uv with n < 0
    assert L.b200gs_uv_grid_bwd(g, 1, 1, None, 0, D, D, None) != 0
    assert L.b200gs_uv_grid_bwd(g, 8, 8, None, 0, None, D, None) != 0


# grids whose float count overflows int: (2, 46341, 1.0) and (2, 1, 70000.0) hold about 8.6e9 and 9.8e9 floats, (1, 46341, 1.0)
# 4.3e9; summed in int their counts wrap to 18,560, 1,210,345,440 and a negative number.  Then a per_level_scale whose level-1 scale
# is infinite in fp32.
OVERFLOW = [(2, 46341, 1.0), (2, 1, 70000.0), (1, 46341, 1.0), (2, 16, 3e38), (16, 16, 2.0)]

# the grid configurations the GPU boundary tests sweep (tests/test_gpu_visibility_boundaries.py), with the levels whose last pixel
# column and row reach corner res_l and wrap through the %: the fp32 scale has a fractional part >= 0.5, or none
SWEEP_WRAPS = {
    (4, 16, 1.405): [0, 2],
    (8, 16, 1.405): [0, 2, 5, 7],
    (12, 16, 1.405): [0, 2, 5, 7, 8, 10, 11],
    (16, 16, 1.405): [0, 2, 5, 7, 8, 10, 11, 12, 14, 15],
    (8, 16, 2.0): list(range(8)),
    (8, 1, 2.0): list(range(8)),
    (4, 1, 1.5): [0, 1],
    (12, 16, 1.5): [0, 1, 2, 3, 4, 10, 11],
    (16, 4, 1.5): [0, 1, 2, 3, 6, 8, 9, 10, 11, 12, 14, 15],
}


@pytest.mark.parametrize("cfg", OVERFLOW)
def test_grids_past_the_float_cap_are_refused(L, cfg):
    from b200gs import _lib
    from b200gs.visibility import UVGridEncoding, _dense_grid_floats
    g = ctypes.byref(_lib.B200gsUvGrid(*cfg))
    assert L.b200gs_uv_grid_params(g) == 0
    assert _dense_grid_floats(*cfg) > 2 ** 31 - 1
    # both entry points, on the pixel grid and on given coordinates, refuse it before any CUDA call (D is never dereferenced)
    assert L.b200gs_uv_grid_fwd(g, 8, 8, None, 0, D, 1, None, 0, D, None) != 0
    assert L.b200gs_uv_grid_fwd(g, 0, 0, D, 4, D, 1, None, 0, D, None) != 0
    assert L.b200gs_uv_grid_bwd(g, 8, 8, None, 0, D, D, None) != 0
    assert L.b200gs_uv_grid_bwd(g, 0, 0, D, 4, D, D, None) != 0
    with pytest.raises(NotImplementedError, match="at most 2"):
        UVGridEncoding(*cfg)


def test_grid_just_under_the_float_cap_is_counted_exactly(L):
    """one level of res 32767 holds 2 * 1,073,676,296 = 2,147,352,592 floats, under INT32_MAX; res 32768 is over it"""
    from b200gs import _lib
    assert L.b200gs_uv_grid_params(ctypes.byref(_lib.B200gsUvGrid(1, 32767, 1.0))) == 2 * ((32767 * 32767 + 7) // 8 * 8) == V.n_params(1, 32767, 1.0)
    assert L.b200gs_uv_grid_params(ctypes.byref(_lib.B200gsUvGrid(1, 32768, 1.0))) == 0


@pytest.mark.parametrize("cfg", list(SWEEP_WRAPS), ids=str)
def test_sweep_grid_sizes_agree(L, cfg):
    from b200gs import _lib, ops
    from b200gs.visibility import _dense_grid_floats
    n = L.b200gs_uv_grid_params(ctypes.byref(_lib.B200gsUvGrid(*cfg)))
    assert n > 0 and n == V.n_params(*cfg) == _dense_grid_floats(*cfg) == ops.uv_grid_params(*cfg)


@pytest.mark.parametrize("cfg", list(SWEEP_WRAPS), ids=str)
def test_wrapping_levels(cfg):
    lv = V.levels(*cfg)
    frac_wraps = [l for l, (s, _, _, _) in enumerate(lv) if float(s) - np.floor(float(s)) >= 0.5 or float(s) == np.floor(float(s))]
    last_wraps = [l for l, (s, res, _, _) in enumerate(lv) if int(np.floor(np.float32(s) + np.float32(0.5))) + 1 == res]
    assert frac_wraps == last_wraps == SWEEP_WRAPS[cfg]


def test_wrapping_levels_near_a_half():
    """fp32 scales two ulp under a half do not wrap although exact arithmetic would; an exact half and an integer do"""
    under = lambda x: float(np.float32(x) - 2 * np.spacing(np.float32(x)))
    s = [float(x[0]) for x in V.levels(12, 16, 1.5)]
    assert s[5] == under(120.5) == 120.49998474121094 and 5 not in SWEEP_WRAPS[(12, 16, 1.5)]
    s = [float(x[0]) for x in V.levels(16, 4, 1.5)]
    assert s[3] == 12.5 and 3 in SWEEP_WRAPS[(16, 4, 1.5)]
    assert s[5] == under(29.375) and 5 not in SWEEP_WRAPS[(16, 4, 1.5)]
    lv = V.levels(8, 1, 2.0)
    assert (float(lv[0][0]), lv[0][1], lv[0][2]) == (0.0, 1, 8)           # every pixel in one cell with frac 0.5
    assert [float(x[0]) for x in V.levels(8, 16, 2.0)] == [16.0 * 2 ** l - 1 for l in range(8)]
    assert V.levels(8, 16, 1.405)[0][0] == 15.0 and abs(float(V.levels(8, 16, 1.405)[1][0]) % 1 - 0.48) < 1e-5


def mlp(feat=16, n_freq=-1, neurons=64, layers=3, n_out=1, flags=(0, 0, 0), null_weight=False):
    from b200gs import _lib
    m = _lib.B200gsAppearanceMlp(feat, n_freq, neurons, layers, n_out, *flags, feat + 128, feat + 128)
    for l in range(layers):
        m.weights[l] = None if null_weight else 16
        m.biases[l] = 16
    return ctypes.byref(m)


def test_visibility_mlp_entry_points(L):
    assert L.b200gs_visibility_mlp_workspace_bytes(16, 64, 3) > 0
    assert L.b200gs_visibility_mlp_workspace_bytes(16, 128, 4) > 0
    for shape in [(12, 64, 3), (40, 64, 3), (16, 32, 3), (16, 64, 1), (16, 64, 5)]:
        assert L.b200gs_visibility_mlp_workspace_bytes(*shape) == 0
    assert L.b200gs_visibility_mlp_fwd(mlp(), 0, None, None, None) == 0                 # n == 0: nothing to do
    for m in [mlp(n_out=3), mlp(n_freq=4), mlp(flags=(1, 0, 0)), mlp(flags=(0, 0, 1)), mlp(feat=12), mlp(null_weight=True)]:
        assert L.b200gs_visibility_mlp_fwd(m, 10, D, D, None) != 0
    assert L.b200gs_visibility_mlp_fwd(mlp(), 10, None, D, None) != 0
    assert L.b200gs_visibility_mlp_fwd(mlp(), -1, D, D, None) != 0
    ws = L.b200gs_visibility_mlp_workspace_bytes(16, 64, 3)
    assert L.b200gs_visibility_mlp_bwd(mlp(), 10, D, D, D, D, ws - 4, D, None) == -3     # workspace too small
    assert L.b200gs_visibility_mlp_bwd(mlp(), 10, D, D, ctypes.c_void_p(24), D, ws, D, None) != 0
    assert L.b200gs_visibility_mlp_bwd(mlp(), 10, D, D, D, D, ws, None, None) != 0
    # the appearance entry points keep their accept set: one output is refused there
    assert L.b200gs_appearance_mlp_workspace_bytes(16, -1, 64, 3, 1) == 0


def test_vis_loss_entry_points(L):
    W, H = 50, 37
    blocks = L.b200gs_vis_loss_blocks(W, H)
    assert blocks == 3 * 4 * 3
    for g in (0, 1):
        assert L.b200gs_vis_loss_workspace_bytes(W, H, g) == ((4 if g else 3) * 3 * W * H + 3 * blocks) * 4
    assert L.b200gs_vis_loss_workspace_bytes(0, H, 0) == 0 and L.b200gs_vis_loss_blocks(W, 0) == 0
    ws = L.b200gs_vis_loss_workspace_bytes(W, H, 1)
    assert L.b200gs_vis_loss_fwd(0, H, D, D, D, None, 1, D, ws, None) != 0
    assert L.b200gs_vis_loss_fwd(W, H, D, None, D, None, 1, D, ws, None) != 0
    assert L.b200gs_vis_loss_fwd(W, H, D, D, None, None, 1, D, ws, None) != 0
    assert L.b200gs_vis_loss_fwd(W, H, D, D, D, None, 1, D, ws - 4, None) == -3
    assert L.b200gs_vis_loss_bwd(W, H, D, D, D, None, D, ws - 4, 0.2, 0.2, None, D, D, None) == -3
    assert L.b200gs_vis_loss_bwd(W, H, D, D, D, None, D, ws, 0.2, 0.2, None, None, D, None) != 0


def test_config_fields_and_defaults_follow_the_reference():
    from b200gs import visibility as B
    from b200gs.metrics import B200VanillaMetrics, B200VisibilityMapMetrics
    assert [(f.name, f.default) for f in dataclasses.fields(B.UVEncodingConfig)] == [
        ("n_levels", 8), ("base_resolution", 16), ("per_level_scale", 1.405)]
    m = B.ModelConfig()
    assert (m.n_images, m.n_gaussian_feature_dims, m.n_appearance_embedding_dims, m.is_view_dependent, m.n_view_direction_frequencies,
            m.n_transient_embedding_dims) == (-1, 64, 128, False, 4, 128)
    assert (m.appearance_network.n_neurons, m.appearance_network.n_layers, m.appearance_network.skip_layers) == (64, 3, [])
    assert (m.visibility_network.n_neurons, m.visibility_network.n_layers, m.visibility_network.skip_layers) == (64, 3, [])
    o = B.OptimizationConfig()
    assert (o.gamma_eps, o.eps, o.max_steps, o.appearance_warm_up, o.transient_warm_up) == (1e-6, 1e-15, 30_000, 1000, 2000)
    assert [(getattr(o, k).lr_init, getattr(o, k).lr_final_factor) for k in
            ("appearance_embedding", "appearance_network", "transient_embedding", "uv_encoding", "visibility_network")] == [
        (2e-3, 0.1), (1e-3, 0.1), (2e-3, 0.1), (2e-3, 0.1), (1e-3, 0.1)]
    metric = B200VisibilityMapMetrics()
    assert isinstance(metric, B200VanillaMetrics) and metric.vis_reg_factor == 0.2 and metric.lambda_dssim == 0.2
    with pytest.raises(NotImplementedError):
        B200VisibilityMapMetrics(rgb_diff_loss="l2").instantiate()


def test_state_dict_keys_and_optimizer_groups(L):
    from b200gs import visibility as B
    r = B.B200GSplatAppearanceEmbeddingVisibilityMapRenderer(B.ModelConfig(n_images=2), B.OptimizationConfig())
    r.setup("fit")
    sd = r.state_dict()
    expect = ["model.appearance_embedding.weight"]
    expect += [f"model.appearance_network.output_layers.{i}.{p}" for i in (0, 2, 4) for p in ("weight", "bias")]
    expect += ["model.transient_embedding.weight", "model.uv_encodings.0.params", "model.uv_encodings.1.params"]
    expect += [f"model.visibility_network.output_layers.{i}.{p}" for i in (0, 2, 4) for p in ("weight", "bias")]
    assert sorted(sd) == sorted(expect)
    assert sd["model.uv_encodings.0.params"].shape == (121760,) and sd["model.appearance_network.output_layers.0.weight"].shape == (64, 192)
    assert sd["model.visibility_network.output_layers.0.weight"].shape == (64, 144)
    assert sd["model.visibility_network.output_layers.4.weight"].shape == (1, 64)
    assert float(sd["model.uv_encodings.1.params"].abs().max()) <= 1e-4
    # a checkpoint loads into a renderer that has not been set up
    r2 = B.B200GSplatAppearanceEmbeddingVisibilityMapRenderer(B.ModelConfig(), B.OptimizationConfig())
    r2.load_state_dict(sd)
    assert torch.equal(r2.model.uv_encodings[1].params, sd["model.uv_encodings.1.params"])
    opts, scheds = r.training_setup(None)
    assert [o.param_groups[0]["name"] for o in opts] == ["appearance_embedding", "appearance_network", "transient_embedding",
                                                          "uv_encoding", "visibility_network"]
    assert [o.defaults["eps"] for o in opts] == [1e-15] * 5
    assert [s.lr_lambdas[0](1000 + 30_000) for s in scheds[:2]] == pytest.approx([0.1, 0.1])
    assert [s.lr_lambdas[0](1500) for s in scheds] == pytest.approx([0.1 ** (500 / 30_000), 0.1 ** (500 / 30_000), 1, 1, 1])
    with pytest.raises(NotImplementedError):
        B.B200VisibilityMapModel(B.ModelConfig(n_images=1, visibility_network=B.VisibilityNetworkConfig(skip_layers=[1])))


def test_tinycudann_hook_leaves_sys_modules_alone_until_imported():
    import sys
    from b200gs import compat
    sys.modules.pop("tinycudann", None)         # another test may have installed with force=True
    sys.meta_path[:] = [f for f in sys.meta_path if getattr(f, "name", None) != "tinycudann"]
    compat.install()
    assert "tinycudann" not in sys.modules
    import tinycudann
    try:
        with pytest.raises(NotImplementedError):
            tinycudann.Encoding(n_input_dims=3, encoding_config={"otype": "DenseGrid"})
        with pytest.raises(NotImplementedError):
            tinycudann.Encoding(n_input_dims=2, encoding_config={"otype": "DenseGrid", "interpolation": "Nearest"})
        with pytest.raises(NotImplementedError):
            tinycudann.NetworkWithInputEncoding(2, 1, {}, {})
        e = tinycudann.Encoding(n_input_dims=2, encoding_config={"otype": "DenseGrid", "n_levels": 8, "base_resolution": 16,
                                                                 "per_level_scale": 1.405}, seed=3, dtype=torch.float)
        assert e.n_output_dims == 16 and e.params.shape == (121760,)
    finally:
        sys.modules.pop("tinycudann", None)
