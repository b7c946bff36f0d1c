"""SWAG in-the-wild appearance without a GPU: the float64 oracle (oracle/swag_oracle.py) against recordings of the unmodified
reference SWAGRenderer / SWAGModel (tests/golden/swag.npz, swag.json, make_golden_swag.py), the hash grid's level table and
known-answer corner indices, the C ABI's argument checks (all made before any CUDA call) and the b200gs.swag plug-in's config,
parameter tree, optimizer and refusals."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import swag_oracle as S

Z = np.load(os.path.join(GOLDEN, "swag.npz"))
META = json.load(open(os.path.join(GOLDEN, "swag.json")))
EINVAL, ENOSPACE = -1, -3


def golden_table(n):
    i = torch.arange(n, dtype=torch.float64)
    return (0.6 * torch.sin(i * 0.7071) + 0.2 * torch.cos(i * 0.0173)).float()


# ---- the oracle against the recorded reference ---------------------------------------------------------------------------------
@pytest.mark.parametrize("case", META["cases"], ids=lambda c: c["name"])
def test_oracle_reproduces_the_reference(case):
    name, degree, u = case["name"], case["degree"], case["u"]
    t = lambda k: torch.from_numpy(Z[k]).double().requires_grad_(True)      # noqa: E731
    means, features, logits = t("means"), t("features"), t("logits")
    table = golden_table(S.n_params()).double().requires_grad_(True)
    emb = t("embedding")
    ws = [t(f"theta.{i}.weight") for i in (0, 2, 4)]
    bs = [t(f"theta.{i}.bias") for i in (0, 2, 4)]
    c, o = S.swag(degree, means, torch.from_numpy(Z["campos"]).double(), features, table, emb[4], ws, bs, torch.sigmoid(logits)[:, 0],
                  0.5 if u is None else u, np.array(META["bbox_min"], np.float32), np.array(META["bbox_size"], np.float32))
    ((c * torch.from_numpy(Z["cot_c"]).double()).sum() + (o * torch.from_numpy(Z["cot_o"]).double()).sum()).backward()
    p = name + "."
    assert np.abs(c.detach().numpy() - Z[p + "colours"]).max() <= 2e-5
    assert np.abs(o.detach().numpy() - Z[p + "opacities"]).max() <= 2e-5

    def close(got, key, tol=2e-4):
        ref = Z[p + key]
        assert np.abs(got - ref).max() <= tol * max(1.0, np.abs(ref).max()), key
    close(np.zeros(Z[p + "v_means"].shape) if means.grad is None else means.grad.numpy(), "v_means")     # degree 0: no direction
    close(features.grad.numpy(), "v_features")
    close(logits.grad.numpy(), "v_logits")
    close(emb.grad.numpy(), "v_embedding")
    for i, (w, b) in zip((0, 2, 4), zip(ws, bs)):
        close(w.grad.numpy(), f"v_theta.{i}.weight")
        close(b.grad.numpy(), f"v_theta.{i}.bias")
    g = np.zeros(table.numel())
    g[Z[p + "v_table_idx"]] = Z[p + "v_table_val"]
    assert np.abs(table.grad.numpy() - g).max() <= 2e-4 * max(1.0, np.abs(g).max())


def test_the_recording_has_the_effective_config_not_the_apparent_one():
    """swag_model.GridEncodingConfig's `n_levels = 12` has no annotation: the field keeps 8, and so does the recorded encoder"""
    assert META["grid_encoding_n_levels"] == 8
    c = META["encoder_config"]
    assert (c["otype"], c["n_levels"], c["n_features_per_level"], c["log2_hashmap_size"], c["base_resolution"]) == ("HashGrid", 8, 4, 19, 16)
    assert c["per_level_scale"] == pytest.approx(2.0, abs=1e-12)
    assert META["state_dict"]["swag_model.grid_encoding.params"] == [11_681_792]
    assert META["state_dict"]["swag_model.theta.0.weight"] == [64, 59]
    assert META["calls"][0]["n_input_dims"] == 3


# ---- the grid --------------------------------------------------------------------------------------------------------------------
def test_level_table_and_parameter_count():
    lv = S.levels()
    assert [(r, s, o) for _, r, s, o in lv] == [(16, 4096, 0), (32, 32768, 4096), (64, 262144, 36864), (128, 524288, 299008),
                                                (256, 524288, 823296), (512, 524288, 1347584), (1024, 524288, 1871872),
                                                (2048, 524288, 2396160)]
    assert S.n_params() == 4 * (4096 + 32768 + 262144 + 5 * 524288) == 11_681_792
    assert S.n_params(n_levels=12) == 20_070_400 and S.n_params(n_features_per_level=2) == 5_840_896


def test_library_parameter_count_matches_the_oracle():
    from b200gs import ops
    for g in ({}, dict(n_levels=16, n_features_per_level=2, log2_hashmap_size=12, base_resolution=20, per_level_scale=1.38),
              dict(n_levels=3, log2_hashmap_size=24, base_resolution=8, per_level_scale=1.5), dict(n_levels=1, base_resolution=1, per_level_scale=1.0)):
        assert ops.hash_grid_params(**g) == S.n_params(**g), g
    for bad in (dict(n_levels=0), dict(n_levels=17), dict(n_features_per_level=8), dict(n_features_per_level=1), dict(log2_hashmap_size=25),
                dict(base_resolution=0), dict(per_level_scale=0.9), dict(per_level_scale=float("inf")),
                dict(n_levels=16, base_resolution=2 ** 30, per_level_scale=4.0)):
        assert ops.hash_grid_params(**bad) == 0, bad


def test_known_answer_corner_indices():
    """tcnn's grid_index on hashed and wrapped (negative / past the last vertex) corners, computed by hand in Python integers"""
    cells = lambda *c: np.array([[v % 2 ** 32 for v in c]], dtype=np.uint64)          # noqa: E731  (uint32 wrap of negatives)
    assert S.grid_index(cells(-1, 5, 7), 128, 524288)[0] == 195225              # level 3: 128^3 > 2^19, hashed
    assert S.grid_index(cells(128, 0, 3), 128, 524288)[0] == 460351
    assert S.grid_index(cells(3, -2, -1), 128, 524288)[0] == 304374
    assert S.grid_index(cells(-1, 0, 0), 16, 4096)[0] == 4095                  # level 0: dense, 2^32 - 1 wraps mod 4096
    assert S.grid_index(cells(16, 15, 15), 16, 4096)[0] == 0                   # one past the last vertex
    assert S.grid_index(cells(0, -1, 0), 16, 4096)[0] == 4080
    assert S.grid_index(cells(32, 32, 32), 32, 32768)[0] == 1056
    assert S.grid_index(cells(-1, -1, -1), 64, 262144)[0] == 257983
    # through the cell selection: x = -0.1 on level 0 (scale 15) gives pos = -1 exactly, cell 2^32 - 1, frac 0
    idx, w = S.corners(np.array([[-0.1, 0.0, 0.0]], np.float32))[0]
    assert int(idx[0, 0]) == 4095 and float(w[0, 0]) == pytest.approx(0.25)
    assert float(w[0, 1]) == 0.0                                                 # the corner at cell + 1 along x has weight frac = 0


# ---- the C ABI's refusals (checked before any CUDA call) --------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    from b200gs import _lib
    return _lib


def _grid(L, **kw):
    g = dict(S.DEFAULT_GRID)
    g.update(kw)
    return L.B200gsHashGrid(g["n_levels"], g["n_features_per_level"], g["log2_hashmap_size"], g["base_resolution"], g["per_level_scale"])


def _err(L):
    return L.lib().b200gs_last_error().decode()


P = 4096      # a fake device address: never dereferenced, every call below is refused first


def test_swag_inputs_refusals(L):
    lib = L.lib()
    fwd = lambda g, degree=3, n=10, row=40, shs=P, means=P, table=P, x0=P, cl=P, split=0, stride=16: lib.b200gs_swag_inputs_fwd(  # noqa: E731
        ctypes.byref(g), degree, n, means, P, shs, P, stride, split, P, table, row, x0, cl, None)
    assert fwd(_grid(L, n_levels=17)) == EINVAL and "unsupported grid" in _err(L)
    assert fwd(_grid(L, n_features_per_level=3)) == EINVAL and "n_features_per_level 2 or 4" in _err(L)
    assert fwd(_grid(L, log2_hashmap_size=25)) == EINVAL
    assert fwd(_grid(L), row=34) == EINVAL and "row_stride" in _err(L)
    assert fwd(_grid(L), row=80) == EINVAL and "row_stride" in _err(L)
    assert fwd(_grid(L), degree=5) == EINVAL and "degree must be 0..4" in _err(L)
    assert fwd(_grid(L), stride=15) == EINVAL and "sh_stride" in _err(L)
    assert fwd(_grid(L), split=2) == EINVAL and "sh_split" in _err(L)
    assert fwd(_grid(L), n=-1) == EINVAL and "n out of range" in _err(L)
    assert fwd(_grid(L), means=None) == EINVAL and "NULL" in _err(L)
    assert fwd(_grid(L), x0=None) == EINVAL and "NULL" in _err(L)
    assert fwd(_grid(L), cl=None) == EINVAL and "NULL" in _err(L)
    assert fwd(_grid(L), table=P + 4) == EINVAL and "aligned" in _err(L)
    assert lib.b200gs_swag_inputs_fwd(None, 3, 10, P, P, P, P, 16, 0, P, P, 40, P, P, None) == EINVAL and "grid is NULL" in _err(L)
    bwd = lambda g, n=10, v_table=P, v_means=P, v_x0=P: lib.b200gs_swag_inputs_bwd(  # noqa: E731
        ctypes.byref(g), 3, n, P, P, P, P, 16, 1, P, P, v_x0, 40, P, P, v_means, v_table, None)
    assert bwd(_grid(L), v_table=None) == EINVAL and "NULL" in _err(L)
    assert bwd(_grid(L), v_means=None) == EINVAL and "NULL" in _err(L)
    assert bwd(_grid(L), v_x0=None) == EINVAL and "NULL v_x0" in _err(L)
    assert bwd(_grid(L, n_levels=0)) == EINVAL and "unsupported grid" in _err(L)


def _mlp(L, feat=40, hidden=64, layers=3, n_out=4, epilogue=2, n_freq=-1, normalize=0):
    m = L.B200gsAppearanceMlp(feat, n_freq, hidden, layers, n_out, normalize, 0, epilogue, 59, 59)
    for l in range(min(layers, 4)):
        m.weights[l], m.biases[l] = P, P
    return m


def test_swag_mlp_refusals(L):
    lib = L.lib()
    fwd = lambda m, in_dim=35, n=10, T=0.1, eps=1e-8, u=P, col=P: lib.b200gs_swag_mlp_fwd(  # noqa: E731
        ctypes.byref(m), in_dim, n, P, P, u, T, eps, col, P, None)
    assert fwd(_mlp(L, epilogue=1)) == EINVAL and "epilogue 2" in _err(L)
    assert fwd(_mlp(L, n_out=3)) == EINVAL and "n_out 4" in _err(L)
    assert fwd(_mlp(L, n_freq=4)) == EINVAL and "n_freq -1" in _err(L)
    assert fwd(_mlp(L, normalize=1)) == EINVAL
    assert fwd(_mlp(L, feat=36)) == EINVAL and "multiple of 8" in _err(L)
    assert fwd(_mlp(L, hidden=32)) == EINVAL and "n_neurons 64 or 128" in _err(L)
    assert fwd(_mlp(L, layers=5)) == EINVAL
    assert fwd(_mlp(L), in_dim=41) == EINVAL and "in_dim" in _err(L)
    assert fwd(_mlp(L), in_dim=32) == EINVAL and "in_dim" in _err(L)
    assert fwd(_mlp(L), T=0.0) == EINVAL and "temperature" in _err(L)
    assert fwd(_mlp(L), eps=-1.0) == EINVAL and "eps" in _err(L)
    assert fwd(_mlp(L), T=float("inf")) == EINVAL
    assert fwd(_mlp(L), u=None) == EINVAL and "NULL x0, base_opacity or u" in _err(L)
    assert fwd(_mlp(L), col=None) == EINVAL and "NULL colour or opacity" in _err(L)
    m = _mlp(L)
    m.weights[1] = None
    assert fwd(m) == EINVAL and "NULL weight" in _err(L)
    assert lib.b200gs_swag_mlp_fwd(None, 35, 10, P, P, P, 0.1, 1e-8, P, P, None) == EINVAL and "mlp is NULL" in _err(L)
    bwd = lambda m, ws=P, ws_bytes=1 << 30, v_x0=P, v_params=P: lib.b200gs_swag_mlp_bwd(  # noqa: E731
        ctypes.byref(m), 35, 10, P, P, P, 0.1, 1e-8, P, P, v_x0, P, ws, ws_bytes, v_params, None)
    assert bwd(_mlp(L), v_params=None) == EINVAL and "NULL v_params" in _err(L)
    assert bwd(_mlp(L), ws=None) == EINVAL and "workspace" in _err(L)
    assert bwd(_mlp(L), v_x0=P + 4) == EINVAL and "16-byte aligned" in _err(L)
    assert bwd(_mlp(L), ws_bytes=16) == ENOSPACE and "workspace too small" in _err(L)
    assert lib.b200gs_swag_mlp_workspace_bytes(40, 64, 3) == lib.b200gs_appearance_mlp_workspace_bytes(40, -1, 64, 3, 4) > 0
    assert lib.b200gs_swag_mlp_workspace_bytes(36, 64, 3) == 0 and lib.b200gs_swag_mlp_workspace_bytes(40, 32, 3) == 0


def test_appearance_entry_points_keep_their_messages(L):
    """the appearance and visibility networks' accept set is unchanged by the SWAG epilogue"""
    lib = L.lib()
    m = _mlp(L, feat=36, epilogue=1, n_out=3)
    assert lib.b200gs_appearance_mlp_fwd(ctypes.byref(m), 10, P, None, P, None, None, None, P, None, None, None) == EINVAL
    assert _err(L) == "b200gs_appearance_mlp_fwd: feat_dim must be a positive multiple of 8"
    m = _mlp(L, feat=16, epilogue=2, n_out=4)
    assert lib.b200gs_visibility_mlp_fwd(ctypes.byref(m), 10, P, P, None) == EINVAL
    assert _err(L) == "b200gs_visibility_mlp_fwd: a visibility network has n_freq -1, n_out 1 and no normalisation or epilogue"


# ---- the plug-in -----------------------------------------------------------------------------------------------------------------
def _renderer():
    from b200gs.swag import B200SWAGModel, B200SWAGRenderer, EmbeddingConfig
    r = B200SWAGRenderer(embedding=EmbeddingConfig(num_embeddings=6))
    pc = torch.from_numpy(Z["point_cloud"])
    r.set_bbox(pc.min(0).values, pc.max(0).values)
    r.swag_model = B200SWAGModel(r.network_config, r.grid_encoding_config, r.embedding_config)
    return r


def test_plug_in_config_matches_the_reference():
    from b200gs import swag
    d = META["defaults"]
    assert swag.GridEncodingConfig().n_levels == META["grid_encoding_n_levels"] == 8
    enc = swag.GridEncodingConfig().get_encoder_config(3)
    assert {k: (float(v) if isinstance(v, (float, np.floating)) else v) for k, v in enc.items()} == META["encoder_config"]
    assert vars(swag.NetworkConfig()) == d["network"] and vars(swag.EmbeddingConfig()) == d["embedding"]
    assert vars(swag.GridEncodingOptimizationConfig()) == d["optimization"]
    r = swag.B200SWAGRenderer()
    assert (r.temperature, r.eps) == (d["temperature"], d["eps"])
    r = _renderer()
    assert r.bbox_min.tolist() == META["bbox_min"] and r.bbox_size.tolist() == META["bbox_size"]


def test_plug_in_state_dict_and_optimizer_match_the_reference():
    r = _renderer()
    assert {k: list(v.shape) for k, v in r.state_dict().items()} == META["state_dict"]
    r.load_state_dict({k: torch.zeros(v) for k, v in META["state_dict"].items()})          # a reference checkpoint loads
    opt, sched = r.training_setup(None)
    o = META["optimizer"]
    assert [g["name"] for g in opt.param_groups] == o["names"] and len(opt.param_groups[0]["params"]) == o["n_params"]
    assert opt.param_groups[0]["lr"] == o["lr"] and opt.defaults["eps"] == o["eps"]
    assert {str(s): sched.lr_lambdas[0](s) for s in (0, 1, 15_000, 30_000, 45_000)} == pytest.approx({k: v for k, v in o["lambda"].items()})
    assert list(r.uniform_sampler.sample((1,)).shape) == META["uniform_sample_shape"]


def test_plug_in_refusals():
    import sys
    from b200gs import compat, swag
    with pytest.raises(NotImplementedError, match="hashgrid encoding only"):
        swag.GridEncodingConfig(type="densegrid").get_encoder_config(3)
    with pytest.raises(NotImplementedError, match="n_features_per_level 2 or 4"):
        swag.HashGridEncoding({"otype": "HashGrid", "n_features_per_level": 8})
    with pytest.raises(NotImplementedError, match="linear interpolation"):
        swag.HashGridEncoding({"otype": "HashGrid", "interpolation": "Nearest"})
    with pytest.raises(NotImplementedError, match="n_neurons 64 or 128"):
        swag.B200SWAGModel(swag.NetworkConfig(n_neurons=32), swag.GridEncodingConfig(log2_hashmap_size=4), swag.EmbeddingConfig(4, 8))
    sys.modules.pop("tinycudann", None)
    compat.install(force=True)
    try:
        import tinycudann as tcnn
        e = tcnn.Encoding(n_input_dims=3, encoding_config=swag.GridEncodingConfig(log2_hashmap_size=10).get_encoder_config(3))
        assert isinstance(e, swag.HashGridEncoding) and e.n_output_dims == 32 and e.params.numel() == S.n_params(log2_hashmap_size=10)
        assert float(e.params.detach().abs().max()) <= 1e-4
        for n_in, cfg in ((2, {"otype": "HashGrid"}), (3, {"otype": "DenseGrid"}), (3, {"otype": "HashGrid", "interpolation": "Nearest"})):
            with pytest.raises(NotImplementedError):
                tcnn.Encoding(n_input_dims=n_in, encoding_config=cfg)
        with pytest.raises(NotImplementedError, match="float32"):
            tcnn.Encoding(n_input_dims=3, encoding_config={"otype": "HashGrid"}, dtype=torch.half)
        with pytest.raises(NotImplementedError):
            tcnn.Network(n_input_dims=3, n_output_dims=4, network_config={})
        with pytest.raises(NotImplementedError):
            tcnn.NetworkWithInputEncoding(3, 4, {}, {})
    finally:
        sys.modules.pop("tinycudann", None)
