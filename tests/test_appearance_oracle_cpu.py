"""The appearance colour pass without a GPU: the float64 oracle (oracle/appearance_oracle.py) against recordings of the reference's
own Model and renderer (tests/golden/appearance.npz, make_golden_appearance.py), the parameter tree of B200AppearanceModel, the
shapes it refuses, and the argument validation of the C entry points."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import appearance_oracle as O

Z = np.load(os.path.join(GOLDEN, "appearance.npz"))
VARIANTS = {
    "default": {},
    "view_dependent": {"is_view_dependent": True},
    "normalize": {"normalize": True},
    "with_opacity": {"with_opacity": True},
    "embedding128": {"n_appearance_embedding_dims": 128},
}
APPEARANCE_ID = 2


def golden_state(name, dtype=torch.float64):
    """(embedding.weight, weights, biases) of a recorded configuration, leaves that require grad"""
    st = {k[len(name) + 7:]: torch.from_numpy(Z[k]).to(dtype) for k in Z.files if k.startswith(name + ".state.")}
    n = len([k for k in st if k.endswith(".weight")]) - 1
    leaf = lambda t: t.clone().requires_grad_(True)
    return (leaf(st["embedding.weight"]), [leaf(st[f"network.output_layers.{2 * i}.weight"]) for i in range(n)],
            [leaf(st[f"network.output_layers.{2 * i}.bias"]) for i in range(n)])


def golden_inputs(dtype=torch.float64):
    x = {k[3:]: torch.from_numpy(Z[k]) for k in Z.files if k.startswith("in.")}
    return {k: (v.to(dtype) if v.dtype == torch.float32 else v) for k, v in x.items()}


def n_freq_of(kw):
    return 4 if kw.get("is_view_dependent") else -1


def close(got, want, what, tol=2e-6):
    """float32 round-off of the recording: relative to the tensor's largest entry"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, what
    assert np.abs(got - want).max() <= tol * max(np.abs(want).max(), 1.0), (what, np.abs(got - want).max())


def param_grads(emb, ws, bs):
    g = {"embedding.weight": emb.grad}
    for i, (w, b) in enumerate(zip(ws, bs)):
        g[f"network.output_layers.{2 * i}.weight"], g[f"network.output_layers.{2 * i}.bias"] = w.grad, b.grad
    return g


@pytest.mark.parametrize("name", list(VARIANTS))
def test_oracle_reproduces_the_reference_model(name):
    kw, x = VARIANTS[name], golden_inputs()
    emb, ws, bs = golden_state(name)
    mask = x["mask"]
    feats = x["features"][mask].clone().requires_grad_(True)
    dirs = torch.nn.functional.normalize(x["means"][mask].float() - x["cam_center"].float(), dim=-1).double()
    y = O.mlp(feats, emb[APPEARANCE_ID], ws, bs, dirs, n_freq_of(kw), kw.get("normalize", False))
    (y * x["cot_model"][mask][:, :y.shape[1]]).sum().backward()
    close(y.detach(), Z[f"{name}.model.out"], "out")
    close(feats.grad, Z[f"{name}.model.v_features"], "v_features")
    for k, g in param_grads(emb, ws, bs).items():
        close(g, Z[f"{name}.model.grad.{k}"], k)


@pytest.mark.parametrize("name", list(VARIANTS))
def test_oracle_reproduces_the_reference_colours(name):
    kw, x = VARIANTS[name], golden_inputs()
    emb, ws, bs = golden_state(name)
    mask = x["mask"]
    feats, base, raw = (x[k].clone().requires_grad_(True) for k in ("features", "base", "raw_opacity"))
    rgbs, opacities, offsets = O.colors(feats, mask, base, x["means"], x["cam_center"], raw, emb[APPEARANCE_ID], ws, bs, n_freq_of(kw),
                                        kw.get("normalize", False))
    loss = (rgbs * x["cot_rgbs"]).sum()
    if offsets is not None:
        loss = loss + (opacities * x["cot_opacities"]).sum() + (offsets * x["cot_offsets"]).sum()
    loss.backward()
    want = Z[f"{name}.colors.rgbs"]
    assert (want[mask.numpy()] == 0).any() and (want[mask.numpy()] == 1).any()        # both clamps are exercised
    # a colour within round-off of a clamp bound may fall on either side in float32: none of the recorded ones does
    close(rgbs.detach(), want, "rgbs")
    close(feats.grad, Z[f"{name}.colors.v_features"], "v_features")
    close(base.grad, Z[f"{name}.colors.v_base"], "v_base")
    if offsets is not None:
        close(opacities.detach(), Z[f"{name}.colors.opacities"], "opacities")
        close(offsets.detach()[mask], Z[f"{name}.colors.offsets"], "offsets")
        close(raw.grad, Z[f"{name}.colors.v_raw_opacity"], "v_raw_opacity")
    for k, g in param_grads(emb, ws, bs).items():
        close(g, Z[f"{name}.colors.grad.{k}"], k)


@pytest.fixture(scope="module")
def L():
    from b200gs import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


@pytest.mark.parametrize("name", list(VARIANTS))
def test_state_dict_matches_the_reference(L, name):
    from b200gs.appearance import B200GSplatAppearanceEmbeddingRenderer, ModelConfig
    renderer = B200GSplatAppearanceEmbeddingRenderer(model=ModelConfig(n_appearances=1, **VARIANTS[name])).instantiate()
    state = {"model." + k[len(name) + 7:]: torch.from_numpy(Z[k]) for k in Z.files if k.startswith(name + ".state.")}
    renderer.load_state_dict(state, strict=True)          # sizes the embedding from the checkpoint, as the reference
    assert list(renderer.state_dict().keys()) == list(Z[f"{name}.keys"])
    assert renderer.config.model.n_appearances == 4
    for k, v in renderer.state_dict().items():
        assert torch.equal(v, state[k])


@pytest.mark.parametrize("kw", [{"tcnn": True}, {"skip_layers": [1]}, {"n_neurons": 32}, {"n_neurons": 256}, {"n_layers": 1}, {"n_layers": 5},
                                {"n_gaussian_feature_dims": 60}, {"n_gaussian_feature_dims": 1024}])
def test_unsupported_shapes_raise(L, kw):
    from b200gs.appearance import B200AppearanceModel, ModelConfig
    with pytest.raises(NotImplementedError):
        B200AppearanceModel(ModelConfig(n_appearances=2, **kw))


def test_supported_shapes_build(L):
    from b200gs.appearance import B200AppearanceModel, ModelConfig
    for kw in ({"n_neurons": 128}, {"n_layers": 2}, {"n_layers": 4, "is_view_dependent": True}, {"n_neurons": 128, "n_layers": 4, "is_view_dependent": True},
               {"n_gaussian_feature_dims": 32, "n_view_direction_frequencies": 6, "is_view_dependent": True}):
        B200AppearanceModel(ModelConfig(n_appearances=2, **kw))


D = ctypes.c_void_p(16)    # non-NULL dummy; never dereferenced here


def mlp_struct(**kw):
    from b200gs._lib import B200gsAppearanceMlp
    f = dict(feat_dim=64, n_freq=-1, n_neurons=64, n_layers=3, n_out=3, normalize=0, normalize_dirs=0, epilogue=1, w0_stride=96, w0_pe_col=96)
    f.update(kw)
    m = B200gsAppearanceMlp(**f)
    for l in range(f["n_layers"] if 0 < f["n_layers"] <= 4 else 0):
        m.weights[l], m.biases[l] = 16, 16
    return m


def fwd(L, m, n=10, features=D, base=D, dirs=D, raw=D, out=D, offsets=D, opacities=D):
    return L.b200gs_appearance_mlp_fwd(ctypes.byref(m) if m is not None else None, n, features, None, base, dirs, None, raw, out, offsets,
                                       opacities, None)


def bwd(L, m, n=10, features=D, base=D, dirs=D, raw=D, v_out=D, v_base=D, v_features=D, v_raw=D, ws=D, ws_bytes=1 << 30, v_params=D):
    return L.b200gs_appearance_mlp_bwd(ctypes.byref(m) if m is not None else None, n, features, None, base, dirs, None, raw, v_out, None, None,
                                       v_base, v_features, v_raw, ws, ws_bytes, v_params, None)


@pytest.mark.parametrize("call", [fwd, bwd], ids=["fwd", "bwd"])
def test_abi_rejects_bad_arguments(L, call):
    err = L.b200gs_last_error
    before = L.b200gs_launch_count()
    assert call(L, None) == -1 and b"mlp is NULL" in err()
    for f in (0, 60, -8):
        assert call(L, mlp_struct(feat_dim=f)) == -1 and b"multiple of 8" in err()
    for h in (32, 96, 256):
        assert call(L, mlp_struct(n_neurons=h)) == -1 and b"n_neurons" in err()
    for layers in (1, 5):
        assert call(L, mlp_struct(n_layers=layers)) == -1 and b"n_layers" in err()
    for o in (2, 5):
        assert call(L, mlp_struct(n_out=o)) == -1 and b"n_out" in err()
    assert call(L, mlp_struct(feat_dim=1024, w0_stride=1056, w0_pe_col=1056)) == -1 and b"shared memory" in err()
    assert call(L, mlp_struct(w0_stride=63)) == -1 and b"w0_stride" in err()
    assert call(L, mlp_struct(n_freq=4, w0_stride=96 + 27, w0_pe_col=97)) == -1 and b"w0_stride" in err()
    assert call(L, mlp_struct(), n=-1) == -1 and b"n out of range" in err()
    m = mlp_struct()
    m.weights[1] = None
    assert call(L, m) == -1 and b"NULL weight" in err()
    assert call(L, mlp_struct(), features=None) == -1 and b"NULL features" in err()
    assert call(L, mlp_struct(), base=None) == -1 and b"NULL base_rgb" in err()
    assert call(L, mlp_struct(n_freq=4, w0_stride=123), dirs=None) == -1 and b"NULL dirs" in err()
    assert call(L, mlp_struct(n_out=4), raw=None) == -1 and b"NULL raw_opacity" in err()
    assert L.b200gs_launch_count() == before


def test_abi_output_pointers_and_workspace(L):
    err = L.b200gs_last_error
    assert fwd(L, mlp_struct(), out=None) == -1 and b"NULL out" in err()
    assert fwd(L, mlp_struct(n_out=4), offsets=None) == -1 and b"NULL opacity output" in err()
    assert fwd(L, mlp_struct(), n=0, features=None, base=None, out=None) == 0          # no row: nothing is read, no launch
    assert bwd(L, mlp_struct(), v_params=None) == -1 and b"NULL v_params" in err()
    assert bwd(L, mlp_struct(), v_out=None) == -1 and b"NULL v_out" in err()
    assert bwd(L, mlp_struct(), v_base=None) == -1 and b"NULL v_base_rgb" in err()
    assert bwd(L, mlp_struct(n_out=4), v_raw=None) == -1 and b"NULL v_raw_opacity" in err()
    assert bwd(L, mlp_struct(), v_features=ctypes.c_void_p(20)) == -1 and b"aligned" in err()
    need = L.b200gs_appearance_mlp_workspace_bytes(64, -1, 64, 3, 3)
    assert need == 132 * 4 * (64 * 64 + 64 * 64 + 3 * 64 + 64 + 64 + 3)
    assert bwd(L, mlp_struct(), ws_bytes=need - 1) == -3 and b"workspace too small" in err()
    assert L.b200gs_appearance_mlp_workspace_bytes(64, 4, 64, 3, 4) == 132 * 4 * (64 * 96 + 64 * 64 + 4 * 64 + 64 + 64 + 4)
    for bad in ((60, -1, 64, 3, 3), (64, -1, 48, 3, 3), (64, -1, 64, 5, 3), (64, -1, 64, 3, 2), (1024, -1, 64, 3, 3)):
        assert L.b200gs_appearance_mlp_workspace_bytes(*bad) == 0
