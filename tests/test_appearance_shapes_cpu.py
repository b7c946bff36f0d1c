"""The appearance network at every shape the library accepts, without a GPU: a restatement of the kernels' shared-memory layout and
warp count (csrc/appearance.cu app_layout / app_warps) against the accept set and workspace size of the C entry points over the
whole shape grid, and the float64 oracle against the reference recorded at shapes other than the default
(tests/golden/appearance_shapes.npz, make_golden_appearance_shapes.py): outputs, gradients, state_dict keys and the model loading
the recorded state."""
import math
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import appearance_oracle as O
from oracle.appearance_oracle import SHAPE_ROWS as N, SHAPES, network_shape, sample_index

APPEARANCE_ID = 2
ZS = np.load(os.path.join(GOLDEN, "appearance_shapes.npz"))
SMEM_LIMIT = 227 * 1024          # opt-in dynamic shared memory per block of sm_90
MAX_CTAS = 132                   # persistent CTAs, and partial weight-gradient blocks
QUEUE = 512                      # ring of compacted row indices


def pe_width(n_freq):
    return 0 if n_freq < 0 else 3 * (2 * n_freq + 1)


def k0p(feat_dim, n_freq):
    return (feat_dim + pe_width(n_freq) + 7) // 8 * 8


def n_params(feat_dim, n_freq, n_neurons, n_layers, n_out):
    ins = [k0p(feat_dim, n_freq)] + [n_neurons] * (n_layers - 1)
    outs = [n_neurons] * (n_layers - 1) + [n_out]
    return sum(o * i for o, i in zip(outs, ins)) + sum(outs)


def smem_floats(shape, warps, bwd):
    """app_layout(...).total: the floats of dynamic shared memory of a CTA of `warps` warps (R = 16 warps rows per tile)"""
    feat_dim, n_freq, H, L, _ = shape
    R = 16 * warps
    ins = [k0p(feat_dim, n_freq)] + [H] * (L - 1)
    out_pad = [H] * (L - 1) + [8]            # the output layer is kept as 8 rows
    total = sum(o * (i + 4) for o, i in zip(out_pad, ins)) + sum(out_pad)         # weights (row stride + 4) and biases
    total += R * (ins[0] + 4)                                                        # x0
    total += (L - 1 if bwd else min(L - 1, 2)) * R * (H + 4)                         # hidden activations: the forward ping-pongs
    total += (R * 12 if bwd else 0) + R + R + QUEUE + 8                              # dz, norms, row list, ring, warp counts
    return total


def warps_of(shape, bwd):
    """app_warps: the most warps (8, 4, 2, 1) whose tile fits shared memory, 0 when none does"""
    for w in (8, 4, 2, 1):
        if smem_floats(shape, w, bwd) * 4 <= SMEM_LIMIT:
            return w
    return 0


def accepted(shape):
    feat_dim, n_freq, H, L, n_out = shape
    return (8 <= feat_dim <= 1024 and feat_dim % 8 == 0 and n_freq <= 16 and H in (64, 128) and 2 <= L <= 4 and n_out in (3, 4)
            and warps_of(shape, True) > 0)


def launch(shape, bwd):
    """(threads per CTA, dynamic shared memory bytes, tile rows R, chunk rows) of a K20 (bwd False) or K21 launch"""
    w = warps_of(shape, bwd)
    return 32 * w, smem_floats(shape, w, bwd) * 4, 16 * w, 32 * w


GRID = [(f, nf, h, l, o) for f in range(8, 1025, 8) for nf in range(-1, 17) for h in (64, 128) for l in (2, 3, 4) for o in (3, 4)]


@pytest.fixture(scope="module")
def L():
    from b200gs import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def test_restated_layout_is_the_accept_set_and_the_workspace(L):
    n_ok, pairs = 0, set()
    for s in GRID:
        got = int(L.b200gs_appearance_mlp_workspace_bytes(*s))
        if accepted(s):
            assert got == MAX_CTAS * n_params(*s) * 4, s
            fwd, bwd = warps_of(s, False), warps_of(s, True)
            assert fwd >= bwd and smem_floats(s, bwd, True) * 4 <= 232448, s
            pairs.add((fwd, bwd))
            n_ok += 1
        else:
            assert got == 0, s
    # shapes just outside the grid are refused too
    for s in ((1032, -1, 64, 2, 3), (0, -1, 64, 3, 3), (64, 17, 64, 3, 3), (64, -1, 96, 3, 3), (64, -1, 64, 1, 3), (64, -1, 64, 3, 5)):
        assert int(L.b200gs_appearance_mlp_workspace_bytes(*s)) == 0, s
    assert n_ok > 0 and pairs == {(8, 8), (8, 4), (4, 4), (4, 2), (2, 2), (2, 1), (1, 1)}


def visibility_accepted(feat_dim, n_neurons, n_layers):
    """the visibility network: an appearance network with no view direction and one output, on 8, 16, 24 or 32 grid features"""
    return feat_dim in (8, 16, 24, 32) and n_neurons in (64, 128) and 2 <= n_layers <= 4 and warps_of((feat_dim, -1, n_neurons, n_layers, 1), True) > 0


VISIBILITY_GRID = [(f, h, l) for f in range(0, 49, 4) for h in (32, 64, 96, 128) for l in range(1, 6)]


def test_restated_layout_is_the_visibility_accept_set_and_workspace(L):
    """the one-output layout keeps the output layer as 8 rows, so its tiles are those of the same network with 3 or 4 outputs; the
    workspace holds the one-output parameter count per persistent CTA"""
    n_ok = 0
    for f, h, l in VISIBILITY_GRID:
        got = int(L.b200gs_visibility_mlp_workspace_bytes(f, h, l))
        if visibility_accepted(f, h, l):
            s = (f, -1, h, l, 1)
            assert got == MAX_CTAS * n_params(*s) * 4, s
            assert launch(s, False) == launch((f, -1, h, l, 3), False) and launch(s, True) == launch((f, -1, h, l, 3), True), s
            assert warps_of(s, False) >= warps_of(s, True) > 0, s
            n_ok += 1
        else:
            assert got == 0, (f, h, l)
    assert n_ok == 4 * 2 * 3


def test_restated_layout_examples():
    """the warp counts the kernels' comments and DESIGN.md quote, and the widest accepted first layers"""
    assert (warps_of((64, -1, 64, 3, 3), False), warps_of((64, -1, 64, 3, 3), True)) == (8, 8)
    assert (warps_of((128, -1, 64, 4, 3), False), warps_of((128, -1, 64, 4, 3), True)) == (8, 4)
    assert (warps_of((112, -1, 128, 3, 3), False), warps_of((112, -1, 128, 3, 3), True)) == (4, 2)
    assert (warps_of((64, -1, 128, 4, 3), False), warps_of((64, -1, 128, 4, 3), True)) == (2, 1)
    widest = {(h, l): max(f for f in range(8, 1025, 8) if accepted((f, -1, h, l, 3))) for h in (64, 128) for l in (2, 3, 4)}
    assert widest == {(64, 2): 688, (64, 3): 616, (64, 4): 552, (128, 2): 368, (128, 3): 232, (128, 4): 104}


# ---- the reference recorded at other shapes ------------------------------------------------------------------------------------

def shape_case(name):
    """(ModelConfig overrides, network shape, float64 inputs, (embedding.weight, weights, biases) as float64 leaves)"""
    kw, seed = SHAPES[name]
    shape = network_shape(kw)
    x = {k: (v.double() if v.is_floating_point() else v) for k, v in O.shape_inputs(N, shape[0], seed).items()}
    st = O.shape_state(*shape, seed=seed)
    n = shape[3]
    leaf = lambda t: t.double().clone().requires_grad_(True)
    return kw, shape, x, (leaf(st["embedding.weight"]), [leaf(st[f"network.output_layers.{2 * i}.weight"]) for i in range(n)],
                          [leaf(st[f"network.output_layers.{2 * i}.bias"]) for i in range(n)])


def shape_state(name):
    kw, seed = SHAPES[name]
    return O.shape_state(*network_shape(kw), seed=seed)


def close(got, want, what, tol=2e-6):
    """float32 round-off of the recording: relative to the tensor's largest entry"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, what
    assert np.abs(got - want).max() <= tol * max(np.abs(want).max(), 1.0), (what, np.abs(got - want).max())


def sampled(t):
    return t.detach().reshape(-1)[torch.from_numpy(sample_index(t.numel()))]


def param_grads(emb, ws, bs):
    g = {"embedding.weight": emb.grad}
    for i, (w, b) in enumerate(zip(ws, bs)):
        g[f"network.output_layers.{2 * i}.weight"], g[f"network.output_layers.{2 * i}.bias"] = w.grad, b.grad
    return g


@pytest.mark.parametrize("name", list(SHAPES))
def test_rebuilt_state_is_the_recorded_one(name):
    st = shape_state(name)
    assert list(st) == [k[len("model."):] for k in ZS[f"{name}.keys"]]
    assert np.array_equal(np.array([math.fsum(v.double().flatten().tolist()) for v in st.values()]), ZS[f"{name}.state_sums"])     # exactly rounded sums


@pytest.mark.parametrize("name", list(SHAPES))
def test_oracle_reproduces_the_reference_model_at_other_shapes(name):
    kw, shape, x, (emb, ws, bs) = shape_case(name)
    mask = x["mask"]
    feats = x["features"][mask].clone().requires_grad_(True)
    dirs = torch.nn.functional.normalize(x["means"][mask].float() - x["cam_center"].float(), dim=-1).double()
    y = O.mlp(feats, emb[APPEARANCE_ID], ws, bs, dirs, shape[1], kw.get("normalize", False))
    (y * x["cot_model"][mask][:, :y.shape[1]]).sum().backward()
    close(y.detach(), ZS[f"{name}.model.out"], "out")
    close(sampled(feats.grad), ZS[f"{name}.model.v_features"], "v_features")
    for k, g in param_grads(emb, ws, bs).items():
        close(sampled(g), ZS[f"{name}.model.grad.{k}"], k)


@pytest.mark.parametrize("name", list(SHAPES))
def test_oracle_reproduces_the_reference_colours_at_other_shapes(name):
    kw, shape, x, (emb, ws, bs) = shape_case(name)
    mask = x["mask"]
    feats, base, raw = (x[k].clone().requires_grad_(True) for k in ("features", "base", "raw_opacity"))
    rgbs, opacities, offsets = O.colors(feats, mask, base, x["means"], x["cam_center"], raw, emb[APPEARANCE_ID], ws, bs, shape[1],
                                        kw.get("normalize", False))
    loss = (rgbs * x["cot_rgbs"]).sum()
    if offsets is not None:
        loss = loss + (opacities * x["cot_opacities"]).sum() + (offsets * x["cot_offsets"]).sum()
    loss.backward()
    want = ZS[f"{name}.colors.rgbs"]
    assert (want[mask.numpy()] == 0).any() and (want[mask.numpy()] == 1).any()        # both clamps are exercised
    close(rgbs.detach(), want, "rgbs")
    close(sampled(feats.grad), ZS[f"{name}.colors.v_features"], "v_features")
    close(base.grad, ZS[f"{name}.colors.v_base"], "v_base")
    assert (offsets is not None) == kw.get("with_opacity", False)
    if offsets is not None:
        assert (ZS[f"{name}.colors.opacities"] == 1).any()                              # the opacity clamp too
        close(opacities.detach(), ZS[f"{name}.colors.opacities"], "opacities")
        close(offsets.detach()[mask], ZS[f"{name}.colors.offsets"], "offsets")
        close(raw.grad, ZS[f"{name}.colors.v_raw_opacity"], "v_raw_opacity")
    for k, g in param_grads(emb, ws, bs).items():
        close(sampled(g), ZS[f"{name}.colors.grad.{k}"], k)


@pytest.mark.parametrize("name", list(SHAPES))
def test_state_dict_matches_the_reference_at_other_shapes(L, name):
    from b200gs.appearance import B200AppearanceModel, B200GSplatAppearanceEmbeddingRenderer, ModelConfig
    kw = SHAPES[name][0]
    state = shape_state(name)
    renderer = B200GSplatAppearanceEmbeddingRenderer(model=ModelConfig(n_appearances=1, **kw)).instantiate()
    renderer.load_state_dict({"model." + k: v for k, v in state.items()}, strict=True)
    assert list(renderer.state_dict().keys()) == list(ZS[f"{name}.keys"])
    assert renderer.config.model.n_appearances == 4
    model = B200AppearanceModel(ModelConfig(n_appearances=4, **kw))
    model.load_state_dict(state, strict=True)
    for k, v in model.state_dict().items():
        assert torch.equal(v, state[k])
