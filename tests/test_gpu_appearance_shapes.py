"""The appearance kernels (csrc/appearance.cu K20-K22) at network shapes other than the default, against the float64 oracle
(oracle/appearance_oracle.py): every warp count of the forward and the backward tile (8, 4, 2, 1; the 128-neuron and wide
networks fall back to fewer warps to fit shared memory), forward and backward at different warp counts, 64 and 128 neurons, 2 to
4 layers, feature widths from 8 to the widest accepted, 3 and 4 outputs, no view direction and 0 to 16 frequencies, with and
without normalisation.  Each shape runs at the row counts where its own tile (R = 16 x warps rows) and chunk (32 x warps rows)
change behaviour, with and without the colour epilogue.  Also: the launch configuration against the restated layout, determinism
of the weight gradients, the launch count without host synchronisation, the model on the reference recordings at other shapes
(tests/golden/appearance_shapes.npz) and the renderer with a 128-neuron, 4-layer network."""
import json
import os
import tempfile

import pytest
import torch

from oracle import appearance_oracle as O
from test_appearance_shapes_cpu import APPEARANCE_ID, SHAPES, ZS, launch, network_shape, param_grads, sample_index, shape_state, warps_of

pytestmark = pytest.mark.gpu
DEV = "cuda"

# name: (feat_dim, n_freq, n_neurons, n_layers, n_out, normalize); the warp counts (forward, backward) are those of warps_of
KERNEL_SHAPES = {
    "f8_l2_normalize": (8, -1, 64, 2, 3, True),              # (8, 8): one k-step, lanes 8..31 hold no feature
    "f32_freq6": (32, 6, 64, 3, 3, False),                   # (8, 8): 32 + 39 = 71 columns, padded to 72
    "f64_freq0_opacity": (64, 0, 64, 3, 4, False),            # (8, 8): PE = d only, 67 -> 72
    "f128_l4": (128, -1, 64, 4, 3, False),                    # (8, 4): four layers, the forward's buffers wrap
    "h128_f112": (112, -1, 128, 3, 3, False),                 # (4, 2)
    "h128_l2_freq4_normalize": (128, 4, 128, 2, 3, True),     # (4, 4): one hidden buffer, normalisation on a fallback tile
    "h128_l4_opacity": (64, -1, 128, 4, 4, False),            # (2, 1)
    "h128_freq16_opacity": (64, 16, 128, 3, 4, False),        # (2, 2): angle doubling up to 2^15 d
    "h128_l4_widest": (104, -1, 128, 4, 3, False),            # (1, 1)
    "h64_widest": (688, -1, 64, 2, 3, False),                 # (1, 1): the widest first layer of all
    "h64_l3_widest_normalize": (616, -1, 64, 3, 3, True),     # (1, 1)
    "h128_widest_opacity": (368, -1, 128, 2, 4, False),       # (1, 1): the widest 128-neuron first layer
}
WARPS = {"f8_l2_normalize": (8, 8), "f32_freq6": (8, 8), "f64_freq0_opacity": (8, 8), "f128_l4": (8, 4), "h128_f112": (4, 2),
         "h128_l2_freq4_normalize": (4, 4), "h128_l4_opacity": (2, 1), "h128_freq16_opacity": (2, 2), "h128_l4_widest": (1, 1),
         "h64_widest": (1, 1), "h64_l3_widest_normalize": (1, 1), "h128_widest_opacity": (1, 1)}
MILLION = ("h128_l4_widest", "h128_l2_freq4_normalize")      # a 1-warp and a 4-warp shape at a million rows


def net(name):
    return KERNEL_SHAPES[name][:5]


def seed_of(name):
    return 100 + list(KERNEL_SHAPES).index(name)


def cases(name):
    """row-count cases of a shape, from the tile R and the chunk of its forward and of its backward launch"""
    (_, _, rf, cf), (_, _, rb, cb) = launch(net(name), False), launch(net(name), True)
    out = ["rows0", "rows1"]
    for R, ch in ((rf, cf), (rb, cb)):
        out += [f"rows{v}_in{ch}" for v in (R - 1, R, R + 1)] + [f"all{ch + 1}"]
    out += ["masked_cta", "null_mask", "many"] + (["1M"] if name in MILLION else [])
    return list(dict.fromkeys(out))


def make_case(name, case, seed=3):
    """(N, mask or None) for a named row-count case of a shape"""
    (_, _, _, cf), (_, _, _, cb) = launch(net(name), False), launch(net(name), True)
    g = torch.Generator().manual_seed(seed)
    if case == "null_mask":
        return 3 * cf + 5, None
    if case == "masked_cta":          # the second CTA's first chunk of either kernel is all masked out, and so is its only one
        mask = torch.rand(3 * cf, generator=g) < 0.66
        mask[min(cf, cb):2 * max(cf, cb)] = False
        return 3 * cf, mask
    if case == "many":                # every one of the 132 CTAs walks three chunks or more, in both kernels
        n = 3 * 132 * cf + 17
        return n, torch.rand(n, generator=g) < 0.66
    if case == "1M":
        return 1_000_000, torch.rand(1_000_000, generator=g) < 0.66
    if case.startswith("all"):        # a full first chunk (two tiles) for the first CTA and one row for the second
        n = int(case[3:])
        return n, torch.ones(n, dtype=torch.bool)
    v, span = (int(case[4:]), cf) if "_in" not in case else map(int, case[4:].split("_in"))
    n = 2 * span + 5
    mask = torch.zeros(n, dtype=torch.bool)
    mask[torch.randperm(span, generator=g)[:v]] = True        # all of them in the first CTA's first chunk
    return n, mask


def make_inputs(n, feat_dim, seed=5):
    g = torch.Generator().manual_seed(seed)
    return {"features": torch.randn(n, feat_dim, generator=g), "means": torch.randn(n, 3, generator=g) * 2, "cam": torch.tensor([0.3, -4.0, 1.5]),
            "base": torch.rand(n, 3, generator=g) * 1.8 - 0.9, "raw": torch.rand(n, generator=g),
            "cot_rgbs": torch.randn(n, 3, generator=g), "cot_opacities": torch.randn(n, generator=g), "cot_offsets": torch.randn(n, generator=g),
            "cot_out": torch.randn(n, 4, generator=g)}


def unit_dirs(x):
    """the view directions as Model.forward receives them: normalised in float32"""
    return torch.nn.functional.normalize(x["means"] - x["cam"], dim=-1)


def state(name):
    """(embedding.weight, weights, biases) as float64 leaves"""
    F, n_freq, H, L, n_out = net(name)
    st = O.shape_state(F, n_freq, H, L, n_out, seed=seed_of(name))
    leaf = lambda t: t.double().clone().requires_grad_(True)
    return (leaf(st["embedding.weight"]), [leaf(st[f"network.output_layers.{2 * i}.weight"]) for i in range(L)],
            [leaf(st[f"network.output_layers.{2 * i}.bias"]) for i in range(L)])


def hidden_preactivations(features, dirs, emb_row, ws, bs, n_freq, normalize):
    """float64 pre-activations of every hidden unit of the given rows, and the sigmoid outputs"""
    f = features.double()
    e = emb_row.detach().reshape(1, -1).repeat(f.shape[0], 1)
    if normalize:
        f, e = torch.nn.functional.normalize(f, dim=-1), torch.nn.functional.normalize(e, dim=-1)
    parts = [f, e] + ([O.positional_encoding(dirs.double(), n_freq)] if n_freq >= 0 else [])
    h, pre = torch.cat(parts, dim=-1), []
    for l, (w, b) in enumerate(zip(ws, bs)):
        h = h @ w.detach().T + b.detach()
        if l < len(ws) - 1:
            pre.append(h)
            h = torch.relu(h)
    return torch.cat(pre, dim=-1), torch.sigmoid(h)


def grad_close(got, want, what, tol=1e-4):
    got, want = got.detach().cpu().double(), want.detach().double()
    scale = float(want.abs().max())
    if scale == 0:
        assert float(got.abs().max()) == 0, what
    else:
        assert float((got - want).abs().max()) <= tol * scale, (what, float((got - want).abs().max()) / scale)


def max_abs(got, want):
    return float((got.detach().cpu().double() - want.detach()).abs().max())


def kernel_dirs(name, x):
    """(dirs, cam, normalize_dirs) handed to the colour kernels, and the float64 directions the oracle uses (None: it normalises
    means - cam itself).  At 16 frequencies sin(2^15 d) moves by 2e-3 for a one-ulp change of d, so the kernels get float32 unit
    directions and the oracle those same values: the test then measures the encoding and the network, not float32 round-off of
    the normalisation."""
    if net(name)[1] >= 8:
        d = unit_dirs(x)
        return d, None, False, d.double()
    return x["means"], x["cam"], True, None


def test_warp_counts_of_the_shapes():
    assert {k: (warps_of(net(k), False), warps_of(net(k), True)) for k in KERNEL_SHAPES} == WARPS
    assert {w for p in WARPS.values() for w in p} == {8, 4, 2, 1}
    assert {p[0] for p in WARPS.values()} == {p[1] for p in WARPS.values()} == {8, 4, 2, 1}


@pytest.mark.parametrize("name,case", [(k, c) for k in KERNEL_SHAPES for c in cases(k)])
def test_kernels_at_every_shape_against_float64_oracle(name, case):
    from b200gs import ops
    F, n_freq, H, L, n_out = net(name)
    normalize, with_opacity = KERNEL_SHAPES[name][5], n_out == 4
    n, mask = make_case(name, case)
    x = make_inputs(n, F, seed=5 + seed_of(name))
    emb, ws, bs = state(name)
    full = torch.ones(n, dtype=torch.bool) if mask is None else mask
    dirs, cam, normalize_dirs, oracle_dirs = kernel_dirs(name, x)

    # Move the inputs off the decision boundaries, where float32 and float64 may choose differently (see test_gpu_appearance.py):
    # rows with a hidden pre-activation within 3e-6 of zero leave the mask, or, without a mask, get their features moved until
    # none is left; a colour within 1e-4 of a clamp bound and an opacity sum within 1e-4 of 1 are moved by 0.01.
    def ambiguous():
        rows = full.nonzero().squeeze(-1)
        near = torch.zeros(rows.numel(), dtype=torch.bool)
        for d in (unit_dirs(x), oracle_dirs if oracle_dirs is not None else torch.nn.functional.normalize(x["means"].double() - x["cam"].double(), dim=-1)):
            pre, s = hidden_preactivations(x["features"][rows], d[rows], emb[APPEARANCE_ID], ws, bs, n_freq, normalize)
            near |= (pre.abs() < 3e-6).any(dim=-1)
        return rows[near], s
    amb, s = ambiguous()
    assert amb.numel() <= 2 + n // 200
    if mask is not None:
        mask[amb] = False
    else:
        for _ in range(3):
            if amb.numel() == 0:
                break
            x["features"][amb] = x["features"][amb] * 1.01 + 0.01
            amb, s = ambiguous()
        assert amb.numel() == 0
    amb, s = ambiguous()
    assert amb.numel() == 0
    colour = x["base"].double()[full] + 0.5 + (s[:, :3] * 2 - 1)
    near = (colour.abs() < 1e-4) | ((colour - 1).abs() < 1e-4)
    x["base"][full] = torch.where(near, x["base"][full] + 0.01, x["base"][full])
    if with_opacity:
        near_o = ((x["raw"].double()[full] + s[:, 3]) - 1).abs() < 1e-4
        x["raw"][full] = torch.where(near_o, x["raw"][full] - 0.01, x["raw"][full])
    x["raw"] = torch.where((x["raw"] - 1).abs() < 1e-4, x["raw"] - 0.01, x["raw"])
    hidden = ~full
    t = lambda v: v.detach().float().to(DEV).requires_grad_(True)

    # the renderer's path: colour epilogue, dense rows, a mask
    feats, base, raw = (x[k].double().requires_grad_(True) for k in ("features", "base", "raw"))
    r_rgbs, r_opac, r_off = O.colors(feats, full, base, x["means"].double(), x["cam"].double(), raw, emb[APPEARANCE_ID], ws, bs, n_freq, normalize,
                                     view_dirs=oracle_dirs)
    loss = (r_rgbs * x["cot_rgbs"]).sum()
    if with_opacity:
        loss = loss + (r_opac * x["cot_opacities"]).sum() + (r_off * x["cot_offsets"]).sum()
    if loss.requires_grad:
        loss.backward()
    g_feats, g_base, g_raw = t(x["features"]), t(x["base"]), t(x["raw"])
    g_emb, g_ws, g_bs = t(emb), [t(w) for w in ws], [t(b) for b in bs]
    e = g_emb[APPEARANCE_ID]
    if normalize:
        e = torch.nn.functional.normalize(e, dim=-1)
    out = ops.appearance_mlp(g_feats, e, g_ws, g_bs, dirs=dirs.to(DEV), cam=None if cam is None else cam.to(DEV), n_freq=n_freq, normalize=normalize,
                             normalize_dirs=normalize_dirs, mask=None if mask is None else mask.to(DEV), base_rgb=g_base,
                             raw_opacity=g_raw if with_opacity else None)
    rgbs, opacities, offsets = out if with_opacity else (out, None, None)
    k_loss = (rgbs * x["cot_rgbs"].to(DEV)).sum()
    if with_opacity:
        k_loss = k_loss + (opacities * x["cot_opacities"].to(DEV)).sum() + (offsets * x["cot_offsets"].to(DEV)).sum()
    k_loss.backward()
    torch.cuda.synchronize()

    assert max_abs(rgbs, r_rgbs) <= 2e-5
    if int(full.sum()) >= 127:
        live = r_rgbs.detach()[full]
        assert bool((live == 0).any()) and bool((live == 1).any())          # both clamps are active somewhere
    assert not rgbs.detach().cpu()[hidden].any() and not g_feats.grad.cpu()[hidden].any() and not g_base.grad.cpu()[hidden].any()
    zero = lambda t_, like: torch.zeros_like(like).double() if t_ is None else t_
    grad_close(g_feats.grad, zero(feats.grad, x["features"]), "v_features")
    grad_close(g_base.grad, zero(base.grad, x["base"]), "v_base_rgb")
    if with_opacity:
        assert max_abs(opacities, r_opac) <= 2e-5 and max_abs(offsets, r_off) <= 2e-5
        assert not offsets.detach().cpu()[hidden].any()
        grad_close(g_raw.grad, zero(raw.grad, x["raw"]), "v_raw_opacity")
    want = param_grads(emb, ws, bs)
    for k, g in param_grads(g_emb, g_ws, g_bs).items():
        grad_close(g, zero(want[k], g.cpu()), k)

    # Model.forward's path: no epilogue, the sigmoid outputs of every row (zeros outside the mask), unit directions as given
    for p in [emb] + ws + bs:
        p.grad = None
    d = unit_dirs(x)
    feats = x["features"].double().requires_grad_(True)
    s = torch.zeros(n, n_out, dtype=torch.float64)
    s[full] = O.mlp(feats[full], emb[APPEARANCE_ID], ws, bs, d.double()[full], n_freq, normalize)
    if s.requires_grad:
        (s * x["cot_out"][:, :n_out]).sum().backward()
    g_feats = t(x["features"])
    g_emb, g_ws, g_bs = t(emb), [t(w) for w in ws], [t(b) for b in bs]
    e = g_emb[APPEARANCE_ID]
    if normalize:
        e = torch.nn.functional.normalize(e, dim=-1)
    y = ops.appearance_mlp(g_feats, e, g_ws, g_bs, dirs=d.to(DEV), n_freq=n_freq, normalize=normalize, mask=None if mask is None else mask.to(DEV))
    assert y.shape == (n, n_out)
    (y * x["cot_out"][:, :n_out].to(DEV)).sum().backward()
    torch.cuda.synchronize()
    assert max_abs(y, s) <= 2e-5
    assert not y.detach().cpu()[hidden].any() and not g_feats.grad.cpu()[hidden].any()
    grad_close(g_feats.grad, zero(feats.grad, x["features"]), "v_features (no epilogue)")
    want = param_grads(emb, ws, bs)
    for k, g in param_grads(g_emb, g_ws, g_bs).items():
        grad_close(g, zero(want[k], g.cpu()), k + " (no epilogue)")


def _kernel_launches(fn):
    """[(kernel name, block, dynamic shared memory bytes, grid)] of the CUDA kernels fn launches, from a torch.profiler trace"""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    return [(e["name"], e["args"]["block"], e["args"]["shared memory"], e["args"]["grid"]) for e in events
            if e.get("cat") == "kernel" and "appearance" in e.get("name", "")]


@pytest.mark.parametrize("name", list(KERNEL_SHAPES))
def test_launch_configuration_is_the_restated_layout(name):
    from b200gs import ops
    F, n_freq, H, L, n_out = net(name)
    normalize = KERNEL_SHAPES[name][5]
    n = 1000
    x = make_inputs(n, F)
    emb, ws, bs = state(name)
    t = lambda v: v.detach().float().to(DEV).requires_grad_(True)
    feats, g_ws, g_bs = t(x["features"]), [t(w) for w in ws], [t(b) for b in bs]
    e = emb.detach()[APPEARANCE_ID].float().to(DEV)

    def run():
        y = ops.appearance_mlp(feats, e, g_ws, g_bs, dirs=unit_dirs(x).to(DEV), n_freq=n_freq, normalize=normalize)
        y.sum().backward()
    seen = _kernel_launches(run)
    fwd = [k for k in seen if "appearance_mlp_fwd_kernel" in k[0]]
    bwd = [k for k in seen if "appearance_mlp_bwd_kernel" in k[0]]
    assert len(fwd) == len(bwd) == 1 and len([k for k in seen if "appearance_reduce_kernel" in k[0]]) == 1, seen
    for (_, block, smem, grid), is_bwd in ((fwd[0], False), (bwd[0], True)):
        threads, smem_bytes, _, _ = launch(net(name), is_bwd)
        assert list(block) == [threads, 1, 1] and threads == 32 * WARPS[name][is_bwd], (name, is_bwd, block)
        assert smem == smem_bytes <= 232448, (name, is_bwd, smem, smem_bytes)
        assert list(grid) == [min(132, -(-n // threads)), 1, 1], (name, is_bwd, grid)


@pytest.mark.parametrize("name", ["h128_l4_widest", "f128_l4", "h128_f112"])
def test_weight_gradients_are_deterministic_at_fallback_shapes(name):
    from b200gs import ops
    F, n_freq, H, L, n_out = net(name)
    normalize = KERNEL_SHAPES[name][5]
    n, mask = make_case(name, "many")
    x = make_inputs(n, F)
    emb, ws, bs = state(name)
    t = lambda v: v.detach().float().to(DEV).requires_grad_(True)
    g_emb, g_ws, g_bs = t(emb), [t(w) for w in ws], [t(b) for b in bs]
    feats, base, cot = x["features"].to(DEV), x["base"].to(DEV), x["cot_rgbs"].to(DEV)
    runs = []
    for _ in range(2):
        for p in [g_emb] + g_ws + g_bs:
            p.grad = None
        rgbs = ops.appearance_mlp(feats, g_emb[APPEARANCE_ID], g_ws, g_bs, dirs=x["means"].to(DEV), cam=x["cam"].to(DEV), n_freq=n_freq,
                                  normalize=normalize, normalize_dirs=True, mask=mask.to(DEV), base_rgb=base)
        (rgbs * cot).sum().backward()
        runs.append([p.grad.clone() for p in [g_emb] + g_ws + g_bs])
    assert all(torch.equal(a, b) for a, b in zip(*runs)) and all(bool(g.abs().sum() > 0) for g in runs[0])


def test_launch_count_and_no_host_synchronisation_on_a_fallback_tile():
    from b200gs import _lib, ops
    name = "h128_l4_opacity"            # forward 2 warps, backward 1
    F, n_freq, H, L, n_out = net(name)
    Lb = _lib.lib()
    emb, ws, bs = state(name)
    t = lambda v: v.detach().float().to(DEV).requires_grad_(True)
    g_emb, g_ws, g_bs = t(emb), [t(w) for w in ws], [t(b) for b in bs]
    deltas = []
    for n in (1000, 300_000):
        x = make_inputs(n, F)
        feats, base, raw = t(x["features"]), t(x["base"]), t(x["raw"])
        cot = torch.randn(n, 3, device=DEV)
        for vis in (torch.zeros(n, dtype=torch.bool, device=DEV), torch.rand(n, device=DEV) < 0.66):
            e = g_emb[APPEARANCE_ID]
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                c0 = Lb.b200gs_launch_count()
                rgbs, opacities, offsets = ops.appearance_mlp(feats, e, g_ws, g_bs, mask=vis, base_rgb=base, raw_opacity=raw)
                c1 = Lb.b200gs_launch_count()
                torch.autograd.backward([rgbs, opacities], [cot, torch.ones_like(opacities)], inputs=[feats, base, raw, g_emb] + g_ws + g_bs)
                c2 = Lb.b200gs_launch_count()
            finally:
                torch.cuda.set_sync_debug_mode("default")
            deltas.append((c1 - c0, c2 - c1))
    assert set(deltas) == {(ops.APPEARANCE_FWD_LAUNCHES, ops.APPEARANCE_BWD_LAUNCHES)} == {(1, 2)}


# ---- the reference recordings at other shapes ------------------------------------------------------------------------------------

def _sampled(t):
    return t.detach().cpu().reshape(-1)[torch.from_numpy(sample_index(t.numel()))]


@pytest.mark.parametrize("name", list(SHAPES))
def test_model_equals_the_reference_recording_at_other_shapes(name):
    from b200gs.appearance import B200AppearanceModel, ModelConfig
    kw, seed = SHAPES[name]
    x = O.shape_inputs(96, network_shape(kw)[0], seed)
    mask = x["mask"]
    model = B200AppearanceModel(ModelConfig(n_appearances=4, **kw))
    model.load_state_dict(shape_state(name), strict=True)
    model = model.to(DEV)
    feats = x["features"][mask].to(DEV).requires_grad_(True)
    dirs = torch.nn.functional.normalize(x["means"][mask] - x["cam_center"], dim=-1).to(DEV)
    y = model(feats, torch.tensor([APPEARANCE_ID], dtype=torch.int32, device=DEV), dirs)
    (y * x["cot_model"][mask][:, :y.shape[1]].to(DEV)).sum().backward()
    torch.cuda.synchronize()
    assert float((y.detach().cpu() - torch.from_numpy(ZS[f"{name}.model.out"])).abs().max()) <= 2e-5
    grad_close(_sampled(feats.grad), torch.from_numpy(ZS[f"{name}.model.v_features"]), "v_features")
    for k, p in model.named_parameters():
        grad_close(_sampled(p.grad), torch.from_numpy(ZS[f"{name}.model.grad.{k}"]), k)


def test_renderer_with_a_128_neuron_4_layer_network_against_oracle_and_v1_blend():
    from b200gs.appearance import B200GSplatAppearanceEmbeddingRenderer, ModelConfig
    from b200gs.v1 import B200GSplatV1Renderer
    from test_gpu_appearance import _scene
    name = "neurons128_layers4_view_opacity"
    kw = SHAPES[name][0]
    pc, cam = _scene()
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    r = B200GSplatAppearanceEmbeddingRenderer(model=ModelConfig(n_appearances=4, **kw)).instantiate()
    st = shape_state(name)
    r.load_state_dict({"model." + k: v for k, v in st.items()}, strict=True)
    r = r.to(DEV)
    assert (warps_of(network_shape(kw), False), warps_of(network_shape(kw), True)) == (1, 1)      # 96-wide first layer, 4 layers
    handed = {}
    get_opacities = r.get_opacities

    def spy(*a, **k):
        handed["opacities"], handed["rgbs"] = get_opacities(*a, **k)
        return handed["opacities"], handed["rgbs"]
    r.get_opacities = spy
    out = r(cam, pc, bg, warm_up=False)
    vis = out["visibility_filter"]
    assert 0 < int(vis.sum()) < vis.numel()
    n = kw["n_layers"]
    ws = [st[f"network.output_layers.{2 * i}.weight"].double() for i in range(n)]
    bs = [st[f"network.output_layers.{2 * i}.bias"].double() for i in range(n)]
    base = r.sh_colors(cam, pc, vis).detach().cpu().double()
    want = O.colors(pc.get_appearance_features().detach().cpu().double(), vis.cpu(), base, pc.get_xyz.detach().cpu().double(),
                    cam.camera_center.cpu().double(), pc.get_opacities().squeeze(-1).detach().cpu().double(),
                    st["embedding.weight"].double()[APPEARANCE_ID], ws, bs, network_shape(kw)[1], False)
    assert float((handed["rgbs"].detach().cpu().double() - want[0]).abs().max()) <= 2e-5
    assert float((handed["opacities"].detach().cpu().double() - want[1]).abs().max()) <= 2e-5

    plain = B200GSplatV1Renderer(separate_sh=True).instantiate().to(DEV)        # the same blend, handed those colours and opacities
    plain.get_rgbs = lambda *a, **k: handed["rgbs"].detach()
    plain.get_opacities = lambda camera, model, projections, visibility, status, **k: (handed["opacities"].detach(), status)
    assert torch.equal(plain(cam, pc, bg)["render"], out["render"])
    out["render"].sum().backward()
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in r.model.parameters())
    assert bool(torch.isfinite(pc.appearance_features.grad).all()) and not pc.appearance_features.grad[~vis].any()
