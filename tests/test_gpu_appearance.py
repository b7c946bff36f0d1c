"""The appearance colour pass on the GPU (csrc/appearance.cu, b200gs.appearance) against the float64 oracle
(oracle/appearance_oracle.py) and the reference's recorded outputs (tests/golden/appearance.npz): the kernels for every recorded
configuration at the row counts where the compaction and the row tile change behaviour, the model on the recorded compact rows,
the renderer against the plain gsplat-v1 renderer, determinism of the weight gradients, the launch count and the absence of
host synchronisation."""
import numpy as np
import pytest
import torch

from oracle import appearance_oracle as O
from test_appearance_oracle_cpu import APPEARANCE_ID, VARIANTS, Z, golden_inputs, golden_state, n_freq_of, param_grads

pytestmark = pytest.mark.gpu
DEV = "cuda"
TILE_ROWS = 128          # rows of one CTA tile for the 64-neuron networks: 8 warps x 16
CHUNK = 256              # rows one CTA scans per step


def make_case(case, seed=3):
    """(N, mask or None) for a named row-count case"""
    g = torch.Generator().manual_seed(seed)
    if case == "null_mask":
        return TILE_ROWS + 1, None
    if case == "masked_cta":          # rows [256, 512) are the second CTA's only chunk: it has nothing to do
        mask = torch.rand(3 * CHUNK, generator=g) < 0.66
        mask[CHUNK:2 * CHUNK] = False
        return 3 * CHUNK, mask
    if case == "1M":
        return 1_000_000, torch.rand(1_000_000, generator=g) < 0.66
    v, n = int(case), 400
    mask = torch.zeros(n, dtype=torch.bool)
    mask[torch.randperm(n, generator=g)[:v]] = True
    return n, mask


def make_inputs(n, seed=5):
    g = torch.Generator().manual_seed(seed)
    return {"features": torch.randn(n, 64, generator=g), "means": torch.randn(n, 3, generator=g) * 2, "cam": torch.tensor([0.3, -4.0, 1.5]),
            "base": torch.rand(n, 3, generator=g) * 1.8 - 0.9, "raw": torch.rand(n, generator=g),
            "cot_rgbs": torch.randn(n, 3, generator=g), "cot_opacities": torch.randn(n, generator=g), "cot_offsets": torch.randn(n, generator=g)}


def hidden_preactivations(x, mask, emb_row, ws, bs, n_freq, normalize):
    """float64 pre-activations of every hidden unit of the masked rows, and the sigmoid outputs"""
    f = x["features"].double()[mask]
    e = emb_row.detach().reshape(1, -1).repeat(f.shape[0], 1)
    if normalize:
        f, e = torch.nn.functional.normalize(f, dim=-1), torch.nn.functional.normalize(e, dim=-1)
    parts = [f, e]
    if n_freq >= 0:
        d = torch.nn.functional.normalize(x["means"][mask] - x["cam"], dim=-1).double()
        parts.append(O.positional_encoding(d, n_freq))
    h, pre = torch.cat(parts, dim=-1), []
    for l, (w, b) in enumerate(zip(ws, bs)):
        h = h @ w.detach().T + b.detach()
        if l < len(ws) - 1:
            pre.append(h)
            h = torch.relu(h)
    return torch.cat(pre, dim=-1), torch.sigmoid(h)


def run_kernels(x, mask, emb, ws, bs, n_freq, normalize, with_opacity):
    from b200gs import ops
    t = lambda v: v.detach().float().to(DEV).requires_grad_(True)
    feats, base, raw = t(x["features"]), t(x["base"]), t(x["raw"])
    emb_g, ws_g, bs_g = t(emb), [t(w) for w in ws], [t(b) for b in bs]
    e = emb_g[APPEARANCE_ID]
    if normalize:
        e = torch.nn.functional.normalize(e, dim=-1)
    out = ops.appearance_mlp(feats, e, ws_g, bs_g, dirs=x["means"].to(DEV), cam=x["cam"].to(DEV), n_freq=n_freq, normalize=normalize,
                             normalize_dirs=True, mask=None if mask is None else mask.to(DEV), base_rgb=base,
                             raw_opacity=raw if with_opacity else None)
    if with_opacity:
        rgbs, opacities, offsets = out
        loss = (rgbs * x["cot_rgbs"].to(DEV)).sum() + (opacities * x["cot_opacities"].to(DEV)).sum() + (offsets * x["cot_offsets"].to(DEV)).sum()
    else:
        rgbs, opacities, offsets = out, None, None
        loss = (rgbs * x["cot_rgbs"].to(DEV)).sum()
    loss.backward()
    torch.cuda.synchronize()
    return rgbs, opacities, offsets, feats.grad, base.grad, raw.grad, param_grads(emb_g, ws_g, bs_g)


def grad_close(got, want, what, tol=1e-4):
    got, want = got.detach().cpu().double(), want.detach().double()
    scale = float(want.abs().max())
    if scale == 0:
        assert float(got.abs().max()) == 0, what
    else:
        assert float((got - want).abs().max()) <= tol * scale, (what, float((got - want).abs().max()) / scale)


def max_abs(got, want):
    return float((got.detach().cpu().double() - want.detach()).abs().max())


CASES = ["0", "1", str(TILE_ROWS - 1), str(TILE_ROWS), str(TILE_ROWS + 1), "null_mask", "masked_cta"]


@pytest.mark.parametrize("case,name", [(c, v) for v in VARIANTS for c in CASES] + [("1M", "default"), ("1M", "with_opacity"), ("1M", "view_dependent")])
def test_kernels_against_float64_oracle(case, name):
    kw = VARIANTS[name]
    n_freq, normalize, with_opacity = n_freq_of(kw), kw.get("normalize", False), kw.get("with_opacity", False)
    n, mask = make_case(case)
    x = make_inputs(n)
    emb, ws, bs = golden_state(name)
    full = torch.ones(n, dtype=torch.bool) if mask is None else mask
    # Move the inputs off the decision boundaries, where float32 and float64 may choose differently.  A hidden unit whose
    # pre-activation is within 3e-6 of zero may be on in one precision and off in the other, which changes that row's share of
    # every gradient by the unit's whole contribution (at a million rows the weight-gradient sums then differ by ~1e-3): such
    # rows (a few hundred in a million) are masked out.  A colour within 1e-4 of a clamp bound and an opacity sum within 1e-4 of
    # 1 are moved by 0.01.
    pre, s = hidden_preactivations(x, full, emb[APPEARANCE_ID], ws, bs, n_freq, normalize)
    if mask is not None:
        ambiguous = full.nonzero().squeeze(-1)[(pre.abs() < 3e-6).any(dim=-1)]
        assert ambiguous.numel() <= 2 + n // 1000
        mask[ambiguous] = False
        pre, s = hidden_preactivations(x, full, emb[APPEARANCE_ID], ws, bs, n_freq, normalize)
    colour = x["base"].double()[full] + 0.5 + (s[:, :3] * 2 - 1)
    near = (colour.abs() < 1e-4) | ((colour - 1).abs() < 1e-4)
    x["base"][full] = torch.where(near, x["base"][full] + 0.01, x["base"][full])
    if with_opacity:
        near_o = ((x["raw"].double()[full] + s[:, 3]) - 1).abs() < 1e-4
        x["raw"][full] = torch.where(near_o, x["raw"][full] - 0.01, x["raw"][full])
    x["raw"] = torch.where((x["raw"] - 1).abs() < 1e-4, x["raw"] - 0.01, x["raw"])

    feats, base, raw = (x[k].double().requires_grad_(True) for k in ("features", "base", "raw"))
    r_rgbs, r_opac, r_off = O.colors(feats, full, base, x["means"].double(), x["cam"].double(), raw, emb[APPEARANCE_ID], ws, bs, n_freq, normalize)
    loss = (r_rgbs * x["cot_rgbs"]).sum()
    if with_opacity:
        loss = loss + (r_opac * x["cot_opacities"]).sum() + (r_off * x["cot_offsets"]).sum()
    if loss.requires_grad:
        loss.backward()
    rgbs, opacities, offsets, v_feats, v_base, v_raw, grads = run_kernels(x, mask, emb, ws, bs, n_freq, normalize, with_opacity)

    assert max_abs(rgbs, r_rgbs) <= 2e-5
    live = r_rgbs.detach()[full]
    if int(full.sum()) >= TILE_ROWS - 1:
        assert bool((live == 0).any()) and bool((live == 1).any())          # both clamps are active somewhere
    hidden = ~full
    assert not rgbs.detach().cpu()[hidden].any() and not v_feats.cpu()[hidden].any() and not v_base.cpu()[hidden].any()
    zero = lambda t: torch.zeros_like(x["features"]).double() if t is None else t
    grad_close(v_feats, zero(feats.grad), "v_features")
    grad_close(v_base, zero(base.grad)[:, :3] if base.grad is not None else torch.zeros(n, 3).double(), "v_base_rgb")
    if with_opacity:
        assert max_abs(opacities, r_opac) <= 2e-5 and max_abs(offsets, r_off) <= 2e-5
        assert not offsets.detach().cpu()[hidden].any()
        grad_close(v_raw, raw.grad if raw.grad is not None else torch.zeros(n).double(), "v_raw_opacity")
    want = param_grads(emb, ws, bs)
    for k, g in grads.items():
        grad_close(g, want[k] if want[k] is not None else torch.zeros_like(g).cpu().double(), k)


@pytest.mark.parametrize("name", list(VARIANTS))
def test_model_equals_the_reference_recording(name):
    from b200gs.appearance import B200AppearanceModel, ModelConfig
    x = golden_inputs(torch.float32)
    mask = x["mask"]
    model = B200AppearanceModel(ModelConfig(n_appearances=4, **VARIANTS[name]))
    model.load_state_dict({k[len(name) + 7:]: torch.from_numpy(Z[k]) for k in Z.files if k.startswith(name + ".state.")}, strict=True)
    model = model.to(DEV)
    feats = x["features"][mask].to(DEV).requires_grad_(True)
    dirs = torch.nn.functional.normalize(x["means"][mask] - x["cam_center"], dim=-1).to(DEV)
    y = model(feats, torch.tensor([APPEARANCE_ID], dtype=torch.int32, device=DEV), dirs)
    (y * x["cot_model"][mask][:, :y.shape[1]].to(DEV)).sum().backward()
    torch.cuda.synchronize()
    assert float((y.detach().cpu() - torch.from_numpy(Z[f"{name}.model.out"])).abs().max()) <= 2e-5
    grad_close(feats.grad, torch.from_numpy(Z[f"{name}.model.v_features"]), "v_features")
    for k, p in model.named_parameters():
        grad_close(p.grad, torch.from_numpy(Z[f"{name}.model.grad.{k}"]), k)
    empty = model(feats[:0].detach(), torch.tensor([APPEARANCE_ID], device=DEV), dirs[:0])
    assert empty.shape == (0, model.n_output_dims)


def _scene(n=4096, W=256, H=192):
    from b200gs.scene import SyntheticGaussians, make_ring_cameras, make_scene

    class AppearanceGaussians(SyntheticGaussians):
        def __init__(self, raw):
            super().__init__(raw)
            self.appearance_features = torch.nn.Parameter(torch.randn(raw["means"].shape[0], 64, generator=torch.Generator().manual_seed(9)))

        def get_appearance_features(self):
            return self.appearance_features

    pc = AppearanceGaussians(make_scene(n, 5, mean_scale=0.05)).to(DEV)
    cam = make_ring_cameras(W, H)[3].to_device(DEV)
    cam.appearance_id = torch.tensor([APPEARANCE_ID], dtype=torch.int32, device=DEV)
    return pc, cam


def _renderer(name):
    from b200gs.appearance import B200GSplatAppearanceEmbeddingRenderer, ModelConfig
    r = B200GSplatAppearanceEmbeddingRenderer(model=ModelConfig(n_appearances=4, **VARIANTS[name])).instantiate()
    r.load_state_dict({"model." + k[len(name) + 7:]: torch.from_numpy(Z[k]) for k in Z.files if k.startswith(name + ".state.")}, strict=True)
    return r.to(DEV)


@pytest.mark.parametrize("name", ["default", "view_dependent", "with_opacity"])
def test_renderer_against_oracle_and_v1_blend(name):
    from b200gs.v1 import B200GSplatV1Renderer
    kw = VARIANTS[name]
    pc, cam = _scene()
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    r = _renderer(name)
    handed = {}
    get_opacities = r.get_opacities

    def spy(*a, **k):
        handed["opacities"], handed["rgbs"] = get_opacities(*a, **k)
        return handed["opacities"], handed["rgbs"]
    r.get_opacities = spy
    out = r(cam, pc, bg, warm_up=False)
    vis = out["visibility_filter"]
    assert 0 < int(vis.sum()) < vis.numel()
    emb, ws, bs = golden_state(name)
    base = r.sh_colors(cam, pc, vis).detach().cpu().double()
    want = O.colors(pc.get_appearance_features().detach().cpu().double(), vis.cpu(), base, pc.get_xyz.detach().cpu().double(),
                    cam.camera_center.cpu().double(), pc.get_opacities().squeeze(-1).detach().cpu().double(), emb[APPEARANCE_ID].detach(),
                    [w.detach() for w in ws], [b.detach() for b in bs], n_freq_of(kw), kw.get("normalize", False))
    assert float((handed["rgbs"].detach().cpu().double() - want[0]).abs().max()) <= 2e-5
    assert float((handed["opacities"].detach().cpu().double() - want[1]).abs().max()) <= 2e-5

    plain = B200GSplatV1Renderer(separate_sh=True).instantiate().to(DEV)        # the same blend, handed those colours and opacities
    plain.get_rgbs = lambda *a, **k: handed["rgbs"].detach()
    plain.get_opacities = lambda camera, model, projections, visibility, status, **k: (handed["opacities"].detach(), status)
    assert torch.equal(plain(cam, pc, bg)["render"], out["render"])
    out["render"].sum().backward()
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in r.model.parameters())
    assert bool(torch.isfinite(pc.appearance_features.grad).all()) and not pc.appearance_features.grad[~vis].any()


def test_renderer_before_warm_up_is_the_v1_renderer():
    from b200gs.v1 import B200GSplatV1Renderer
    pc, cam = _scene()
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    r = _renderer("default")
    r.config.optimization.warm_up = 10
    out = r.training_forward(3, None, cam, pc, bg)
    ref = B200GSplatV1Renderer(separate_sh=True).instantiate().to(DEV)(cam, pc, bg)
    assert torch.equal(out["render"], ref["render"]) and torch.equal(out["alpha"], ref["alpha"])
    past = r.training_forward(10, None, cam, pc, bg)
    assert not torch.equal(past["render"], ref["render"])


def _colour_pass(r, pc, cam, vis, warm_up=False):
    rgbs, opacities, _ = r._get_rgbs_and_opacities(cam, pc, None, vis, None, warm_up=warm_up)
    return rgbs, opacities


def test_weight_gradients_are_deterministic():
    pc, cam = _scene(n=200_000)
    r = _renderer("with_opacity")
    vis = torch.rand(200_000, generator=torch.Generator().manual_seed(1)).to(DEV) < 0.66
    cot = torch.randn(200_000, 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    runs = []
    for _ in range(2):
        r.zero_grad()
        rgbs, opacities = _colour_pass(r, pc, cam, vis)
        ((rgbs * cot).sum() + opacities.sum()).backward()
        runs.append([p.grad.clone() for p in r.model.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*runs)) and all(bool(g.abs().sum() > 0) for g in runs[0])


def test_launch_count_and_no_host_synchronisation():
    from b200gs import _lib, ops
    L = _lib.lib()
    r = _renderer("with_opacity")
    deltas = []
    for n in (1000, 300_000):
        pc, cam = _scene(n=n)
        cot = torch.randn(n, 3, device=DEV)
        for vis in (torch.zeros(n, dtype=torch.bool, device=DEV), torch.rand(n, device=DEV) < 0.66):
            feats, xyz, raw = pc.get_appearance_features(), pc.get_xyz.detach(), pc.get_opacities().squeeze(-1)
            base = r.sh_colors(cam, pc, vis)
            lin = r.model.linears()
            e = r.model.embedding_row(cam.appearance_id)
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                c0 = L.b200gs_launch_count()
                rgbs, opacities, offsets = ops.appearance_mlp(feats, e, [m.weight for m in lin], [m.bias for m in lin], dirs=xyz, cam=cam.camera_center,
                                                              n_freq=-1, mask=vis, base_rgb=base, raw_opacity=raw)
                c1 = L.b200gs_launch_count()
                torch.autograd.backward([rgbs, opacities], [cot, torch.ones_like(opacities)], inputs=[feats] + list(r.model.parameters()))
                c2 = L.b200gs_launch_count()
            finally:
                torch.cuda.set_sync_debug_mode("default")
            deltas.append((c1 - c0, c2 - c1))
    assert set(deltas) == {(ops.APPEARANCE_FWD_LAUNCHES, ops.APPEARANCE_BWD_LAUNCHES)} == {(1, 2)}
    # and the renderer's whole colour pass (masked SH + fused colours) is free of host synchronisation too
    pc, cam = _scene()
    vis = torch.rand(4096, device=DEV) < 0.5
    cot = torch.randn(4096, 3, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        rgbs, opacities = _colour_pass(r, pc, cam, vis)
        ((rgbs * cot).sum() + opacities.sum()).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
