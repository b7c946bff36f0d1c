"""K49 / K50 (csrc/swag.cu) and the SWAG MLP epilogue of K20 / K21 (csrc/appearance.cu) through ops.hash_grid_encode,
ops.swag_colours_and_opacities and b200gs.swag.B200SWAGRenderer on the GPU, against the float64 oracle (oracle/swag_oracle.py) and
the reference's own torch steps on the compat stand-ins."""
import math
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import swag_oracle as S

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def rel(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30)) if b.numel() else 0.0


GRIDS = {   # name: grid (dense-only, mixed and all-hashed levels, F 2 and 4)
    "default": dict(n_levels=8, n_features_per_level=4, log2_hashmap_size=19, base_resolution=16, per_level_scale=2.0),
    "dense_f4": dict(n_levels=3, n_features_per_level=4, log2_hashmap_size=24, base_resolution=8, per_level_scale=1.5),
    "dense_f2": dict(n_levels=4, n_features_per_level=2, log2_hashmap_size=24, base_resolution=4, per_level_scale=2.0),
    "mixed_f2": dict(n_levels=6, n_features_per_level=2, log2_hashmap_size=14, base_resolution=12, per_level_scale=1.7),
    "hashed_f4": dict(n_levels=5, n_features_per_level=4, log2_hashmap_size=10, base_resolution=16, per_level_scale=1.3),
    "hashed_f2_16": dict(n_levels=16, n_features_per_level=2, log2_hashmap_size=12, base_resolution=20, per_level_scale=1.38),
    "one_level": dict(n_levels=1, n_features_per_level=4, log2_hashmap_size=1, base_resolution=1, per_level_scale=1.0),
}


def grid_points(n, grid, seed=0):
    """fp32 points: uniform in [-0.5, 1.5] (outside the unit box too), with vertices of level 1, 0, 1 and negatives first"""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, generator=g) * 2 - 0.5
    lv = S.levels(**grid)
    special = [[0, 0, 0], [1, 1, 1], [1, 0, 1], [-1e-3, 0.5, 2.0], [-3.25, -0.75, 1.0]]
    scale = float(lv[min(1, len(lv) - 1)][0])
    if scale > 0:
        special += [[(k - 0.5) / scale] * 3 for k in (0, 1, 3)]      # pos = k exactly: on a vertex
    k = min(n, len(special))
    if k:
        x[:k] = torch.tensor(special[:k], dtype=torch.float32)
    return x


@pytest.mark.parametrize("name", sorted(GRIDS))
@pytest.mark.parametrize("n", [0, 1, 3000])
def test_hash_grid_encode_matches_the_oracle(name, n):
    from b200gs import ops
    grid = GRIDS[name]
    x = grid_points(n, grid, seed=n)
    nparams = S.n_params(**grid)
    assert ops.hash_grid_params(**grid) == nparams
    table = (torch.rand(nparams, generator=torch.Generator().manual_seed(1)) * 2 - 1)
    t = table.to(DEV).requires_grad_(True)
    enc = ops.hash_grid_encode(t, x.to(DEV), **grid)
    width = grid["n_levels"] * grid["n_features_per_level"]
    assert enc.shape == (n, width)
    cot = torch.randn(n, width, generator=torch.Generator().manual_seed(2))
    enc.backward(cot.to(DEV))
    t64 = table.double().requires_grad_(True)
    ref = S.encode(t64, x.numpy(), **grid)
    (ref * cot.double()).sum().backward()
    if n:
        assert (enc.detach().cpu().double() - ref.detach()).abs().max() <= 2e-6
    assert (t.grad.cpu().double() - t64.grad).abs().max() <= 1e-5 * max(1.0, float(t64.grad.abs().max()))


def test_hash_grid_encode_at_one_million_points():
    from b200gs import ops
    grid = GRIDS["default"]
    n = 1_000_000
    x = grid_points(n, grid, seed=5)
    table = torch.rand(S.n_params(**grid), generator=torch.Generator().manual_seed(3)) * 2 - 1
    t = table.to(DEV).requires_grad_(True)
    enc = ops.hash_grid_encode(t, x.to(DEV), **grid)
    cot = torch.randn(n, 32, generator=torch.Generator().manual_seed(4))
    enc.backward(cot.to(DEV))
    t64 = table.double().requires_grad_(True)
    ref = S.encode(t64, x.numpy(), **grid)
    (ref * cot.double()).sum().backward()
    assert (enc.detach().cpu().double() - ref.detach()).abs().max() <= 2e-6
    assert (t.grad.cpu().double() - t64.grad).abs().max() <= 2e-5 * float(t64.grad.abs().max())


# ---- the whole node ------------------------------------------------------------------------------------------------------------
def node_inputs(n, degree, grid, seed=0, stride=16, hidden=64, layers=3, emb=24):
    g = torch.Generator().manual_seed(seed)
    campos = torch.randn(3, generator=g)
    means = campos + torch.randn(n, 3, generator=g) * 2.0
    bbox_min, bbox_max = (means.min(0).values, means.max(0).values) if n > 1 else (campos - 2, campos + 2)
    bbox_size = (bbox_max - bbox_min) * 1.1
    bbox_min = bbox_min + 0.2 * bbox_size        # a smaller box: some Gaussians outside it
    dc = torch.randn(n, 1, 3, generator=g) * 0.8
    rest = torch.randn(n, stride - 1, 3, generator=g) * 0.3
    enc_dim = grid["n_levels"] * grid["n_features_per_level"]
    table = (torch.rand(S.n_params(**grid), generator=g) * 2 - 1) * 0.5
    in_dim = 3 + enc_dim + emb
    ws, bs, k = [], [], in_dim
    for l in range(layers):
        out = 4 if l == layers - 1 else hidden
        ws.append(torch.randn(out, k, generator=g) / math.sqrt(k))
        bs.append(torch.randn(out, generator=g) * 0.1)
        k = out
    embedding = torch.randn(emb, generator=g)
    base = torch.rand(n, generator=g)
    v_col, v_op = torch.randn(n, 3, generator=g), torch.randn(n, generator=g)
    return dict(means=means, campos=campos, bbox_min=bbox_min, bbox_size=bbox_size, dc=dc, rest=rest, table=table, ws=ws, bs=bs,
                embedding=embedding, base=base, v_col=v_col, v_op=v_op)


def run_node(d, degree, layout, grid, u, temperature=0.1):
    from b200gs import ops
    P = {k: (v.to(DEV).requires_grad_(True) if isinstance(v, torch.Tensor) else [t.to(DEV).requires_grad_(True) for t in v])
         for k, v in d.items() if k in ("means", "dc", "rest", "table", "ws", "bs", "embedding", "base")}
    colour = {"shs_dc": P["dc"], "shs_rest": P["rest"]} if layout == "split" else {"features": torch.cat([P["dc"], P["rest"]], 1)}
    bbox = torch.cat([d["bbox_min"], d["bbox_size"]]).to(DEV)
    c, o = ops.swag_colours_and_opacities(degree, P["means"], d["campos"].to(DEV), P["base"], torch.tensor([u], device=DEV), P["table"],
                                          P["embedding"], P["ws"], P["bs"], bbox=bbox, temperature=temperature, **grid, **colour)
    torch.autograd.backward([c, o], [d["v_col"].to(DEV), d["v_op"].to(DEV)])
    return c, o, P


def run_oracle(d, degree, grid, u, temperature=0.1):
    P = {k: (v.double().requires_grad_(True) if isinstance(v, torch.Tensor) else [t.double().requires_grad_(True) for t in v])
         for k, v in d.items() if k in ("means", "dc", "rest", "table", "ws", "bs", "embedding", "base")}
    feats = torch.cat([P["dc"], P["rest"]], 1)
    c, o = S.swag(degree, P["means"], d["campos"].double(), feats, P["table"], P["embedding"], P["ws"], P["bs"], P["base"], u,
                  d["bbox_min"].numpy(), d["bbox_size"].numpy(), temperature=temperature, **grid)
    torch.autograd.backward([c, o], [d["v_col"].double(), d["v_op"].double()])
    return c, o, P


def compare(got, ref, tol_out=2e-4, tol_grad=2e-3):
    c, o, P = got
    rc, ro, RP = ref
    assert (c.detach().cpu().double() - rc.detach()).abs().max() <= tol_out
    assert (o.detach().cpu().double() - ro.detach()).abs().max() <= tol_out
    for k in ("means", "dc", "rest", "table", "embedding", "base"):
        if RP[k].grad is None:      # degree 0: the colour does not depend on the direction
            assert float(P[k].grad.abs().max()) == 0.0, k
        else:
            assert rel(P[k].grad, RP[k].grad) <= tol_grad, k
    for k in ("ws", "bs"):
        for l, (a, b) in enumerate(zip(P[k], RP[k])):
            assert rel(a.grad, b.grad) <= tol_grad, (k, l)


@pytest.mark.parametrize("degree", [0, 1, 2, 3])
@pytest.mark.parametrize("layout", ["split", "features"])
def test_node_matches_the_oracle(degree, layout):
    grid = GRIDS["default"]
    d = node_inputs(1500, degree, grid, seed=degree)
    compare(run_node(d, degree, layout, grid, 0.5), run_oracle(d, degree, grid, 0.5))


@pytest.mark.parametrize("u", [0.5, 1e-3, 0.999])
@pytest.mark.parametrize("temperature", [0.1, 0.7])
def test_node_epilogue_u_and_temperature(u, temperature):
    grid = GRIDS["mixed_f2"]
    d = node_inputs(1200, 3, grid, seed=11)
    compare(run_node(d, 3, "split", grid, u, temperature), run_oracle(d, 3, grid, u, temperature))


@pytest.mark.parametrize("name", ["dense_f4", "hashed_f4", "hashed_f2_16"])
def test_node_at_other_grids(name):
    grid = GRIDS[name]
    d = node_inputs(800, 2, grid, seed=7)
    compare(run_node(d, 2, "features", grid, 0.3), run_oracle(d, 2, grid, 0.3))


def test_node_with_zero_gumbel_output_and_opacity_clamped_exactly_at_zero():
    """o3 = 0 (abs has gradient 0 there) and u = 0.5: sigmoid(10 log(1e-8)) is 0 in fp32, so with base opacity 0 the clamp argument
    is exactly 0 and, by clamp_min's rule, passes the gradient to the base opacity; nothing reaches o3's weights."""
    grid = GRIDS["dense_f2"]
    d = node_inputs(500, 1, grid, seed=3)
    d["ws"][-1][3].zero_()
    d["bs"][-1][3] = 0.0
    d["base"].zero_()
    c, o, P = run_node(d, 1, "split", grid, 0.5)
    assert torch.equal(o.detach().cpu(), torch.zeros(500))
    assert torch.equal(P["base"].grad.cpu(), d["v_op"])
    assert float(P["ws"][-1].grad[3].abs().max()) == 0.0 and float(P["bs"][-1].grad[3].abs().max()) == 0.0
    rc, ro, RP = run_oracle(d, 1, grid, 0.5)
    assert (c.detach().cpu().double() - rc.detach()).abs().max() <= 2e-4


def test_embedding_columns_of_the_first_weight_get_their_gradient():
    """W_0's columns 35..58 (the image embedding, folded into b_0) and 0..34 against the oracle; the row padding 35..39 never reads
    them"""
    grid = GRIDS["default"]
    d = node_inputs(700, 3, grid, seed=21)
    d["ws"][0][:, 35:40] = 50.0                   # would wreck the output if the kernels read them as row columns
    got, ref = run_node(d, 3, "split", grid, 0.5), run_oracle(d, 3, grid, 0.5)
    compare(got, ref)
    g, r = got[2]["ws"][0].grad.cpu().double(), ref[2]["ws"][0].grad
    assert rel(g[:, 35:], r[:, 35:]) <= 2e-3 and rel(g[:, :35], r[:, :35]) <= 2e-3


@pytest.mark.parametrize("n", [0, 1, 33, 1_000_000])
def test_node_sizes(n):
    grid = GRIDS["default"]
    d = node_inputs(n, 3, grid, seed=n % 97)
    got = run_node(d, 3, "split", grid, 0.4)
    assert got[0].shape == (n, 3) and got[1].shape == (n,)
    if n == 0:
        return
    if n > 100_000:     # the oracle on a sample of rows: the row outputs do not depend on each other
        idx = torch.randperm(n, generator=torch.Generator().manual_seed(0))[:4000]
        sub = dict(d)
        for k in ("means", "dc", "rest", "base", "v_col", "v_op"):
            sub[k] = d[k][idx]
        rc, ro, _ = run_oracle(sub, 3, grid, 0.4)
        assert (got[0].detach().cpu()[idx].double() - rc.detach()).abs().max() <= 2e-4
        assert (got[1].detach().cpu()[idx].double() - ro.detach()).abs().max() <= 2e-4
        assert all(bool(torch.isfinite(t.grad).all()) for t in (got[2]["means"], got[2]["table"], got[2]["rest"]))
    else:
        compare(got, run_oracle(d, 3, grid, 0.4))


def test_launch_counts_and_no_host_synchronisation():
    from b200gs import _lib, ops
    grid = GRIDS["default"]
    d = node_inputs(20_000, 3, grid, seed=4)
    L = _lib.lib()
    means = d["means"].to(DEV).requires_grad_(True)
    dc, rest = d["dc"].to(DEV).requires_grad_(True), d["rest"].to(DEV).requires_grad_(True)
    table = d["table"].to(DEV).requires_grad_(True)
    ws = [w.to(DEV).requires_grad_(True) for w in d["ws"]]
    bs = [b.to(DEV).requires_grad_(True) for b in d["bs"]]
    emb, base = d["embedding"].to(DEV).requires_grad_(True), d["base"].to(DEV).requires_grad_(True)
    bbox, campos, u = torch.cat([d["bbox_min"], d["bbox_size"]]).to(DEV), d["campos"].to(DEV), torch.tensor([0.3], device=DEV)
    vc, vo = d["v_col"].to(DEV), d["v_op"].to(DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        c0 = L.b200gs_launch_count()
        c, o = ops.swag_colours_and_opacities(3, means, campos, base, u, table, emb, ws, bs, bbox=bbox, shs_dc=dc, shs_rest=rest, **grid)
        c1 = L.b200gs_launch_count()
        torch.autograd.backward([c, o], [vc, vo])
        c2 = L.b200gs_launch_count()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert (c1 - c0, c2 - c1) == (ops.SWAG_FWD_LAUNCHES, ops.SWAG_BWD_LAUNCHES) == (2, 3)


# ---- the renderer against the reference's own steps ------------------------------------------------------------------------------
def _model(n, seed=0):
    from b200gs.scene import SyntheticGaussians, make_scene
    return SyntheticGaussians(make_scene(n, seed, mean_scale=0.05)).to(DEV)


def _renderer(xyz):
    from b200gs.swag import B200SWAGRenderer, EmbeddingConfig
    r = B200SWAGRenderer(embedding=EmbeddingConfig(num_embeddings=8))
    r.set_bbox(xyz.min(0).values, xyz.max(0).values)
    from b200gs.swag import B200SWAGModel
    r.swag_model = B200SWAGModel(r.network_config, r.grid_encoding_config, r.embedding_config).to(DEV)
    with torch.no_grad():
        r.swag_model.grid_encoding.params.uniform_(-0.3, 0.3, generator=torch.Generator(device=DEV).manual_seed(0))
    return r


def _reference_steps(r, cam, pc, bg, u):
    """SWAGRenderer.forward with SWAGModel.forward, as the reference writes them, on compat's tinycudann Encoding (the same table)
    and B200VanillaRenderer.render: eval_gaussian_model_sh, the bbox normalisation, grid, repeat, concat, theta, the Gumbel sigmoid."""
    from b200gs import compat
    from b200gs.renderers import B200VanillaRenderer
    from oracle.gs_oracle import sh_basis
    sys.modules.pop("tinycudann", None)
    compat.install(force=True)
    try:
        import tinycudann as tcnn
        enc = tcnn.Encoding(n_input_dims=3, encoding_config=r.grid_encoding_config.get_encoder_config(3))
        enc = enc.to(DEV)
        with torch.no_grad():
            enc.params.copy_(r.swag_model.grid_encoding.params)
    finally:
        sys.modules.pop("tinycudann", None)
    xyz = pc.get_xyz
    shs_view = pc.get_features.transpose(1, 2).view(-1, 3, (pc.max_sh_degree + 1) ** 2)
    dir_pp = xyz - cam.camera_center.repeat(pc.get_features.shape[0], 1)
    dirs = dir_pp / dir_pp.norm(dim=1, keepdim=True)
    ncoef = (pc.active_sh_degree + 1) ** 2
    rgb = (sh_basis(pc.active_sh_degree, dirs).unsqueeze(1) * shs_view[:, :, :ncoef]).sum(-1)
    colors = torch.clamp_min(rgb + 0.5, 0.0)
    x = (xyz.detach() - r.bbox_min.to(DEV)) / r.bbox_size.to(DEV)
    x_emb = enc(x).to(colors.dtype)
    m = r.swag_model
    image_emb = m.image_embedding(torch.tensor([int(cam.appearance_id)], dtype=torch.int, device=DEV)).repeat((colors.shape[0], 1))
    out = m.theta(torch.concat([colors, x_emb, image_emb], dim=-1))
    c, d = torch.sigmoid(out[:, :3]), out[:, -1]
    var = torch.sigmoid(1 / r.temperature * (torch.log(torch.abs(d) + r.eps) + torch.log(u + r.eps) - torch.log(1 - u + r.eps)))
    opacity = torch.clamp_min(pc.get_opacity.squeeze(-1) - var, 0).unsqueeze(-1)
    return B200VanillaRenderer.render(means3D=xyz, opacity=opacity, scales=pc.get_scaling, rotations=pc.get_rotation, features=None,
                                      active_sh_degree=pc.active_sh_degree, viewpoint_camera=cam, bg_color=bg, colors_precomp=c), enc


@pytest.mark.parametrize("u", [None, 0.8])
def test_renderer_matches_the_reference_steps(u):
    from b200gs.scene import make_ring_cameras
    W, H = 128, 96
    cam = make_ring_cameras(W, H)[3].to_device(DEV)
    cam.appearance_id = torch.tensor(5, device=DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    cot = (torch.rand(3, H, W, generator=torch.Generator().manual_seed(1)) * 2 - 1).to(DEV)
    outs, grads = [], []
    pc0 = _model(3000, seed=2)
    r = _renderer(pc0.get_xyz.detach().cpu())
    ut = None if u is None else torch.tensor([u], device=DEV)
    for path in ("b200gs", "reference"):
        pc = _model(3000, seed=2)
        for p in r.swag_model.parameters():
            p.grad = None
        if path == "b200gs":
            out = r(cam, pc, bg, u=ut)
            tab = r.swag_model.grid_encoding.params
        else:
            out, enc = _reference_steps(r, cam, pc, bg, torch.tensor(0.5, device=DEV) if ut is None else ut)
            tab = enc.params
        (out["render"] * cot).sum().backward()
        outs.append(out["render"].detach())
        g = {k: v.grad.clone() for k, v in pc.gaussians.items()}
        g["table"] = tab.grad.clone()
        for name, p in r.swag_model.named_parameters():
            if "grid_encoding" not in name:
                g[name] = p.grad.clone()
        grads.append(g)
    assert (outs[0] - outs[1]).abs().max() <= 2e-4
    for k in grads[1]:
        assert rel(grads[0][k], grads[1][k]) <= 5e-3, k


def test_renderer_trains_a_step_with_the_swag_baseline_arguments():
    """configs/swag_baseline.yaml's init_args (embedding.num_embeddings 1536) through setup, training_setup and training_forward"""
    import types
    from b200gs.scene import make_ring_cameras
    from b200gs.swag import B200SWAGRenderer, EmbeddingConfig
    pc = _model(2000, seed=4)
    xyz = pc.get_xyz.detach().cpu().numpy()
    module = types.SimpleNamespace(trainer=types.SimpleNamespace(datamodule=types.SimpleNamespace(
        dataparser_outputs=types.SimpleNamespace(point_cloud=types.SimpleNamespace(xyz=xyz)))))
    r = B200SWAGRenderer(embedding=EmbeddingConfig(num_embeddings=1536))
    r.setup("fit", module)
    r = r.to(DEV)
    assert r.swag_model.grid_encoding.params.numel() == 11_681_792
    opt, sched = r.training_setup(module)
    cam = make_ring_cameras(96, 64)[0].to_device(DEV)
    cam.appearance_id = torch.tensor(1500, device=DEV)
    before = [p.detach().clone() for p in r.swag_model.parameters()]
    out = r.training_forward(0, module, cam, pc, torch.zeros(3, device=DEV))
    out["render"].mean().backward()
    opt.step()
    sched.step()
    assert all(bool(torch.isfinite(p.grad).all()) for p in r.swag_model.parameters() if p.grad is not None)
    assert any(not torch.equal(a, b) for a, b in zip(before, r.swag_model.parameters()))
    assert bool(torch.isfinite(pc.gaussians["means"].grad).all())


# ---- replay of the recorded reference (tests/golden/swag.npz, make_golden_swag.py) ---------------------------------------------
def _golden():
    import json
    return np.load(os.path.join(GOLDEN, "swag.npz")), json.load(open(os.path.join(GOLDEN, "swag.json")))


@pytest.mark.parametrize("case", ["d3_eval", "d3_u02", "d1_u09", "d0_eval"])
def test_golden_recording_replayed_through_the_plug_in(case):
    from b200gs import ops
    Z, meta = _golden()
    c = next(x for x in meta["cases"] if x["name"] == case)
    t = lambda k: torch.from_numpy(Z[k]).to(DEV).requires_grad_(True)      # noqa: E731
    means, features, logits, emb = t("means"), t("features"), t("logits"), t("embedding")
    ws = [t(f"theta.{i}.weight") for i in (0, 2, 4)]
    bs = [t(f"theta.{i}.bias") for i in (0, 2, 4)]
    i = torch.arange(S.n_params(), dtype=torch.float64)
    table = (0.6 * torch.sin(i * 0.7071) + 0.2 * torch.cos(i * 0.0173)).float().to(DEV).requires_grad_(True)
    bbox = torch.tensor(meta["bbox_min"] + meta["bbox_size"], dtype=torch.float32, device=DEV)
    u = torch.tensor([0.5 if c["u"] is None else c["u"]], device=DEV)
    col, op = ops.swag_colours_and_opacities(c["degree"], means, torch.from_numpy(Z["campos"]).to(DEV), torch.sigmoid(logits)[:, 0], u,
                                             table, emb[4], ws, bs, bbox=bbox, features=features)
    ((col * torch.from_numpy(Z["cot_c"]).to(DEV)).sum() + (op * torch.from_numpy(Z["cot_o"]).to(DEV)).sum()).backward()
    p = case + "."
    assert np.abs(col.detach().cpu().numpy() - Z[p + "colours"]).max() <= 2e-4
    assert np.abs(op.detach().cpu().numpy() - Z[p + "opacities"]).max() <= 2e-4

    def close(got, key, tol=3e-3):
        ref = Z[p + key]
        assert np.abs(got.detach().cpu().numpy() - ref).max() <= tol * max(1e-3, np.abs(ref).max()), key
    if c["degree"] > 0:
        close(means.grad, "v_means")
    close(features.grad, "v_features")
    close(logits.grad, "v_logits")
    close(emb.grad, "v_embedding")
    for k, (w, b) in zip((0, 2, 4), zip(ws, bs)):
        close(w.grad, f"v_theta.{k}.weight")
        close(b.grad, f"v_theta.{k}.bias")
    g = torch.zeros(table.numel(), dtype=torch.float32)
    g[torch.from_numpy(Z[p + "v_table_idx"])] = torch.from_numpy(Z[p + "v_table_val"])
    assert float((table.grad.cpu() - g).abs().max()) <= 3e-3 * float(g.abs().max())
