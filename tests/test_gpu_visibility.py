"""Transient visibility map kernels (csrc/visibility.cu; the visibility MLP on csrc/appearance.cu) on the GPU against the float64
oracle (oracle/visibility_oracle.py): the DenseGrid encoding K32 and its gradient K33, including the pixels whose corners wrap;
the one-output MLP; the masked L1 + SSIM K34/K35 with and without a dataset mask and with and without the visibility gradient; at
1920x1080, 800x600, 37x50, 2x64 and 64x2.  Also: the grid -> MLP -> loss chain against the float64 chain, the plug-in renderer and
metric end to end, the tinycudann stand-in, out-of-range ids, bit-identical backwards, launch counts and no host synchronisation."""
import types

import numpy as np
import pytest
import torch

from oracle import visibility_oracle as V
from oracle.appearance_oracle import mlp as oracle_mlp

pytestmark = pytest.mark.gpu
DEV = "cuda"
SIZES = [(1920, 1080), (800, 600), (37, 50), (2, 64), (64, 2)]      # (W, H)
N_IMAGES = 3


def rel(a, ref):
    a, ref = np.asarray(a, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    return np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-30)


def grids(seed, n=N_IMAGES):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(V.n_params(), generator=g) * 2 - 1 for _ in range(n)]


@pytest.mark.parametrize("W,H", SIZES)
def test_uv_grid_matches_the_oracle(W, H):
    from b200gs import ops
    host = grids(W + H)
    dev = [p.to(DEV).requires_grad_(True) for p in host]
    app_id = torch.tensor([1], dtype=torch.int64, device=DEV)
    enc = ops.uv_grid_encode(dev, app_id, width=W, height=H, selected=1)
    v_enc = torch.rand(H * W, 16, generator=torch.Generator().manual_seed(5)) * 2 - 1
    enc.backward(v_enc.to(DEV))
    u, v = V.pixel_uv(W, H)
    p64 = host[1].double().requires_grad_(True)
    ref = V.encode(p64, u, v)
    (ref * v_enc.double()).sum().backward()
    assert np.abs(enc.detach().cpu().double().numpy() - ref.detach().numpy()).max() <= 1e-6
    assert rel(dev[1].grad.cpu(), p64.grad) <= 1e-4
    assert dev[0].grad is None and dev[2].grad is None      # only the selected image's grid gets a gradient
    # the last column and row reach corner res_l on levels 0, 2, 5 and 7 and wrap through the %; they are held to the same bar
    last = enc.detach().cpu().double().numpy().reshape(H, W, 16)
    ref_last = ref.detach().numpy().reshape(H, W, 16)
    assert np.abs(last[:, -1] - ref_last[:, -1]).max() <= 1e-6 and np.abs(last[-1] - ref_last[-1]).max() <= 1e-6


def test_uv_grid_with_the_id_on_the_host():
    from b200gs import ops
    host = grids(3)
    enc = ops.uv_grid_encode([p.to(DEV) for p in host], 2, width=37, height=50)
    u, v = V.pixel_uv(37, 50)
    assert np.abs(enc.cpu().double().numpy() - V.encode(host[2].double(), u, v).numpy()).max() <= 1e-6


@pytest.mark.parametrize("app_id", [N_IMAGES, -1, 1 << 40])
def test_out_of_range_id_gives_nan(app_id):
    from b200gs import ops
    enc = ops.uv_grid_encode([p.to(DEV) for p in grids(4)], torch.tensor(app_id, device=DEV), width=37, height=50)
    assert torch.isnan(enc).all()


def mlp_case(n, n_neurons=64, n_layers=3, seed=0):
    torch.manual_seed(seed)
    dims = [16 + 128] + [n_neurons] * (n_layers - 1) + [1]
    lin = [torch.nn.Linear(a, b) for a, b in zip(dims[:-1], dims[1:])]
    weights = [l.weight.detach() * 2 for l in lin]
    biases = [l.bias.detach() * 2 for l in lin]
    g = torch.Generator().manual_seed(seed + 1)
    return torch.randn(n, 16, generator=g) * 0.5, torch.randn(128, generator=g), weights, biases, torch.randn(n, generator=g)


def kink_rows(enc, emb, weights, biases, eps=1e-5):
    """Rows with a hidden pre-activation within eps of 0 in float64: there fp32 may take the other side of the ReLU, which moves that
    row's input gradient by a whole term.  Their cotangent is zeroed in both arms."""
    h = torch.cat([enc.double(), emb.double().reshape(1, -1).expand(enc.shape[0], -1)], 1)
    near = torch.zeros(enc.shape[0], dtype=torch.bool)
    for w, b in zip(weights[:-1], biases[:-1]):
        pre = h @ w.double().T + b.double()
        near |= (pre.abs() < eps).any(1)
        h = pre.relu()
    return near


@pytest.mark.parametrize("n,n_neurons,n_layers", [(1920 * 1080, 64, 3), (800 * 600, 64, 3), (37 * 50, 128, 2), (128, 64, 4), (1, 64, 3)])
def test_visibility_mlp_matches_the_oracle(n, n_neurons, n_layers):
    from b200gs import ops
    enc, emb, weights, biases, cot = mlp_case(n, n_neurons, n_layers)
    near = kink_rows(enc, emb, weights, biases)
    assert int(near.sum()) <= max(1, n // 200)
    cot[near] = 0
    d = [t.to(DEV).requires_grad_(True) for t in [enc, emb] + weights + biases]
    L = len(weights)
    out = ops.visibility_mlp(d[0], d[1], d[2:2 + L], d[2 + L:])
    out.backward(cot.to(DEV))
    r = [t.double().requires_grad_(True) for t in [enc, emb] + weights + biases]
    ref = oracle_mlp(r[0], r[1], r[2:2 + L], r[2 + L:])[:, 0]
    (ref * cot.double()).sum().backward()
    assert np.abs(out.detach().cpu().double().numpy() - ref.detach().numpy()).max() <= 2e-5
    for a, b in zip(d, r):
        assert rel(a.grad.cpu(), b.grad) <= 1e-4


def loss_case(W, H, masked, seed=0):
    g = torch.Generator().manual_seed(seed)
    image, gt = torch.rand(3, H, W, generator=g), torch.rand(3, H, W, generator=g)
    vis = torch.rand(1, H, W, generator=g)
    mask = (torch.rand(H, W, generator=g) < 0.8) if masked else None
    return image, gt, vis, mask


@pytest.mark.parametrize("W,H", SIZES)
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("vis_grad", [True, False])
def test_masked_loss_matches_the_oracle(W, H, masked, vis_grad):
    from b200gs import ops
    image, gt, vis, mask = loss_case(W, H, masked)
    i = image.to(DEV).requires_grad_(True)
    v = vis.to(DEV).requires_grad_(vis_grad)
    loss, stats = ops.visibility_l1_ssim_loss(i, gt.to(DEV), v, None if mask is None else mask.to(DEV), 0.2, 0.2)
    loss.backward()
    ri, rv = image.double().requires_grad_(True), vis.double().requires_grad_(True)
    ref, l1, s, reg = V.masked_loss(ri, gt.double(), rv, mask, 0.2, 0.2)
    ref.backward()
    assert abs(float(loss) - float(ref)) < 2e-6
    assert abs(float(stats[0]) - float(l1)) < 1e-6 and abs(float(stats[1]) - float(s)) < 5e-6 and abs(float(stats[2]) - float(reg)) < 1e-6
    assert rel(i.grad.cpu(), ri.grad) < 1e-3
    if vis_grad:
        assert rel(v.grad.cpu(), rv.grad) < 1e-3
    else:
        assert v.grad is None


def chain(W, H, app_id, masked, dev, dtype, state):
    """grid -> visibility MLP -> masked loss; returns the loss and the leaves"""
    from b200gs import ops
    host_grids, emb, weights, biases, image, gt, mask = state
    leaves = [t.to(dev, dtype).requires_grad_(True) for t in host_grids + [emb] + weights + biases + [image]]
    G, E = leaves[:N_IMAGES], leaves[N_IMAGES]
    L = len(weights)
    Ws, Bs, img = leaves[N_IMAGES + 1:N_IMAGES + 1 + L], leaves[N_IMAGES + 1 + L:-1], leaves[-1]
    m = None if mask is None else mask.to(dev)
    if dev == DEV:
        enc = ops.uv_grid_encode(G, torch.tensor([app_id], device=DEV), width=W, height=H, selected=app_id)
        vis = ops.visibility_mlp(enc, E, Ws, Bs).reshape(1, H, W)
        loss, _ = ops.visibility_l1_ssim_loss(img, gt.to(dev), vis, m)
    else:
        vis = V.visibility(G[app_id], E, Ws, Bs, W, H).reshape(1, H, W)
        loss = V.masked_loss(img, gt.to(dtype), vis, m)[0]
    loss.backward()
    return loss, leaves


def chain_state(W, H, masked, seed=3):
    enc, emb, weights, biases, _ = mlp_case(1, seed=seed)
    host = [p * 0.5 for p in grids(seed)]
    image, gt, _, mask = loss_case(W, H, masked, seed)
    return host, emb, weights, biases, image, gt, mask


# small images: every pixel's gradient reaches the grid, so one fp32 ReLU kink (see kink_rows) would move it
@pytest.mark.parametrize("W,H,masked", [(160, 120, True), (37, 50, False)])
def test_grid_mlp_loss_chain_matches_the_float64_chain(W, H, masked):
    state = chain_state(W, H, masked)
    loss, fused = chain(W, H, 2, masked, DEV, torch.float32, state)
    ref_loss, ref = chain(W, H, 2, masked, "cpu", torch.float64, state)
    assert abs(float(loss) - float(ref_loss)) < 1e-5
    for k, (a, b) in enumerate(zip(fused, ref)):
        if b.grad is None:
            assert a.grad is None, k
        else:
            assert rel(a.grad.cpu(), b.grad) < 1e-3, k


def test_two_backwards_give_bit_identical_gradients():
    state = chain_state(1920, 1080, True)
    first = chain(1920, 1080, 1, True, DEV, torch.float32, state)[1]
    second = chain(1920, 1080, 1, True, DEV, torch.float32, state)[1]
    for a, b in zip(first, second):
        assert (a.grad is None and b.grad is None) or torch.equal(a.grad, b.grad)


def test_no_host_synchronisation_and_launch_counts():
    from b200gs import _lib, ops
    Lb = _lib.lib()
    W, H = 128, 96
    state = chain_state(W, H, True)
    chain(W, H, 0, True, DEV, torch.float32, state)         # builds the grid-pointer table once
    host_grids, emb, weights, biases, image, gt, mask = state
    G = [p.to(DEV).requires_grad_(True) for p in host_grids]
    E = emb.to(DEV).requires_grad_(True)
    Ws = [w.to(DEV).requires_grad_(True) for w in weights]
    Bs = [b.to(DEV).requires_grad_(True) for b in biases]
    img, gt_d, m = image.to(DEV).requires_grad_(True), gt.to(DEV), mask.to(DEV)
    app_id = torch.tensor([0], device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        n0 = Lb.b200gs_launch_count()
        enc = ops.uv_grid_encode(G, app_id, width=W, height=H, selected=0)
        vis = ops.visibility_mlp(enc, E, Ws, Bs).reshape(1, H, W)
        loss, _ = ops.visibility_l1_ssim_loss(img, gt_d, vis, m)
        n1 = Lb.b200gs_launch_count()
        loss.backward()
        n2 = Lb.b200gs_launch_count()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert n1 - n0 == ops.UV_GRID_FWD_LAUNCHES + ops.VISIBILITY_MLP_FWD_LAUNCHES + ops.VISIBILITY_LOSS_FWD_LAUNCHES == 3
    assert n2 - n1 == ops.UV_GRID_BWD_LAUNCHES + ops.VISIBILITY_MLP_BWD_LAUNCHES + ops.VISIBILITY_LOSS_BWD_LAUNCHES == 4
    assert torch.isfinite(G[0].grad).all() and torch.isfinite(img.grad).all()


def test_tinycudann_stand_in_encodes_given_coordinates():
    import sys
    from b200gs import compat
    compat.install()
    import tinycudann as tcnn
    try:
        enc = tcnn.Encoding(n_input_dims=2, encoding_config={"otype": "DenseGrid", "n_levels": 8, "base_resolution": 16,
                                                             "per_level_scale": 1.405}, seed=0, dtype=torch.float).to(DEV)
        assert enc.n_output_dims == 16 and enc.params.numel() == 121760
        u, v = V.pixel_uv(64, 48)
        uv = torch.from_numpy(np.stack([u, v], 1))
        out = enc(uv.to(DEV))
        cot = torch.rand(out.shape, generator=torch.Generator().manual_seed(2))
        out.backward(cot.to(DEV))
        p64 = enc.params.detach().cpu().double().requires_grad_(True)
        ref = V.encode(p64, u, v)
        (ref * cot.double()).sum().backward()
        assert np.abs(out.detach().cpu().double().numpy() - ref.detach().numpy()).max() <= 1e-6
        assert rel(enc.params.grad.cpu(), p64.grad) <= 1e-4
        with pytest.raises(NotImplementedError):
            tcnn.Encoding(n_input_dims=2, encoding_config={"otype": "HashGrid"})
        with pytest.raises(NotImplementedError):
            tcnn.Network(n_input_dims=2, n_output_dims=1, network_config={})
    finally:
        sys.modules.pop("tinycudann", None)


class _Model:
    """The attributes of AppearanceFeatureGaussian the renderer reads"""

    def __init__(self, raw, feats):
        from b200gs.scene import activate
        self.act = {k: v.to(DEV).requires_grad_(True) for k, v in activate(raw).items()}
        self.feats = feats.to(DEV).requires_grad_(True)
        self.active_sh_degree = 0
        self.get_xyz, self.get_scaling, self.get_rotation = self.act["means"], self.act["scales"], self.act["rotations"]
        self.get_opacity, self.get_features = self.act["opacities"], self.act["shs"]

    def get_appearance_features(self):
        return self.feats


def test_renderer_and_metric_end_to_end():
    from b200gs.metrics import B200VisibilityMapMetrics
    from b200gs.scene import make_ring_cameras, make_scene
    from b200gs.visibility import B200GSplatAppearanceEmbeddingVisibilityMapRenderer, ModelConfig, OptimizationConfig
    W, H = 128, 96
    raw = make_scene(2048, 7, mean_scale=0.05)
    pc = _Model(raw, torch.randn(2048, 64, generator=torch.Generator().manual_seed(1)) * 0.1)
    cam = make_ring_cameras(W, H)[1].to_device(DEV)
    cam.appearance_id = torch.tensor([2], dtype=torch.int32, device=DEV)
    r = B200GSplatAppearanceEmbeddingVisibilityMapRenderer(ModelConfig(n_images=N_IMAGES), OptimizationConfig())
    r.setup("fit")
    r.to(DEV)
    opts, scheds = r.training_setup(None)
    assert [o.param_groups[0]["name"] for o in opts] == ["appearance_embedding", "appearance_network", "transient_embedding",
                                                          "uv_encoding", "visibility_network"]
    module = types.SimpleNamespace(device=torch.device(DEV))
    out = r.training_forward(5000, module, cam, pc, torch.tensor([0.1, 0.2, 0.3], device=DEV))
    assert out["render"].shape == (3, H, W) and out["visibility"].shape == (1, H, W) and out["extra_image"] is out["visibility"]
    metric = B200VisibilityMapMetrics().instantiate()
    metric.setup("fit", None)
    gt = torch.rand(3, H, W, generator=torch.Generator().manual_seed(9)).to(DEV)
    metrics, pbar = metric.get_train_metrics(None, pc, 5000, (cam, ("x", gt, None), None), out)
    assert set(metrics) == set(pbar) == {"loss", "rgb_diff", "ssim", "vis_reg"}
    metrics["loss"].backward()
    m = r.model
    assert m.uv_encodings[2].params.grad is not None and m.uv_encodings[0].params.grad is None and m.uv_encodings[1].params.grad is None
    assert m.transient_embedding.weight.grad[2].abs().sum() > 0 and m.appearance_embedding.weight.grad[2].abs().sum() > 0
    assert all(p.grad is not None for p in m.visibility_network.parameters()) and pc.feats.grad.abs().sum() > 0
    # the map is the chain of the ops on the same parameters
    lin = [x for x in m.visibility_network.output_layers if isinstance(x, torch.nn.Linear)]
    ref = V.visibility(m.uv_encodings[2].params.detach().cpu().double(), m.transient_embedding.weight[2].detach().cpu().double(),
                       [x.weight.detach().cpu().double() for x in lin], [x.bias.detach().cpu().double() for x in lin], W, H)
    assert np.abs(out["visibility"][0].detach().cpu().double().numpy() - ref.numpy()).max() <= 2e-5
    # warm-ups: ones maps
    assert torch.equal(r.training_forward(10, module, cam, pc, torch.zeros(3, device=DEV))["visibility"], torch.ones(1, H, W, device=DEV))
    assert torch.equal(r.training_forward(1500, module, cam, pc, torch.zeros(3, device=DEV))["visibility"], torch.ones(1, H, W, device=DEV))


# ---- recordings of the reference's own renderer and metric (tests/golden/visibility.npz, make_golden_visibility.py) ------------
def _golden():
    import json
    import os
    from conftest import GOLDEN
    return np.load(os.path.join(GOLDEN, "visibility.npz")), json.load(open(os.path.join(GOLDEN, "visibility.json")))


@pytest.mark.parametrize("k", range(4))
def test_reference_cases_replayed_through_the_plug_in(k):
    from b200gs.metrics import B200VisibilityMapMetrics
    from b200gs.visibility import B200GSplatAppearanceEmbeddingVisibilityMapRenderer, ModelConfig, OptimizationConfig
    Z, META = _golden()
    case = META["cases"][k]
    W, H, aid, name = case["W"], case["H"], case["aid"], case["name"]
    r = B200GSplatAppearanceEmbeddingVisibilityMapRenderer(ModelConfig(n_images=N_IMAGES), OptimizationConfig())
    r.load_state_dict({key: V.golden_param(key[len("model."):], s).to(DEV) for key, s in META["state_dict"].items()})
    m = r.model
    render, gt, mask = V.golden_inputs(W, H, len(name) + W)
    render = render.to(DEV).requires_grad_(True)
    vis = m.visibility_forward(W, H, torch.tensor([aid], device=DEV), aid).unsqueeze(0)
    if not case["vis_grad"]:
        vis = vis.detach()
    metric = B200VisibilityMapMetrics().instantiate()
    metric.setup("fit", None)
    metrics, pbar = metric.get_train_metrics(None, None, 5000, (None, ("img", gt.to(DEV), mask.to(DEV) if case["masked"] else None), None),
                                             {"render": render, "visibility": vis})
    metrics["loss"].backward()
    p = name + "."
    assert pbar == case["pbar"]
    assert np.abs(vis.detach()[0].cpu().double().numpy() - Z[p + "visibility"]).max() <= 2e-5
    for key in ("loss", "rgb_diff", "ssim", "vis_reg"):
        assert abs(float(metrics[key]) - float(Z[p + key])) <= 5e-6, key
    assert rel(render.grad.cpu(), Z[p + "v_render"]) <= 1e-3
    if case["vis_grad"]:
        assert rel(m.transient_embedding.weight.grad[aid].cpu(), Z[p + "v_transient"]) <= 1e-3
        for key, t in m.visibility_network.named_parameters():
            assert rel(t.grad.cpu(), Z[f"{p}v_vnet.{key}"]) <= 1e-3, key
        g = m.uv_encodings[aid].params.grad.cpu().double()
        assert abs(float(g @ V.golden_probe(g.numel())) - case["grid_grad_probe"]) <= 1e-3 * abs(case["grid_grad_probe"])
        assert [i for i in range(N_IMAGES) if m.uv_encodings[i].params.grad is not None] == case["grids_with_grad"]


def test_reference_renderer_replayed_through_compat():
    """The reference's visibility_forward made these tinycudann calls; repeated through compat's Encoding, followed by the
    reference's own torch steps (repeat, concat, network), they give the recorded map and, from the recorded visibility gradient,
    the recorded gradients of the transient embedding, the network and the grid."""
    import sys
    from b200gs import compat
    Z, META = _golden()
    sys.modules.pop("tinycudann", None)
    compat.install()
    import tinycudann as tcnn
    try:
        encs = torch.nn.ModuleList([tcnn.Encoding(n_input_dims=e["n_input_dims"], encoding_config=e["encoding_config"], seed=e["seed"],
                                                  dtype=torch.float32) for e in META["encodings"]]).to(DEV)
        for i, e in enumerate(encs):
            e.params.data.copy_(V.golden_param(f"uv_encodings.{i}.params", e.params.shape))
        state = {key[len("model."):]: V.golden_param(key[len("model."):], s).to(DEV).requires_grad_(True)
                 for key, s in META["state_dict"].items() if "uv_encodings" not in key}
        calls = [c for c in META["calls"] if c["call"] == "Encoding.forward"]
        for case, call in zip(META["cases"], calls):
            if not case["vis_grad"]:
                continue
            W, H, aid, p = case["W"], case["H"], case["aid"], case["name"] + "."
            u, v = V.pixel_uv(W, H)
            x = torch.from_numpy(np.stack([u, v], 1))
            assert call["sum"] == float(x.double().sum()) and call["shape"] == list(x.shape)
            for t in list(state.values()) + list(encs.parameters()):
                t.grad = None
            enc = encs[aid](x.to(DEV))
            transient = state["transient_embedding.weight"][aid].reshape(1, -1).repeat(W * H, 1)
            h = torch.concat([enc, transient], dim=-1)
            for i in (0, 2, 4):
                h = h @ state[f"visibility_network.output_layers.{i}.weight"].T + state[f"visibility_network.output_layers.{i}.bias"]
                h = torch.relu(h) if i < 4 else torch.sigmoid(h)
            vis = h.reshape(H, W)
            assert np.abs(vis.detach().cpu().double().numpy() - Z[p + "visibility"]).max() <= 2e-5
            vis.backward(torch.from_numpy(Z[p + "v_visibility"]).to(DEV))
            assert rel(state["transient_embedding.weight"].grad[aid].cpu(), Z[p + "v_transient"]) <= 1e-3
            for i in (0, 2, 4):
                for t in ("weight", "bias"):
                    key = f"visibility_network.output_layers.{i}.{t}"
                    assert rel(state[key].grad.cpu(), Z[f"{p}v_vnet.output_layers.{i}.{t}"]) <= 1e-3, key
            g = encs[aid].params.grad.cpu().double()
            assert abs(float(g @ V.golden_probe(g.numel())) - case["grid_grad_probe"]) <= 1e-3 * abs(case["grid_grad_probe"])
            assert int((g != 0).sum()) == case["grid_grad_nonzero"]
    finally:
        sys.modules.pop("tinycudann", None)
