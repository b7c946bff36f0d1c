"""K51 / K52 (csrc/gs4d.cu) through ops.gs4d_repack_planes / ops.gs4d_deform and b200gs.gs4d.B200VanillaGS4DRenderer on the GPU,
against the float64 oracle (oracle/gs4d_oracle.py) and the reference's own VanillaGS4DRenderer recorded on the CPU
(tests/golden/make_golden_gs4d.py)."""
import itertools
import math
import os

import numpy as np
import pytest
import torch

from oracle import gs4d_oracle as O
from oracle import gs_oracle as G
from test_gs4d_cpu import MG, META, ZS, load_case, network

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HEADS = ("dx", "ds", "dr", "dshs")
AABB = torch.tensor([[1.4, 0.9, 1.1], [-1.2, -1.0, -0.8]])          # xyz_max, xyz_min


def max_abs(got, want):
    return float((got.detach().cpu().double() - want.detach().cpu().double()).abs().max()) if want.numel() else 0.0


def make_net(C, L, W, D, seed, res_scale=1):
    """random planes of per-axis sizes that differ (an axis swap shows), trunk and all four heads"""
    g = torch.Generator().manual_seed(seed)
    base = (7, 6, 5, 4)
    res = [tuple(r * (l + 1) * res_scale if d < 3 else r + l for d, r in enumerate(base)) for l in range(L)]
    grids = [[torch.rand(1, C, r[b], r[a], generator=g) + 0.5 for a, b in O.PLANES] for r in res]
    lin = lambda o, i: (torch.randn(o, i, generator=g) / math.sqrt(i), torch.randn(o, generator=g) * 0.1)  # noqa: E731
    trunk = [lin(W, C * L)] + ([lin(W, W)] if D == 2 else [])
    heads = {h: (lin(W, W), lin(o, W)) for h, o in zip(HEADS, (3, 3, 4, 48))}
    return grids, res, trunk, heads


def points(n, seed):
    """p uniform in [-1.3, 1.3] per axis, with p at, just inside and beyond +-1 on every axis first; as means in the aabb's frame"""
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(n, 3, generator=g) * 2.6 - 1.3
    special = torch.tensor(list(itertools.product((-1.5, -1.0, -0.999, 0.0, 0.999, 1.0, 1.5), repeat=3)), dtype=torch.float32)
    k = min(n, special.shape[0])
    p[:k] = special[:k]
    hi, lo = AABB[0], AABB[1]
    return hi + (p + 1) / 2 * (lo - hi)


def gaussians(n, seed):
    g = torch.Generator().manual_seed(seed + 100)
    return dict(means=points(n, seed), scales=torch.randn(n, 3, generator=g) * 0.5 - 3, quats=torch.randn(n, 4, generator=g),
                dc=torch.randn(n, 1, 3, generator=g) * 0.4, rest=torch.randn(n, 15, 3, generator=g) * 0.2)


def dev_net(grids, trunk, heads):
    from b200gs import ops
    planes = ops.gs4d_repack_planes([[p.to(DEV) for p in level] for level in grids])
    d = lambda wb: tuple(t.to(DEV) for t in wb)  # noqa: E731
    return planes, [d(wb) for wb in trunk], {h: (d(a), d(b)) for h, (a, b) in heads.items()}


def run(gs, t, planes, trunk, heads, apply_rotation=False):
    from b200gs import ops
    with torch.no_grad():
        return ops.gs4d_deform(gs["means"].to(DEV), gs["scales"].to(DEV), gs["quats"].to(DEV), t, planes, AABB.to(DEV), trunk, heads,
                               shs_dc=gs["dc"].to(DEV), shs_rest=gs["rest"].to(DEV), apply_rotation=apply_rotation)


def oracle_parts(gs, t, grids, trunk, heads, rows=None):
    sel = (lambda x: x) if rows is None else (lambda x: x[rows])
    h = O.trunk_forward(O.features(sel(gs["means"]), t, AABB, grids), trunk)
    return h, {name: O.head_forward(h, hd) for name, hd in heads.items()}


def check_outputs(out, gs, deltas, flags, apply_rotation, rows=None, bar=2e-5):
    sel = (lambda x: x) if rows is None else (lambda x: x[rows])
    m, s, q, dc, rest = (sel(o.cpu()) for o in out)
    want_m = sel(gs["means"]).double() + (deltas["dx"] if "dx" in flags else 0)
    want_s = sel(gs["scales"]).double() + (deltas["ds"] if "ds" in flags else 0)
    q0 = sel(gs["quats"]).double()
    want_q = (O.quaternion_multiply_normalized(q0, deltas["dr"]) if apply_rotation else q0 + deltas["dr"]) if "dr" in flags else q0
    assert max_abs(m, want_m) <= bar and max_abs(s, want_s) <= bar and max_abs(q, want_q) <= bar
    if "dx" not in flags:
        assert torch.equal(m, sel(gs["means"]))
    if "dr" not in flags:
        assert torch.equal(q, sel(gs["quats"]))
    shs0 = torch.cat([sel(gs["dc"]), sel(gs["rest"])], 1).double()
    if "dshs" in flags:
        want = shs0 + deltas["dshs"].reshape(-1, 16, 3)
        assert max_abs(torch.cat([dc, rest], 1), want) <= bar
    else:
        assert torch.equal(torch.cat([dc, rest], 1).double(), shs0)


SHAPES = [(W, D, C, L) for W in (64, 128) for D in (0, 1, 2) for C in (16, 32) for L in (1, 2, 3, 4)]


@pytest.mark.parametrize("W,D,C,L", SHAPES, ids=[f"w{w}_d{d}_c{c}_l{l}" for w, d, c, l in SHAPES])
def test_kernel_at_every_accepted_shape_and_head_combination(W, D, C, L):
    n, t = 333, 0.4
    grids, res, trunk, heads = make_net(C, L, W, D, seed=W + 10 * D + 100 * C + L)
    gs = gaussians(n, seed=L)
    planes, dtrunk, dheads = dev_net(grids, trunk, heads)
    _, deltas = oracle_parts(gs, t, grids, trunk, heads)
    assert float(deltas["dx"].abs().max()) > 0.05             # the heads move the parameters visibly
    for mask in range(16):
        flags = [h for i, h in enumerate(HEADS) if mask >> i & 1]
        for apply_rotation in ((False, True) if "dr" in flags else (False,)):
            out = run(gs, t, planes, dtrunk, {h: dheads[h] for h in flags}, apply_rotation)
            check_outputs(out, gs, deltas, flags, apply_rotation)


@pytest.mark.parametrize("n", [1, 15, 16, 17, 127, 128, 129, 1_000_003])
def test_row_counts_at_tile_edges(n):
    t = 0.75
    grids, res, trunk, heads = make_net(32, 4, 64, 1, seed=7, res_scale=4)
    gs = gaussians(n, seed=3)
    planes, dtrunk, dheads = dev_net(grids, trunk, heads)
    out = run(gs, t, planes, dtrunk, dheads, apply_rotation=True)
    torch.cuda.synchronize()
    rows = torch.arange(n) if n < 5000 else torch.cat([torch.arange(0, n, 997), torch.arange(n - 300, n)])
    _, deltas = oracle_parts(gs, t, grids, trunk, heads, rows=rows)
    check_outputs(out, gs, deltas, HEADS, True, rows=rows)
    assert all(bool(torch.isfinite(o).all()) for o in out)


@pytest.mark.parametrize("t", [0.0, 1.0, 0.3, -0.4, 1.6])
def test_coordinates_at_inside_and_beyond_the_border_on_every_axis(t):
    """every combination of p in {-1.5, -1, -0.999, 0, 0.999, 1, 1.5} on x, y, z, and t on, inside and beyond the time axis' ends;
    plus points on the nodes of every level"""
    grids, res, trunk, heads = make_net(16, 3, 128, 2, seed=11)
    gs = gaussians(343, seed=5)
    nodes = []
    for r in res:
        for j in range(0, max(r[:3]), 2):
            nodes.append([-1 + 2 * min(j, rr - 1) / (rr - 1) for rr in r[:3]])
    p = torch.tensor(nodes, dtype=torch.float32)
    extra = AABB[0] + (p + 1) / 2 * (AABB[1] - AABB[0])
    gs["means"] = torch.cat([gs["means"], extra])
    k = extra.shape[0]
    for key in ("scales", "quats", "dc", "rest"):
        gs[key] = torch.cat([gs[key], gs[key][:k]])
    planes, dtrunk, dheads = dev_net(grids, trunk, heads)
    out = run(gs, t, planes, dtrunk, dheads)
    _, deltas = oracle_parts(gs, t, grids, trunk, heads)
    check_outputs(out, gs, deltas, HEADS, False)


def test_repack_is_channel_last():
    from b200gs import ops
    grids, res, _, _ = make_net(16, 2, 64, 1, seed=2)
    planes = ops.gs4d_repack_planes([[p.to(DEV) for p in level] for level in grids]).planes.cpu()
    want = torch.cat([p[0].permute(1, 2, 0).reshape(-1) for level in grids for p in level])
    assert torch.equal(planes, want)


def test_grad_enabled_inputs_are_refused():
    grids, res, trunk, heads = make_net(16, 1, 64, 1, seed=1)
    planes, dtrunk, dheads = dev_net(grids, trunk, heads)
    gs = gaussians(20, seed=1)
    from b200gs import ops
    means = gs["means"].to(DEV).requires_grad_(True)
    with pytest.raises(RuntimeError, match="forward only"):
        ops.gs4d_deform(means, gs["scales"].to(DEV), gs["quats"].to(DEV), 0.5, planes, AABB.to(DEV), dtrunk, dheads,
                        shs_dc=gs["dc"].to(DEV), shs_rest=gs["rest"].to(DEV))
    w = dtrunk[0][0].clone().requires_grad_(True)
    with pytest.raises(RuntimeError, match="forward only"):
        ops.gs4d_deform(gs["means"].to(DEV), gs["scales"].to(DEV), gs["quats"].to(DEV), 0.5, planes, AABB.to(DEV), [(w, dtrunk[0][1])],
                        dheads, shs_dc=gs["dc"].to(DEV), shs_rest=gs["rest"].to(DEV))
    with torch.no_grad():
        ops.gs4d_deform(means, gs["scales"].to(DEV), gs["quats"].to(DEV), 0.5, planes, AABB.to(DEV), dtrunk, dheads,
                        shs_dc=gs["dc"].to(DEV), shs_rest=gs["rest"].to(DEV))


def test_one_launch_and_no_host_synchronisation():
    from b200gs import _lib, ops
    grids, res, trunk, heads = make_net(32, 2, 64, 1, seed=4)
    planes, dtrunk, dheads = dev_net(grids, trunk, heads)
    gs = {k: v.to(DEV) for k, v in gaussians(5000, seed=2).items()}
    t, aabb = torch.tensor([0.5], device=DEV), AABB.to(DEV)
    L = _lib.lib()
    with torch.no_grad():
        ops.gs4d_deform(gs["means"], gs["scales"], gs["quats"], t, planes, aabb, dtrunk, dheads, shs_dc=gs["dc"], shs_rest=gs["rest"])
        torch.cuda.synchronize()
        c0 = L.b200gs_launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            ops.gs4d_deform(gs["means"], gs["scales"], gs["quats"], t, planes, aabb, dtrunk, dheads, shs_dc=gs["dc"],
                            shs_rest=gs["rest"])
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert L.b200gs_launch_count() - c0 == ops.GS4D_FWD_LAUNCHES == 1


# ---- the renderer on checkpoints in the reference's format ---------------------------------------------------------------------
def _renderer(tmp_path, name):
    from b200gs.gs4d import B200GS4DDeformNetwork, B200VanillaGS4DRenderer
    cfg, sd, p, t = load_case(name)
    MG.write_checkpoint(str(tmp_path), cfg, sd, p["means"].shape[0])
    return B200VanillaGS4DRenderer(str(tmp_path), MG.ITERATION, DEV), cfg, sd, p, t


def _model(p):
    from b200gs.scene import SyntheticGaussians
    return SyntheticGaussians(p).to(DEV)


@pytest.mark.parametrize("name", sorted(MG.CASES))
def test_renderer_matches_the_reference_recording(tmp_path, name):
    r, cfg, sd, p, t = _renderer(tmp_path, name)
    from b200gs.scene import make_ring_cameras
    cam = make_ring_cameras(128, 96)[2].to_device(DEV)
    cam.time = torch.tensor([t], device=DEV)
    pc = _model(p)
    (m, s, q, dc, rest), raw = r.deform(cam, pc)
    bar = 2e-5
    assert max_abs(m, torch.from_numpy(ZS[f"{name}.out.means3D"])) <= bar
    assert max_abs(s.exp(), torch.from_numpy(ZS[f"{name}.out.scales"])) <= bar
    assert max_abs(torch.nn.functional.normalize(q), torch.from_numpy(ZS[f"{name}.out.rotations"])) <= bar
    assert max_abs(torch.cat([dc, rest], 1), torch.from_numpy(ZS[f"{name}.out.features"])) <= bar
    assert max_abs(torch.sigmoid(raw["opacities"]), torch.from_numpy(ZS[f"{name}.out.opacity"])) <= 2.5e-7         # torch sigmoid, CPU against GPU: 2 ulp


@pytest.mark.parametrize("name", ["default", "hypernerf_like", "small_rotation"])
def test_renderer_image_against_the_oracle_render(tmp_path, name):
    from b200gs.scene import make_ring_cameras
    r, cfg, sd, p, t = _renderer(tmp_path, name)
    W, H = 128, 96
    cam = make_ring_cameras(W, H)[5]
    ov = G.make_view(cam.R, cam.T, float(cam.fx), float(cam.fy), float(cam.cx), float(cam.cy), W, H)
    cam = cam.to_device(DEV)
    cam.time = torch.tensor([t], device=DEV)
    bg = torch.tensor([0.1, 0.2, 0.3])
    out = r(cam, _model(p), bg.to(DEV))
    assert set(out) == {"render", "depth", "viewspace_points", "visibility_filter", "radii"} and out["depth"] is None
    grids, trunk, heads = network(cfg, sd)
    d = O.deform(p["means"], p["scales"], p["rotations"], t, sd["deformation_net.grid.aabb"], grids, trunk, heads,
                 shs=torch.cat([p["shs_dc"], p["shs_rest"]], 1), apply_rotation=cfg.apply_rotation)
    a = O.activate(d, p["opacities"])
    ref = G.render(G.MODE_VANILLA, a["means"], a["scales"], a["rotations"], a["opacities"], a["shs"], ov, bg.double())
    vis = out["visibility_filter"].cpu()
    assert 0 < int(vis.sum()) and out["radii"].shape == (p["means"].shape[0],)
    assert float(out["render"].detach().cpu().double().sub(ref["render"]).abs().max()) <= 2e-4
    assert float(out["render"].abs().max()) > 0.05
    assert out["viewspace_points"].shape == p["means"].shape and out["viewspace_points"].requires_grad


def test_renderer_refuses_a_pre_activated_model(tmp_path):
    r, cfg, sd, p, t = _renderer(tmp_path, "small_d1")
    pc = _model(p)
    pc.is_pre_activated = True
    from b200gs.scene import make_ring_cameras
    cam = make_ring_cameras(64, 48)[0].to_device(DEV)
    cam.time = torch.tensor([t], device=DEV)
    with pytest.raises(ValueError, match="pre-activated"):
        r(cam, pc, torch.zeros(3, device=DEV))
