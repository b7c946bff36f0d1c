"""K47 / K48 (csrc/glossy.cu) through ops.glossy_sh and B200GlossyRendererModule on the GPU, against the float64 oracle
(oracle/glossy_oracle.py) and the recorded reference modules (tests/golden/glossy.npz).

Clamp decisions: a sample whose oracle value lies within AMBIGUOUS (8 * 2^-23, relative to the rounding scale of its sum) of a clamp
bound may fall either way in fp32 (DESIGN.md §2, threshold flips).  For those samples the oracle takes the kernel's decision, read
from the dc gradient (basis_0 * cotangent, zero exactly when the kernel clamped), and they must be rare.  Every other clamped
sample must get exactly zero gradient."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import glossy_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def make_inputs(n, degree, layout, mask_kind, k_rest=None, stride=None, seed=0, at_camera=True):
    """float32 CPU tensors: means, campos, op dc / rest, colour (split pair, features or None), mask, cotangents"""
    g = torch.Generator().manual_seed(seed)
    need = (degree + 1) ** 2
    k_rest = need - 1 if k_rest is None else k_rest
    stride = max(need, 16) if stride is None else stride
    campos = torch.randn(3, generator=g)
    means = campos + torch.randn(n, 3, generator=g) * 2.0
    if at_camera and n > 0:
        means[0] = campos                                       # the zero direction
    dc = torch.randn(n, 1, 1, generator=g) * 1.5
    rest = torch.randn(n, k_rest, 1, generator=g) * 0.6
    colour = None
    if layout == "split":
        colour = (torch.randn(n, 1, 3, generator=g), torch.randn(n, stride - 1, 3, generator=g) * 0.5)
    elif layout == "features":
        colour = torch.randn(n, stride, 3, generator=g) * 0.5
    mask = {"none": None, "false": torch.zeros(n, dtype=torch.bool), "mixed": torch.rand(n, generator=g) < 0.6}[mask_kind]
    v_rgb, v_op = torch.randn(n, 3, generator=g), torch.randn(n, generator=g)
    return means, campos, dc, rest, colour, mask, v_rgb, v_op


def _mx(t):
    return float(t.abs().max()) if t.numel() else 0.0


def run_kernels(degree, means, campos, dc, rest, colour, mask, v_rgb, v_op):
    from b200gs import ops
    dc, rest = dc.to(DEV).requires_grad_(True), rest.to(DEV).requires_grad_(True)
    kw, params = {}, [dc, rest]
    if isinstance(colour, tuple):
        kw = {"shs_dc": colour[0].to(DEV).requires_grad_(True), "shs_rest": colour[1].to(DEV).requires_grad_(True)}
        params += [kw["shs_dc"], kw["shs_rest"]]
    elif colour is not None:
        kw = {"features": colour.to(DEV).requires_grad_(True)}
        params += [kw["features"]]
    rgb, op = ops.glossy_sh(degree, means.to(DEV), campos.to(DEV), dc, rest, mask=None if mask is None else mask.to(DEV), **kw)
    outs, cots = [op], [v_op.to(DEV)]
    if rgb is not None:
        outs.append(rgb)
        cots.append(v_rgb.to(DEV))
    torch.autograd.backward(outs, cots)
    return (None if rgb is None else rgb.detach().cpu()), op.detach().cpu(), [p.grad.cpu() for p in params]


def check_against_oracle(degree, means, campos, dc, rest, colour, mask, v_rgb, v_op, tol=2e-6):
    """runs the kernels, compares with the oracle (the kernel's clamp decision on ambiguous samples); returns the kernel outputs"""
    rgb, op, grads = run_kernels(degree, means, campos, dc, rest, colour, mask, v_rgb, v_op)
    n, need = means.shape[0], (degree + 1) ** 2
    d64 = lambda t: t.double().requires_grad_(True)                                     # noqa: E731
    p64 = [d64(dc), d64(rest)] + ([d64(c) for c in colour] if isinstance(colour, tuple) else [] if colour is None else [d64(colour)])
    col64 = None if colour is None else (tuple(p64[2:]) if isinstance(colour, tuple) else p64[2])
    first = O.glossy(degree, means.double(), campos.double(), p64[0].detach(), p64[1].detach(),
                     None if col64 is None else (tuple(c.detach() for c in col64) if isinstance(col64, tuple) else col64.detach()), mask)
    near_o = O.near_bound(first["raw_opacity"], first["scale_opacity"], 0.0, 1.0)
    pass_o = torch.where(near_o, grads[0][:, 0, 0] != 0, (first["raw_opacity"] >= 0) & (first["raw_opacity"] <= 1))
    pass_c = near_c = None
    if colour is not None:
        near_c = O.near_bound(first["raw_rgb"], first["scale_rgb"], 0.0)
        if mask is not None:
            near_c &= mask[:, None]
        pass_c = torch.where(near_c, grads[2][:, 0, :] != 0, first["raw_rgb"] >= 0)    # the colour dc row, in both layouts
    assert int(near_o.sum()) + (0 if near_c is None else int(near_c.sum())) <= 2 + n // 1000
    ref = O.glossy(degree, means.double(), campos.double(), p64[0], p64[1], col64, mask, pass_opacity=pass_o, pass_rgb=pass_c)
    outs, cots = [ref["opacity"]], [v_op.double()]
    if colour is not None:
        outs.append(ref["rgb"])
        cots.append(v_rgb.double())
    torch.autograd.backward(outs, cots)

    assert _mx(op.double() - ref["opacity"].detach()) <= tol * max(_mx(first["scale_opacity"]), 1.0)
    if colour is None:
        assert rgb is None
    else:
        assert _mx(rgb.double() - ref["rgb"].detach()) <= tol * max(_mx(first["scale_rgb"]), 1.0)
    for k, (got, p) in enumerate(zip(grads, p64)):
        want = torch.zeros_like(p) if p.grad is None else p.grad
        err = _mx(got.double() - want)
        assert err <= 4 * tol * max(_mx(want), 1.0), (k, err)
    if n > 0:       # the opacity dc gradient is zero exactly where the oracle's is
        assert torch.equal(grads[0] == 0, p64[0].grad == 0)
    # exact zeros: blocked opacity rows, rest rows beyond the degree, masked and clamped colour entries
    blocked = ~pass_o
    assert not grads[0][blocked].any() and not grads[1][blocked].any() and not grads[1][:, need - 1:].any()
    if colour is not None:
        v_col = torch.cat(grads[2:], dim=1)                                 # [n, stride, 3] in coefficient order
        assert not v_col[:, need:].any()
        if mask is not None:
            assert not v_col[~mask].any() and bool((rgb[~mask] == 0.5).all())
        assert not v_col.permute(0, 2, 1)[~pass_c].any()
    return rgb, op, grads


@pytest.mark.parametrize("mask_kind", ["none", "false", "mixed"])
@pytest.mark.parametrize("layout", ["split", "features"])
@pytest.mark.parametrize("degree", [0, 1, 2, 3, 4])
def test_against_oracle(degree, layout, mask_kind):
    stride = 25 if degree == 4 else 16
    check_against_oracle(degree, *make_inputs(257, degree, layout, mask_kind, k_rest=stride - 1, stride=stride, seed=degree))


@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 1 << 20])
def test_sizes(n):
    check_against_oracle(3, *make_inputs(n, 3, "split", "mixed", seed=n % 97))


@pytest.mark.parametrize("degree,k_rest,layout,stride", [(1, 15, "features", 16), (2, 24, "split", 25), (3, 24, "features", 25),
                                                         (0, 15, "split", 16), (3, 60, "split", 16)])
def test_storage_longer_than_the_degree_needs(degree, k_rest, layout, stride):
    """extra opacity rows and colour coefficients get exactly zero gradient; 25-coefficient colour at degree 3 and a 60-row opacity
    rest are wider than the 16-coefficient kernel's staging rows and take the per-thread stores"""
    check_against_oracle(degree, *make_inputs(300, degree, layout, "mixed", k_rest=k_rest, stride=stride, seed=7))


def test_colour_off_gives_identical_opacity():
    means, campos, dc, rest, colour, mask, v_rgb, v_op = make_inputs(5000, 3, "split", "mixed", seed=4)
    rgb0, op0, g0 = check_against_oracle(3, means, campos, dc, rest, None, mask, v_rgb, v_op)
    rgb1, op1, g1 = run_kernels(3, means, campos, dc, rest, colour, mask, v_rgb, v_op)
    assert rgb0 is None and rgb1 is not None
    assert torch.equal(op0, op1) and torch.equal(g0[0], g1[0]) and torch.equal(g0[1], g1[1])


def test_repeats_launches_and_no_host_sync():
    from b200gs import _lib, ops
    L = _lib.lib()
    for layout in ("split", "features"):
        means, campos, dc, rest, colour, mask, v_rgb, v_op = make_inputs(300_000, 3, layout, "mixed", seed=9)
        runs = [run_kernels(3, means, campos, dc, rest, colour, mask, v_rgb, v_op) for _ in range(2)]
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
        assert all(torch.equal(a, b) for a, b in zip(runs[0][2], runs[1][2]))
        dcd, restd = dc.to(DEV).requires_grad_(True), rest.to(DEV).requires_grad_(True)
        kw = ({"shs_dc": colour[0].to(DEV).requires_grad_(True), "shs_rest": colour[1].to(DEV).requires_grad_(True)} if layout == "split"
              else {"features": colour.to(DEV).requires_grad_(True)})
        md, cd, maskd, vr, vo = means.to(DEV), campos.to(DEV), mask.to(DEV), v_rgb.to(DEV), v_op.to(DEV)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            c0 = L.b200gs_launch_count()
            rgb, op = ops.glossy_sh(3, md, cd, dcd, restd, mask=maskd, **kw)
            c1 = L.b200gs_launch_count()
            torch.autograd.backward([rgb, op], [vr, vo])
            c2 = L.b200gs_launch_count()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert (c1 - c0, c2 - c1) == (ops.GLOSSY_FWD_LAUNCHES, ops.GLOSSY_BWD_LAUNCHES) == (1, 1)


# ---- the recorded reference modules ------------------------------------------------------------------------------------------
Z = np.load(os.path.join(GOLDEN, "glossy.npz"))


def _gz(key):
    return torch.from_numpy(Z[key])


def _glossy_model(n=None, scene=None, degree=3):
    """A stand-in with the reference GlossyGaussianModel's property names: opacities [N,1,1] (SH dc) and opacity_rest [N,15,1]."""
    from b200gs.scene import SyntheticGaussians, make_scene

    class GlossyGaussians(SyntheticGaussians):
        def get_opacities(self):
            return 0.28209479177387814 * self.gaussians["opacities"][:, 0] + 0.5

    raw = make_scene(n, 5, mean_scale=0.05) if scene is None else scene
    g = torch.Generator().manual_seed(21)
    m = raw["means"].shape[0]
    raw = dict(raw)
    raw["opacities"] = torch.randn(m, 1, 1, generator=g) * 1.2 + 0.4
    raw["opacity_rest"] = torch.randn(m, 15, 1, generator=g) * 0.4
    return GlossyGaussians(raw, active_sh_degree=degree)


@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_golden_replay(degree):
    from b200gs import ops
    from b200gs.glossy import B200GlossyRenderer
    w = _gz("w").to(DEV)
    for key in ("model", "renderer"):
        dc, rest = _gz("op_dc").to(DEV).requires_grad_(True), _gz("op_rest").to(DEV).requires_grad_(True)
        if key == "model":
            _, op = ops.glossy_sh(degree, _gz("means").to(DEV), _gz("campos").to(DEV), dc, rest)
            want = _gz(f"renderer_{degree}_opacity")            # the kernel clamps; the recorded model output is unclamped
        else:
            model = _glossy_model(scene={"means": _gz("means"), "shs_dc": torch.zeros(96, 1, 3), "shs_rest": torch.zeros(96, 15, 3),
                                         "scales": torch.zeros(96, 3), "rotations": torch.ones(96, 4)}, degree=degree).to(DEV)
            with torch.no_grad():
                model.gaussians["opacities"].copy_(_gz("op_dc"))
                model.gaussians["opacity_rest"].copy_(_gz("op_rest"))
            dc, rest = model.gaussians["opacities"], model.gaussians["opacity_rest"]
            r = B200GlossyRenderer(separate_sh=True, tile_based_culling=True).instantiate().to(DEV)
            r._rgb_requested = False
            cam = type("Cam", (), {"camera_center": _gz("campos").to(DEV)})()
            op, status = r.get_opacities(cam, model, None, torch.ones(96, dtype=torch.bool, device=DEV), None)
            assert status is None
            want = _gz(f"renderer_{degree}_opacity")
        (op * w).sum().backward()
        assert float((op.detach().cpu() - want).abs().max()) <= 4e-6, key
        assert float((dc.grad.cpu() - _gz(f"renderer_{degree}_v_dc")).abs().max()) <= 1e-5, key
        assert float((rest.grad.cpu() - _gz(f"renderer_{degree}_v_rest")).abs().max()) <= 1e-5, key
        raw = _gz(f"model_{degree}_opacity").reshape(-1)
        inside = (raw > 1e-5) & (raw < 1 - 1e-5)
        assert float((op.detach().cpu()[inside] - raw[inside]).abs().max()) <= 4e-6


# ---- end to end: the renderer against the v1 render with the oracle's hooks restated in torch -----------------------------------
def _oracle_hooks_renderer(config):
    from b200gs.v1 import B200GSplatV1RendererModule

    class TorchGlossy(B200GSplatV1RendererModule):
        def get_opacities(self, camera, gm, projections, visibility_filter, status, **kwargs):
            out = O.glossy(gm.active_sh_degree, gm.get_xyz, camera.camera_center, gm.gaussians["opacities"], gm.gaussians["opacity_rest"],
                           colour=(gm.get_shs_dc(), gm.get_shs_rest()), mask=visibility_filter)
            return out["opacity"], out["rgb"]

        def get_rgbs(self, camera, gm, projections, visibility_filter, status, **kwargs):
            return status

    return TorchGlossy(config)


@pytest.mark.parametrize("anti_aliased", [True, False])
@pytest.mark.parametrize("culling", [True, False])
def test_end_to_end_against_the_torch_hooks(anti_aliased, culling):
    from b200gs.glossy import B200GlossyRenderer
    from b200gs.scene import make_ring_cameras
    cfg = B200GlossyRenderer(separate_sh=True, tile_based_culling=culling, anti_aliased=anti_aliased)
    cam = make_ring_cameras(256, 192)[2].to_device(DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    cot = torch.randn(3, 192, 256, generator=torch.Generator().manual_seed(3)).to(DEV)
    results = []
    for renderer in (cfg.instantiate(), _oracle_hooks_renderer(cfg)):
        pc = _glossy_model(4096).to(DEV)
        out = renderer.to(DEV)(cam, pc, bg)
        vis = out["visibility_filter"]
        assert 0 < int(vis.sum()) < vis.numel()
        (out["render"] * cot).sum().backward()
        results.append((out["render"].detach(), out["opacities"].detach(), {k: p.grad.clone() for k, p in pc.gaussians.items()}))
    (img, opac, grads), (img_t, opac_t, grads_t) = results
    assert float((img - img_t).abs().max()) <= 1e-5
    assert float((opac - opac_t).abs().max()) <= 2e-6
    for k in ("opacities", "opacity_rest", "shs_dc", "shs_rest", "means", "scales", "rotations"):
        scale = float(grads_t[k].abs().max()) + 1e-12
        assert float((grads[k] - grads_t[k]).abs().max()) <= 1e-4 * scale, (k, float((grads[k] - grads_t[k]).abs().max()) / scale)


def test_render_without_rgb_skips_the_colour():
    from b200gs.glossy import B200GlossyRenderer
    from b200gs.scene import make_ring_cameras
    cam = make_ring_cameras(128, 96)[1].to_device(DEV)
    pc = _glossy_model(2048).to(DEV)
    r = B200GlossyRenderer(separate_sh=True, tile_based_culling=True).instantiate().to(DEV)
    depth = r(cam, pc, torch.zeros(3, device=DEV), render_types=["acc_depth"])
    full = r(cam, pc, torch.zeros(3, device=DEV), render_types=["rgb", "acc_depth"])
    assert depth["render"] is None and full["render"] is not None
    assert torch.equal(depth["opacities"], full["opacities"])
