"""gsplat v1 drop-in (b200gs/compat/gsplat_v1.py): the reference's GSplatV1Renderer call sequence on the b200gs kernels.

tests/golden/make_golden_v1_dropin.py ran the reference's unmodified GSplatV1Renderer (internal/renderers/gsplat_v1_renderer.py)
with recording stand-ins and stored, per option set, the calls it made into gsplat.  `reference_forward` below is that
renderer's forward written out against the gsplat names ``b200gs.compat.install()`` registers; the first test checks it makes
exactly the recorded calls, with the contract's shapes and dtypes on every argument and return.  The others check the drop-in
against the plug-in ``B200GSplatV1Renderer`` (images bit for bit, gradients to atomic-order rounding), the float64 oracle, and the keys / offsets / split-SH kernels at
their boundaries.
"""
import importlib
import json
import math
import os
import zlib

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import gs_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
AMBIGUOUS = 5e-4
ATOMIC_NOISE = 5e-5     # the same gradient terms summed in another atomic order (as in test_gpu_blend_channels.py)
OPTIONS = [(False, False), (False, True), (True, False), (True, True)]     # (separate_sh, tile_based_culling)


def _golden():
    with open(os.path.join(GOLDEN, "dropin_v1.json")) as f:
        return json.load(f)


def _gsplat(log=None):
    """The gsplat names the reference imported, resolved through the modules install() registers; `log` records every call."""
    from b200gs import compat
    compat.install()
    fns = {}
    for mod, attr in _golden()["imported"]:
        if not mod.startswith("gsplat"):
            continue
        fn = getattr(importlib.import_module(mod), attr)
        if log is not None:
            fn = (lambda f, name: lambda *a, **k: log.append((name, a, k, f(*a, **k))) or log[-1][3])(fn, attr)
        fns[attr] = fn
    return fns


def reference_forward(g, separate_sh, culling, cam, pc, bg, render_types, block_size=16):
    """GSplatV1RendererModule.forward (gsplat_v1_renderer.py:137-348) with GSplatV1's helpers (:370-603) for these render types."""
    viewmats = cam.world_to_camera.T.unsqueeze(0)
    Ks = torch.tensor([[[float(cam.fx), 0., float(cam.cx)], [0., float(cam.fy), float(cam.cy)], [0., 0., 1.]]], dtype=torch.float, device=DEV)
    img_width, img_height = int(cam.width), int(cam.height)
    projections = g["fully_fused_projection"](pc.get_means(), None, pc.get_rotations(), pc.get_scales(), viewmats=viewmats, Ks=Ks,
                                              width=img_width, height=img_height, eps2d=0.3, calc_compensations=True, packed=False,
                                              radius_clip=0.0, camera_model="pinhole")
    radii, means2d, depths, conics, compensations = projections
    visibility_filter = radii.squeeze(0) > 0
    opacities = pc.get_opacities().squeeze(-1).unsqueeze(0) * compensations
    tw, th = math.ceil(img_width / float(block_size)), math.ceil(img_height / float(block_size))
    if culling:
        tiles_per_gauss, isect_ids, flatten_ids = g["isect_tiles_tile_based_culling"](means2d, radii, depths, conics, opacities.detach(), block_size,
                                                                                      tw, th, packed=False, n_cameras=1, camera_ids=None,
                                                                                      gaussian_ids=None)
        isect_offsets, flatten_ids = g["isect_offset_encode_tile_based_culling"](isect_ids, flatten_ids, 1, tw, th)
    else:
        tiles_per_gauss, isect_ids, flatten_ids = g["isect_tiles"](means2d, radii, depths, block_size, tw, th, packed=False, n_cameras=1,
                                                                   camera_ids=None, gaussian_ids=None)
        isect_offsets = g["isect_offset_encode"](isect_ids, 1, tw, th)
    means2d = means2d.squeeze(0)

    def rasterize(colors, background, opac=opacities, absgrad=True):
        c, a = g["rasterize_to_pixels"](means2d=means2d, conics=conics, colors=colors.unsqueeze(0), opacities=opac, image_width=img_width,
                                        image_height=img_height, tile_size=block_size, isect_offsets=isect_offsets, flatten_ids=flatten_ids,
                                        backgrounds=background.unsqueeze(0), absgrad=absgrad)
        return c.squeeze(0), a.squeeze(0)

    out = {"viewspace_points": means2d, "visibility_filter": visibility_filter, "radii": radii.squeeze(0),
           "isects": (tiles_per_gauss, isect_ids, flatten_ids, isect_offsets)}
    feats, bgs, slices, n = [], [], {}, 0
    if "rgb" in render_types:
        dirs = pc.get_xyz.detach() - cam.camera_center
        if separate_sh:
            rgbs = g["spherical_harmonics_decomposed"](pc.active_sh_degree, dirs, pc.get_shs_dc(), pc.get_shs_rest(), visibility_filter)
        else:
            rgbs = g["spherical_harmonics"](pc.active_sh_degree, dirs, pc.get_features, visibility_filter)
        feats.append(torch.clamp(rgbs + 0.5, min=0.0)); bgs.append(bg); slices["render"] = (n, n + 3); n += 3
    if {"alpha", "acc_depth", "exp_depth"} & set(render_types):
        feats.append(depths[0].unsqueeze(-1)); bgs.append(torch.zeros((1,), device=DEV)); slices["acc_depth"] = (n, n + 1); n += 1
    if "normal" in render_types:
        from b200gs.v1 import build_rotation
        normals = build_rotation(pc.get_rotations())[:, :3, -1]
        facing = torch.einsum("ij,ij->i", normals, pc.get_means() - cam.camera_center) > 0
        feats.append(normals * torch.where(facing, -1., 1.).unsqueeze(-1)); bgs.append(torch.zeros((3,), device=DEV))
        slices["normal"] = (n, n + 3); n += 3
    rendered, alpha = rasterize(torch.concat(feats, dim=-1), torch.concat(bgs, dim=-1))
    rendered, alpha = rendered.permute(2, 0, 1), alpha.squeeze(-1).unsqueeze(0)
    for k, (a, b) in slices.items():
        out[k] = rendered[a:b]
    out["alpha"], out["acc_vis"] = alpha, means2d.has_hit_any_pixels
    if "exp_depth" in render_types:
        out["exp_depth"] = torch.where(alpha > 0, out["acc_depth"] / alpha, out["acc_depth"].detach().max())
    zero1 = torch.zeros((1,), dtype=torch.float, device=DEV)
    if "inverse_depth" in render_types:
        out["inverse_depth"] = rasterize(1. / (depths[0].clamp_min(0.) + 1e-8).unsqueeze(-1), zero1)[0].permute(2, 0, 1)
    if "hard_depth" in render_types:
        out["hard_depth"] = rasterize(depths[0].unsqueeze(-1), zero1, opac=opacities + (1 - opacities.detach()), absgrad=False)[0].permute(2, 0, 1)
    return out


def _setup(n=4096, W=256, H=192, seed=5, pose=3, ms=0.05):
    from b200gs.scene import SyntheticGaussians, make_ring_cameras, make_scene
    raw = make_scene(n, seed, mean_scale=ms)
    return raw, SyntheticGaussians(raw).to(DEV), make_ring_cameras(W, H)[pose].to_device(DEV)


def _describe(a, sizes):
    if torch.is_tensor(a):
        return {"shape": list(a.shape), "dtype": str(a.dtype).replace("torch.", "")}
    if isinstance(a, (tuple, list)):
        return {"seq": [_describe(x, sizes) for x in a]}
    return {"value": a}


def _concrete(d, sizes):
    """A recorded descriptor with N / H / W / I replaced by this run's sizes and the requires_grad flag (a property of the stand-ins)
    dropped."""
    if "shape" in d:
        return {"shape": [sizes[s] if isinstance(s, str) else s for s in d["shape"]], "dtype": d["dtype"]}
    if "seq" in d:
        return {"seq": [_concrete(x, sizes) for x in d["seq"]]}
    return d


@pytest.mark.parametrize("separate_sh,culling", OPTIONS)
def test_reference_call_sequence_and_contract_shapes(separate_sh, culling):
    rec = _golden()
    calls = rec["renders"][f"sh{int(separate_sh)}_cull{int(culling)}"]["calls"]
    raw, model, cam = _setup(rec["N"], rec["W"], rec["H"], 4, 2)
    log = []
    out = reference_forward(_gsplat(log), separate_sh, culling, cam, model, torch.tensor([0.1, 0.2, 0.3], device=DEV), rec["render_types"])
    sizes = {"N": rec["N"], "H": rec["H"], "W": rec["W"], "I": int(out["isects"][1].shape[0])}
    assert [c[0] for c in log] == [c["fn"] for c in calls]
    for (fn, args, kw, ret), c in zip(log, calls):
        assert [_describe(a, sizes) for a in args] == [_concrete(a, sizes) for a in c["args"]], fn
        assert {k: _describe(v, sizes) for k, v in kw.items()} == {k: _concrete(v, sizes) for k, v in c["kwargs"].items()}, fn
        ret = ret if isinstance(ret, tuple) else (ret,)
        assert [_describe(r, sizes) for r in ret] == [_concrete(r, sizes) for r in c["returns"]], fn


def _cotangents(out, seed=1):
    gen = torch.Generator().manual_seed(seed)
    return {k: (torch.rand(out[k].shape, generator=gen) * 2 - 1).to(DEV) for k in
            ("render", "alpha", "acc_depth", "normal", "exp_depth", "inverse_depth", "hard_depth")}


def _run(fn, model, cot=None):
    for p in model.parameters():
        p.grad = None
    out = fn()
    out["viewspace_points"].retain_grad()
    cot = cot or _cotangents(out)
    sum((out[k] * c).sum() for k, c in cot.items()).backward()
    grads = {k: p.grad.clone() for k, p in model.gaussians.items()}
    return out, grads, cot


@pytest.mark.parametrize("separate_sh,culling", OPTIONS)
def test_bit_identical_to_plugin(separate_sh, culling):
    from b200gs.v1 import B200GSplatV1Renderer
    raw, model, cam = _setup()
    bg = torch.tensor([0.2, 0.1, 0.5], device=DEV)
    types = _golden()["render_types"]
    g = _gsplat()
    ref, g_ref, cot = _run(lambda: reference_forward(g, separate_sh, culling, cam, model, bg, types), model)
    plug = B200GSplatV1Renderer(separate_sh=separate_sh, tile_based_culling=culling).instantiate().to(DEV)
    out, g_out, _ = _run(lambda: plug(cam, model, bg, render_types=types), model, cot)
    for k in ("render", "alpha", "acc_depth", "normal", "exp_depth", "inverse_depth", "hard_depth", "radii", "acc_vis", "visibility_filter"):
        assert torch.equal(out[k], ref[k]), k
    # K7 accumulates the per-Gaussian gradients with float atomics from every tile the Gaussian is listed in, so their summation
    # order (and last bits) is not fixed from one backward to the next, for either path: the gradients agree to that rounding
    def close(a, b):
        return float((a - b).abs().max()) <= ATOMIC_NOISE * float(b.abs().max())

    assert close(out["viewspace_points"].grad, ref["viewspace_points"].grad)
    assert close(out["viewspace_points"].absgrad, ref["viewspace_points"].absgrad)
    for k in g_out:
        assert close(g_out[k], g_ref[k]), k
    # the contract's isect tensors against the plug-in's binning of the same view
    tiles_per_gauss, isect_ids, flatten_ids, isect_offsets = ref["isects"]
    b = out["isects"].binning
    assert torch.equal(tiles_per_gauss, out["isects"][0].int()) and torch.equal(flatten_ids, b.sorted_ids[:b.total])
    assert isect_ids.dtype == torch.int64 and isect_offsets.dtype == torch.int32 and flatten_ids.dtype == torch.int32


def _np_offset_encode(keys, n_tiles):
    """gsplat's isect_offset_encode for one camera, in numpy: the first index of each tile, the next start for empty tiles."""
    return np.searchsorted(np.asarray(keys) >> 32, np.arange(n_tiles), side="left").astype(np.int32)


def _is_subsequence(sub, full):
    it = iter(full.tolist())
    return all(any(x == y for y in it) for x in sub.tolist())


@pytest.mark.parametrize("separate_sh,culling", OPTIONS)
def test_against_float64_oracle(separate_sh, culling):
    """rgb render and every gradient against the float64 oracle (DESIGN §2's bars), isect_ids / offsets / flatten_ids against
    the oracle's stable sort."""
    from b200gs.scene import activate, make_ring_cameras
    raw, model, cam = _setup()
    bg = torch.tensor([0.2, 0.1, 0.5], device=DEV)
    W, H = int(cam.width), int(cam.height)
    out = reference_forward(_gsplat(), separate_sh, culling, cam, model, bg, ["rgb"])
    cot = torch.rand(3, H, W, generator=torch.Generator().manual_seed(1)) * 2 - 1
    (out["render"] * cot.to(DEV)).sum().backward()
    c = make_ring_cameras(W, H)[3]
    ov = O.make_view(c.R, c.T, float(c.fx), float(c.fy), float(c.cx), float(c.cy), W, H)
    leaves = {k: v.double().requires_grad_(True) for k, v in raw.items()}     # the model's raw parameters, activated as it does
    act = activate(leaves)
    margins = []
    ref = O.render(O.MODE_GSPLAT, act["means"], act["scales"], act["rotations"], act["opacities"], act["shs"], ov, bg.cpu().double(),
                   margins=margins)
    (ref["render"] * cot.double()).sum().backward()
    err = (out["render"].detach().cpu().double() - ref["render"].detach()).abs().max(dim=0).values
    ambiguous = margins[0] < AMBIGUOUS
    assert int(((err > 1e-4) & ~ambiguous).sum()) == 0 and int(ambiguous.sum()) <= err.numel() // 20
    for k, p in model.gaussians.items():
        gref = leaves[k].grad
        assert float((p.grad.cpu().double() - gref).abs().max()) <= 1e-3 * float(gref.abs().max()), k
    # isect_ids / flatten_ids / offsets
    _, isect_ids, flatten_ids, isect_offsets = out["isects"]
    keys = isect_ids.cpu()
    assert bool((keys[1:] >= keys[:-1]).all())
    n_tiles = ((W + 15) // 16) * ((H + 15) // 16)
    if culling:
        assert _is_subsequence(keys, ref["sorted_keys"]) and keys.shape[0] < ref["sorted_keys"].shape[0]
    else:
        assert torch.equal(keys, ref["sorted_keys"]) and torch.equal(flatten_ids.cpu(), ref["sorted_ids"])
    assert np.array_equal(isect_offsets.cpu().numpy().reshape(-1), _np_offset_encode(keys.numpy(), n_tiles))


def _rects(xy, r, gx, gy):
    rmin = torch.stack([((xy[:, 0] - r) / 16).int().clamp(0, gx), ((xy[:, 1] - r) / 16).int().clamp(0, gy)], -1)
    rmax = torch.stack([(((xy[:, 0] + r) / 16).int() + 1).clamp(0, gx), (((xy[:, 1] + r) / 16).int() + 1).clamp(0, gy)], -1)
    tiles = torch.where(r > 0, (rmax - rmin).prod(-1), torch.zeros_like(r)).int()
    return rmin, rmax, tiles


BOUNDARY_CASES = {          # name: (W, H, n, how the splats are placed)
    "no_visible": (64, 48, 50, "none"),
    "empty_first_and_last_tiles": (80, 64, 300, "middle"),
    "single_tile": (16, 16, 40, "any"),
    "single_tile_partial": (11, 7, 40, "any"),
    "not_multiple_of_16": (77, 53, 500, "any"),
    "1x1": (1, 1, 20, "any"),
    "17x1": (17, 1, 40, "any"),
    "1x300": (1, 300, 300, "any"),
    "15x17": (15, 17, 60, "any"),
    "4000x16": (4000, 16, 3000, "any"),
}


@pytest.mark.parametrize("case", sorted(BOUNDARY_CASES))
def test_isect_keys_and_offsets_at_boundaries(case):
    from b200gs.compat import gsplat_v1 as G
    W, H, n, how = BOUNDARY_CASES[case]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    gen = torch.Generator().manual_seed(zlib.crc32(case.encode()))
    xy = torch.rand(n, 2, generator=gen) * torch.tensor([W, H]).float()
    if how == "middle":       # every rect inside tiles 1 .. n_tiles - 2
        xy = torch.tensor([W / 2, H / 2]) + (torch.rand(n, 2, generator=gen) - 0.5) * 8
    r = torch.randint(1, 12, (n,), generator=gen, dtype=torch.int32)
    if how == "none":
        r.zero_()
    depth = torch.rand(n, generator=gen) * 10 + 0.1
    depth[::7] = depth[3]                                   # equal depths: ties ordered by id
    rmin, rmax, tiles = _rects(xy, r, gx, gy)
    keys_ref, ids_ref = O.build_sort_keys(depth.double(), rmin, rmax, tiles, gx)
    skeys, sids, _ = O.sort_and_ranges(keys_ref, ids_ref, gx * gy)
    tpg, keys, flat = G.isect_tiles(xy[None].to(DEV), r[None].to(DEV), depth[None].to(DEV), 16, gx, gy)
    offsets = G.isect_offset_encode(keys, 1, gx, gy)
    assert torch.equal(tpg.cpu()[0], tiles)
    assert keys.dtype == torch.int64 and flat.dtype == torch.int32 and offsets.shape == (1, gy, gx)
    assert torch.equal(keys.cpu(), skeys) and torch.equal(flat.cpu(), sids)
    assert np.array_equal(offsets.cpu().numpy().reshape(-1), _np_offset_encode(skeys.numpy(), gx * gy))
    if how == "none":
        assert keys.numel() == 0 and flat.numel() == 0 and int(offsets.abs().sum()) == 0
    if how == "middle":
        o = offsets.reshape(-1).cpu()
        assert int(o[0]) == 0 and int(o[-1]) == keys.numel() and int(o[1]) == 0       # empty first tile(s) / empty last tile
    # the offsets come from the keys handed over alone: any sorted key set, including tiles past the grid and gaps
    arbitrary = torch.sort(torch.randint(0, gx * gy + 2, (97,), generator=gen).long() << 32 | 5).values
    got = G.isect_offset_encode(arbitrary.to(DEV), 1, gx, gy).cpu().numpy().reshape(-1)
    assert np.array_equal(got, _np_offset_encode(arbitrary.numpy(), gx * gy))


SH_STORAGE = {0: (16, 1), 1: (16, 4), 2: (16, 9), 3: (16, 16), 4: (25, 25)}


@pytest.mark.parametrize("degree", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("mask_kind", ["none", "partial", "all_false"])
def test_split_sh(degree, mask_kind):
    from b200gs import ops
    n = 1000
    gen = torch.Generator().manual_seed(degree * 10 + len(mask_kind))
    for k in SH_STORAGE[degree]:
        dirs = torch.randn(n, 3, generator=gen) * 3
        coeffs = torch.randn(n, k, 3, generator=gen)
        mask = {"none": None, "partial": torch.rand(n, generator=gen) < 0.6, "all_false": torch.zeros(n, dtype=torch.bool)}[mask_kind]
        keep = torch.ones(n, dtype=torch.bool) if mask is None else mask
        cot = torch.rand(n, 3, generator=gen) * 2 - 1
        dc = coeffs[:, :1].contiguous().to(DEV).requires_grad_(True)
        rest = coeffs[:, 1:].contiguous().to(DEV).requires_grad_(True)
        d = dirs.to(DEV).requires_grad_(True)
        rgb = ops.spherical_harmonics_decomposed(degree, d, dc, rest, None if mask is None else mask.to(DEV))
        (rgb * cot.to(DEV)).sum().backward()
        # the concatenated kernel: bit-identical on unmasked rows
        cc = coeffs.to(DEV).requires_grad_(True)
        d2 = dirs.to(DEV).requires_grad_(True)
        rgb2 = ops.spherical_harmonics(degree, d2, cc)
        (rgb2 * cot.to(DEV)).sum().backward()
        kk = keep.to(DEV)
        assert torch.equal(rgb[kk], rgb2[kk])
        assert torch.equal(dc.grad[kk], cc.grad[kk, :1]) and torch.equal(rest.grad[kk], cc.grad[kk, 1:])
        assert torch.equal(d.grad[kk], d2.grad[kk])
        # masked rows: zeros
        assert int(rgb[~kk].abs().sum()) == 0 and int(dc.grad[~kk].abs().sum()) == 0 and int(rest.grad[~kk].abs().sum()) == 0
        assert int(d.grad[~kk].abs().sum()) == 0
        # float64 oracle on the unmasked rows
        dd = dirs.double().requires_grad_(True)
        sh = coeffs.double().requires_grad_(True)
        ref = O.eval_sh(degree, sh, dd / dd.norm(dim=-1, keepdim=True))
        (ref[keep] * cot.double()[keep]).sum().backward()
        if bool(keep.any()):
            assert float((rgb.detach().cpu().double()[keep] - ref.detach()[keep]).abs().max()) < 1e-4 * max(1.0, float(ref.abs().max()))
            gcat = torch.cat((dc.grad, rest.grad), dim=1).cpu().double()
            assert float((gcat - sh.grad).abs().max()) <= 1e-3 * float(sh.grad.abs().max())
            if degree > 0:
                assert float((d.grad.cpu().double() - dd.grad).abs().max()) <= 1e-3 * float(dd.grad.abs().max())


def test_split_sh_without_rest():
    """dc only (k_rest = 0, a degree-0 model): rest may be an empty tensor."""
    from b200gs import ops
    n = 300
    dirs, dc = torch.randn(n, 3, device=DEV), torch.randn(n, 1, 3, device=DEV, requires_grad=True)
    rest = torch.zeros(n, 0, 3, device=DEV, requires_grad=True)
    rgb = ops.spherical_harmonics_decomposed(0, dirs, dc, rest)
    rgb.sum().backward()
    assert torch.equal(rgb, ops.spherical_harmonics(0, dirs, dc.detach()))
    assert torch.allclose(dc.grad, torch.full_like(dc.grad, 0.28209479177387814))


def test_two_camera_projection_equals_two_single_calls():
    from b200gs.compat import gsplat_v1 as G
    from b200gs.scene import activate, make_ring_cameras, make_scene
    act = {k: v.to(DEV) for k, v in activate(make_scene(3000, 2, mean_scale=0.05)).items()}
    cams = [c.to_device(DEV) for c in make_ring_cameras(200, 150)[1:3]]
    viewmats = torch.stack([c.world_to_camera.T for c in cams])
    Ks = torch.tensor([[[float(c.fx), 0., float(c.cx)], [0., float(c.fy), float(c.cy)], [0., 0., 1.]] for c in cams], device=DEV)
    gen = torch.Generator().manual_seed(3)

    def params():
        return [act[k].clone().requires_grad_(True) for k in ("means", "rotations", "scales")]

    m, q, s = params()
    both = G.fully_fused_projection(m, None, q, s, viewmats, Ks, 200, 150, calc_compensations=True)
    cots = [torch.rand(t.shape, generator=gen).to(DEV) if t.dtype.is_floating_point else None for t in both]
    sum((t * c).sum() for t, c in zip(both, cots) if c is not None).backward()
    grads2 = [m.grad, q.grad, s.grad]
    acc = [0, 0, 0]
    for c in range(2):
        m1, q1, s1 = params()
        one = G.fully_fused_projection(m1, None, q1, s1, viewmats[c:c + 1], Ks[c:c + 1], 200, 150, calc_compensations=True)
        for t2, t1 in zip(both, one):
            assert torch.equal(t2[c:c + 1], t1)
        sum((t * cc[c:c + 1]).sum() for t, cc in zip(one, cots) if cc is not None).backward()
        acc = [a + p.grad for a, p in zip(acc, (m1, q1, s1))]
    for a, b in zip(acc, grads2):
        assert torch.equal(a, b)


def test_launch_count_of_the_new_kernels():
    """keys, offsets and split SH each add exactly one launch."""
    from b200gs import ops
    from b200gs._lib import lib
    from b200gs.compat import gsplat_v1 as G
    L = lib()
    xy, r, d = torch.rand(1, 100, 2, device=DEV) * 64, torch.full((1, 100), 5, dtype=torch.int32, device=DEV), torch.rand(1, 100, device=DEV) + 1
    b0 = ops.bin_gaussians(1, 64, 64, xy[0], d[0], r[0])
    n0 = L.b200gs_launch_count()
    keys = ops.isect_keys(b0, d[0])
    n1 = L.b200gs_launch_count()
    G.isect_offset_encode(keys, 1, 4, 4)
    n2 = L.b200gs_launch_count()
    ops.spherical_harmonics_decomposed(3, torch.randn(100, 3, device=DEV), torch.randn(100, 1, 3, device=DEV), torch.randn(100, 15, 3, device=DEV))
    torch.cuda.synchronize()
    assert (n1 - n0, n2 - n1, L.b200gs_launch_count() - n2) == (1, 1, 1)


# ---- GSplatAppearanceEmbeddingRenderer past warm-up (gsplat_appearance_embedding_renderer.py) ---------------------------------
def _appearance_golden():
    with open(os.path.join(GOLDEN, "dropin_v1_appearance.json")) as f:
        rec = json.load(f)
    return rec, torch.from_numpy(np.load(os.path.join(GOLDEN, "dropin_v1_appearance.npz"))["colors"])


def appearance_forward(g, cam, pc, bg, colors, block_size=16):
    """GSplatAppearanceEmbeddingRendererModule.forward past warm-up for the rgb render: GSplatV1RendererModule.forward (:137-287) with
    get_opacities -> _get_rgbs_and_opacities (:217-286).  The appearance MLP is the reference's torch code; its output colours, as
    recorded, come in as `colors` [N,3]."""
    viewmats = cam.world_to_camera.T.unsqueeze(0)
    Ks = torch.tensor([[[float(cam.fx), 0., float(cam.cx)], [0., float(cam.fy), float(cam.cy)], [0., 0., 1.]]], dtype=torch.float, device=DEV)
    img_width, img_height = int(cam.width), int(cam.height)
    radii, means2d, depths, conics, compensations = g["fully_fused_projection"](
        pc.get_means(), None, pc.get_rotations(), pc.get_scales(), viewmats=viewmats, Ks=Ks, width=img_width, height=img_height, eps2d=0.3,
        calc_compensations=True, packed=False, radius_clip=0.0, camera_model="pinhole")
    visibility_filter = radii.squeeze(0) > 0
    view_directions = torch.nn.functional.normalize(pc.get_xyz.detach()[visibility_filter] - cam.camera_center, dim=-1)
    base_rgbs = g["spherical_harmonics_decomposed"](pc.active_sh_degree, view_directions, dc=pc.get_shs_dc()[visibility_filter],
                                                    coeffs=pc.get_shs_rest()[visibility_filter]) + 0.5      # selective_sh (:204-215)
    opacities = pc.get_opacities().squeeze(-1).unsqueeze(0) * compensations
    tw, th = math.ceil(img_width / float(block_size)), math.ceil(img_height / float(block_size))
    _, isect_ids, flatten_ids = g["isect_tiles"](means2d, radii, depths, block_size, tw, th, packed=False, n_cameras=1, camera_ids=None,
                                                 gaussian_ids=None)
    isect_offsets = g["isect_offset_encode"](isect_ids, 1, tw, th)
    means2d = means2d.squeeze(0)
    img, alpha = g["rasterize_to_pixels"](means2d=means2d, conics=conics, colors=colors.unsqueeze(0), opacities=opacities, image_width=img_width,
                                          image_height=img_height, tile_size=block_size, isect_offsets=isect_offsets, flatten_ids=flatten_ids,
                                          backgrounds=bg.unsqueeze(0), absgrad=True)
    return {"render": img.squeeze(0).permute(2, 0, 1), "alpha": alpha.squeeze(0).squeeze(-1).unsqueeze(0), "viewspace_points": means2d,
            "visibility_filter": visibility_filter, "base_rgbs": base_rgbs, "view_directions": view_directions, "isect_ids": isect_ids}


def test_appearance_renderer_call_sequence_and_contract_shapes():
    rec, colors = _appearance_golden()
    raw, model, cam = _setup(rec["N"], rec["W"], rec["H"], 4, 2)
    log = []
    out = appearance_forward(_gsplat(log), cam, model, torch.tensor([0.1, 0.2, 0.3], device=DEV), colors.to(DEV))
    sizes = {"N": rec["N"], "H": rec["H"], "W": rec["W"], "I": int(out["isect_ids"].shape[0]), "V": int(out["visibility_filter"].sum())}
    assert [c[0] for c in log] == [c["fn"] for c in rec["calls"]]
    for (fn, args, kw, ret), c in zip(log, rec["calls"]):
        assert [_describe(a, sizes) for a in args] == [_concrete(a, sizes) for a in c["args"]], fn
        assert {k: _describe(v, sizes) for k, v in kw.items()} == {k: _concrete(v, sizes) for k, v in c["kwargs"].items()}, fn
        ret = ret if isinstance(ret, tuple) else (ret,)
        assert [_describe(r, sizes) for r in ret] == [_concrete(r, sizes) for r in c["returns"]], fn


def test_appearance_renderer_against_float64_oracle():
    """The render of the recorded MLP colours and every gradient (geometry and colours) against the float64 oracle with those colours
    as precomputed colours; the SH of the gathered visible rows (no mask) and its dc / rest gradients against O.eval_sh."""
    from b200gs.scene import activate, make_ring_cameras
    rec, colors = _appearance_golden()
    W, H = rec["W"], rec["H"]
    raw, model, cam = _setup(rec["N"], W, H, 4, 2)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    col = colors.to(DEV).requires_grad_(True)
    out = appearance_forward(_gsplat(), cam, model, bg, col)
    gen = torch.Generator().manual_seed(7)
    cot = torch.rand(3, H, W, generator=gen) * 2 - 1
    cot_sh = torch.rand(out["base_rgbs"].shape, generator=gen) * 2 - 1
    ((out["render"] * cot.to(DEV)).sum() + (out["base_rgbs"] * cot_sh.to(DEV)).sum()).backward()

    c = make_ring_cameras(W, H)[2]
    ov = O.make_view(c.R, c.T, float(c.fx), float(c.fy), float(c.cx), float(c.cy), W, H)
    leaves = {k: v.double().requires_grad_(True) for k, v in raw.items()}
    act = activate(leaves)
    col_d = colors.double().requires_grad_(True)
    margins = []
    ref = O.render(O.MODE_GSPLAT, act["means"], act["scales"], act["rotations"], act["opacities"], None, ov, bg.cpu().double(),
                   colors_precomp=col_d, margins=margins)
    vis = out["visibility_filter"].cpu()
    assert int(((ref["radii"] > 0) != vis).sum()) <= 1       # a radius within rounding of an integer may differ (test_gpu_parity.py)
    dirs = out["view_directions"].detach().cpu().double()
    ref_sh = O.eval_sh(3, act["shs"][vis], dirs) + 0.5
    ((ref["render"] * cot.double()).sum() + (ref_sh * cot_sh.double()).sum()).backward()
    err = (out["render"].detach().cpu().double() - ref["render"].detach()).abs().max(dim=0).values
    ambiguous = margins[0] < AMBIGUOUS
    assert int(((err > 1e-4) & ~ambiguous).sum()) == 0 and int(ambiguous.sum()) <= max(8, err.numel() // 20)
    assert float((out["base_rgbs"].detach().cpu().double() - ref_sh.detach()).abs().max()) < 1e-5 * max(1.0, float(ref_sh.abs().max()))
    assert float((col.grad.cpu().double() - col_d.grad).abs().max()) <= 1e-3 * float(col_d.grad.abs().max())
    for k, p in model.gaussians.items():
        gref = leaves[k].grad
        assert float((p.grad.cpu().double() - gref).abs().max()) <= 1e-3 * float(gref.abs().max()), k
    assert int(model.gaussians["shs_rest"].grad[~vis.to(DEV)].abs().sum()) == 0       # only the gathered rows get an SH gradient
