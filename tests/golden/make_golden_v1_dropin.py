"""Record the gsplat-v1 calls of the reference's own GSplatV1Renderer, for tests/test_gpu_v1_dropin.py and
tests/test_v1_dropin_abi_cpu.py:
    python tests/golden/make_golden_v1_dropin.py <reference checkout>   -> tests/golden/dropin_v1.json, dropin_v1_appearance.{json,npz}

Runs GSplatV1Renderer (internal/renderers/gsplat_v1_renderer.py) unmodified on the CPU, with the reference's own VanillaGaussian
model and Cameras, for separate_sh in {False, True} x tile_based_culling in {False, True} and every render type the renderer
composites in one or several rasterize calls.  The gsplat names it imports are recording stand-ins that return random tensors of
the contract's shapes.  For each render the file stores the sequence of calls: function, positional and keyword arguments
(tensors as shape with N / H / W / I for the Gaussian count, image size and pair count, dtype and requires_grad; other
values as they are), and the shapes of what the reference then reads from the returns.  It also stores every
(module, attribute) the reference imported from gsplat, viser and lightning.

It then records GSplatAppearanceEmbeddingRenderer past warm-up on the reference's AppearanceFeatureGaussian model (the same
tensors plus seeded appearance features, 4 appearances, seeded MLP weights): its call sequence, with V for the number of
Gaussians the projection stand-in marks visible, and the colours its appearance MLP hands to rasterize_to_pixels."""
import inspect
import json
import math
import os
import sys
import types
import typing

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, sys.argv[1]]

N, W, H, POSE, SEED, I = 300, 80, 56, 2, 4, 37      # I: the pair count the isect stand-ins return
RENDER_TYPES = ["rgb", "alpha", "acc_depth", "normal", "exp_depth", "inverse_depth", "hard_depth"]
gen = torch.Generator().manual_seed(0)
imported = []
calls = []
colors = []     # the colours each rasterize_to_pixels call received


V = None       # the number of Gaussians the projection stand-in marks visible (rows of the appearance renderer's gathered SH call)


def sym(d):
    return {N: "N", H: "H", W: "W", I: "I", V: "V"}.get(int(d), int(d))


def describe(a):
    if torch.is_tensor(a):
        return {"shape": [sym(d) for d in a.shape], "dtype": str(a.dtype).replace("torch.", ""), "grad": bool(a.requires_grad)}
    if isinstance(a, (tuple, list)):
        return {"seq": [describe(x) for x in a]}
    return {"value": a}


def record(fn, args, kwargs, out):
    outs = out if isinstance(out, tuple) else (out,)
    calls.append({"fn": fn, "args": [describe(a) for a in args], "kwargs": {k: describe(v) for k, v in kwargs.items()},
                  "returns": [describe(o) for o in outs]})
    return out


def rnd(*shape):
    return torch.rand(*shape, generator=gen) + 0.5


def bound(fn, args, kw):
    """The arguments of a gsplat call by name (the stand-ins record them exactly as passed)."""
    return inspect.signature(fn).bind(*args, **kw).arguments


def _ffp(means, covars, quats, scales, viewmats, Ks, width, height, **kw):
    pass


def fully_fused_projection(*args, **kw):
    a = bound(_ffp, args, kw)
    c, n = a["viewmats"].shape[0], a["means"].shape[0]
    out = (torch.randint(0, 3, (c, n), generator=gen, dtype=torch.int32), rnd(c, n, 2).requires_grad_(), rnd(c, n), rnd(c, n, 3), rnd(c, n))
    global V
    V = int((out[0] > 0).sum())
    assert V not in (N, H, W, I)
    return record("fully_fused_projection", args, kw, out)


def _isect_out(means2d, tile_width, tile_height):
    ids = torch.sort(torch.randint(0, tile_width * tile_height, (I,), generator=gen).long() << 32).values
    return torch.ones(1, means2d.shape[1], dtype=torch.int32), ids, torch.randint(0, means2d.shape[1], (I,), generator=gen, dtype=torch.int32)


def _it(means2d, radii, depths, tile_size, tile_width, tile_height, **kw):
    pass


def _itc(means2d, radii, depths, conics, opacities, tile_size, tile_width, tile_height, **kw):
    pass


def isect_tiles(*args, **kw):
    a = bound(_it, args, kw)
    return record("isect_tiles", args, kw, _isect_out(a["means2d"], a["tile_width"], a["tile_height"]))


def isect_tiles_tile_based_culling(*args, **kw):
    a = bound(_itc, args, kw)
    return record("isect_tiles_tile_based_culling", args, kw, _isect_out(a["means2d"], a["tile_width"], a["tile_height"]))


def isect_offset_encode(isect_ids, n_cameras, tile_width, tile_height):
    out = torch.zeros(n_cameras, tile_height, tile_width, dtype=torch.int32)
    return record("isect_offset_encode", (isect_ids, n_cameras, tile_width, tile_height), {}, out)


def isect_offset_encode_tile_based_culling(isect_ids, flatten_ids, n_cameras, tile_width, tile_height):
    out = (torch.zeros(n_cameras, tile_height, tile_width, dtype=torch.int32), flatten_ids)
    return record("isect_offset_encode_tile_based_culling", (isect_ids, flatten_ids, n_cameras, tile_width, tile_height), {}, out)


def spherical_harmonics(*args, **kw):
    return record("spherical_harmonics", args, kw, rnd(args[1].shape[0], 3))


def spherical_harmonics_decomposed(*args, **kw):
    # SH values around 0 (the renderers add 0.5), so the appearance MLP's colours spread over [0, 1] instead of clamping
    return record("spherical_harmonics_decomposed", args, kw, torch.rand(args[1].shape[0], 3, generator=gen) * 0.6 - 0.3)


def rasterize_to_pixels(**kw):
    colors.append(kw["colors"].detach().clone())
    kw["means2d"].has_hit_any_pixels = torch.ones(kw["means2d"].shape[0], dtype=torch.bool)
    out = (rnd(1, kw["image_height"], kw["image_width"], kw["colors"].shape[-1]), rnd(1, kw["image_height"], kw["image_width"], 1))
    return record("rasterize_to_pixels", (), kw, out)


class Recording(types.ModuleType):
    """A stand-in module that logs every name imported from it."""

    def __init__(self, name, **attrs):
        super().__init__(name)
        self._attrs = attrs

    def __getattr__(self, nm):
        attrs = self.__dict__.get("_attrs", {})
        if nm.startswith("__") or nm not in attrs:
            raise AttributeError(nm)
        if (self.__name__, nm) not in imported:
            imported.append((self.__name__, nm))
        return attrs[nm]


def install_stubs():
    torch.Any = typing.Any      # gsplat_appearance_embedding_renderer.py:347 annotates with torch.Any
    for name, attrs in (
            ("gsplat", {}), ("gsplat.cuda", {}),
            ("gsplat.cuda._wrapper", dict(fully_fused_projection=fully_fused_projection, isect_offset_encode=isect_offset_encode,
                                          isect_tiles=isect_tiles, spherical_harmonics=spherical_harmonics)),
            ("gsplat.sh_decomposed", dict(spherical_harmonics_decomposed=spherical_harmonics_decomposed)),
            ("gsplat.cuda.isect_tiles_tile_based_culling", dict(isect_tiles_tile_based_culling=isect_tiles_tile_based_culling,
                                                                isect_offset_encode_tile_based_culling=isect_offset_encode_tile_based_culling)),
            ("gsplat.v0_interfaces", dict(rasterize_to_pixels=rasterize_to_pixels)),
            ("viser", dict(ViserServer=type("ViserServer", (), {}))),
            ("lightning", dict(LightningModule=type("LightningModule", (), {}))),
            ("diff_gaussian_rasterization", dict(GaussianRasterizationSettings=object, GaussianRasterizer=object))):
        m = Recording(name, **attrs)
        if name == "gsplat" or name == "gsplat.cuda":
            m.__path__ = []
        sys.modules[name] = m


def reference_camera(Cameras):
    from b200gs.scene import ring_pose
    rot, trans = ring_pose(POSE)
    fx = 0.5 * W / math.tan(math.radians(39.6) * 0.5)
    return Cameras(R=rot[None], T=trans[None], fx=torch.tensor([fx]), fy=torch.tensor([fx]), cx=torch.tensor([W / 2.0]),
                   cy=torch.tensor([H / 2.0]), width=torch.tensor([W], dtype=torch.int32), height=torch.tensor([H], dtype=torch.int32),
                   appearance_id=torch.zeros(1, dtype=torch.int32), normalized_appearance_id=torch.zeros(1), distortion_params=None,
                   camera_type=torch.zeros(1, dtype=torch.int32))[0]


def main():
    install_stubs()
    from internal.cameras.cameras import Cameras
    from internal.models.appearance_feature_gaussian import AppearanceFeatureGaussian
    from internal.models.vanilla_gaussian import VanillaGaussian
    from internal.renderers.gsplat_appearance_embedding_renderer import GSplatAppearanceEmbeddingRenderer, ModelConfig
    from internal.renderers.gsplat_v1_renderer import GSplatV1Renderer
    from b200gs.scene import make_scene

    raw = make_scene(N, SEED, mean_scale=0.05)
    model = VanillaGaussian(sh_degree=3).instantiate()
    model.setup_from_tensors({k: v.clone() for k, v in raw.items()})
    model.active_sh_degree = 3
    cam = reference_camera(Cameras)
    bg = torch.tensor([0.1, 0.2, 0.3])
    renders = {}
    for separate_sh in (False, True):
        for culling in (False, True):
            calls.clear()
            r = GSplatV1Renderer(separate_sh=separate_sh, tile_based_culling=culling).instantiate()
            out = r(cam, model, bg, render_types=RENDER_TYPES)
            renders[f"sh{int(separate_sh)}_cull{int(culling)}"] = {
                "calls": list(calls), "outputs": {k: describe(v) for k, v in out.items() if torch.is_tensor(v)}}
    with open(os.path.join(HERE, "dropin_v1.json"), "w") as f:
        json.dump({"N": N, "W": W, "H": H, "I": I, "render_types": RENDER_TYPES, "imported": imported, "renders": renders}, f,
                  separators=(",", ":"))
    print({k: [c["fn"] for c in v["calls"]] for k, v in renders.items()}, imported)

    # GSplatAppearanceEmbeddingRenderer past warm-up: colours from its appearance MLP (4 appearances, seeded weights) on the
    # model's appearance features, the SH of the visible rows gathered and evaluated without a mask (selective_sh)
    torch.manual_seed(SEED)
    app_model = AppearanceFeatureGaussian(sh_degree=3, appearance_feature_init_type="normal").instantiate()
    app_model.setup_from_tensors({**{k: v.clone() for k, v in raw.items()},
                                  "appearance_features": torch.randn(N, 64, generator=torch.Generator().manual_seed(SEED))})
    app_model.active_sh_degree = 3
    renderer = GSplatAppearanceEmbeddingRenderer(model=ModelConfig(n_appearances=4)).instantiate()
    renderer._setup_model()
    renderer.eval()
    calls.clear()
    colors.clear()
    out = renderer(cam, app_model, bg, warm_up=False)
    assert len(colors) == 1 and colors[0].shape == (1, N, 3)
    with open(os.path.join(HERE, "dropin_v1_appearance.json"), "w") as f:
        json.dump({"N": N, "W": W, "H": H, "I": I, "V": V, "calls": list(calls), "imported": imported,
                   "outputs": {k: describe(v) for k, v in out.items() if torch.is_tensor(v)}}, f, separators=(",", ":"))
    np.savez_compressed(os.path.join(HERE, "dropin_v1_appearance.npz"), colors=colors[0][0].numpy())
    print("appearance", [c["fn"] for c in calls], "V =", V)


if __name__ == "__main__":
    main()
