"""Drop-in evidence for the feature renderers: the calls the reference's own ``GSplatContrastiveFeatureRenderer`` (SegAnyGS; the
Feature3DGS renderer makes the same rasterize_gaussians call per 32-channel batch) makes to gsplat, replayed through
``b200gs.compat.gsplat_v0`` on the GPU, against the float64 oracle.

tests/golden/make_golden_feature_dropin.py ran the unmodified reference class on the CPU with recording stand-ins for gsplat, at
feature_map_width -1 and 256 (the rescaled intrinsics and image size of a reduced feature map), with 32-dimensional unit-norm
semantic features and the 32-entry zero background of SegAnySplatting.  The model is frozen, as SegAnySplatting freezes it: the
projection carries no gradient, the render takes the features-only backward, and only the features receive a gradient.
"""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import gs_oracle as O
from test_gpu_blend_channels import _assert_channels
from test_gpu_parity import _rel
import test_gpu_reference_dropin as T

pytestmark = pytest.mark.gpu
DEV = "cuda"
D = 32
FEATURE_MAP_WIDTHS = (-1, 256)


def semantic_features(n, dev):
    """SegAnySplatting.get_processed_semantic_features hands over unit-norm rows"""
    g = torch.Generator().manual_seed(17)
    return torch.nn.functional.normalize(torch.randn(n, D, generator=g), dim=-1).to(dev)


def replay(width, model, cam, bg, feats):
    """The recorded calls of one render through b200gs.compat.gsplat_v0.  -> (returned dict, args and kwargs of each call)"""
    from b200gs.compat import gsplat_v0
    with open(os.path.join(GOLDEN, "dropin_contrastive.json")) as f:
        rec = json.load(f)["renders"][str(width)]
    data = np.load(os.path.join(GOLDEN, "dropin_contrastive.npz"))
    outs, calls = [], []

    def names():
        d = T.named_tensors(model, cam, bg, outs)
        d["semantic_features"] = feats
        return d

    def value(a, nm):
        if "ref" in a:
            return nm[a["ref"]]
        if "data" in a:
            return torch.from_numpy(data[a["data"]]).to(DEV)
        return a["value"]

    for call in rec["calls"]:
        nm = names()
        args = [value(a, nm) for a in call["args"]]
        kw = {k: value(a, nm) for k, a in call["kwargs"].items()}
        out = getattr(gsplat_v0, call["fn"])(*args, **kw)
        outs.append(tuple(out) if isinstance(out, (tuple, list)) else (out,))
        calls.append((call["fn"], args, kw))
    nm = names()
    return {k: (None if a is None else value(a, nm)) for k, a in rec["returns"].items()}, calls


def _tile_lists(xy, depth, radii, w, h):
    """gsplat's full tile rects (min = int((p - r)/16), max = int((p + r)/16) + 1, clamped), depth-sorted per tile"""
    gx, gy = (w + 15) // 16, (h + 15) // 16
    r = radii.float()
    rmin = torch.stack([((xy[:, 0] - r) / 16).int().clamp(0, gx), ((xy[:, 1] - r) / 16).int().clamp(0, gy)], dim=1)
    rmax = torch.stack([((xy[:, 0] + r) / 16).int().add(1).clamp(0, gx), ((xy[:, 1] + r) / 16).int().add(1).clamp(0, gy)], dim=1)
    tiles = ((rmax - rmin).prod(dim=1) * (radii > 0)).int()
    keys, ids = O.build_sort_keys(depth, rmin, rmax, tiles, gx)
    _, sids, ranges = O.sort_and_ranges(keys, ids, gx * gy)
    return sids, ranges


@pytest.mark.parametrize("width", FEATURE_MAP_WIDTHS)
def test_reference_contrastive_feature_renderer_runs_on_b200gs(width):
    raw, model, cam = T.setup(DEV)
    for p in model.gaussians.values():
        p.requires_grad_(False)
    feats = semantic_features(raw["means"].shape[0], DEV).requires_grad_(True)
    bg = torch.zeros(D, device=DEV)
    out, calls = replay(width, model, cam, bg, feats)
    assert [c[0] for c in calls] == ["project_gaussians", "rasterize_gaussians"]
    h, w = (T.H, T.W) if width < 0 else (int(width * T.H / T.W), width)
    img = out["render"]
    assert img.shape == (D, h, w)
    assert torch.equal(out["visibility_filter"], out["radii"] > 0) and int(out["radii"].gt(0).sum()) > 0
    assert out["viewspace_points_grad_scale"] == 0.5 * max(h, w)
    assert not out["viewspace_points"].requires_grad            # frozen geometry: nothing to differentiate in the projection
    cot = (torch.rand(D, h, w, generator=torch.Generator().manual_seed(3)) * 2 - 1).to(DEV)
    (img * cot).sum().backward()
    assert all(p.grad is None for p in model.gaussians.values())

    # the float64 oracle on the rasterize call's own (fp32) inputs
    _, args, kw = calls[1]
    xys, depths, radii, conics, _, colors, opac = (a.detach().cpu() for a in args[:7])
    assert colors.shape == (xys.shape[0], D) and kw["background"].shape == (D,) and (kw["img_height"], kw["img_width"]) == (h, w)
    sids, ranges = _tile_lists(xys, depths, radii, w, h)
    f64 = feats.detach().cpu().double().requires_grad_(True)
    margins = []
    ref_img, ref_alpha, _ = O.blend(O.MODE_GSPLAT, xys.double(), conics.double(), opac.reshape(-1).double(), f64, sids, ranges,
                                    bg.cpu().double(), w, h, margins=margins)
    (ref_img * cot.cpu().double()).sum().backward()
    _assert_channels(img, ref_img.detach(), margins[0], f"contrastive feature_map_width={width}")
    assert _rel(feats.grad, f64.grad) < 1e-3, f"feature gradient {_rel(feats.grad, f64.grad):.3e}"
