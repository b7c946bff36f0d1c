"""Record what the reference's GSplatContrastiveFeatureRenderer (SegAnyGS, internal/renderers/gsplat_contrastive_feature_renderer.py)
hands to gsplat, for tests/test_gpu_feature_dropin.py:
    python tests/golden/make_golden_feature_dropin.py <reference checkout>   -> tests/golden/dropin_contrastive.{json,npz}

Runs GSplatContrastiveFeatureRenderer.forward unmodified on the CPU, at feature_map_width -1 (the camera's size) and 256 (the
rescaled feature map), with the reference's own VanillaGaussian model and Cameras, 32-dimensional unit-norm semantic features
(what SegAnySplatting.get_processed_semantic_features hands over) and its 32-entry zero background, while ``gsplat`` is the
recording stand-in of make_golden_dropin.py.  The features are named (tests/test_gpu_feature_dropin.py rebuilds them from a
seed), not stored."""
import json
import math
import os
import sys

import numpy as np
import torch

import make_golden_dropin as G   # noqa: E402  (puts the repository, tests/ and the reference checkout on sys.path)
import test_gpu_feature_dropin as F  # noqa: E402
import test_gpu_reference_dropin as T  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


class FeatureRecorder(G.Recorder):
    def __init__(self, model, cam, bg, feats):
        super().__init__(model, cam, bg)
        self.feats = feats

    def describe(self, a):
        if torch.is_tensor(a) and a.shape == self.feats.shape and torch.equal(a.detach(), self.feats):
            return {"ref": "semantic_features"}
        return super().describe(a)


def rasterize_gaussians(*args, **kw):
    """the stand-in of gsplat.rasterize.rasterize_gaussians at the size the renderer asks for (the feature map may be rescaled)"""
    img = G.rnd(kw["img_height"], kw["img_width"], args[5].shape[-1])
    out = (img, G.rnd(kw["img_height"], kw["img_width"])) if kw.get("return_alpha") else (img,)
    G.R.record("rasterize_gaussians", args, kw, out)
    return out if kw.get("return_alpha") else img


def main():
    G.install_stubs()
    sys.modules["gsplat.rasterize"].rasterize_gaussians = rasterize_gaussians
    from internal.cameras.cameras import Cameras
    from internal.models.vanilla_gaussian import VanillaGaussian
    from internal.renderers.gsplat_contrastive_feature_renderer import GSplatContrastiveFeatureRenderer
    from b200gs.scene import ring_pose

    raw, ours, our_cam = T.setup("cpu")
    model = VanillaGaussian(sh_degree=3).instantiate()
    model.setup_from_tensors({k: v.clone() for k, v in raw.items()})
    model.active_sh_degree = 3
    rot, trans = ring_pose(T.POSE)
    fx = 0.5 * T.W / math.tan(math.radians(39.6) * 0.5)
    cam = Cameras(R=rot[None], T=trans[None], fx=torch.tensor([fx]), fy=torch.tensor([fx]), cx=torch.tensor([T.W / 2.0]),
                  cy=torch.tensor([T.H / 2.0]), width=torch.tensor([T.W], dtype=torch.int32),
                  height=torch.tensor([T.H], dtype=torch.int32), appearance_id=torch.zeros(1, dtype=torch.int32),
                  normalized_appearance_id=torch.zeros(1), distortion_params=None,
                  camera_type=torch.zeros(1, dtype=torch.int32))[0]
    feats = F.semantic_features(raw["means"].shape[0], "cpu")
    bg = torch.zeros(F.D)                                   # SegAnySplatting.bg_color
    renders, data = {}, {}
    for width in F.FEATURE_MAP_WIDTHS:
        G.R = FeatureRecorder(ours, our_cam, bg, feats)
        returned = GSplatContrastiveFeatureRenderer(feature_map_width=width)(cam, model, bg, semantic_features=feats)
        rets = {k: (None if v is None else G.R.describe(v)) for k, v in returned.items()}
        prefix = f"w{width}_"
        for call in G.R.calls:
            for a in list(call["args"]) + list(call["kwargs"].values()):
                if "data" in a:
                    a["data"] = prefix + a["data"]
        data.update({prefix + k: v for k, v in G.R.data.items()})
        renders[str(width)] = {"calls": G.R.calls, "returns": rets}
        print(width, [c["fn"] for c in G.R.calls], "stored:", {k: v.shape for k, v in G.R.data.items()})
    with open(os.path.join(HERE, "dropin_contrastive.json"), "w") as f:
        json.dump({"renders": renders}, f, separators=(",", ":"))
    np.savez_compressed(os.path.join(HERE, "dropin_contrastive.npz"), **data)


if __name__ == "__main__":
    main()
