"""Record the reference's own appearance network and colour epilogue, for tests/test_appearance_oracle_cpu.py and
tests/test_gpu_appearance.py:
    python tests/golden/make_golden_appearance.py <reference checkout>   -> tests/golden/appearance.npz

Runs, on the CPU and unmodified, Model (internal/renderers/gsplat_appearance_embedding_renderer.py:50-93) on compact rows and
GSplatAppearanceEmbeddingRendererModule._get_rgbs_and_opacities (:239-295) on dense rows with a visibility mask, for five
configurations: the default, is_view_dependent, normalize, with_opacity and a 128-dim embedding.  The gsplat imports are the
stand-ins of make_golden_v1_dropin.py; the renderer's SH call returns the rows of a seeded `base` tensor, so its gradient is
recorded too.  Weights are nn.Linear's seeded initialisation times 2 (so the sigmoids leave 0.5), the base colours span
[-0.9, 0.9] (both clamps of the colour are active) and the raw opacities [0, 1] (so is the opacity's).  The file holds the shared
inputs and cotangents and, per configuration, the state_dict, every output and every gradient."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_v1_dropin as stubs  # noqa: E402  (puts the repository and the reference checkout on sys.path)

N, F_DIM, N_APPEARANCES, APPEARANCE_ID, SEED = 96, 64, 4, 2, 11
VARIANTS = {
    "default": {},
    "view_dependent": {"is_view_dependent": True},
    "normalize": {"normalize": True},
    "with_opacity": {"with_opacity": True},
    "embedding128": {"n_appearance_embedding_dims": 128},
}


def inputs():
    g = torch.Generator().manual_seed(SEED)
    return {
        "features": torch.randn(N, F_DIM, generator=g),
        "mask": torch.rand(N, generator=g) < 0.66,
        "means": torch.randn(N, 3, generator=g) * 2,
        "cam_center": torch.tensor([0.3, -4.0, 1.5]),
        "base": torch.rand(N, 3, generator=g) * 1.8 - 0.9,
        "raw_opacity": torch.rand(N, generator=g),
        "cot_model": torch.randn(N, 4, generator=g),          # rows of the mask, first 3 | 4 columns
        "cot_rgbs": torch.randn(N, 3, generator=g),
        "cot_opacities": torch.randn(N, generator=g),
        "cot_offsets": torch.randn(N, generator=g),
    }


def main():
    stubs.install_stubs()
    import internal.renderers.gsplat_appearance_embedding_renderer as R

    x = inputs()
    mask = x["mask"]
    out = {f"in.{k}": v.numpy() for k, v in x.items()}
    appearance = torch.tensor([APPEARANCE_ID], dtype=torch.int32)
    camera = types.SimpleNamespace(camera_center=x["cam_center"], appearance_id=appearance)
    for name, kw in VARIANTS.items():
        torch.manual_seed(SEED)
        renderer = R.GSplatAppearanceEmbeddingRenderer(model=R.ModelConfig(n_appearances=N_APPEARANCES, **kw)).instantiate()
        renderer._setup_model()
        model = renderer.model
        with torch.no_grad():
            for k, p in model.named_parameters():
                if k.endswith("weight") and "network" in k:
                    p.mul_(2.0)
        out[f"{name}.keys"] = np.array(list(renderer.state_dict().keys()))
        for k, v in model.state_dict().items():
            out[f"{name}.state.{k}"] = v.numpy().copy()

        # Model.forward on the compact rows
        feats = x["features"][mask].clone().requires_grad_(True)
        dirs = torch.nn.functional.normalize(x["means"][mask] - x["cam_center"], dim=-1)
        y = model(feats, appearance, dirs)
        (y * x["cot_model"][mask][:, :y.shape[1]]).sum().backward()
        out[f"{name}.model.out"] = y.detach().numpy()
        out[f"{name}.model.v_features"] = feats.grad.numpy()
        for k, p in model.named_parameters():
            out[f"{name}.model.grad.{k}"] = p.grad.numpy().copy()
        model.zero_grad()

        # the renderer's colours and opacities on the dense rows
        feats = x["features"].clone().requires_grad_(True)
        base = x["base"].clone().requires_grad_(True)
        raw = x["raw_opacity"].clone().requires_grad_(True)
        R.spherical_harmonics_decomposed = lambda deg, dirs, dc, coeffs, masks=None: base[mask]
        pc = types.SimpleNamespace(get_opacities=lambda: raw.unsqueeze(-1), get_xyz=x["means"], is_pre_activated=False, active_sh_degree=3,
                                   get_shs_dc=lambda: torch.zeros(N, 1, 3), get_shs_rest=lambda: torch.zeros(N, 15, 3),
                                   get_appearance_features=lambda: feats, n_gaussians=N)
        rgbs, opacities, offsets = renderer._get_rgbs_and_opacities(camera, pc, (None, torch.zeros(N, 2)), mask, None)
        loss = (rgbs * x["cot_rgbs"]).sum()
        if offsets is not None:
            loss = loss + (opacities * x["cot_opacities"]).sum() + (offsets * x["cot_offsets"][mask]).sum()
        loss.backward()
        out[f"{name}.colors.rgbs"] = rgbs.detach().numpy()
        out[f"{name}.colors.v_features"] = feats.grad.numpy()
        out[f"{name}.colors.v_base"] = base.grad.numpy()
        if offsets is not None:
            out[f"{name}.colors.opacities"] = opacities.detach().numpy()
            out[f"{name}.colors.offsets"] = offsets.detach().numpy()          # compact: the rows of the mask
            out[f"{name}.colors.v_raw_opacity"] = raw.grad.numpy()
        for k, p in model.named_parameters():
            out[f"{name}.colors.grad.{k}"] = p.grad.numpy().copy()
        pre = x["base"][mask] + 0.5 + (y.detach()[:, :3] * 2 - 1)
        print(name, "V =", int(mask.sum()), "clamped at 0:", int((pre < 0).sum()), "at 1:", int((pre > 1).sum()))
    np.savez_compressed(os.path.join(HERE, "appearance.npz"), **out)


if __name__ == "__main__":
    main()
