"""Record the reference's own appearance network and colour epilogue at network shapes other than the default, for
tests/test_appearance_shapes_cpu.py and tests/test_gpu_appearance_shapes.py:
    python tests/golden/make_golden_appearance_shapes.py <reference checkout>   -> tests/golden/appearance_shapes.npz

Runs, on the CPU and unmodified, Model (internal/renderers/gsplat_appearance_embedding_renderer.py:50-93) on compact rows and
GSplatAppearanceEmbeddingRendererModule._get_rgbs_and_opacities (:239-295) on dense rows with a visibility mask, as
make_golden_appearance.py does, for the configurations in oracle.appearance_oracle.SHAPES: 128 neurons, 2 and 4 layers, a 32- and an 8-wide feature, 0 and
6 view-direction frequencies, with and without opacity and normalisation.  The parameters and inputs are not stored: they are
rebuilt from a deterministic sequence by oracle.appearance_oracle.shape_state / shape_inputs (weights are nn.Linear's range times 2,
so the sigmoids leave 0.5; the base colours span [-0.9, 0.9] and the raw opacities [0, 1), so both colour clamps and the opacity
clamp are active) and loaded into the reference's model.  Stored per configuration: the renderer's state_dict keys, the sum of
each parameter (the rebuilt state is the one recorded), every output and v_base, and the entries of sample_index of v_features
and of each parameter gradient."""
import math
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_v1_dropin as stubs  # noqa: E402  (puts the repository and the reference checkout on sys.path)

N_APPEARANCES, APPEARANCE_ID = 4, 2


def main():
    stubs.install_stubs()
    import internal.renderers.gsplat_appearance_embedding_renderer as R
    from oracle.appearance_oracle import SHAPE_ROWS as N, SHAPES, network_shape, sample_index, shape_inputs, shape_state

    out = {}
    appearance = torch.tensor([APPEARANCE_ID], dtype=torch.int32)
    for name, (kw, seed) in SHAPES.items():
        feat_dim, n_freq, n_neurons, n_layers, n_out = network_shape(kw)
        x = shape_inputs(N, feat_dim, seed)
        mask = x["mask"]
        camera = types.SimpleNamespace(camera_center=x["cam_center"], appearance_id=appearance)
        renderer = R.GSplatAppearanceEmbeddingRenderer(model=R.ModelConfig(n_appearances=N_APPEARANCES, **kw)).instantiate()
        renderer._setup_model()
        model = renderer.model
        model.load_state_dict(shape_state(feat_dim, n_freq, n_neurons, n_layers, n_out, seed=seed), strict=True)
        out[f"{name}.keys"] = np.array(list(renderer.state_dict().keys()))
        out[f"{name}.state_sums"] = np.array([math.fsum(v.double().flatten().tolist()) for v in model.state_dict().values()])

        # Model.forward on the compact rows
        feats = x["features"][mask].clone().requires_grad_(True)
        dirs = torch.nn.functional.normalize(x["means"][mask] - x["cam_center"], dim=-1)
        y = model(feats, appearance, dirs)
        (y * x["cot_model"][mask][:, :y.shape[1]]).sum().backward()
        out[f"{name}.model.out"] = y.detach().numpy()
        out[f"{name}.model.v_features"] = feats.grad.numpy().reshape(-1)[sample_index(feats.numel())]
        for k, p in model.named_parameters():
            out[f"{name}.model.grad.{k}"] = p.grad.numpy().reshape(-1)[sample_index(p.numel())]
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
        out[f"{name}.colors.v_features"] = feats.grad.numpy().reshape(-1)[sample_index(feats.numel())]
        out[f"{name}.colors.v_base"] = base.grad.numpy()
        if offsets is not None:
            out[f"{name}.colors.opacities"] = opacities.detach().numpy()
            out[f"{name}.colors.offsets"] = offsets.detach().numpy()          # compact: the rows of the mask
            out[f"{name}.colors.v_raw_opacity"] = raw.grad.numpy()
        for k, p in model.named_parameters():
            out[f"{name}.colors.grad.{k}"] = p.grad.numpy().reshape(-1)[sample_index(p.numel())]

        # a colour or an opacity sum within float32 round-off of a clamp bound could fall on either side: none may
        pre = x["base"][mask].double() + 0.5 + (y.detach()[:, :3].double() * 2 - 1)
        assert bool((pre < 0).any()) and bool((pre > 1).any()), name
        assert float(torch.minimum(pre.abs(), (pre - 1).abs()).min()) > 1e-4, name
        if offsets is not None:
            assert float(((x["raw_opacity"][mask].double() + y.detach()[:, 3].double()) - 1).abs().min()) > 1e-4, name
        print(name, "V =", int(mask.sum()), "clamped at 0:", int((pre < 0).sum()), "at 1:", int((pre > 1).sum()))
    np.savez_compressed(os.path.join(HERE, "appearance_shapes.npz"), **out)


if __name__ == "__main__":
    main()
