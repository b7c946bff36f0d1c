"""The float64 exposure oracle (oracle/exposure_oracle.py) against the reference's unmodified ExposureProcessorModule
(tests/golden/exposure.npz, made by tests/golden/make_golden_exposure.py); the b200gs.exposure plug-in's config fields and defaults,
state_dict keys, initial values and optimizer groups against the recorded ones."""
import dataclasses
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import exposure_oracle as O

Z = np.load(os.path.join(GOLDEN, "exposure.npz"))
META = json.load(open(os.path.join(GOLDEN, "exposure.json")))


def case_inputs(case):
    H, W = case["image"]
    return O.inputs(H, W, case["with_bias"], case["shade_correction_size"] if case["shade_correction"] else 0, case["seed"],
                    META["n_appearances"])


@pytest.mark.parametrize("case", META["cases"], ids=lambda c: c["key"])
def test_oracle_matches_the_reference_module(case):
    render, params, shade, v_out = case_inputs(case)
    k = case["key"]
    out, v_render, v_params, v_shade = O.vjp(render, params, case["appearance_id"], shade, v_out, with_bias=case["with_bias"])
    assert np.abs(out - Z[f"{k}_out"]).max() <= 1e-5
    assert np.abs(v_render - Z[f"{k}_v_render"]).max() <= 1e-5 * np.abs(v_render).max()
    row = case["appearance_id"]
    assert np.abs(v_params[row] - Z[f"{k}_v_params"][row]).max() <= 1e-4 * np.abs(v_params[row]).max()
    others = [i for i in range(params.shape[0]) if i != row]
    assert not v_params[others].any() and not Z[f"{k}_v_params"][others].any()
    if case["shade_correction"]:
        assert np.abs(v_shade - Z[f"{k}_v_shade"]).max() <= 1e-4 * np.abs(v_shade).max()
    else:
        assert f"{k}_v_shade" not in Z


def test_inputs_cover_the_clamp_and_gamma_ranges():
    """Across the recorded cases: scaled pixels below 0, above 1 and exactly on 0 and on 1, and gammas below and above 1."""
    below = above = zero = one = 0
    gammas = set()
    for case in META["cases"]:
        render, params, shade, _ = case_inputs(case)
        a = torch.sigmoid(torch.from_numpy(params[case["appearance_id"]]))
        x = a[:3, None, None] * 5.0 * torch.from_numpy(render)
        if shade is not None:
            x = x * O.shade_map(torch.from_numpy(shade[0]).double(), *render.shape[1:]).float()
        if case["with_bias"]:
            x = x + (a[3:6, None, None] * 2. - 1.)
        below, above = below + int((x < 0).sum()), above + int((x > 1).sum())
        zero, one = zero + int((x == 0).sum()), one + int((x == 1).sum())
        gammas.add(float(a[-1]) * 5.0)
    assert below > 0 and above > 0 and zero > 0 and one > 0
    assert min(gammas) < 1 < max(gammas)
    assert {c["appearance_id"] for c in META["cases"]} >= {0, META["n_appearances"] - 1}


def test_size_one_axes_follow_torch():
    """An image one pixel tall or wide samples the map's first row or column (torch's source scale 0), which F.interpolate
    confirms in float64."""
    shade0 = torch.from_numpy(O.inputs(3, 3, False, 9, 5)[2][0]).double()
    M = torch.sigmoid(shade0)
    M = M / M.max()
    for H, W in ((1, 17), (13, 1), (1, 1), (40, 31)):
        ref = torch.nn.functional.interpolate(M[None, None], size=(H, W), mode="bilinear", align_corners=True)[0, 0]
        assert torch.allclose(O.shade_map(shade0, H, W), ref, rtol=0, atol=1e-12)


def test_config_fields_and_defaults_match_the_reference():
    from b200gs.exposure import B200ExposureProcessor
    assert {f.name: f.default for f in dataclasses.fields(B200ExposureProcessor)} == META["config"]
    with pytest.raises(AssertionError):
        B200ExposureProcessor(max_gray_scale=1.0).instantiate()
    with pytest.raises(AssertionError):
        B200ExposureProcessor(max_gamma=0.5).instantiate()


@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("shade", [False, True])
def test_state_dict_initial_values_and_optimizer_match_the_reference(with_bias, shade):
    from b200gs.exposure import B200ExposureProcessor
    k = f"b{int(with_bias)}_c{int(shade)}"
    proc = B200ExposureProcessor(with_bias=with_bias, shade_correction=shade, shade_correction_size=16).instantiate()
    proc.init_exposures(META["n_appearances"], "cpu")
    sd = proc.state_dict()
    assert {n: {"shape": list(v.shape), "dtype": str(v.dtype)} for n, v in sd.items()} == META["state_dict"][k]
    for n, v in sd.items():
        assert torch.equal(v, torch.from_numpy(Z[f"sd_{k}_{n}"]))
    # a reference checkpoint loads, re-initialising to its number of appearances
    ckpt = {n: torch.from_numpy(Z[f"sd_{k}_{n}"])[:3].clone() if n == "exposure_parameters" else torch.from_numpy(Z[f"sd_{k}_{n}"])
            for n in sd}
    other = B200ExposureProcessor(with_bias=with_bias, shade_correction=shade, shade_correction_size=16).instantiate()
    other.load_state_dict(ckpt)
    assert other.exposure_parameters.shape[0] == 3 and torch.equal(other.exposure_parameters, ckpt["exposure_parameters"])
    opt, sched = proc.training_setup(None)
    rec = META["training_setup"][k]
    assert (type(opt).__name__, type(sched).__name__) == (rec["optimizer"], rec["scheduler"])
    got = [{"name": g["name"], "lr": g["lr"], "shapes": [list(p.shape) for p in g["params"]], "betas": list(g["betas"]),
            "eps": g["eps"]} for g in opt.param_groups]
    assert got == rec["groups"]
    lrs = [[g["initial_lr"] * sched.lr_lambdas[0](it) for g in opt.param_groups] for it in rec["lr_at"]["iterations"]]
    np.testing.assert_allclose(lrs, rec["lr_at"]["lr"], rtol=1e-12)


def test_setup_counts_the_appearance_groups():
    import types
    from b200gs.exposure import B200ExposureProcessor
    proc = B200ExposureProcessor(with_bias=True).instantiate()
    outputs = types.SimpleNamespace(appearance_group_ids={"a": (0, 0.0), "b": (4, 1.0), "c": (2, 0.5)})
    pl = types.SimpleNamespace(device=torch.device("cpu"),
                               trainer=types.SimpleNamespace(datamodule=types.SimpleNamespace(dataparser_outputs=outputs)))
    proc.setup("fit", pl_module=pl)
    assert tuple(proc.exposure_parameters.shape) == (5, 7)
