"""B200MCMCDensityController is the reference's MCMCDensityControllerImpl with the position noise routed to b200gs.mcmc.  Needs a
gaussian-splatting-lightning checkout, named by the B200GS_REFERENCE environment variable (skipped without one); `lightning`
is stubbed, and no device is used (the noise kernel is replaced by a recorder).  Without the reference, instantiate() fails
with an ImportError that names it."""
import os
import sys
import types

import pytest
import torch

REFERENCE = os.environ.get("B200GS_REFERENCE", "")
needs_reference = pytest.mark.skipif(not os.path.isfile(os.path.join(REFERENCE, "internal", "density_controllers", "mcmc_density_controller.py")),
                                reason="set B200GS_REFERENCE to a gaussian-splatting-lightning checkout")


@pytest.fixture
def reference(monkeypatch):
    from b200gs import compat, mcmc, renderers  # noqa: F401  (imported before the reference is on sys.path: they keep their own bases)
    before = set(sys.modules)
    lightning = types.ModuleType("lightning")
    lightning.LightningModule = type("LightningModule", (), {})
    monkeypatch.setitem(sys.modules, "lightning", lightning)
    monkeypatch.syspath_prepend(REFERENCE)
    # the controller module imports gsplat.relocation at load time: instantiate() must have installed it before the first import
    yield lambda: __import__("internal.density_controllers.mcmc_density_controller", fromlist=["*"])
    for name in set(sys.modules) - before:
        if name == "internal" or name.startswith(("internal.", "gsplat", "diff_gaussian_rasterization", "simple_knn")):
            del sys.modules[name]


class _Module:
    def is_final_step(self):
        return True

    gaussian_optimizers = [types.SimpleNamespace(param_groups=[{"name": "opacities", "lr": 0.05}]),
                           types.SimpleNamespace(param_groups=[{"name": "scales", "lr": 0.005}, {"name": "means", "lr": 1.6e-4}])]


@needs_reference
def test_instantiate_returns_the_reference_impl_with_our_relocation(reference):
    from b200gs import mcmc
    from b200gs.mcmc import B200MCMCDensityController
    cfg = B200MCMCDensityController(cap_max=1000)
    assert (cfg.noise_lr, cfg.densify_from_iter, cfg.densify_until_iter, cfg.densification_interval, cfg.min_opacity, cfg.N_max) \
        == (5e5, 500, 25_000, 100, 0.005, 51)
    impl = cfg.instantiate()
    ref = reference()
    assert isinstance(impl, ref.MCMCDensityControllerImpl)
    assert ref.compute_relocation is mcmc.compute_relocation
    assert sys.modules["gsplat.relocation"].compute_relocation is mcmc.compute_relocation


@needs_reference
def test_add_xyz_noise_calls_the_fused_kernel_with_the_means_lr(reference, monkeypatch):
    from b200gs import mcmc
    from b200gs.scene import SyntheticGaussians, make_scene
    calls = []
    monkeypatch.setattr(mcmc, "add_position_noise", lambda *args, **kw: calls.append((args, kw)))
    impl = mcmc.B200MCMCDensityController(cap_max=1000, noise_lr=1234.0).instantiate()
    model = SyntheticGaussians(make_scene(16, 0))
    impl._add_xyz_noise({}, None, model, 7, _Module())
    assert len(calls) == 1
    args, kw = calls[0]
    g = model.gaussians
    assert args[0] is g["means"] and args[1] is g["scales"] and args[2] is g["rotations"] and args[3] is g["opacities"]
    assert args[4:] == (1234.0, 1.6e-4) and not kw


@needs_reference
def test_other_models_keep_the_reference_formula(reference, monkeypatch):
    from b200gs import mcmc
    from b200gs.scene import SyntheticGaussians, make_scene
    monkeypatch.setattr(mcmc, "add_position_noise", lambda *a, **k: pytest.fail("the fused kernel needs the vanilla activations"))

    class FilteredGaussians(SyntheticGaussians):     # a model the fused renderer path does not accept either
        @property
        def means(self):
            return self.gaussians["means"]

    model = FilteredGaussians(make_scene(16, 0))
    before = model.means.detach().clone()
    mcmc.B200MCMCDensityController(cap_max=1000).instantiate()._add_xyz_noise({}, None, model, 7, _Module())
    assert not torch.equal(model.means.detach(), before)


def test_instantiate_without_the_reference_names_it(monkeypatch):
    from b200gs.mcmc import B200MCMCDensityController
    monkeypatch.setitem(sys.modules, "internal.density_controllers.mcmc_density_controller", None)   # import -> ImportError
    with pytest.raises(ImportError, match="internal.density_controllers.mcmc_density_controller"):
        B200MCMCDensityController(cap_max=1000).instantiate()
