"""Drop-in modules carrying the names the reference imports from its CUDA pip dependencies.

``install()`` aliases them in ``sys.modules`` so that the UNMODIFIED reference renderers
(``internal/renderers/vanilla_renderer.py:14``, ``gsplat_renderer.py:2-4``, ``gsplat_v1_renderer.py:8-20``) run on the b200gs
kernels:

    import b200gs.compat; b200gs.compat.install()
    from internal.renderers.vanilla_renderer import VanillaRenderer   # now backed by libb200gs.so
"""
import importlib.abc
import importlib.util
import sys
import types

import torch


def install(force: bool = False):
    from . import diff_gaussian_rasterization as dgr
    from . import gsplat_v0, gsplat_v1

    def put(name, module):
        if force or name not in sys.modules:
            sys.modules[name] = module

    put("diff_gaussian_rasterization", dgr)
    # simple_knn._C.distCUDA2 (internal/models/vanilla_gaussian.py:122-124)
    from .. import ops
    knn = types.ModuleType("simple_knn")
    knn.__path__ = []
    knn_c = types.ModuleType("simple_knn._C")
    knn_c.distCUDA2 = ops.knn_mean_dist2
    knn._C = knn_c
    put("simple_knn", knn)
    put("simple_knn._C", knn_c)
    pkg = types.ModuleType("gsplat")
    pkg.__path__ = []  # mark as package
    pkg.project_gaussians = gsplat_v0.project_gaussians
    pkg.rasterize_gaussians = gsplat_v0.rasterize_gaussians
    pkg.spherical_harmonics = gsplat_v0.spherical_harmonics
    put("gsplat", pkg)
    for sub, names in (("v0_interfaces", ("project_gaussians", "rasterize_gaussians")),
                       ("project_gaussians", ("project_gaussians",)),
                       ("rasterize", ("rasterize_gaussians",)),
                       ("sh", ("spherical_harmonics",))):
        m = types.ModuleType(f"gsplat.{sub}")
        for nm in names:
            setattr(m, nm, getattr(gsplat_v0, nm))
        if sub == "v0_interfaces":     # gsplat_v1_renderer.py:20
            m.rasterize_to_pixels = gsplat_v1.rasterize_to_pixels
        put(f"gsplat.{sub}", m)
    # gsplat v1 (gsplat_v1_renderer.py:8-20)
    cuda = types.ModuleType("gsplat.cuda")
    cuda.__path__ = []
    pkg.cuda = cuda
    for sub, names in (("cuda._wrapper", ("fully_fused_projection", "isect_tiles", "isect_offset_encode", "spherical_harmonics")),
                       ("cuda.isect_tiles_tile_based_culling", ("isect_tiles_tile_based_culling", "isect_offset_encode_tile_based_culling")),
                       ("sh_decomposed", ("spherical_harmonics_decomposed",))):
        m = types.ModuleType(f"gsplat.{sub}")
        for nm in names:
            setattr(m, nm, getattr(gsplat_v1, nm))
        setattr(cuda if sub.startswith("cuda.") else pkg, sub.split(".")[-1], m)
        put(f"gsplat.{sub}", m)
    put("gsplat.cuda", cuda)
    # gsplat.relocation.compute_relocation (internal/density_controllers/mcmc_density_controller.py:13)
    from .. import mcmc
    reloc = types.ModuleType("gsplat.relocation")
    reloc.compute_relocation = mcmc.compute_relocation
    put("gsplat.relocation", reloc)
    # fused_bilagrid (internal/output_processors/bilagrid.py:40, BilagridProcessor with fused: true, the default)
    from .. import bilagrid
    fb = types.ModuleType("fused_bilagrid")
    for nm in ("BilateralGrid", "slice", "total_variation_loss"):
        setattr(fb, nm, getattr(bilagrid, nm))
    put("fused_bilagrid", fb)
    # fused_ssim.fused_ssim (internal/metrics/vanilla_metrics.py:35-39 with fused_ssim: true; the Taming density controller): made
    # when first imported, through an import hook, so install() itself leaves sys.modules as it was
    if force:
        sys.modules["fused_ssim"] = _fused_ssim_module()
    elif "fused_ssim" not in sys.modules and not any(isinstance(f, _OnImport) and f.name == "fused_ssim" for f in sys.meta_path):
        sys.meta_path.insert(0, _OnImport("fused_ssim", _fused_ssim_module))
    # tinycudann.Encoding, 2-D DenseGrid only (gsplat_appearance_embedding_visibility_map_renderer.py:4,114-124), the same way
    if force:
        sys.modules["tinycudann"] = _tcnn_module()
    elif "tinycudann" not in sys.modules and not any(isinstance(f, _OnImport) and f.name == "tinycudann" for f in sys.meta_path):
        sys.meta_path.insert(0, _OnImport("tinycudann", _tcnn_module))
    # gsplat.utils.depth_to_normal (internal/metrics/normal_reg.py:3, VanillaWithNormalRegMetrics), the same way
    if force:
        sys.modules["gsplat.utils"] = _gsplat_utils_module()
    elif "gsplat.utils" not in sys.modules and not any(isinstance(f, _OnImport) and f.name == "gsplat.utils" for f in sys.meta_path):
        sys.meta_path.insert(0, _OnImport("gsplat.utils", _gsplat_utils_module))


def _fused_ssim_module():
    from .. import metrics
    fs = types.ModuleType("fused_ssim")
    fs.fused_ssim = metrics.fused_ssim
    return fs


def _gsplat_utils_module():
    from .. import metrics
    m = types.ModuleType("gsplat.utils")
    m.depth_to_normal = metrics.depth_to_normal
    return m


def _tcnn_module():
    from ..visibility import UVGridEncoding

    class Encoding(UVGridEncoding):
        """tinycudann.Encoding for n_input_dims 2 and otype DenseGrid with linear interpolation and 2 features per level, on K32/K33;
        anything else raises.  The initial values are uniform(-1e-4, 1e-4) from torch's generator, not tcnn's pcg32 stream."""

        def __init__(self, n_input_dims, encoding_config, seed=1337, dtype=None):
            c = dict(encoding_config)
            if n_input_dims != 2 or str(c.get("otype", "")).lower() not in ("densegrid", "dense") or \
                    str(c.get("interpolation", "Linear")).lower() != "linear" or int(c.get("n_features_per_level", 2)) != 2 or \
                    dtype not in (None, torch.float32):
                raise NotImplementedError(f"b200gs provides tinycudann.Encoding for 2-D float32 DenseGrid with linear interpolation "
                                          f"and 2 features per level only, got n_input_dims={n_input_dims}, {c}, dtype={dtype}")
            super().__init__(c.get("n_levels", 16), c.get("base_resolution", 16), c.get("per_level_scale", 2.0))

    def refuse(name):
        def init(self, *args, **kwargs):
            raise NotImplementedError(f"b200gs provides no tinycudann.{name}: only Encoding with a 2-D DenseGrid")
        return type(name, (), {"__init__": init})

    m = types.ModuleType("tinycudann")
    m.Encoding = Encoding
    m.Network = refuse("Network")
    m.NetworkWithInputEncoding = refuse("NetworkWithInputEncoding")
    return m


class _OnImport(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    """Import hook that builds the module `name` with `make()` when it is first imported."""

    def __init__(self, name, make):
        self.name, self.make = name, make

    def find_spec(self, fullname, path, target=None):
        return importlib.util.spec_from_loader(fullname, self) if fullname == self.name else None

    def create_module(self, spec):
        return self.make()

    def exec_module(self, module):
        pass
