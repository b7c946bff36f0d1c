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
from collections import namedtuple

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
    # tinycudann.Encoding, 2-D DenseGrid (gsplat_appearance_embedding_visibility_map_renderer.py:4,114-124) and 3-D HashGrid
    # (swag_model.py:82-86), the same way
    if force:
        sys.modules["tinycudann"] = _tcnn_module()
    elif "tinycudann" not in sys.modules and not any(isinstance(f, _OnImport) and f.name == "tinycudann" for f in sys.meta_path):
        sys.meta_path.insert(0, _OnImport("tinycudann", _tcnn_module))
    # gsplat.utils.depth_to_normal (internal/metrics/normal_reg.py:3, VanillaWithNormalRegMetrics), the same way
    if force:
        sys.modules["gsplat.utils"] = _gsplat_utils_module()
    elif "gsplat.utils" not in sys.modules and not any(isinstance(f, _OnImport) and f.name == "gsplat.utils" for f in sys.meta_path):
        sys.meta_path.insert(0, _OnImport("gsplat.utils", _gsplat_utils_module))
    # pytorch3d.ops.knn_points (internal/metrics/appearance_feature_similarity_regularization_metrics.py:8, segany_splatting.py:276),
    # the same way; pytorch3d.ops.iou_box3d (partition_lod_renderer.py:8) raises ImportError on import
    for name, make in (("pytorch3d", _pytorch3d_module), ("pytorch3d.ops", _pytorch3d_ops_module),
                       ("pytorch3d.ops.iou_box3d", _pytorch3d_refused)):
        if force and make is not _pytorch3d_refused:
            sys.modules[name] = make()
        elif name not in sys.modules and not any(isinstance(f, _OnImport) and f.name == name for f in sys.meta_path):
            sys.meta_path.insert(0, _OnImport(name, make))      # the refusal always goes through the hook, so it names what exists
    if force:
        sys.modules["pytorch3d"].ops = sys.modules["pytorch3d.ops"]


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


KNN = namedtuple("KNN", ["dists", "idx", "knn"])


def knn_points(p1, p2, lengths1=None, lengths2=None, norm: int = 2, K: int = 1, version: int = -1, return_nn: bool = False,
               return_sorted: bool = True):
    """pytorch3d.ops.knn_points on ``ops.knn_points`` (one search per batch entry): p1 [B,S,3] and p2 [B,N,3] float32 CUDA,
    ``lengths1`` / ``lengths2`` None, ``norm`` 2, ``return_sorted`` True, ``return_nn`` False, 1 <= K <= min(32, N), and no
    gradient (inputs that require grad while grad is enabled are refused).  ``version`` is ignored.  Returns KNN(dists [B,S,K] squared
    distances, idx [B,S,K] int64, None), ascending."""
    from .. import ops
    unsupported = []
    if lengths1 is not None or lengths2 is not None:
        unsupported.append("lengths1 / lengths2")
    if norm != 2:
        unsupported.append(f"norm={norm}")
    if return_nn:
        unsupported.append("return_nn=True")
    if not return_sorted:
        unsupported.append("return_sorted=False")
    if torch.is_grad_enabled() and (p1.requires_grad or p2.requires_grad):
        unsupported.append("inputs that require grad")
    if unsupported:
        raise NotImplementedError(f"b200gs's pytorch3d.ops.knn_points does not support {', '.join(unsupported)}: it provides norm=2, "
                                  "return_sorted=True, return_nn=False and lengths=None without gradients")
    if p1.dim() != 3 or p2.dim() != 3 or p1.shape[0] != p2.shape[0]:
        raise ValueError(f"p1 and p2 must be [B, S, 3] and [B, N, 3], got {tuple(p1.shape)} and {tuple(p2.shape)}")
    results = [ops.knn_points(p1[b], p2[b], K) for b in range(p1.shape[0])]
    return KNN(torch.stack([r[0] for r in results]), torch.stack([r[1] for r in results]), None)


def _pytorch3d_module():
    m = types.ModuleType("pytorch3d")
    m.__path__ = []
    return m


def _pytorch3d_ops_module():
    m = types.ModuleType("pytorch3d.ops")
    m.__path__ = []
    m.knn_points = knn_points
    m.KNN = KNN
    return m


def _pytorch3d_refused():
    raise ImportError("b200gs provides only pytorch3d.ops.knn_points; pytorch3d.ops.iou_box3d (partition_lod_renderer.py) is not "
                      "provided")


def _tcnn_module():
    from ..visibility import UVGridEncoding

    class Encoding(UVGridEncoding):
        """tinycudann.Encoding for n_input_dims 2 and otype DenseGrid with linear interpolation and 2 features per level, on K32/K33,
        and for n_input_dims 3 and otype HashGrid (swag.HashGridEncoding, K49/K50; the grids swag.grid_kwargs accepts); anything
        else raises.  The initial values are uniform(-1e-4, 1e-4) from torch's generator, not tcnn's pcg32 stream, and a hash grid
        is float32, not half."""

        def __new__(cls, n_input_dims, encoding_config, seed=1337, dtype=None):
            if n_input_dims == 3 and str(dict(encoding_config).get("otype", "")).lower() == "hashgrid":
                from ..swag import HashGridEncoding
                if dtype not in (None, torch.float32):
                    raise NotImplementedError(f"b200gs provides tinycudann.Encoding for float32 grids only, got dtype={dtype}")
                return HashGridEncoding(encoding_config)       # not an Encoding: __init__ below is not called
            return super().__new__(cls)

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
            raise NotImplementedError(f"b200gs provides no tinycudann.{name}: only Encoding with a 2-D DenseGrid or a 3-D HashGrid")
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
