"""Drop-in modules carrying the names the reference imports from its CUDA pip dependencies.

``install()`` aliases them in ``sys.modules`` so that the UNMODIFIED reference renderers
(``internal/renderers/vanilla_renderer.py:14``, ``gsplat_renderer.py:2-4``, ``gsplat_v1_renderer.py:8-20``) run on the b200gs
kernels:

    import b200gs.compat; b200gs.compat.install()
    from internal.renderers.vanilla_renderer import VanillaRenderer   # now backed by libb200gs.so
"""
import sys
import types


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
