"""gsplat v1 operator surface backed by libb200gs.so: the names the reference's ``GSplatV1`` helpers import
(``internal/renderers/gsplat_v1_renderer.py:8-20``) with the argument names, defaults, shapes and return tuples of those call
sites.  ``install()`` registers them as ``gsplat.cuda._wrapper``, ``gsplat.sh_decomposed``,
``gsplat.cuda.isect_tiles_tile_based_culling`` and ``gsplat.v0_interfaces.rasterize_to_pixels``, so ``GSplatV1Renderer`` and every
renderer built on it run unmodified.

Costs of the gsplat contract that the fused plug-ins (``b200gs.v1``, ``b200gs.renderers``) do not pay:
  - ``isect_ids`` / ``flatten_ids`` have the exact pair count, so ``isect_tiles`` bins synchronously: one host wait per view, as
    gsplat's own ``isect_tiles`` performs;
  - ``viewmats`` / ``Ks`` are read back once per ``fully_fused_projection`` call (25 floats per camera).

Options without a b200gs implementation raise instead of returning something else: ``covars``, ``packed``, ``sparse_grad``,
camera models other than pinhole, ``radius_clip``, a finite ``far_plane``, ``tile_size`` other than 16, more than one camera in
``isect_tiles`` / ``rasterize_to_pixels``, and ``viewmats`` / ``Ks`` that require a gradient (there is no pose gradient).
"""
import math

import torch

from .. import ops
from .._lib import MODE_GSPLAT, TILE
from ..v1 import camera_views, tiles_per_gauss

spherical_harmonics = ops.spherical_harmonics
spherical_harmonics_decomposed = ops.spherical_harmonics_decomposed

_FAR_PLANE = 1e10


def fully_fused_projection(means, covars, quats, scales, viewmats, Ks, width, height, eps2d=0.3, near_plane=0.01, far_plane=_FAR_PLANE,
                           radius_clip=0.0, packed=False, sparse_grad=False, calc_compensations=False, camera_model="pinhole"):
    """-> (radii [C,N] int32, means2d [C,N,2], depths [C,N], conics [C,N,3], compensations [C,N] or None).

    K1 per camera (``ops.project_gaussians``); the backward is each camera's K8, summed by autograd."""
    if covars is not None:
        raise NotImplementedError("b200gs projects from quats and scales; covars is unsupported")
    if packed or sparse_grad:
        raise NotImplementedError("b200gs: packed / sparse_grad projection is unsupported")
    if camera_model != "pinhole":
        raise NotImplementedError("b200gs projects pinhole cameras only")
    if radius_clip != 0:
        raise NotImplementedError("b200gs: radius_clip is unsupported")
    if far_plane != _FAR_PLANE:
        raise NotImplementedError("b200gs: far_plane is unsupported")
    if viewmats.requires_grad or Ks.requires_grad:
        raise NotImplementedError("b200gs has no camera-pose gradient: viewmats and Ks must not require grad")
    if viewmats.dim() != 3 or viewmats.shape[1:] != (4, 4) or Ks.shape != (viewmats.shape[0], 3, 3):
        raise ValueError("viewmats must be [C,4,4] and Ks [C,3,3]")
    outs = []
    for view in camera_views(viewmats, Ks, int(width), int(height)):
        view = ops._copy_view(view, eps2d=float(eps2d), near_plane=float(near_plane))
        xys, depths, radii, conics, comp, _, _ = ops.project_gaussians(means, scales, 1.0, quats, None, 0, 0, 0, 0, view.height, view.width,
                                                                       view=view)
        outs.append((radii, xys, depths, conics, comp))
    radii, means2d, depths, conics, comp = (torch.stack(t) for t in zip(*outs))
    return radii, means2d, depths, conics, (comp if calc_compensations else None)


def _isect(means2d, radii, depths, tile_size, tile_width, tile_height, sort, packed, n_cameras, camera_ids, gaussian_ids, conics=None,
           opacities=None):
    if tile_size != TILE:
        raise ValueError(f"b200gs supports tile_size {TILE} only")
    if packed or camera_ids is not None or gaussian_ids is not None:
        raise NotImplementedError("b200gs: packed intersections are unsupported")
    if not sort:
        raise NotImplementedError("b200gs lists intersections sorted only")
    if n_cameras != 1 or means2d.dim() != 3 or means2d.shape[0] != 1:
        raise NotImplementedError("b200gs intersects one camera per call (C = 1)")
    tw, th = int(tile_width), int(tile_height)
    xy, d, r = means2d.reshape(-1, 2).detach().contiguous(), depths.reshape(-1).detach().contiguous(), radii.reshape(-1).contiguous()
    if conics is None:
        binning = ops.bin_gaussians(MODE_GSPLAT, tw * TILE, th * TILE, xy, d, r)
    else:
        binning = ops.bin_gaussians(MODE_GSPLAT, tw * TILE, th * TILE, xy, d, r, conics.reshape(-1, 3).detach().contiguous(),
                                    opacities.reshape(-1).detach().contiguous())
    keys = ops.isect_keys(binning, d)
    return tiles_per_gauss(xy, r, tw, th, tile_size).to(torch.int32), keys, binning.sorted_ids[:keys.shape[0]]


def isect_tiles(means2d, radii, depths, tile_size, tile_width, tile_height, sort=True, packed=False, n_cameras=1, camera_ids=None,
                gaussian_ids=None):
    """-> (tiles_per_gauss [1,N] int32, isect_ids [I] int64, flatten_ids [I] int32): every tile of each 3-sigma rect, front to back.
    isect_ids are the keys of our list order, (tile << 32) | float_bits(depth), equal to gsplat's sorted keys; gsplat's radix sort
    need not order equal keys by Gaussian id, ours does.  Bins synchronously (the exact pair count)."""
    return _isect(means2d, radii, depths, tile_size, tile_width, tile_height, sort, packed, n_cameras, camera_ids, gaussian_ids)


def isect_tiles_tile_based_culling(means2d, radii, depths, conics, opacities, tile_size, tile_width, tile_height, sort=True, packed=False,
                                   n_cameras=1, camera_ids=None, gaussian_ids=None):
    """isect_tiles with exact tile culling: only (tile, Gaussian) pairs whose tile can see alpha >= 1/255 are listed, and only they
    carry keys.  tiles_per_gauss still counts the whole rect."""
    return _isect(means2d, radii, depths, tile_size, tile_width, tile_height, sort, packed, n_cameras, camera_ids, gaussian_ids,
                  conics, opacities)


def isect_offset_encode(isect_ids, n_cameras, tile_width, tile_height):
    """-> isect_offsets [1, tile_height, tile_width] int32: index of the first key of each tile (the next start for empty tiles)."""
    if n_cameras != 1:
        raise NotImplementedError("b200gs intersects one camera per call (C = 1)")
    return ops.isect_offsets(isect_ids, int(tile_width) * int(tile_height)).reshape(1, int(tile_height), int(tile_width))


def isect_offset_encode_tile_based_culling(isect_ids, flatten_ids, n_cameras, tile_width, tile_height):
    """-> (isect_offsets [1,th,tw], flatten_ids): the culled lists hold no dropped pairs, so flatten_ids is returned as it is."""
    return isect_offset_encode(isect_ids, n_cameras, tile_width, tile_height), flatten_ids


def rasterize_to_pixels(means2d, conics, colors, opacities, image_width, image_height, tile_size, isect_offsets, flatten_ids, backgrounds=None,
                        absgrad=False, **kwargs):
    """means2d [N,2], conics [1,N,3], colors [1,N,D], opacities [1,N], backgrounds [1,D] -> (colors [1,H,W,D], alphas [1,H,W,1]).

    The per-tile lists are [isect_offsets[t], isect_offsets[t+1]) of flatten_ids (the last tile ends at len(flatten_ids)); the
    blend is ``ops.rasterize_binned`` (groups of <= 4 channels).  Sets ``means2d.has_hit_any_pixels`` (bool [N]) now and
    ``means2d.absgrad`` after the backward when absgrad."""
    if tile_size != TILE:
        raise ValueError(f"b200gs supports tile_size {TILE} only")
    if means2d.dim() != 2 or colors.dim() != 3 or colors.shape[0] != 1 or isect_offsets.shape[0] != 1:
        raise NotImplementedError("b200gs rasterizes one camera per call: means2d [N,2], colors [1,N,D], isect_offsets [1,th,tw]")
    W, H = int(image_width), int(image_height)
    if isect_offsets.shape[1:] != (math.ceil(H / TILE), math.ceil(W / TILE)):
        raise ValueError("isect_offsets do not match the image size")
    for name, t in (("isect_offsets", isect_offsets), ("flatten_ids", flatten_ids)):
        if not t.is_cuda or t.device != means2d.device or t.dtype not in (torch.int32, torch.int64):
            raise ValueError(f"{name} must be an integer tensor on the device of means2d")
    starts = isect_offsets.reshape(-1).to(torch.int32)
    ends = torch.cat((starts[1:], starts.new_full((1,), flatten_ids.shape[0])))
    binning = ops.Binning(flatten_ids.to(torch.int32).contiguous(), torch.stack((starts, ends), dim=-1).contiguous(), int(flatten_ids.shape[0]))
    image, alpha, hits = ops.rasterize_binned(means2d, conics.reshape(-1, 3), colors[0], opacities.reshape(-1), binning, H, W,
                                              None if backgrounds is None else backgrounds.reshape(-1), absgrad=absgrad, want_hits=True)
    means2d.has_hit_any_pixels = hits.bool()
    return image.unsqueeze(0), alpha.unsqueeze(-1).unsqueeze(0)
