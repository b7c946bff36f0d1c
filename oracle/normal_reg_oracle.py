"""Float64 oracle of the depth-normal consistency term (K39-K42, csrc/normal_reg.cu): NormalRegModuleMixin.get_normal_reg_metrics
(internal/metrics/normal_reg.py:27-38) and gsplat's utils.depth_to_normal.

``depth_to_points`` / ``depth_to_normal`` restate gsplat's published ``utils.py`` in torch for any dtype and device: rays
R ((x - cx + 0.5) / fx, (y - cy + 0.5) / fy, 1), points o + depth * ray, normals normalize(cross(p[y+1,x] - p[y-1,x],
p[y,x+1] - p[y,x-1])) with F.normalize's max(|v|, 1e-12), zero-padded by one pixel.  The golden recorder hands them to the
reference's module as ``gsplat.utils.depth_to_normal``.  gsplat is a pip dependency pinned to a yzslab/gsplat commit that is not
part of the reference repository, so equality with that commit's own output is unpinned (as for fused_ssim).

``loss`` and ``vjp`` are the term and its gradient in float64; ``origin_free`` is the kernels' formulation (the camera origin cancels
in the differences and is never added), available in float32 to measure what fp32 arithmetic costs on the same input.  ``case``
generates seeded depth maps, cameras, alphas and normal maps."""
import numpy as np
import torch
import torch.nn.functional as F

KINDS = ("plane", "sphere", "noise", "flat", "zero")


def depth_to_points(depths, camtoworlds, Ks, z_depth=True):
    """gsplat utils.depth_to_points: depths [..., H, W, 1], camtoworlds [..., 4, 4], Ks [..., 3, 3] -> points [..., H, W, 3]"""
    height, width = depths.shape[-3:-1]
    x, y = torch.meshgrid(torch.arange(width, device=depths.device, dtype=depths.dtype),
                          torch.arange(height, device=depths.device, dtype=depths.dtype), indexing="xy")
    fx, fy, cx, cy = Ks[..., 0, 0], Ks[..., 1, 1], Ks[..., 0, 2], Ks[..., 1, 2]
    camera_dirs = F.pad(torch.stack([(x - cx[..., None, None] + 0.5) / fx[..., None, None],
                                     (y - cy[..., None, None] + 0.5) / fy[..., None, None]], dim=-1), (0, 1), value=1.0)
    directions = torch.einsum("...ij,...hwj->...hwi", camtoworlds[..., :3, :3], camera_dirs)
    origins = camtoworlds[..., :3, -1]
    if not z_depth:
        directions = F.normalize(directions, dim=-1)
    return origins[..., None, None, :] + depths * directions


def depth_to_normal(depths, camtoworlds, Ks, z_depth=True):
    """gsplat utils.depth_to_normal: [..., H, W, 1] depths -> [..., H, W, 3] normals, 0 on the one-pixel border"""
    points = depth_to_points(depths, camtoworlds, Ks, z_depth=z_depth)
    dx = torch.cat([points[..., 2:, 1:-1, :] - points[..., :-2, 1:-1, :]], dim=-3)
    dy = torch.cat([points[..., 1:-1, 2:, :] - points[..., 1:-1, :-2, :]], dim=-2)
    normals = F.normalize(torch.cross(dx, dy, dim=-1), dim=-1)
    return F.pad(normals, (0, 0, 1, 1, 1, 1), value=0.0)


def _cross_origin_free(depth, R, K):
    """cross(R a, R b) [H-2, W-2, 3] with a, b the camera-space differences d' c' - d c: the origin never enters"""
    H, W = depth.shape
    x = torch.arange(W, dtype=depth.dtype, device=depth.device)
    y = torch.arange(H, dtype=depth.dtype, device=depth.device)
    u = (x - K[0, 2] + 0.5) / K[0, 0]
    v = (y - K[1, 2] + 0.5) / K[1, 1]
    dt, db, dl, dr = depth[:-2, 1:-1], depth[2:, 1:-1], depth[1:-1, :-2], depth[1:-1, 2:]
    uu, vv = u[None, 1:-1], v[1:-1, None]
    a = torch.stack([uu * db - uu * dt, v[2:, None] * db - v[:-2, None] * dt, db - dt], dim=-1)
    b = torch.stack([u[None, 2:] * dr - u[None, :-2] * dl, vv * dr - vv * dl, dr - dl], dim=-1)
    return torch.cross(a @ R.T, b @ R.T, dim=-1)


def origin_free(depth, w2c, K, alpha):
    """n_d [3,H,W] as the kernels compute it, in depth's dtype: R = inverse of w2c's 3x3 block"""
    H, W = depth.shape
    out = torch.zeros((H, W, 3), dtype=depth.dtype, device=depth.device)
    if H >= 3 and W >= 3:
        R = torch.linalg.inv(w2c[:3, :3].to(torch.float64)).to(depth.dtype)
        out[1:-1, 1:-1] = F.normalize(_cross_origin_free(depth, R, K.to(depth.dtype)), dim=-1)
    return out.permute(2, 0, 1) * alpha


def normals_from_depth(depth, w2c, K, alpha, dtype=torch.float64):
    """the reference's n_d [3,H,W]: depth_to_normal(depth, inv(w2c), K) * alpha, in dtype (float64: the oracle).  An image with a
    side of 1 gives zeros: gsplat's slicing and padding would return a side of 2 there, a map of the wrong shape."""
    d, w, k, a = (t.to(dtype) for t in (depth, w2c, K, alpha))
    if min(depth.shape) < 3:
        return torch.zeros((3, *depth.shape), dtype=dtype, device=depth.device)
    return depth_to_normal(d[..., None], torch.linalg.inv(w), k).permute(2, 0, 1) * a


def cross_norm(depth, w2c, K):
    """|cross| [H,W] in float64 (0 on the border): how close each pixel is to F.normalize's 1e-12 floor"""
    H, W = depth.shape
    out = torch.zeros((H, W), dtype=torch.float64, device=depth.device)
    if H >= 3 and W >= 3:
        R = torch.linalg.inv(w2c[:3, :3].double())
        out[1:-1, 1:-1] = _cross_origin_free(depth.double(), R, K.double()).norm(dim=-1)
    return out


def loss(normal, depth, alpha, w2c, K, weight):
    """weight mean(1 - sum_c normal n_d), float64 scalar tensor"""
    n_d = normals_from_depth(depth, w2c, K, alpha)
    return (1 - (normal.double() * n_d).sum(0)).mean() * weight


def vjp(depth, alpha, w2c, K, weight, v_loss=1.0):
    """d loss / d normal [3,H,W] in float64"""
    H, W = depth.shape
    return -float(v_loss) * weight / (H * W) * normals_from_depth(depth, w2c, K, alpha)


def rotation(seed):
    """a random proper rotation, float64"""
    q, r = np.linalg.qr(np.random.default_rng(seed).standard_normal((3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def camera(H, W, seed, translation=3.0):
    """(w2c [4,4], K [3,3]) float32: a random rotation, a translation of size ~translation, fx ~ 0.9 W"""
    rng = np.random.default_rng(seed + 1)
    w2c = np.eye(4)
    w2c[:3, :3] = rotation(seed)
    w2c[:3, 3] = rng.uniform(-1, 1, 3) * translation
    f = 0.9 * max(W, H, 2) * rng.uniform(0.8, 1.2)
    K = np.array([[f, 0, W / 2 + rng.uniform(-2, 2)], [0, f * rng.uniform(0.95, 1.05), H / 2 + rng.uniform(-2, 2)], [0, 0, 1]])
    return torch.from_numpy(w2c.astype(np.float32)), torch.from_numpy(K.astype(np.float32))


def plane_depth(H, W, K, plane_cam, offset):
    """z depth [H,W] of the camera-space plane n . p = offset (n = plane_cam), and the closed-form n_d [3,H,W] in camera space"""
    Kd = K.double()
    x = torch.arange(W, dtype=torch.float64)
    y = torch.arange(H, dtype=torch.float64)
    u = ((x - Kd[0, 2] + 0.5) / Kd[0, 0])[None, :].expand(H, W)
    v = ((y - Kd[1, 2] + 0.5) / Kd[1, 1])[:, None].expand(H, W)
    n = torch.as_tensor(plane_cam, dtype=torch.float64)
    n = n / n.norm()
    ndotc = n[0] * u + n[1] * v + n[2]
    depth = offset / ndotc
    # the cross product of the image-aligned differences points back at the camera: -sign(n . ray) n
    return depth, -torch.sign(ndotc)[None] * n[:, None, None]


def plane_normals(kind, H, W, seed, translation=3.0):
    """closed-form world-space n_d [3,H,W] (alpha 1, 0 on the border) of case(kind, H, W, seed) for kind plane or flat"""
    w2c, K = camera(H, W, seed, translation)
    n_cam = plane_depth(H, W, K, (0.0, 0.0, 1.0) if kind == "flat" else (0.3, -0.4, 1.0), 2.5)[1]
    n = torch.einsum("ij,jhw->ihw", torch.linalg.inv(w2c.double())[:3, :3], n_cam)
    out = torch.zeros_like(n)
    out[:, 1:-1, 1:-1] = n[:, 1:-1, 1:-1]
    return out


def case(kind, H, W, seed, translation=3.0, alpha="random"):
    """(depth [H,W], alpha [H,W], normal [3,H,W], w2c [4,4], K [3,3]) float32 CPU tensors.  kind: plane (a tilted plane), sphere (a
    sphere in front of the camera on a plane background), noise (uniform depth in [1, 5]), flat (constant depth) or zero (all 0).
    alpha: "random" (uniform [0, 1)), 0 or 1."""
    rng = np.random.default_rng(seed + 2)
    w2c, K = camera(H, W, seed, translation)
    if kind in ("plane", "flat"):
        normal_cam = (0.0, 0.0, 1.0) if kind == "flat" else (0.3, -0.4, 1.0)
        depth = plane_depth(H, W, K, normal_cam, 2.5)[0]
    elif kind == "sphere":
        depth = plane_depth(H, W, K, (0.1, 0.2, 1.0), 6.0)[0]
        Kd = K.double()
        x = torch.arange(W, dtype=torch.float64)
        y = torch.arange(H, dtype=torch.float64)
        ray = torch.stack(torch.broadcast_tensors(((x - Kd[0, 2] + 0.5) / Kd[0, 0])[None, :], ((y - Kd[1, 2] + 0.5) / Kd[1, 1])[:, None],
                                                  torch.ones(1, 1, dtype=torch.float64)), dim=-1)
        center, radius = torch.tensor([0.05, -0.03, 3.0], dtype=torch.float64), 1.0
        bq = (ray * center).sum(-1)
        aq = (ray * ray).sum(-1)
        disc = bq * bq - aq * (center @ center - radius ** 2)
        t = (bq - disc.clamp_min(0).sqrt()) / aq
        depth = torch.where(disc > 0, torch.minimum(t, depth), depth)
    elif kind == "noise":
        depth = torch.from_numpy(rng.uniform(1.0, 5.0, (H, W)))
    elif kind == "zero":
        depth = torch.zeros(H, W, dtype=torch.float64)
    else:
        raise ValueError(kind)
    if alpha == "random":
        a = torch.from_numpy(rng.uniform(0.0, 1.0, (H, W)))
    else:
        a = torch.full((H, W), float(alpha), dtype=torch.float64)
    normal = F.normalize(torch.from_numpy(rng.standard_normal((3, H, W))), dim=0) * torch.from_numpy(rng.uniform(0.5, 1.0, (1, H, W)))
    return depth.float(), a.float(), normal.float(), w2c, K
