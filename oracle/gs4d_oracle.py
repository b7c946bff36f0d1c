"""Float64 restatement of the 4DGS deformation VanillaGS4DRenderer applies every frame (internal/renderers/vanilla_gs4d_renderer.py with
internal/model_components/gs4d_hexplane.py and gs4d_deformation.py), steps 2-5:

    p      = (means - aabb[0]) * 2 / (aabb[1] - aabb[0]) - 1          aabb[0] = xyz_max, aabb[1] = xyz_min: the max corner maps to -1
    f_l    = prod_k bilinear(plane_l^k; (p, t)_{a_k}, (p, t)_{b_k})    k over (0,1), (0,2), (0,3), (1,2), (1,3), (2,3); a: width
    h      = trunk([f_0 | .. | f_{L-1}])                               Linear, then (D - 1) x [ReLU, Linear]
    head   = Linear(ReLU(Linear(ReLU(h))))                             dx [3], ds [3], dr [4], dshs [48]
    means' = means + dx, log_scales' = log_scales + ds, quats' = quats + dr | normalize(quats * dr), shs' = shs + dshs

bilinear is grid_sample with align_corners=True and padding_mode='border': the source index ((x + 1) / 2)(res - 1) is clipped to
[0, res - 1] before the four corners are weighed.  Everything here is computed in float64 from the inputs as given."""
import torch

PLANES = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
HEADS = ("dx", "ds", "dr", "dshs")


def _d(x):
    return torch.as_tensor(x).double()


def normalize_points(means, aabb):
    aabb = _d(aabb)
    return (_d(means) - aabb[0]) * (2.0 / (aabb[1] - aabb[0])) - 1.0


def sample_plane(plane, u, v):
    """bilinear sample of plane [C, H, W] at width coordinate u and height coordinate v (each [N], in [-1, 1] or beyond): [N, C]"""
    plane = _d(plane)
    C, H, W = plane.shape

    def axis(x, size):
        ix = ((x + 1.0) / 2.0 * (size - 1)).clamp(0.0, size - 1)
        i0 = ix.floor()
        f = ix - i0
        i0 = i0.long()
        return i0, (i0 + 1).clamp(max=size - 1), f

    x0, x1, fx = axis(_d(u), W)
    y0, y1, fy = axis(_d(v), H)
    flat = plane.reshape(C, H * W)

    def at(y, x):
        return flat[:, y * W + x].T

    fx, fy = fx[:, None], fy[:, None]
    return at(y0, x0) * (1 - fx) * (1 - fy) + at(y0, x1) * fx * (1 - fy) + at(y1, x0) * (1 - fx) * fy + at(y1, x1) * fx * fy


def hexplane(points4, grids):
    """[f_0 | .. | f_{L-1}] of points4 [N, 4] ((p, t)); grids: L levels of six planes, each [C, res_b, res_a] (or [1, C, ..])"""
    points4 = _d(points4)
    feats = []
    for level in grids:
        prod = 1.0
        for (a, b), plane in zip(PLANES, level):
            plane = _d(plane)
            plane = plane[0] if plane.dim() == 4 else plane
            prod = prod * sample_plane(plane, points4[:, a], points4[:, b])
        feats.append(prod)
    return torch.cat(feats, dim=-1)


def linear(x, wb):
    w, b = wb
    return x @ _d(w).T + _d(b)


def trunk_forward(features, trunk):
    h = linear(features, trunk[0])
    for wb in trunk[1:]:
        h = linear(torch.relu(h), wb)
    return h


def head_forward(h, head):
    hidden, out = head
    return linear(torch.relu(linear(torch.relu(h), hidden)), out)


def quaternion_multiply_normalized(q1, q2):
    w = q1[:, 0] * q2[:, 0] - q1[:, 1] * q2[:, 1] - q1[:, 2] * q2[:, 2] - q1[:, 3] * q2[:, 3]
    x = q1[:, 0] * q2[:, 1] + q1[:, 1] * q2[:, 0] + q1[:, 2] * q2[:, 3] - q1[:, 3] * q2[:, 2]
    y = q1[:, 0] * q2[:, 2] - q1[:, 1] * q2[:, 3] + q1[:, 2] * q2[:, 0] + q1[:, 3] * q2[:, 1]
    z = q1[:, 0] * q2[:, 3] + q1[:, 1] * q2[:, 2] - q1[:, 2] * q2[:, 1] + q1[:, 3] * q2[:, 0]
    q = torch.stack((w, x, y, z), dim=1)
    return q / q.norm(dim=1, keepdim=True)


def features(means, t, aabb, grids):
    p = normalize_points(means, aabb)
    return hexplane(torch.cat([p, torch.full_like(p[:, :1], float(t))], dim=-1), grids)


def deform(means, log_scales, quats, t, aabb, grids, trunk, heads, shs=None, apply_rotation=False):
    """dict of the deformed raw parameters: means, log_scales, quats and (with the dshs head and shs [N, 16, 3]) shs.  ``heads`` maps
    each enabled head name to ((hidden weight, bias), (output weight, bias)); ``trunk`` lists the trunk's (weight, bias)."""
    h = trunk_forward(features(means, t, aabb, grids), trunk)
    out = {"means": _d(means), "log_scales": _d(log_scales), "quats": _d(quats), "shs": None if shs is None else _d(shs)}
    if "dx" in heads:
        out["means"] = out["means"] + head_forward(h, heads["dx"])
    if "ds" in heads:
        out["log_scales"] = out["log_scales"] + head_forward(h, heads["ds"])
    if "dr" in heads:
        dr = head_forward(h, heads["dr"])
        out["quats"] = quaternion_multiply_normalized(out["quats"], dr) if apply_rotation else out["quats"] + dr
    if "dshs" in heads:
        out["shs"] = out["shs"] + head_forward(h, heads["dshs"]).reshape(-1, 16, 3)
    return out


def activate(deformed, opacity_logits):
    """step 5: exp of the scales, normalize of the rotations and sigmoid of the UNdeformed opacity logits"""
    q = deformed["quats"]
    return {"means": deformed["means"], "scales": deformed["log_scales"].exp(), "rotations": q / q.norm(dim=1, keepdim=True).clamp_min(1e-12),
            "opacities": torch.sigmoid(_d(opacity_logits)).reshape(-1, 1), "shs": deformed["shs"]}
