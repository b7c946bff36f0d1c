"""Float64 oracle of the Glossy-Gaussian view-dependent opacity and SH colour (internal/renderers/glossy_renderer.py
``GlossyRendererModule.get_opacities`` / ``get_rgbs`` with ``GlossyGaussianModel.get_view_dep_opacities``,
internal/models/glossy_gaussian.py:66-79).

``glossy(degree, means, campos, op_dc, op_rest, colour=None, mask=None, pass_opacity=None, pass_rgb=None)``:
  dir     = (means - campos) / max(|means - campos|, 1e-12), detached (F.normalize; the reference detaches the means)
  opacity = clamp(sum_k B_k(dir) op_k + 0.5, 0, 1)                 for every row (the reference ignores the masks here)
  rgb     = clamp(sum_k B_k(dir) c_k + 0.5, min=0) on mask rows, 0.5 elsewhere with no gradient (gsplat's masked SH, then the clamp)
with B the basis of ``gs_oracle.sh_basis``.  ``colour`` is ``(shs_dc [N,1,3], shs_rest [N,K-1,3])`` or ``features [N,K,3]``.
The clamps pass the gradient where lo <= x <= hi, torch.clamp's rule.  ``pass_opacity`` [N] / ``pass_rgb`` [N,3] (bool) replace
that decision, for samples the caller found within ``AMBIGUOUS`` of a bound (``near_bound``), where fp32 may decide either way.
Returns a dict: ``opacity`` [N], ``rgb`` [N,3] (None without colour), the unclamped ``raw_opacity`` / ``raw_rgb`` and their rounding
scales ``scale_opacity`` / ``scale_rgb`` (0.5 plus the sum of |term|), all in the inputs' dtype, with autograd to the coefficients.
"""
import torch

from oracle.gs_oracle import sh_basis

AMBIGUOUS = 8 * 2.0 ** -23


def directions(means, campos):
    d = means - campos.reshape(1, 3)
    return d / d.norm(dim=-1, keepdim=True).clamp_min(1e-12)


def _clamp(raw, lo, hi, passes):
    rule = (raw >= lo) if hi is None else ((raw >= lo) & (raw <= hi))
    passes = rule if passes is None else passes
    return torch.where(passes, raw, raw.clamp(lo, hi).detach())


def glossy(degree, means, campos, op_dc, op_rest, colour=None, mask=None, pass_opacity=None, pass_rgb=None):
    ncoef = (degree + 1) ** 2
    dirs = directions(means.detach(), campos.detach())
    B = sh_basis(degree, dirs)                                                       # [N, ncoef]
    op = torch.cat([op_dc[:, :, 0], op_rest[:, :ncoef - 1, 0]], dim=1)              # [N, ncoef]
    terms = B * op
    out = {"raw_opacity": terms.sum(1) + 0.5, "scale_opacity": terms.detach().abs().sum(1) + 0.5}
    out["opacity"] = _clamp(out["raw_opacity"], 0.0, 1.0, pass_opacity)
    out["rgb"] = out["raw_rgb"] = out["scale_rgb"] = None
    if colour is not None:
        coefs = torch.cat(colour, dim=1) if isinstance(colour, (tuple, list)) else colour
        cterms = B[:, :, None] * coefs[:, :ncoef]
        raw = cterms.sum(1) + 0.5
        out["raw_rgb"], out["scale_rgb"] = raw, cterms.detach().abs().sum(1) + 0.5
        rgb = _clamp(raw, 0.0, None, pass_rgb)
        if mask is not None:
            rgb = torch.where(mask.reshape(-1, 1), rgb, torch.full_like(rgb, 0.5).detach())
        out["rgb"] = rgb
    return out


def near_bound(raw, scale, lo, hi=None):
    """Samples within AMBIGUOUS (relative to their rounding scale) of a clamp bound."""
    near = (raw - lo).abs() <= AMBIGUOUS * scale
    if hi is not None:
        near |= (raw - hi).abs() <= AMBIGUOUS * scale
    return near
