"""float64 restatement of the learned exposure correction of internal/output_processors/exposure.py
(ExposureProcessorModule.forward, :112-143), gradients by autograd:

  a = sigmoid(P[id]),  P [n_appearances, 4 | 7]
  M = sigmoid(S[0]) / clamp_min(max(sigmoid(S[0])), 1e-4)         (the max detached)
  m(y, x) = bilinear interpolation of M at (y (s - 1) / (H - 1), x (s - 1) / (W - 1)), written out with torch's
            upsample_bilinear2d(align_corners=True) rule: lower cell floor(src), the upper one clipped to s - 1, and a source
            scale of 0 when the output has one pixel along the axis
  x_c = (a_c max_gray) (r_c m) [+ 2 a_{3+c} - 1],   c = x - (x - clamp(x, 0, 1)).detach(),   out = (c + 1e-5) ^ (a_last max_gamma)

``inputs`` builds seeded float32 test inputs whose parameters are pushed away from their initial values, with pixels that land
below 0, above 1 and on 0 and 1 after scaling, and exposure rows whose gamma lies below and above 1.
"""
import numpy as np
import torch

from oracle.bilagrid_oracle import weyl


def _axis(n_out, s):
    """lower cell, upper cell and upper weight per output pixel of one axis (float64)"""
    scale = (s - 1) / (n_out - 1) if n_out > 1 else 0.0
    src = scale * np.arange(n_out, dtype=np.float64)
    i0 = np.floor(src).astype(np.int64)
    i1 = np.where(i0 < s - 1, i0 + 1, i0)
    return torch.from_numpy(i0), torch.from_numpy(i1), torch.from_numpy(src - i0)


def shade_map(shade0, H, W):
    """m [H, W] from the shade parameter shade0 [s, s] (autograd through it; float64 for the oracle, any dtype and device for the
    torch chains the tests compare against)"""
    s = shade0.shape[-1]
    M = torch.sigmoid(shade0)
    M = M / M.detach().max().clamp_min(1e-4)
    y0, y1, ly = (t.to(M.device) for t in _axis(H, s))
    x0, x1, lx = (t.to(M.device) for t in _axis(W, s))
    ly, lx = ly.to(M.dtype), lx.to(M.dtype)
    ly, lx = ly[:, None], lx[None, :]
    top = (1 - lx) * M[y0][:, x0] + lx * M[y0][:, x1]
    bottom = (1 - lx) * M[y1][:, x0] + lx * M[y1][:, x1]
    return (1 - ly) * top + ly * bottom


def forward(render, params, appearance_id, shade, max_gray_scale=5.0, max_gamma=5.0, with_bias=False):
    """out [3, H, W] (float64 tensors in, autograd through render, params and shade); shade None: no shade correction.  An id
    outside the rows gives a NaN image."""
    if not 0 <= int(appearance_id) < params.shape[0]:
        return torch.full_like(render, float("nan"))
    a = torch.sigmoid(params[int(appearance_id)])
    img = render
    if shade is not None:
        img = img * shade_map(shade[0], render.shape[1], render.shape[2])[None]
    x = a[:3, None, None] * max_gray_scale * img
    if with_bias:
        x = x + (a[3:6, None, None] * 2. - 1.)
    x = x - (x - torch.clamp(x, 0., 1.)).detach()
    return torch.pow(x + 1e-5, a[-1] * max_gamma)


def near_zero(render, params, appearance_id, shade, with_bias=False, max_gray_scale=5.0, eps=1e-3):
    """[3, H, W] mask of the pixels whose scaled value x lies within eps of 0 but not on it, with a bias.  There
    d v_render / dx relative to v_render is |gamma - 1| / (x + 1e-5), and x is a difference of terms of order 0.1-1 that a float32
    evaluation carries to about 1e-7, so v_render is known only to about 1e-2 of itself within 1e-5 of 0 and to 1e-4 of itself
    from eps = 1e-3 on.  Without a bias x is a product, exact to a few float32 roundings of itself, and no pixel is masked."""
    with torch.no_grad():
        r = torch.as_tensor(np.asarray(render, np.float64))
        a = torch.sigmoid(torch.as_tensor(np.asarray(params, np.float64))[int(appearance_id)])
        if shade is not None:
            r = r * shade_map(torch.as_tensor(np.asarray(shade, np.float64))[0], r.shape[1], r.shape[2])[None]
        x = a[:3, None, None] * max_gray_scale * r
        if with_bias:
            x = x + (a[3:6, None, None] * 2. - 1.)
    return ((x.abs() < eps) & (x != 0) & with_bias).numpy()


def vjp(render, params, appearance_id, shade, v_out, **cfg):
    """(out, v_render, v_params, v_shade or None) in float64 numpy for float arrays in"""
    r = torch.as_tensor(np.asarray(render, np.float64)).requires_grad_(True)
    P = torch.as_tensor(np.asarray(params, np.float64)).requires_grad_(True)
    S = None if shade is None else torch.as_tensor(np.asarray(shade, np.float64)).requires_grad_(True)
    out = forward(r, P, appearance_id, S, **cfg)
    out.backward(torch.as_tensor(np.asarray(v_out, np.float64)))
    return out.detach().numpy(), r.grad.numpy(), P.grad.numpy(), None if S is None else S.grad.numpy()


# gamma = sigmoid(P[:, -1]) max_gamma of the rows inputs() builds, for max_gamma = 5: below and above 1, the initial value 1 in
# row 1 and the largest in the last row
ROW_GAMMAS = (0.55, 1.0, 1.7, 0.8, 3.2)


def _logit(p):
    return float(np.log(p / (1 - p)))


def inputs(H, W, with_bias, shade_size, seed, n_appearances=5, max_gray_scale=5.0, max_gamma=5.0):
    """float32 (render [3,H,W], params [n, 4 | 7], shade [1, s, s] or None, v_out [3,H,W]).

    The colour gains a_c max_gray lie in about [0.6, 2.4], biases in about [-0.15, 0.15]; the render is in [-0.05, 1.1) so scaled
    pixels land below 0 and above 1.  Pixels 0-5 of the first row are 0 (x = 0 exactly where the bias of that channel is 0: the
    bias parameter of channel 0 is 0 in every row); pixels 6-11 are 0.4, which a gain of exactly 2.5 (a = 0.5, params 0, in
    channel 1 of every row) scales to 1 in float32 without shade correction.  The shade map is the initial 0.95 plus up to
    +-2 in logit."""
    n_params = 7 if with_bias else 4
    u = weyl((n_appearances, n_params), seed)
    params = np.empty((n_appearances, n_params))
    params[:, :3] = _logit(1. / max_gray_scale) + 2.0 * u[:, :3] - 0.6
    if with_bias:
        params[:, 3:6] = 0.6 * u[:, 3:6] - 0.3
        params[:, 3] = 0.0
    params[:, 1] = 0.0
    gam = np.resize(np.asarray(ROW_GAMMAS), n_appearances)
    params[:, -1] = [_logit(g / max_gamma) for g in gam]
    render = (1.15 * weyl((3, H, W), seed + 1) - 0.05).astype(np.float32)
    flat = render.reshape(3, -1)
    flat[:, :min(6, H * W)] = 0.0
    flat[:, 6:12] = 0.4
    shade = None
    if shade_size > 0:
        shade = (_logit(0.95) + 4.0 * weyl((1, shade_size, shade_size), seed + 2) - 2.0).astype(np.float32)
    v_out = (2.0 * weyl((3, H, W), seed + 3) - 1.0).astype(np.float32)
    return render, params.astype(np.float32), shade, v_out
