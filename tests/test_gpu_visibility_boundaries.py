"""The transient visibility kernels at their boundaries against the float64 oracle (oracle/visibility_oracle.py, oracle/loss_oracle.py).

K32 / K33 (csrc/visibility.cu): every grid configuration of GRID_CONFIGS, whose levels wrap (the last pixel column and row reach
corner res_l, which the % sends to the next row or the start) on different sets of levels, including fp32 scales two ulp under a half
that do not wrap, an exact half, all-integer scales and a level of scale 0 with one cell; images of 2 pixels along an axis, 16 x 16
(every pixel's frac 0.5 at scale 15), 31 x 17 (odd columns on cell boundaries at scale 15), 37 x 50 and 1080p.  Each level is held to
its own bar: the forward within 1e-6 (the last row and column separately), the gradient within max(8 e32, 1e-6) of the level's
largest entry, e32 being the distance of a float32 scatter-add in pixel order from float64; vertices no pixel reaches are exactly
0, two backwards are bit-identical, K33 agrees with the atomic scatter of the same coordinates, and only the selected grid gets a
gradient.

The visibility MLP (csrc/appearance.cu with one output): every accepted shape, at row counts around the forward and backward tile
and past three waves of chunks of the persistent CTAs; each parameter tensor against its own largest entry, and bit-identical
weight gradients across two runs.

K34 / K35: every (H, W) of EDGES^2, 37 x 50, 270 x 480 and 1080p, every content kind of loss_oracle, six visibility maps, five
masks, lambda in {0, 0.2, 1}, vis_reg_factor in {0, 0.2} and the cotangent in {1, 0.37, 0}; each statistic within max(8 e32,
floor) and the image and visibility gradients per pixel class (the 5-pixel border, the tile seams, the interior), each class against
its own largest float64 entry.  Exact identities: visibility 1 without a mask is K9/K10, a mask of all True is no mask, an all-False
mask or a zero visibility leaves only the regulariser, and the visibility gradient does not change the image gradient.

The module prints, per family, the largest error / bar ratio it met."""
import numpy as np
import pytest
import torch

from oracle import loss_oracle as LO
from oracle import visibility_oracle as V
from oracle.appearance_oracle import mlp as oracle_mlp
from test_appearance_shapes_cpu import launch

pytestmark = pytest.mark.gpu
DEV = "cuda"
MARGIN = 8.0
RATIOS = {}              # family -> largest error / bar


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    for family, r in sorted(RATIOS.items()):
        print(f"\n{family}: largest error / bar: {r:.3g}")


def _note(family, err, bar):
    if bar > 0:
        RATIOS[family] = max(RATIOS.get(family, 0.0), err / bar)


# ---- K32 / K33 ------------------------------------------------------------------------------------------------------------------
GRID_CONFIGS = [(4, 16, 1.405), (8, 16, 1.405), (12, 16, 1.405), (16, 16, 1.405), (8, 16, 2.0), (8, 1, 2.0), (4, 1, 1.5),
                (12, 16, 1.5), (16, 4, 1.5)]
GRID_SIZES = [(2, 2), (2, 64), (64, 2), (16, 16), (31, 17), (37, 50)]           # (W, H)
GRID_CASES = ([(c, W, H) for c in GRID_CONFIGS for W, H in GRID_SIZES]
              + [((8, 16, 1.405), 1920, 1080), ((16, 16, 1.405), 1920, 1080)])
F32_EPS = float(np.finfo(np.float32).eps) / 2                                  # unit roundoff


def _level_corners(u, v, level, dev):
    idx, w = V.corners(u, v, [level])[0]
    return (idx - level[3]).to(dev), w.to(dev)


@pytest.mark.parametrize("cfg,W,H", GRID_CASES, ids=[f"{c[0]}-{c[1]}-{c[2]}-{W}x{H}" for c, W, H in GRID_CASES])
def test_uv_grid_levels_against_the_oracle(cfg, W, H):
    from b200gs import ops
    grid = dict(n_levels=cfg[0], base_resolution=cfg[1], per_level_scale=cfg[2])
    n_params, n_levels = V.n_params(*cfg), cfg[0]
    g = torch.Generator(device=DEV).manual_seed(W * 7 + H + 131 * n_levels + cfg[1])
    G = [torch.zeros(n_params, device=DEV).requires_grad_(True) for _ in range(3)]
    with torch.no_grad():
        G[1].uniform_(-1, 1, generator=g)
    v_enc = torch.rand(W * H, 2 * n_levels, device=DEV, generator=g) * 2 - 1
    enc = ops.uv_grid_encode(G, torch.tensor([1], device=DEV), width=W, height=H, selected=1, **grid)
    enc.backward(v_enc)
    k33 = G[1].grad.view(-1, 2)
    assert G[0].grad is None and G[2].grad is None                     # only the selected image's grid gets a gradient
    (again,) = torch.autograd.grad(ops.uv_grid_encode(G, torch.tensor([1], device=DEV), width=W, height=H, selected=1, **grid), G[1], v_enc)
    assert torch.equal(again.view(-1, 2), k33)                          # K33 gathers in a fixed order
    u, v = V.pixel_uv(W, H)
    uv = torch.from_numpy(np.stack([u, v], 1)).to(DEV)
    enc_uv = ops.uv_grid_encode(G, 1, uv=uv, **grid)
    assert torch.equal(enc_uv, enc)                                     # the same fp32 coordinates, the same corners and weights
    (scatter,) = torch.autograd.grad(enc_uv, G[1], v_enc)
    scatter = scatter.view(-1, 2)

    P = G[1].detach().double().view(-1, 2)
    enc64 = enc.detach().double().view(H, W, n_levels, 2)
    d64 = v_enc.double().view(-1, n_levels, 2)
    d32_cpu = v_enc.view(-1, n_levels, 2).cpu()
    for l, level in enumerate(V.levels(*cfg)):
        size, offset = level[2], level[3]
        idx, w = _level_corners(u, v, level, DEV)
        what = (cfg, W, H, l)
        # forward: the level's two columns, and the last column and row on their own
        ref = (P[idx + offset] * w.unsqueeze(-1)).sum(1).view(H, W, 2)
        diff = (enc64[:, :, l] - ref).abs()
        for part in (diff, diff[:, -1], diff[-1]):
            err = float(part.max())
            _note("K32 forward (bar 1e-6)", err, 1e-6)
            assert err <= 1e-6, what
        # backward: float64 scatter, and the float32 scatter in pixel order for e32
        contrib = w.unsqueeze(-1) * d64[:, l].unsqueeze(1)                                  # [n, 4, 2]
        r64 = torch.zeros(size, 2, dtype=torch.float64, device=DEV).index_add_(0, idx.reshape(-1), contrib.reshape(-1, 2))
        src32 = (w.cpu().unsqueeze(-1) * d32_cpu[:, l].double().unsqueeze(1)).float()
        s32 = torch.zeros(size, 2).index_add_(0, idx.cpu().reshape(-1), src32.reshape(-1, 2))
        e32 = float((s32.double() - r64.cpu()).abs().max())
        kl = k33[offset:offset + size]
        scale = float(r64.abs().max())
        err = float((kl.double() - r64).abs().max())
        bar = max(MARGIN * e32, 1e-6 * scale)
        _note("K33 gradient (bar max(8 e32, 1e-6 x level max))", err, bar)
        assert err <= bar, (what, err, e32, scale)
        # exact zeros: vertices no pixel reaches, padding in [res^2, size) included
        reached = torch.zeros(size, dtype=torch.bool, device=DEV)
        reached[idx.reshape(-1)] = True
        assert not kl[~reached].any(), what
        # the atomic scatter of the same coordinates: each sum within the rounding of both orders and of the rounded products
        n_v = torch.bincount(idx.reshape(-1), minlength=size).double().unsqueeze(-1)
        s_abs = torch.zeros(size, 2, dtype=torch.float64, device=DEV).index_add_(0, idx.reshape(-1), contrib.abs().reshape(-1, 2))
        gap = (kl.double() - scatter[offset:offset + size].double()).abs()
        bound = (2 * n_v + 1) * F32_EPS * s_abs
        _note("K33 against the atomic scatter (bar (2 n + 1) u sum|w d|)", float((gap / bound.clamp_min(1e-300)).max()), 1.0)
        assert bool((gap <= bound).all()), (what, float(gap.max()))


# ---- the visibility MLP ------------------------------------------------------------------------------------------------------
MLP_SHAPES = [(f, h, l) for f in (8, 16, 24, 32) for h in (64, 128) for l in (2, 3, 4)]
EMBED = 128


def mlp_rows(f, h, l):
    _, _, r_fwd, chunk_fwd = launch((f, -1, h, l, 1), False)
    _, _, r_bwd, chunk_bwd = launch((f, -1, h, l, 1), True)
    rows = {1, 3 * 132 * chunk_fwd + 17, 3 * 132 * chunk_bwd + 17}
    for r in (r_fwd, r_bwd):
        rows |= {r - 1, r, r + 1}
    return sorted(rows)


def mlp_case(n, f, h, l, seed):
    g = torch.Generator().manual_seed(seed)
    dims = [f + EMBED] + [h] * (l - 1) + [1]
    weights = [(torch.rand(b, a, generator=g) * 2 - 1) * 2 / a ** 0.5 for a, b in zip(dims[:-1], dims[1:])]
    biases = [(torch.rand(b, generator=g) * 2 - 1) * 0.5 for b in dims[1:]]
    return torch.rand(n, f, generator=g) * 2 - 1, torch.randn(EMBED, generator=g), weights, biases, torch.randn(n, generator=g)


def kink_rows(enc, emb, weights, biases, eps=1e-5):
    """rows with a hidden pre-activation within eps of 0 in float64, where fp32 may take the other side of the ReLU"""
    h = torch.cat([enc.double(), emb.double().reshape(1, -1).expand(enc.shape[0], -1)], 1)
    near = torch.zeros(enc.shape[0], dtype=torch.bool, device=enc.device)
    for w, b in zip(weights[:-1], biases[:-1]):
        pre = h @ w.double().T + b.double()
        near |= (pre.abs() < eps).any(1)
        h = pre.relu()
    return near


def contribution_mass(enc, emb, weights, biases, cot):
    """float64, per entry of each gradient (enc, embedding, weights, biases): the sum of the magnitudes of the row contributions it
    adds up.  Where the rows cancel (the output bias sums cot s (1 - s) over every row) the gradient is far smaller than this sum,
    and a float32 sum of the contributions carries rounding of the order of u times it."""
    n = enc.shape[0]
    h = [torch.cat([enc, emb.reshape(1, -1).expand(n, -1)], 1)]
    zs = []
    for w, b in zip(weights, biases):
        zs.append(h[-1] @ w.T + b)
        h.append(zs[-1].relu())
    s = torch.sigmoid(zs[-1])
    delta = cot.reshape(-1, 1) * s * (1 - s)
    gw, gb = [None] * len(weights), [None] * len(weights)
    for i in reversed(range(len(weights))):
        gw[i], gb[i] = delta.abs().T @ h[i].abs(), delta.abs().sum(0)
        if i:
            delta = (delta @ weights[i]) * (zs[i - 1] > 0)
    f = enc.shape[1]
    w0 = weights[0].abs()
    return [delta.abs() @ w0[:, :f], delta.abs().sum(0) @ w0[:, f:]] + gw + gb


@pytest.mark.parametrize("f,h,l", MLP_SHAPES, ids=[f"f{f}-h{h}-l{l}" for f, h, l in MLP_SHAPES])
def test_visibility_mlp_every_shape_and_tile_edge(f, h, l):
    from b200gs import ops
    for n in mlp_rows(f, h, l):
        enc, emb, weights, biases, cot = mlp_case(n, f, h, l, seed=n + 1000 * f + h + l)
        d = [t.to(DEV).requires_grad_(True) for t in [enc, emb] + weights + biases]
        near = kink_rows(d[0].detach(), d[1].detach(), [t.detach() for t in d[2:2 + l]], [t.detach() for t in d[2 + l:]])
        assert int(near.sum()) <= max(1, n // 50), (n, int(near.sum()))
        cot = cot.to(DEV)
        cot[near] = 0
        out = ops.visibility_mlp(d[0], d[1], d[2:2 + l], d[2 + l:])
        out.backward(cot)
        again = torch.autograd.grad(ops.visibility_mlp(d[0], d[1], d[2:2 + l], d[2 + l:]), d[2:], cot)
        for a, b in zip(d[2:], again):
            assert torch.equal(a.grad, b), (n, "weight gradients are bit-identical across runs")
        r = [t.detach().double().requires_grad_(True) for t in d]           # float64 on the GPU
        ref = oracle_mlp(r[0], r[1], r[2:2 + l], r[2 + l:])[:, 0]
        (ref * cot.double()).sum().backward()
        mass = contribution_mass(*[t.detach() for t in r[:2]], [t.detach() for t in r[2:2 + l]], [t.detach() for t in r[2 + l:]],
                                 cot.double())
        err = float((out.detach().double() - ref.detach()).abs().max())
        _note("visibility MLP output (bar 2e-5)", err, 2e-5)
        assert err <= 2e-5, n
        for k, (a, b, m) in enumerate(zip(d, r, mass)):
            # each tensor against its own largest entry, or, where the rows cancel, 8 u times the magnitude of what is summed
            scale = float(b.grad.abs().max())
            bar = torch.clamp(MARGIN * F32_EPS * m.reshape(b.grad.shape), min=1e-4 * scale)
            err = (a.grad.double() - b.grad).abs()
            _note("visibility MLP gradients (bar max(1e-4 x tensor max, 8 u sum|row terms|))", float((err / bar).max()), 1.0)
            assert bool((err <= bar).all()), (n, k, float(err.max()), scale)


# ---- K34 / K35 ---------------------------------------------------------------------------------------------------------------
EDGES = [1, 2, 5, 6, 10, 11, 15, 16, 17, 26, 27, 32, 33]         # test_gpu_loss.EDGES
VIS_KINDS = ("uniform", "binary", "one", "zero", "near_one", "sigmoid")
MASK_KINDS = ("none", "all", "nothing", "random", "seams")
FLOOR = {"l1": 1e-6, "ssim": 5e-6, "loss": 2e-6, "reg": 1e-6}
GRAD_FLOOR = 1e-4


def visibility_map(kind, H, W, g):
    if kind == "uniform":
        return torch.rand(H, W, generator=g)
    if kind == "binary":
        return (torch.rand(H, W, generator=g) < 0.5).float()
    if kind == "one":
        return torch.ones(H, W)
    if kind == "zero":
        return torch.zeros(H, W)
    if kind == "near_one":
        return 1 - 1e-3 * torch.rand(H, W, generator=g)
    y, x = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    return torch.sigmoid(3 * torch.sin(x / 7 + 0.3) * torch.cos(y / 5 - 0.2))


def keep_mask(kind, H, W, g):
    if kind == "none":
        return None
    if kind == "all":
        return torch.ones(H, W, dtype=torch.bool)
    if kind == "nothing":
        return torch.zeros(H, W, dtype=torch.bool)
    if kind == "random":
        return torch.rand(H, W, generator=g) < 0.8
    y, x = torch.arange(H)[:, None], torch.arange(W)[None, :]                     # holes on the 16-pixel tile seams
    return ~((((x % 16 == 0) | (x % 16 == 15)) & (y % 32 < 20)) | (((y % 16 == 0) | (y % 16 == 15)) & (x % 32 >= 12)))


def loss_inputs(kind, vis_kind, mask_kind, H, W, seed):
    img, gt = LO.case(kind, 3, H, W, seed)
    g = torch.Generator().manual_seed(seed + 1)
    return img, gt, visibility_map(vis_kind, H, W, g), keep_mask(mask_kind, H, W, g)


def oracle(img, gt, vis, mask, lam, reg, up, dtype, dev):
    x = img.to(dev, dtype, copy=True).requires_grad_(True)
    w = vis.to(dev, dtype, copy=True).requires_grad_(True)
    with torch.backends.cudnn.flags(enabled=False, allow_tf32=False):
        loss, l1, s, r = V.masked_loss(x, gt.to(dev, dtype), w, None if mask is None else mask.to(dev), lam, reg)
        loss.backward(torch.tensor(up, dtype=dtype, device=dev))
    return {"loss": float(loss.detach()), "l1": float(l1), "ssim": float(s), "reg": float(r), "v_image": x.grad.double(), "v_vis": w.grad.double()}


def kernel(img, gt, vis, mask, lam, reg, up, vis_grad=True):
    from b200gs import ops
    x = img.to(DEV).requires_grad_(True)
    w = vis.to(DEV).requires_grad_(vis_grad)
    loss, stats = ops.visibility_l1_ssim_loss(x, gt.to(DEV), w, None if mask is None else mask.to(DEV), lam, reg)
    loss.backward(torch.tensor(up, device=DEV))
    return {"loss": float(loss), "l1": float(stats[0]), "ssim": float(stats[1]), "reg": float(stats[2]), "v_image": x.grad,
            "v_vis": w.grad, "stats": stats}


def pixel_classes(H, W, dev):
    y, x = torch.arange(H, device=dev)[:, None], torch.arange(W, device=dev)[None, :]
    border = (x < 5) | (x >= W - 5) | (y < 5) | (y >= H - 5)
    seam = ~border & ((x % 16 == 0) | (x % 16 == 15) | (y % 16 == 0) | (y % 16 == 15))
    return {"border": border, "seam": seam, "interior": ~border & ~seam}


def check_loss(kind, vis_kind, mask_kind, H, W, lam=0.2, reg=0.2, up=1.0, seed=0, dev="cpu"):
    img, gt, vis, mask = loss_inputs(kind, vis_kind, mask_kind, H, W, seed)
    r64 = oracle(img, gt, vis, mask, lam, reg, up, torch.float64, dev)
    r32 = oracle(img, gt, vis, mask, lam, reg, up, torch.float32, dev)
    k = kernel(img, gt, vis, mask, lam, reg, up)
    what = (kind, vis_kind, mask_kind, H, W, lam, reg, up)
    for q, floor in FLOOR.items():
        err, e32 = abs(k[q] - r64[q]), abs(r32[q] - r64[q])
        bar = max(MARGIN * e32, floor)
        _note(f"K34 {q} (bar max(8 e32, {floor:g}))", err, bar)
        assert err <= bar, (what, q, k[q], r64[q], e32)
    classes = pixel_classes(H, W, r64["v_image"].device)
    for name in ("v_image", "v_vis"):
        g64 = r64[name]
        got = k[name].to(g64.device).double().reshape(g64.shape)
        d_k, d_32 = (got - g64).abs(), (r32[name] - g64).abs()
        for cls, m in classes.items():
            if not bool(m.any()):
                continue
            m = m.expand_as(g64)
            err, e32, scale = float(d_k[m].max()), float(d_32[m].max()), float(g64.abs()[m].max())
            bar = max(MARGIN * e32, GRAD_FLOOR * scale)
            _note(f"K35 {name} per pixel class (bar max(8 e32, 1e-4 x class max))", err, bar)
            assert err <= bar, (what, name, cls, err, e32, scale)
    return k, (img, gt, vis, mask)


@pytest.mark.parametrize("H", EDGES)
def test_vis_loss_tile_edges(H):
    """every width of EDGES at this height; the content, visibility and mask turn over with the width"""
    for i, W in enumerate(EDGES):
        j = i + EDGES.index(H)
        check_loss(LO.KINDS[j % len(LO.KINDS)], VIS_KINDS[j % len(VIS_KINDS)], MASK_KINDS[j % len(MASK_KINDS)], H, W, seed=H * 100 + W)


@pytest.mark.parametrize("kind", LO.KINDS)
def test_vis_loss_content_visibility_and_mask(kind):
    for vk in VIS_KINDS:
        for mk in MASK_KINDS:
            check_loss(kind, vk, mk, 37, 50, seed=LO.KINDS.index(kind) * 31 + VIS_KINDS.index(vk) * 7 + MASK_KINDS.index(mk))


@pytest.mark.parametrize("kind", LO.KINDS)
def test_vis_loss_lambda_reg_and_cotangent(kind):
    i = 0
    for lam in (0.0, 0.2, 1.0):
        for reg in (0.0, 0.2):
            for up in (1.0, 0.37, 0.0):
                k, _ = check_loss(kind, VIS_KINDS[i % len(VIS_KINDS)], MASK_KINDS[i % len(MASK_KINDS)], 37, 50, lam, reg, up, seed=i)
                if up == 0.0:
                    assert not k["v_image"].any() and not k["v_vis"].any(), "a zero cotangent gives exact zeros"
                i += 1


LARGE = [(270, 480, kind, vk, mk) for kind, vk, mk in (("noise", "uniform", "random"), ("flat", "sigmoid", "seams"),
                                                       ("saturated", "binary", "none"), ("converged", "near_one", "all"))]
LARGE += [(1080, 1920, kind, vk, mk) for kind, vk, mk in (("noise", "sigmoid", "random"), ("flat", "near_one", "seams"),
                                                          ("hdr", "uniform", "none"))]


@pytest.mark.parametrize("H,W,kind,vk,mk", LARGE, ids=[f"{H}x{W}-{k}-{v}-{m}" for H, W, k, v, m in LARGE])
def test_vis_loss_large(H, W, kind, vk, mk):
    """the float64 and fp32 oracles on the GPU"""
    check_loss(kind, vk, mk, H, W, seed=H + W, dev=DEV)


# ---- exact identities --------------------------------------------------------------------------------------------------------
IDENTITY_SIZES = [(1, 1), (16, 16), (17, 33), (37, 50), (270, 480)]


@pytest.mark.parametrize("H,W", IDENTITY_SIZES)
@pytest.mark.parametrize("kind", ["noise", "flat", "saturated"])
def test_visibility_one_without_a_mask_is_the_plain_loss(H, W, kind):
    """w = 1.0 multiplies exactly, and the tile engine and the gradient expression are K9/K10's.  The two kernels are compiled
    separately and round the expression differently in its last places (measured on an H100: up to 2 ulp of the image's largest
    entry), so they are held to 4 ulp of that entry instead of bit equality"""
    from b200gs import ops
    img, gt = LO.case(kind, 3, H, W, H + W)
    for lam, up in ((0.2, 1.0), (1.0, 0.37), (0.0, 1.0)):
        k = kernel(img, gt, torch.ones(H, W), None, lam, 0.2, up)
        x = img.to(DEV).requires_grad_(True)
        loss, _ = ops.l1_ssim_loss(x, gt.to(DEV), lam)
        loss.backward(torch.tensor(up, device=DEV))
        ref = x.grad.cpu().numpy()
        gap = float(np.abs(k["v_image"].cpu().numpy() - ref).max())
        ulp = float(np.spacing(np.abs(ref).max()))
        _note("K35 at visibility 1 against K10 (bar 4 ulp of the largest entry)", gap, 4 * ulp)
        assert gap <= 4 * ulp, (lam, up, gap / ulp)


@pytest.mark.parametrize("H,W", IDENTITY_SIZES)
def test_mask_of_all_true_is_no_mask(H, W):
    img, gt, vis, _ = loss_inputs("noise", "uniform", "none", H, W, 5)
    a = kernel(img, gt, vis, None, 0.2, 0.2, 0.37)
    b = kernel(img, gt, vis, torch.ones(H, W, dtype=torch.bool), 0.2, 0.2, 0.37)
    assert torch.equal(a["stats"], b["stats"]) and a["loss"] == b["loss"]
    assert torch.equal(a["v_image"], b["v_image"]) and torch.equal(a["v_vis"], b["v_vis"])


@pytest.mark.parametrize("H,W", IDENTITY_SIZES)
@pytest.mark.parametrize("case", ["mask_nothing", "vis_zero"])
def test_nothing_weighted_leaves_only_the_regulariser(H, W, case):
    img, gt, vis, _ = loss_inputs("noise", "uniform", "none", H, W, 6)
    if case == "vis_zero":
        vis, mask = torch.zeros(H, W), None
    else:
        mask = torch.zeros(H, W, dtype=torch.bool)
    for reg, up in ((0.2, 1.0), (0.2, 0.37), (0.0, 1.0)):
        k = kernel(img, gt, vis, mask, 0.2, reg, up)
        # every pixel's SSIM is C1 C2 / (C1 C2), formed with the fast reciprocals: 1 within a few ulp
        assert k["l1"] == 0.0 and abs(k["ssim"] - 1.0) <= 1e-6, (k["l1"], k["ssim"])
        assert not k["v_image"].any()
        # -2 f (1 - v) up / (H W) in the kernel's fp32 order; the division may be the fast one (2 ulp)
        f32 = np.float32
        want = -(f32(up) * f32(2) * f32(reg) * (f32(1) - vis.numpy())) / (f32(W) * f32(H))
        got = k["v_vis"].cpu().numpy()
        assert (np.abs(got - want) <= 2 * np.spacing(np.abs(want))).all(), (reg, up, float(np.abs(got - want).max()))


@pytest.mark.parametrize("H,W", IDENTITY_SIZES)
def test_visibility_gradient_leaves_the_image_gradient_alone(H, W):
    for mk in ("none", "random"):
        img, gt, vis, mask = loss_inputs("noise", "uniform", mk, H, W, 7)
        a = kernel(img, gt, vis, mask, 0.2, 0.2, 0.37, vis_grad=True)
        b = kernel(img, gt, vis, mask, 0.2, 0.2, 0.37, vis_grad=False)
        assert b["v_vis"] is None and a["v_vis"] is not None
        assert torch.equal(a["v_image"], b["v_image"]) and torch.equal(a["stats"], b["stats"])
