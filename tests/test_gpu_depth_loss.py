"""Inverse-depth loss K27-K31 (csrc/depth_loss.cu on the tile engine csrc/ssim.cuh; b200gs.metrics.inverse_depth_loss) on the GPU
against the float64 oracle (oracle/depth_loss_oracle.py), at its tile and window edges and on every kind of oracle.case content.

Error model (as tests/test_gpu_loss.py): each quantity (loss, l-term, SSIM, v_pred) stays within max(8 e32, floor), e32 being the
float32 oracle's distance from the float64 oracle on the same input, both on the GPU without cuDNN or TF32.  Near an l1 sign flip
or an E[x^2] - mu^2 cancellation float32 itself cannot do better, so no constant bound fits converged, flat or saturated maps.
Gradients are checked on five pixel classes, each against its own largest float64 entry: the 5-pixel image edge, the ring 5-10
pixels in (where the full-window region ends), tile seams (x or y % 16 in {0, 15}), pred's extremum pixels (which carry the data-
range gradient) and the interior.

Sizes: l1+ssim at every (H, W) in SSIM_EDGES^2; l1 and l2 with and without a mask over L_EDGES^2; every kind x every (loss type,
norm, mask) at MIDDLE; noise, converged and saturated at 1080p; saturated and lone-extremum content at 2160x3840, where the
statistics grid is at its 1024-CTA cap.  Also: the range tie, a flat pred, two flat maps (NaN), sgn(0) = 0, cotangents, masked
pixels, strided maps and masks, argument errors and bit-identical backwards.
"""
import numpy as np
import pytest
import torch

from oracle import depth_loss_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
W_SSIM = 0.2
SSIM_EDGES = [11, 12, 15, 16, 17, 20, 21, 22, 26, 27, 31, 32, 33]     # the full-window region's edge on both sides of a tile seam
L_EDGES = [1, 2, 5, 15, 16, 17, 33]
MIDDLE = [(37, 50), (96, 128), (270, 480), (13, 200), (200, 13)]
COMBOS = [(t, n, m) for t in ("l1", "l2") for n in O.NORMS for m in (False, True)] + [("l1+ssim", n, False) for n in O.NORMS]
MARGIN = 8.0                      # x e32
REL_FLOOR = {"loss": 2e-6, "term": 2e-6}
SSIM_FLOOR = 5e-6
GRAD_FLOOR = 1e-4                 # x the largest |float64 gradient| of the pixel class
RATIOS = {}                       # kind -> [largest error / e32 where 8 e32 is the bound, largest error / bound]


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    for kind, (r, used) in sorted(RATIOS.items()):
        print(f"\nK27-K31 on {kind}: largest kernel error / e32 where 8 e32 > floor: {r:.3g}; largest error / bound: {used:.3g}")


def _note(kind, err, e32, floor):
    r = RATIOS.setdefault(kind, [0.0, 0.0])
    if MARGIN * e32 > floor:
        r[0] = max(r[0], err / e32)
    if max(MARGIN * e32, floor) > 0:
        r[1] = max(r[1], err / max(MARGIN * e32, floor))


def kernel(gt, pred, loss_type, cfg, up=1.0, mask=None):
    """loss, l-term, SSIM and v_pred (float64 numpy) of inverse_depth_loss; the mask, when cfg has one, as a [3,H,W] bool"""
    from b200gs.metrics import inverse_depth_loss
    cfg = dict(cfg)
    if mask is not None:
        cfg["mask"] = mask
    elif cfg.get("mask") is not None:
        cfg["mask"] = torch.from_numpy(np.ascontiguousarray(cfg["mask"]))[None].repeat(3, 1, 1).to(DEV)
    p = (pred if torch.is_tensor(pred) else torch.from_numpy(pred).to(DEV)).detach().requires_grad_(True)
    g = gt if torch.is_tensor(gt) else torch.from_numpy(gt).to(DEV)
    loss, stats = inverse_depth_loss(g, p, loss_type=loss_type, ssim_weight=W_SSIM, **cfg)
    loss.backward(torch.tensor(up, device=DEV))
    s = stats.cpu().double().numpy()
    return {"loss": float(loss.detach()), "term": float(s[0]), "ssim": float(s[1]), "grad": p.grad.cpu().double().numpy()}


def oracle(gt, pred, loss_type, cfg, dtype, tie_share=O.TIE_SHARE):
    loss, term, s, v = O.vjp(gt, pred, DEV, dtype, loss_type=loss_type, ssim_weight=W_SSIM, separable=True, tie_share=tie_share, **cfg)
    return {"loss": loss, "term": term, "ssim": s, "grad": v}


def pixel_classes(pred):
    H, W = pred.shape
    y, x = np.arange(H)[:, None], np.arange(W)[None, :]
    d = np.minimum(np.minimum(x, W - 1 - x), np.minimum(y, H - 1 - y))
    ext = (pred == pred.max()) | (pred == pred.min())
    edge, ring = (d < 5) & ~ext, (d >= 5) & (d < 10) & ~ext
    seam = (d >= 10) & ((x % 16 == 0) | (x % 16 == 15) | (y % 16 == 0) | (y % 16 == 15)) & ~ext
    return {"edge": edge, "ring": ring, "seam": seam, "extremum": ext, "interior": ~(edge | ring | seam | ext)}


def check(kind, gt, pred, loss_type, cfg, up=1.0, mask=None):
    """the kernel against float64: every quantity within max(8 e32, floor), finite wherever the float64 oracle is, masked pixels
    exactly 0; returns the kernel's outputs and the float64 oracle's"""
    r64, r32 = oracle(gt, pred, loss_type, cfg, torch.float64), oracle(gt, pred, loss_type, cfg, torch.float32)
    k = kernel(gt, pred, loss_type, cfg, up, mask)
    what = (kind, pred.shape, loss_type, {q: v for q, v in cfg.items() if q != "mask"}, "mask" in cfg, up)
    for q in ("loss", "term", "ssim"):
        if q == "ssim" and loss_type != "l1+ssim":
            assert np.isnan(k[q]), what
            continue
        if not np.isfinite(r64[q]):
            continue
        assert np.isfinite(k[q]), (what, q)
        err, e32 = abs(k[q] - r64[q]), abs(r32[q] - r64[q])
        floor = SSIM_FLOOR if q == "ssim" else REL_FLOOR[q] * abs(r64[q])
        if q == "loss" and loss_type == "l1+ssim":
            floor += W_SSIM * SSIM_FLOOR                                   # the loss holds w x SSIM
        _note(kind, err, e32, floor)
        assert err <= max(MARGIN * e32, floor), (what, q, k[q], r64[q], e32)
    g64, g32, gk = up * r64["grad"], up * r32["grad"], k["grad"]
    fin = np.isfinite(g64)
    assert np.isfinite(gk[fin]).all(), what
    d_k, d_32 = np.abs(gk - g64) - sign_slack(gt, pred, loss_type, cfg, up), np.abs(g32 - g64)
    for name, m in pixel_classes(pred).items():
        m = m & fin
        if not m.any():
            continue
        err, e32, scale = d_k[m].max(), d_32[m].max(), np.abs(g64[m]).max()
        _note(kind, err, e32, GRAD_FLOOR * scale)
        assert err <= max(MARGIN * e32, GRAD_FLOOR * scale), (what, name, err, e32, scale)
    if cfg.get("mask") is not None:
        assert not gk[~cfg["mask"]].any(), (what, "masked pixels get exactly 0")
    return k, r64


def sign_slack(gt, pred, loss_type, cfg, up):
    """per pixel, the gradient error an l1 sign may add where a' and b' lie within 8 float32 ulps of each other: there the
    float32 maps (the kernel's normalisation constants are rounded, not the oracle's) decide the sign of a' - b', and any of
    -1, 0 and 1 is right"""
    if loss_type == "l2":
        return 0.0
    norm = ("normalized" if cfg.get("normalized") else "median" if cfg.get("median") is not None
            else "mean" if cfg.get("mean_normalization") else "none")
    b = O.normalize_pred(pred, norm, gt)
    a = gt.astype(np.float64) / (gt.astype(np.float64).mean() if norm == "mean" else 1.0)
    if cfg.get("mask") is not None:
        a, b = a * cfg["mask"], b * cfg["mask"]
    chain = {"normalized": 1.0 / (np.ptp(pred.astype(np.float64)) + 1e-8), "median": 1.0 / O.MEDIAN,
             "mean": 1.0 / gt.astype(np.float64).mean(), "none": 1.0}[norm]
    coef = (1.0 - W_SSIM if loss_type == "l1+ssim" else 1.0) / pred.size * chain * abs(up)
    return np.where(np.abs(a - b) <= 2.0 ** -21 * np.maximum(np.abs(a), np.abs(b)), 2.0 * coef * (1 + 1e-6), 0.0)


def seed_of(kind, H, W, i=0):
    return H * 1000 + W + 7919 * O.KINDS.index(kind) + 104729 * i


# ---- sizes ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", SSIM_EDGES)
def test_ssim_tile_and_window_edges(H):
    """l1+ssim at every width of SSIM_EDGES at this height, cycling through the four norms: the full-window region, 5 pixels in
    from the image edge, on either side of a 16-pixel tile seam"""
    for j, W in enumerate(SSIM_EDGES):
        norm = O.NORMS[(SSIM_EDGES.index(H) + j) % 4]
        gt, pred, cfg = O.case("noise", H, W, norm, seed_of("noise", H, W))
        check("noise", gt, pred, "l1+ssim", cfg)


@pytest.mark.parametrize("H", L_EDGES)
def test_l1_l2_tile_edges(H):
    for j, W in enumerate(L_EDGES):
        for i, (loss_type, masked) in enumerate((("l1", False), ("l1", True), ("l2", False), ("l2", True))):
            norm = O.NORMS[(L_EDGES.index(H) + j + i) % 4]
            gt, pred, cfg = O.case("noise", H, W, norm, seed_of("noise", H, W, i), masked=masked)
            check("noise", gt, pred, loss_type, cfg)


@pytest.mark.parametrize("kind", O.KINDS)
@pytest.mark.parametrize("H,W", MIDDLE)
def test_middle_sizes(H, W, kind):
    for i, (loss_type, norm, masked) in enumerate(COMBOS):
        gt, pred, cfg = O.case(kind, H, W, norm, seed_of(kind, H, W, i), masked=masked)
        check(kind, gt, pred, loss_type, cfg)


@pytest.mark.parametrize("kind", ["noise", "converged", "saturated"])
def test_1080p(kind):
    for i, (loss_type, norm, masked) in enumerate(COMBOS):
        gt, pred, cfg = O.case(kind, 1080, 1920, norm, seed_of(kind, 1080, 1920, i), masked=masked)
        check(kind, gt, pred, loss_type, cfg)


FOUR_K = [("l1+ssim", "normalized"), ("l1", "mean"), ("l2", "median")]


@pytest.mark.parametrize("kind", ["saturated", "lone"])
def test_2160x3840_at_the_statistics_grid_cap(kind):
    """8.3 M pixels: K27 runs its 1024-CTA cap (4050 CTAs of 2048 pixels would be needed) and K28 adds a full row of partials"""
    from b200gs import _lib
    H, W = 2160, 3840
    n, tiles = H * W, (H // 16) * (W // 16)
    for t in range(3):
        assert _lib.lib().b200gs_depth_loss_workspace_bytes(H, W, t) == 4 * (16 + 8 * 1024 + 8 * tiles + (3 * n if t == 2 else 0))
    assert -(-n // 2048) > 1024
    for i, (loss_type, norm) in enumerate(FOUR_K):
        gt, pred, cfg = O.case(kind, H, W, norm, seed_of(kind, H, W, i))
        check(kind, gt, pred, loss_type, cfg)


# ---- exact properties -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("norm", ["none", "median", "mean"])
def test_range_tie_gives_pred_its_tie_share_of_the_dr_gradient(norm):
    """range(gt') == range(pred') exactly in float32 and float64.  The oracle's tie rule is O.TIE_SHARE (torch.maximum: half to each
    side); at pred's extremum pixels the kernel's gradient is the untied gradient's dr part times that share.  The rule is open:
    torchmetrics may take Python's max, which gives all of it to gt' on a tie; changing O.TIE_SHARE and the kernel's H_SHARE moves
    this test with it."""
    gt, pred, cfg = O.case("tie", 96, 128, norm, 17)
    k, _ = check("tie", gt, pred, "l1+ssim", cfg)
    lo = oracle(gt, pred, "l1+ssim", cfg, torch.float64, tie_share=0.0)["grad"]      # gt' takes the whole dr gradient
    hi = oracle(gt, pred, "l1+ssim", cfg, torch.float64, tie_share=1.0)["grad"]      # pred' takes it
    ext = (pred == pred.max()) | (pred == pred.min())
    dr_part = hi - lo
    assert not dr_part[~ext].any()
    want = lo + O.TIE_SHARE * dr_part
    for side in (pred == pred.max(), pred == pred.min()):            # the dr part per pixel is 1 / (the number of tied pixels)
        assert np.abs(dr_part[side]).min() > 0
        assert np.abs(k["grad"][side] - want[side]).max() <= 0.02 * np.abs(dr_part[side]).min()


@pytest.mark.parametrize("norm", O.NORMS)
def test_flat_pred(norm):
    """a constant pred: every pixel is at once pred''s max and min, so its two dr terms cancel to 0 (under min-max normalisation
    pred' = 0 with the divisor 1e-8); l1 and l2 too, and sgn(0) = 0 where gt' equals pred' exactly"""
    for i, loss_type in enumerate(("l1+ssim", "l1", "l2")):
        gt, pred, cfg = O.case("flat_pred", 37, 50, norm, 40 + i)
        k, r64 = check("flat_pred", gt, pred, loss_type, cfg)
        if loss_type == "l1":
            eq = (gt == pred) if norm == "mean" else (gt == O.pred32(pred, norm))
            assert eq.sum() > 100 and not k["grad"][eq].any()


@pytest.mark.parametrize("norm", ["none", "normalized", "median"])
def test_two_flat_maps_give_nan(norm):
    """gt' and pred' both flat at 0 under l1+ssim (a view where nothing is rendered and the depth map is empty): dr = 0, so
    C1 = C2 = 0 and SSIM is 0 / 0.  The float64 oracle gives NaN and so must the kernel, not a finite number.  (At a nonzero
    constant the variances E[x^2] - mu^2 are of the order of the float32 window's distance from a unit sum, and whether they round
    to 0 depends on the summation order, so no precision defines the answer there.)"""
    gt = np.zeros((37, 50), np.float32)
    pred = np.full((37, 50), 0.25 if norm == "normalized" else 0.0, np.float32)
    cfg = {"normalized": norm == "normalized", "median": O.MEDIAN if norm == "median" else None}
    r64 = oracle(gt, pred, "l1+ssim", cfg, torch.float64)
    k = kernel(gt, pred, "l1+ssim", cfg)
    assert np.isnan(r64["loss"]) and np.isnan(r64["ssim"]) and np.isnan(r64["grad"]).all()
    assert np.isnan(k["loss"]) and np.isnan(k["ssim"]) and np.isnan(k["grad"]).all()
    assert k["term"] == r64["term"] == 0.0


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("norm", O.NORMS)
def test_l1_subgradient_at_zero_is_zero(norm, masked):
    """where gt' == pred' exactly in float32 (the maps the reference computes), the l1 gradient is exactly 0: torch.abs' sgn(0)"""
    gt, pred, cfg = O.case("converged", 96, 128, norm, 23, masked=masked)
    k, _ = check("converged", gt, pred, "l1", cfg)
    eq = (gt == pred) if norm == "mean" else (gt == O.pred32(pred, norm))
    assert eq.mean() > 1 / 8 and not k["grad"][eq].any()
    assert k["grad"][~eq & cfg.get("mask", True)].all()


CASES_UP = [("saturated", "l1+ssim", "normalized", False), ("converged", "l2", "mean", True), ("noise", "l1", "median", False),
            ("lone", "l1+ssim", "none", False)]


@pytest.mark.parametrize("kind,loss_type,norm,masked", CASES_UP)
def test_cotangents(kind, loss_type, norm, masked):
    """a zero cotangent gives exact zeros; +-2^k scales v_pred bit-exactly; others stay within the error model"""
    gt, pred, cfg = O.case(kind, 96, 128, norm, 31, masked=masked)
    base = kernel(gt, pred, loss_type, cfg)["grad"]
    assert kernel(gt, pred, loss_type, cfg, up=0.0)["grad"].tolist() == np.zeros_like(base).tolist()
    for up in (2.0 ** -3, 2.0 ** 4, -1.0, -(2.0 ** 5)):
        assert np.array_equal(kernel(gt, pred, loss_type, cfg, up=up)["grad"], up * base), up
    for up in (-0.3, 3.0):
        check(kind, gt, pred, loss_type, cfg, up=up)


# ---- layouts and arguments --------------------------------------------------------------------------------------------------
def test_strided_maps_match_their_contiguous_copies():
    """pred as a transposed view and gt as a crop of a larger buffer give the contiguous inputs' results bit for bit"""
    gt, pred, cfg = O.case("saturated", 50, 37, "normalized", 5)
    want = kernel(gt, pred, "l1+ssim", cfg)
    p_t = torch.from_numpy(np.ascontiguousarray(pred.T)).to(DEV).t()
    big = torch.zeros(64, 80, device=DEV)
    big[3:53, 7:44] = torch.from_numpy(gt).to(DEV)
    g_crop = big[3:53, 7:44]
    assert not p_t.is_contiguous() and not g_crop.is_contiguous()
    got = kernel(g_crop, p_t, "l1+ssim", cfg)
    assert got["loss"] == want["loss"] and got["term"] == want["term"] and got["ssim"] == want["ssim"]
    assert np.array_equal(got["grad"], want["grad"])


@pytest.mark.parametrize("loss_type", ["l1", "l2"])
def test_mask_layouts(loss_type):
    """a non-square keep-mask (H != W, so reading it with its two strides swapped would read other pixels) as a [3,H,W] bool, a
    permuted [H,W,3] bool, a uint8 with 255 for keep, a stride-0 expand and a crop of a larger [H,W] buffer: the same results as the
    oracle with the plain mask, bit-identical to each other"""
    H, W = 50, 37
    gt, pred, cfg = O.case("noise", H, W, "mean", 9, masked=True)
    m = torch.from_numpy(cfg["mask"]).to(DEV)
    big = torch.zeros(64, 64, dtype=torch.bool, device=DEV)
    big[:H, :W] = m
    layouts = {
        "repeat": m[None].repeat(3, 1, 1),
        "hwc": m[:, :, None].repeat(1, 1, 3).permute(2, 0, 1),
        "uint8_255": (m.to(torch.uint8) * 255)[None].repeat(3, 1, 1),
        "expand": m[None].expand(3, H, W),
        "crop": big[:H, :W],
    }
    assert layouts["expand"].stride(0) == 0 and layouts["hwc"].stride()[1:] == (3 * W, 3) and layouts["crop"].stride() == (64, 1)
    want, _ = check("noise", gt, pred, loss_type, cfg, mask=layouts["repeat"])
    for name, mask in layouts.items():
        got = kernel(gt, pred, loss_type, cfg, mask=mask)
        assert got["loss"] == want["loss"] and got["term"] == want["term"] and np.array_equal(got["grad"], want["grad"]), name


def test_bad_arguments_raise():
    from b200gs.metrics import inverse_depth_loss
    a = torch.rand(20, 30, device=DEV)
    m = torch.ones(3, 20, 30, dtype=torch.bool, device=DEV)
    for gt, pred in ((a, a[:, :29]), (a[None], a[None]), (a.double(), a), (a, a.double()), (a.cpu(), a), (a, a.cpu()), (a, a.half())):
        with pytest.raises(ValueError):
            inverse_depth_loss(gt, pred)
    for mask in (m[:, :, :29], m.float(), m.cpu(), m[:, :19]):
        with pytest.raises(ValueError):
            inverse_depth_loss(a, a, mask=mask)
    with pytest.raises(ValueError):
        inverse_depth_loss(a[:10], a[:10], loss_type="l1+ssim")
    with pytest.raises(NotImplementedError):
        inverse_depth_loss(a, a, loss_type="l1+ssim", mask=m)


def test_two_backwards_at_2160x3840_are_bit_identical():
    gt, pred, cfg = O.case("saturated", 2160, 3840, "normalized", 3)
    first, second = kernel(gt, pred, "l1+ssim", cfg), kernel(gt, pred, "l1+ssim", cfg)
    assert first["loss"] == second["loss"] and first["term"] == second["term"] and first["ssim"] == second["ssim"]
    assert np.array_equal(first["grad"], second["grad"])
