"""The seeded content of oracle/depth_loss_oracle.case has the property each kind claims, under every normalisation, without a GPU;
and the oracle's options (separable window, device, dtype, tie rule) leave its float64 results where they were."""
import numpy as np
import pytest
import torch

from oracle import depth_loss_oracle as O

SIZES = [(37, 50), (96, 128), (13, 200)]


def maps(kind, H, W, norm, seed=3):
    """gt' and pred' in float32 the way the contract computes them, and in float64"""
    gt, pred, cfg = O.case(kind, H, W, norm, seed)
    a32 = gt / np.float32(np.float64(gt).mean()) if norm == "mean" else gt
    b32 = O.pred32(pred, norm, gt)
    a64 = gt.astype(np.float64) / (gt.astype(np.float64).mean() if norm == "mean" else 1.0)
    b64 = O.normalize_pred(pred, norm, gt)
    return gt, pred, a32, b32, a64, b64


@pytest.mark.parametrize("norm", O.NORMS)
@pytest.mark.parametrize("H,W", SIZES)
def test_every_kind_has_its_property(H, W, norm):
    n = H * W
    for kind in O.KINDS:
        gt, pred, a32, b32, a64, b64 = maps(kind, H, W, norm)
        assert gt.dtype == pred.dtype == np.float32 and gt.shape == pred.shape == (H, W), kind
        assert np.isfinite(gt).all() and np.isfinite(pred).all(), kind
        rb, ra = np.ptp(b64), np.ptp(a64)
        if kind == "noise":
            assert np.abs(a64 - b64).min() >= 1e-3 * rb
        elif kind == "converged":
            assert np.abs(a64 - b64).max() <= 1e-3 * rb
            eq = (gt == pred) if norm == "mean" else (a32 == b32)
            assert eq.mean() >= 1 / 8 and (~eq).mean() >= 0.5
        elif kind == "flat":
            same = (pred[1:-1, 1:-1] == pred[:-2, 1:-1]) & (pred[1:-1, 1:-1] == pred[2:, 1:-1]) & \
                   (pred[1:-1, 1:-1] == pred[1:-1, :-2]) & (pred[1:-1, 1:-1] == pred[1:-1, 2:])
            assert same.mean() >= 0.5 and (pred == 0).sum() >= W and ((gt == pred) if norm == "mean" else (a32 == b32)).mean() > 0.3
            for m in (pred, gt):
                cols = np.nonzero((m[H // 2, 1:] != m[H // 2, :-1]))[0] + 1      # plateau edges along a row miss the tile seams
                assert not ((cols % 16 == 0) & (np.abs(m[H // 2, cols] - m[H // 2, cols - 1]) > 0.02)).any()
        elif kind == "saturated":
            at_max, at_min = pred == pred.max(), pred == pred.min()
            assert at_max.mean() >= 0.05 and at_min.mean() >= 0.05
            assert at_max.reshape(-1)[0] and at_min.reshape(-1)[-1]
            ty, tx = np.nonzero(at_max)
            assert len(set(zip(ty // 16, tx // 16))) >= 0.9 * ((H + 15) // 16) * ((W + 15) // 16)    # in most tiles
            sb = O.stat_blocks(n)
            idx = np.nonzero(at_max.reshape(-1))[0]
            assert len(set((idx // 256) % sb)) == sb                                     # in every statistics CTA
            assert rb > ra
        elif kind == "lone":
            assert (pred == pred.max()).sum() == 1 and (pred == pred.min()).sum() == 1
            assert pred.reshape(-1)[0] == pred.min()
            i = int(np.argmax(pred.reshape(-1)))
            y, x = divmod(i, W)
            assert i == O.last_stat_pixel(n) or (y % 16 in (0, 15) and x % 16 in (0, 15))
            assert rb > ra
        elif kind == "tie":
            assert np.ptp(a32) == np.ptp(b32) and (norm == "mean" or np.ptp(b32) == 1.0)
            if norm != "normalized":
                assert ra == rb
            else:
                assert ra - rb == pytest.approx(1e-8 / np.ptp(pred.astype(np.float64)), rel=1e-6)
        elif kind == "flat_pred":
            assert (pred == pred.reshape(-1)[0]).all() and ra > 0
            assert ((gt == pred) if norm == "mean" else (a32 == b32)).sum() >= n // 11
        elif kind == "hdr":
            assert pred.max() >= 20 and (pred == 0).sum() >= W and np.median(pred) < 1


def test_the_lone_extremum_lands_on_a_seam_or_in_the_last_statistics_cta():
    seen = set()
    for seed in range(8):
        _, pred, _ = O.case("lone", 1080, 1920, "none", seed)
        i = int(np.argmax(pred.reshape(-1)))
        seen.add("last" if i == O.last_stat_pixel(1080 * 1920) else "seam")
    assert seen == {"last", "seam"}
    assert O.stat_blocks(2160 * 3840) == 1024 < -(-2160 * 3840 // 2048)          # 4K fills the statistics grid's cap
    i = O.last_stat_pixel(2160 * 3840)
    assert (i // 256) % 1024 == 1023 and i + 256 * 1024 >= 2160 * 3840


def test_masks_drop_the_first_and_last_pixel():
    for kind in O.KINDS:
        _, _, cfg = O.case(kind, 37, 50, "none", 4, masked=True)
        m = cfg["mask"]
        assert m.dtype == bool and not m.reshape(-1)[0] and not m.reshape(-1)[-1] and 0.6 < m.mean() < 0.9


@pytest.mark.parametrize("loss_type", ["l1", "l2", "l1+ssim"])
@pytest.mark.parametrize("norm", O.NORMS)
def test_options_leave_the_float64_oracle_unchanged(loss_type, norm):
    """the separable window and the explicit device and dtype give the 2-D convolution's float64 results; float32 stays close"""
    gt, pred, cfg = O.case("noise", 37, 50, norm, 11)
    ref = O.vjp(gt, pred, loss_type=loss_type, **cfg)
    sep = O.vjp(gt, pred, "cpu", torch.float64, loss_type=loss_type, separable=True, **cfg)
    f32 = O.vjp(gt, pred, "cpu", torch.float32, loss_type=loss_type, separable=True, **cfg)
    for k in range(3):
        assert sep[k] == pytest.approx(ref[k], rel=1e-13, abs=1e-15, nan_ok=True)
        assert f32[k] == pytest.approx(ref[k], rel=1e-5, abs=1e-6, nan_ok=True)
    assert np.abs(sep[3] - ref[3]).max() <= 1e-12 * np.abs(ref[3]).max()
    assert np.abs(f32[3] - ref[3]).max() <= 1e-4 * np.abs(ref[3]).max()


def test_tie_rule():
    """on an exact tie torch.maximum gives half of the dr gradient to each range; tie_share moves it all to one side"""
    a = torch.tensor([0.0, 1.0, 0.5], dtype=torch.float64, requires_grad=True)
    b = torch.tensor([1.0, 0.25, 0.0], dtype=torch.float64, requires_grad=True)
    for share in (0.5, 0.0, 1.0):
        a.grad = b.grad = None
        O.data_range(a, b, share).backward()
        assert b.grad.tolist() == [share, 0.0, -share] and a.grad.tolist() == [-(1 - share), 1 - share, 0.0]
