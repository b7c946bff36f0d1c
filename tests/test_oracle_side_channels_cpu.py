"""The oracle's blend side channels (gs_oracle.blend(side=...), gs_oracle.absgrad) against brute force, on a scene small
enough for a per-pixel autograd loop: 20 splats over 2x2 tiles of a 24x20 image (partial tiles), an opaque front layer
so that pixels stop at the 1e-4 transmittance cut-off, and opacities at the 0.999 clamp."""
import pytest
import torch

from oracle import gs_oracle as O

W, H = 24, 20


def _tiny_scene(seed=0, n=20):
    """-> xy, conic, opacity [float64], sorted ids and tile ranges (every splat listed in every tile except the last one,
    which is listed nowhere), depth-sorted."""
    g = torch.Generator().manual_seed(seed)
    xy = torch.rand(n, 2, generator=g, dtype=torch.float64) * torch.tensor([W + 8.0, H + 8.0], dtype=torch.float64) - 4.0
    ang = torch.rand(n, generator=g, dtype=torch.float64) * 3.14159
    s = torch.exp(torch.rand(n, 2, generator=g, dtype=torch.float64) * 2.0)            # std 1 - 7.4 px
    c, si = torch.cos(ang), torch.sin(ang)
    a = c * c * s[:, 0] ** 2 + si * si * s[:, 1] ** 2
    b = c * si * (s[:, 0] ** 2 - s[:, 1] ** 2)
    d = si * si * s[:, 0] ** 2 + c * c * s[:, 1] ** 2
    det = a * d - b * b
    conic = torch.stack([d / det, -b / det, a / det], dim=1)
    opacity = torch.rand(n, generator=g, dtype=torch.float64) * 0.9 + 0.05
    centre = torch.tensor([W / 2.0, H / 2.0], dtype=torch.float64)
    # four opaque layers (std 8 px) over the centre: pixels stop behind them, at the alpha clamp; splat n-2, small and
    # behind them, is listed but never composited
    opacity[:4] = 1.0
    conic[:4] = torch.tensor([1.0 / 64, 0.0, 1.0 / 64], dtype=torch.float64)
    xy[:4] = centre + 0.5 * torch.randn(4, 2, generator=g, dtype=torch.float64)
    xy[n - 2], conic[n - 2], opacity[n - 2] = centre, torch.tensor([2.0, 0.0, 2.0], dtype=torch.float64), 0.5
    depth = torch.rand(n, generator=g, dtype=torch.float64)
    depth[:4] *= 0.2
    depth[n - 2] = 2.0
    order = torch.argsort(depth)
    listed = order[order != n - 1].to(torch.int32)
    sids = listed.repeat(4)
    L = listed.numel()
    ranges = torch.tensor([[t * L, (t + 1) * L] for t in range(4)], dtype=torch.int64)
    return xy, conic, opacity, sids, ranges


def _features(n, D, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, D, generator=g, dtype=torch.float64) * torch.logspace(0, 3, D, dtype=torch.float64)


def _leaves(xy, conic, opacity, colors):
    return [t.clone().requires_grad_(True) for t in (xy, conic, opacity, colors)]


@pytest.mark.parametrize("mode", [O.MODE_VANILLA, O.MODE_GSPLAT])
@pytest.mark.parametrize("D", [1, 4])
def test_absgrad_equals_per_pixel_brute_force(mode, D):
    xy0, conic0, op0, sids, ranges = _tiny_scene()
    n = xy0.shape[0]
    bg = torch.linspace(0.2, -0.3, D, dtype=torch.float64)
    gen = torch.Generator().manual_seed(3)
    cot = torch.rand(D, H, W, generator=gen, dtype=torch.float64) * 2 - 1
    cot_a = torch.rand(H, W, generator=gen, dtype=torch.float64) * 2 - 1

    xy, conic, op, col = _leaves(xy0, conic0, op0, _features(n, D, 1))
    side = {}
    img, alpha, _ = O.blend(mode, xy, conic, op, col, sids, ranges, bg, W, H, side=side)
    ((img * cot).sum() + (alpha * cot_a).sum()).backward()
    got = O.absgrad(side["abs_terms"], n)
    assert bool(side["stopped"].any()), "no pixel reaches the transmittance cut-off"
    if mode == O.MODE_GSPLAT:
        assert side["clamped"] > 0, "no sample reaches the alpha clamp"

    # brute force: the gradient of every pixel's own loss, summed in magnitude
    xy, conic, op, col = _leaves(xy0, conic0, op0, _features(n, D, 1))
    img, alpha, _ = O.blend(mode, xy, conic, op, col, sids, ranges, bg, W, H)
    per_pixel = (img * cot).sum(dim=0) + alpha * cot_a
    ref = torch.zeros(n, 2, dtype=torch.float64)
    for yy in range(H):
        for xx in range(W):
            gxy, = torch.autograd.grad(per_pixel[yy, xx], xy, retain_graph=True)
            ref += gxy.abs()
    assert float(ref.max()) > 0
    assert float((got - ref).abs().max()) <= 1e-12 * float(ref.abs().max())
    assert float(ref[-1].abs().max()) == 0.0 and float(got[-1].abs().max()) == 0.0      # the unlisted splat


@pytest.mark.parametrize("mode", [O.MODE_VANILLA, O.MODE_GSPLAT])
def test_hits_equal_contributors_below_n_contrib(mode):
    """hit[g] <=> some pixel composites splat g with non-zero weight at a list position <= that pixel's n_contrib.  The
    weights come from a separate evaluation with one indicator channel per splat (the image is linear in the colours, so
    channel g of that image is splat g's weight in every pixel)."""
    xy, conic, op, sids, ranges = _tiny_scene()
    n = xy.shape[0]
    side = {}
    _, _, ncontrib = O.blend(mode, xy, conic, op, _features(n, 1, 1), sids, ranges, None, W, H, side=side)
    weights, _, nc2 = O.blend(mode, xy, conic, op, torch.eye(n, dtype=torch.float64), sids, ranges, None, W, H)
    assert torch.equal(ncontrib, nc2)
    expect = torch.zeros(n, dtype=torch.bool)
    gx = (W + O.BLOCK - 1) // O.BLOCK
    for yy in range(H):
        for xx in range(W):
            s, e = (int(v) for v in ranges[(yy // O.BLOCK) * gx + xx // O.BLOCK])
            ids = sids[s:e].long()
            k = int(ncontrib[yy, xx])
            w = weights[ids, yy, xx]
            assert bool((w >= 0).all()) and bool((w[k:] == 0).all())                    # nothing composites behind n_contrib
            assert k == 0 or float(w[k - 1]) > 0.0                                         # the entry at n_contrib does
            expect[ids[:k][w[:k] > 0]] = True
    assert torch.equal(side["hit"], expect)
    assert 0 < int(expect.sum()) < n - 1                     # some listed splats are never composited (hidden behind the front)
    m = side["hit_margin"]
    assert bool(torch.isfinite(m[:-1]).all()) and float(m[-1]) == float("inf")
    # a stopped pixel gives the margin of its stopping sample to every splat it never reaches
    assert bool(side["stopped"].any())


@pytest.mark.parametrize("mode", [O.MODE_VANILLA, O.MODE_GSPLAT])
def test_side_channels_leave_outputs_bit_identical(mode):
    xy0, conic0, op0, sids, ranges = _tiny_scene(seed=4)
    n = xy0.shape[0]
    bg = torch.tensor([0.1, -0.4, 0.7], dtype=torch.float64)
    cot = torch.rand(3, H, W, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    outs = []
    for side in (None, {}):
        xy, conic, op, col = _leaves(xy0, conic0, op0, _features(n, 3, 2))
        margins = []
        img, alpha, nc = O.blend(mode, xy, conic, op, col, sids, ranges, bg, W, H, margins=margins, side=side)
        ((img * cot).sum() + alpha.sum()).backward()
        outs.append((img.detach(), alpha.detach(), nc, margins[0], xy.grad, conic.grad, op.grad, col.grad))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
