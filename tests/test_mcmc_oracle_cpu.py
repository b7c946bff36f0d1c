"""The float64 3DGS-MCMC oracle (oracle/mcmc_oracle.py) against exact rational arithmetic, the identities of the relocation, and the
position noise the reference's own controller computed (tests/golden/mcmc_noise.npz, made by tests/golden/make_golden_mcmc.py)."""
import math
import os
from fractions import Fraction

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import mcmc_oracle as M


def _exact_denominator(op: Fraction, N: int) -> Fraction:
    """D with every operation exact except the square roots, which enter as exact rationals of their float64 values."""
    return sum(Fraction(math.comb(i - 1, k) * (-1) ** k) * op ** (k + 1) / Fraction(math.sqrt(k + 1))
               for i in range(1, N + 1) for k in range(i))


@pytest.mark.parametrize("o", [0.005, 0.1, 0.5, 0.9, 0.99])
def test_both_denominator_forms_match_exact_arithmetic(o):
    for N in range(1, 13):
        op = M.relocated_opacity(o, N)
        exact = float(_exact_denominator(Fraction(op), N))
        for form in (M.denominator_double_sum, M.denominator_hockey_stick):
            assert abs(form(op, N) - exact) <= 1e-12 * abs(exact), (o, N, form.__name__)


def test_one_sample_is_the_identity():
    rng = np.random.default_rng(0)
    o = rng.uniform(0.005, 0.999, 64)
    s = rng.uniform(0.001, 1.0, (64, 3))
    for form in ("hockey_stick", "double_sum"):
        new_o, new_s = M.relocation(o, s, np.ones(64, np.int64), 51, form)
        np.testing.assert_allclose(new_o, o, rtol=1e-15)
        np.testing.assert_allclose(new_s, s, rtol=1e-13)


def test_relocated_opacities_compose_back_to_the_original():
    for o in (0.005, 0.1, 0.5, 0.9, 0.99, 1 - 2.0 ** -23):
        for N in range(1, 52):
            op = M.relocated_opacity(o, N)
            assert abs(-math.expm1(N * math.log1p(-op)) - o) <= 1e-14 * o, (o, N)


def test_counts_are_clamped_to_the_table():
    o, s = np.array([0.3, 0.3, 0.3]), np.ones((3, 3))
    new_o, new_s = M.relocation(o, s, [51, 400, 0], 51)
    assert new_o[0] == new_o[1] and new_o[2] == 0.3
    np.testing.assert_array_equal(new_s[0], new_s[1])


def test_noise_oracle_reproduces_the_reference_controller():
    d = np.load(os.path.join(GOLDEN, "mcmc_noise.npz"))
    assert not d["means"].any()     # the recorded update started from zero means: means_after is the noise itself
    delta = M.noise_delta(d["log_scales"], d["raw_quats"], d["opacity_logits"], float(d["noise_lr"] * d["xyz_lr"]), d["z"])
    ref = d["means_after"]
    scale = np.abs(ref).max(axis=1, keepdims=True)
    assert (np.abs(delta - ref) <= 1e-12 * scale).all()
    w = M.noise_weight(d["opacity_logits"])
    assert w.max() > 0.5 and w.min() < 1e-30     # the fixture spans both ends of the noise weight
