"""Numeric edges of the draws from a caller's fp32 logits (shift invariance, tied and extreme magnitudes, the two-way
calibration of the noise) under HOST EMULATION of the CUDA kernels (tests/emu): the tests of
tests/sampling_edges_suite.py at CPU-friendly sizes, and the same shift invariance of the float64 oracle of the draw."""
import numpy as np

from oracle import logits_oracle as LO
from tests import sampling_edges_suite
from tests.backends import collect

collect(globals(), sampling_edges_suite, "emu")


def test_oracle_draw_shift_invariant():
    """The oracle draws on max-subtracted scores: legal logits tied at 0, +-1e30 or +-FLT_MAX give one draw, not the
    lowest index every time, with log_prob -log n; grid logits shifted by 2^20 or -2^40 (exact in float64) give the
    unshifted draw and log_prob exactly."""
    rng = np.random.default_rng(0)
    J = 15
    drawn = set()
    for k in range(200):
        legal = rng.random(J + 1) < 0.7
        legal[rng.integers(J)] = True
        n = int(legal.sum())
        args = (legal, False, 9, k % 7, k)
        a0, lp0, err, _ = LO.draw(np.zeros(J + 1), *args)
        assert not err and legal[a0] and abs(lp0 + np.log(n)) < 1e-12, (k, a0, lp0)
        drawn.add(a0 - int(np.flatnonzero(legal)[0]))
        for v in sampling_edges_suite.TIES:
            assert LO.draw(np.full(J + 1, v), *args)[:3] == (a0, lp0, False), (k, v)
        x = rng.integers(-64, 65, size=J + 1) / 8
        a, lp, _, _ = LO.draw(x, *args)
        for c in (2.0 ** 20, -2.0 ** 40):
            assert LO.draw(x + c, *args)[:2] == (a, lp), (k, c)
    assert len(drawn) > 5, drawn                          # ties are broken by the noise, not by the index
