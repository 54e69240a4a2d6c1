"""The FP16 route's K step with two weight tiles (fn2_conv_tc.cu), restated in numpy.

The activations keep their low half unscaled: hi = fp16(a 2^-e), lo'' = fp16(a 2^-e - hi) (the subtraction is exact in float32),
and a K step accumulates, per 16-slot half, lo'' W_A + hi W_B + hi W_A = 2^(11-e-f) sum a w, so that the stage holds W_A and
W_B only.  e, hi, the weights and the scale-back are those of tests/test_conv_fp16_split_cpu.py.  lo'' W_A equals the earlier
lo' W_C (lo' = fp16(2^11 (a 2^-e - hi)), W_C = w_hi) exactly wherever |a 2^-e| >= 2^-1; below that lo'' meets FP16's subnormal
floor, 2^-24.
"""
import numpy as np
import pytest

from tests.test_conv_fp16_split_cpu import ROWS, channel, exp_bits, pack_f16, row_exp, row_max, split_a, wexp

F32, F16 = np.float32, np.float16


def split_two_tile(a, e):
    """(hi, lo'') of a float32 row for row exponent e, as conv_tc_kernel forms them"""
    with np.errstate(invalid="ignore", over="ignore"):
        x = a.astype(F32) * F32(2.0 ** -e)
        hi = x.astype(F16)
        lo = (x - hi.astype(F32)).astype(F16)
    return hi, lo


def step_dot(a, w):
    """one K step of one output as the two-tile step computes it: per 16-slot half (K slot s holds channel channel(s)),
    lo'' W_A and hi W_B, then hi W_A (float64 sums of exact products), scaled back"""
    f = wexp(np.abs(w).max())
    e = row_exp(row_max(a), f)
    hi, lo = split_two_tile(a, e)
    WA, WB, _ = pack_f16(w, f)
    d = lambda u, v, s: (u[s].astype(np.float64) * v[s].astype(np.float64)).sum()
    halves = [np.array([channel(16 * h + j) for j in range(16)]) for h in range(2)]
    cross = sum(d(lo, WA, s) + d(hi, WB, s) for s in halves)
    return (cross + sum(d(hi, WA, s) for s in halves)) * 2.0 ** (e + f - 11)


@pytest.mark.parametrize("name", sorted(ROWS))
@pytest.mark.parametrize("f", [-100, -40, 0, 13, 100])
def test_split_error_bound(name, f):
    """hi + lo'' reproduces a 2^-e to within 2^-22 |a| + 2^-25 2^e per element: 2^-39 of the row's largest |a| where e is not
    clamped, the absolute resolution the per-layer exponent gives the weights."""
    a = ROWS[name]
    e = row_exp(row_max(a), f)
    if exp_bits(row_max(a)) - 141 > e:
        return                                      # clamped from above: |a| max |w| overflows float32 (the split test's case)
    hi, lo = split_two_tile(a, e)
    assert np.isfinite(hi).all() and np.isfinite(lo).all()
    got = (hi.astype(np.float64) + lo.astype(np.float64)) * 2.0 ** e
    a64 = a.astype(np.float64)
    assert (np.abs(got - a64) <= 2.0 ** -22 * np.abs(a64) + 2.0 ** -25 * 2.0 ** e).all()


@pytest.mark.parametrize("name", sorted(ROWS))
@pytest.mark.parametrize("wscale", [1e-3, 1.0, 1e4])
def test_step_dot(name, wscale):
    """One K step's three products, scaled back, within 2^-20 sum |a w| of the exact dot product (the dropped lo'' w_lo term
    and the two splits), plus the FP16 floor of the row's low halves (2^-25 2^e per element) and of the weights."""
    r = np.random.default_rng(13)
    a = ROWS[name]
    w = (r.standard_normal(32) * wscale).astype(F32)
    got = step_dot(a, w)
    f = wexp(np.abs(w).max())
    e = row_exp(row_max(a), f)
    a64, w64 = a.astype(np.float64), w.astype(np.float64)
    want = (a64 * w64).sum()
    bound = 2.0 ** -20 * (np.abs(a64) * np.abs(w64)).sum() + 2.0 ** -24 * 2.0 ** e * np.abs(w64).sum() \
        + 2.0 ** -34 * 2.0 ** f * np.abs(a64).sum()
    assert abs(got - want) <= bound, (got, want, bound)


def _same_products(a, w):
    """per element of the row a (one output channel's weights w): (lo'' W_A == lo' W_C, |a 2^-e| >= 2^-1)"""
    f = wexp(np.abs(w).max())
    e = row_exp(row_max(a), f)
    hi, lo2 = split_two_tile(a, e)
    hi1, lo1 = split_a(a, e)
    assert np.array_equal(hi.view(np.uint16), hi1.view(np.uint16))
    WA, _, WC = pack_f16(w, f)
    new = lo2.astype(np.float64) * WA.astype(np.float64)             # products of two FP16 values: exact in float64
    old = lo1.astype(np.float64) * WC.astype(np.float64)
    with np.errstate(invalid="ignore"):
        big = np.abs(a.astype(F32) * F32(2.0 ** -e)) >= 0.5
    return (new == old) | (np.isnan(new) & np.isnan(old)), big


@pytest.mark.parametrize("name", sorted(ROWS))
def test_low_half_products_match_three_tiles(name):
    """lo'' W_A == lo' W_C exactly for every element with |a 2^-e| >= 2^-1 of the adversarial rows."""
    w = np.random.default_rng(3).standard_normal(32).astype(F32)
    same, big = _same_products(ROWS[name], w)
    assert same[big].all()


def test_low_half_products_match_three_tiles_random():
    """The same on 10^6 random elements (rows of 32 spanning 2^-40 .. 2^40 around a random magnitude), where the elements
    within 2^-15 of their row's largest |a| all match and those further down may not."""
    r = np.random.default_rng(29)
    n = 10 ** 6 // 32
    a = (r.standard_normal((n, 32)) * 2.0 ** r.uniform(-40, 40, (n, 32)) * 2.0 ** r.integers(-60, 60, (n, 1))).astype(F32)
    w = (r.standard_normal((n, 32)) * 10.0 ** r.uniform(-3, 3, (n, 1))).astype(F32)
    checked = differ = 0
    for i in range(n):
        same, big = _same_products(a[i], w[i])
        assert same[big].all(), i
        near = np.abs(a[i].astype(np.float64)) >= 2.0 ** -15 * float(row_max(a[i]))
        assert big[near].all(), i
        checked += int(big.sum())
        differ += int((~same).sum())
    assert checked > 10 ** 5 and differ > 0             # both regimes occur
