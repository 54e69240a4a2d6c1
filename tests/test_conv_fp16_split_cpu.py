"""The FP16 operand route of the per-tap tensor-core engine (fn2_conv_tc.cu: the NT = 128 layers in plain K-block mode),
restated in numpy, and its error bound on adversarial rows.

Activations, per K step and pixel row (the 32 channels of the step): e from the largest |a| so that |a| 2^-e < 2^15, clamped to
the range that keeps 2^-e, 2^(11-e) and 2^(e+f-11) normal floats (e = 0 when the largest |a| is not finite); hi = fp16(a 2^-e),
lo' = fp16((a 2^-e - hi) 2^11).  Weights, per layer: f from the largest |w| (largest scaled weight in [8, 16)), w_hi = fp16(w 2^-f),
W_A = 2^11 w_hi, W_B = fp16(2^11 (w 2^-f - w_hi)), W_C = w_hi.  A K step accumulates lo' W_C + hi W_B + hi W_A = 2^(11-e-f) sum a w and
scales it back by 2^(e+f-11).  tests/test_conv_fp16_split_gpu.py checks the packing kernel against pack_f16 bit for bit.
"""
import numpy as np
import pytest

F32, F16 = np.float32, np.float16


def exp_bits(x):
    """biased exponent of float32 x"""
    return int(np.asarray(x, F32).view(np.uint32) >> 23)


def pow2(k):
    assert -126 <= k <= 127
    return F32(2.0 ** k)


def wexp(maxabs):
    """tc_f16_wexp: the layer's weight exponent f"""
    E = exp_bits(abs(F32(maxabs)))
    return 0 if E >= 255 else min(max(E - 130, -100), 100)


def row_exp(maxabs, f):
    """the row exponent e of the MMA warpgroups"""
    E = exp_bits(abs(F32(maxabs)))
    return 0 if E == 255 else min(max(E - 141, max(-116, -115 - f)), min(126, 138 - f))


def row_max(a):
    """fmaxf over |a|: a NaN element never wins unless all are NaN"""
    m = np.abs(a.astype(F32))
    return F32(np.nanmax(m)) if not np.isnan(m).all() else F32(np.nan)


def split_a(a, e):
    """(hi, lo') of a float32 row for row exponent e, as the kernel forms them (fmaf(-2048, hi, a 2^(11-e)) is exact)"""
    with np.errstate(invalid="ignore", over="ignore"):
        x = a.astype(F32) * pow2(-e)
        hi = x.astype(F16)
        lo = (a.astype(F32) * pow2(11 - e) - F32(2048) * hi.astype(F32)).astype(F16)
    return hi, lo


def pack_f16(w, f):
    """(W_A, W_B, W_C) of float32 weights for layer exponent f (tc_pack_f16_kernel)"""
    with np.errstate(invalid="ignore", over="ignore"):
        x = w.astype(F32) * pow2(-f)
        hi = x.astype(F16)
        hf = hi.astype(F32)
        return (F32(2048) * hf).astype(F16), ((x - hf) * F32(2048)).astype(F16), hi


def channel(s):
    """tc_f16_channel: K slot -> channel of the 32-channel block"""
    h, j = s >> 4, s & 15
    return 8 * ((j & 7) >> 1) + 4 * h + 2 * (j >> 3) + (j & 1)


def step_dot(a, w):
    """one K step of one output: sum over the row's channels as the three FP16 products compute it (float64 sum of exact
    products), scaled back; a: (32,) activations of one pixel row, w: (32,) weights of one output channel"""
    f = wexp(np.abs(w).max())
    e = row_exp(row_max(a), f)
    hi, lo = split_a(a, e)
    WA, WB, WC = pack_f16(w, f)
    d = lambda u, v: (u.astype(np.float64) * v.astype(np.float64)).sum()
    return (d(lo, WC) + d(hi, WB) + d(hi, WA)) * 2.0 ** (e + f - 11)


# ---- rows ----------------------------------------------------------------------------------------------------------------------
def rows():
    r = np.random.default_rng(7)
    out = {
        "mixed_1e30_1e-30": np.where(r.random(32) < 0.5, 1e30, 1e-30) * r.choice([-1, 1], 32),
        "zeros": np.zeros(32),
        "subnormal": r.uniform(-1, 1, 32) * 1e-39,
        "subnormal_and_normal": np.concatenate([r.uniform(-1, 1, 16) * 1e-40, r.uniform(-1, 1, 16) * 1e-30]),
        "span_1e-20_1e20": 10.0 ** r.uniform(-20, 20, 32) * r.choice([-1, 1], 32),
        "fp16_top": np.full(32, 65519.0) * 2.0 ** r.integers(-30, 30),      # rounds up to 2^16 in FP16 without the scale
        "one_big": np.concatenate([[3e38], r.standard_normal(31)]),
        "gaussian": r.standard_normal(32),
        "tiny_max": r.uniform(-1, 1, 32) * 2.0 ** -120,
    }
    return {k: v.astype(F32) for k, v in out.items()}


ROWS = rows()


@pytest.mark.parametrize("name", sorted(ROWS))
@pytest.mark.parametrize("f", [-100, -40, 0, 13, 100])
def test_split_error_bound(name, f):
    """hi + 2^-11 lo' reproduces a 2^-e to within 2^-22 |a| + 2^-35 2^e per element; the scaled row never overflows FP16."""
    a = ROWS[name]
    e = row_exp(row_max(a), f)
    assert max(-116, -115 - f) <= e <= min(126, 138 - f)
    if exp_bits(row_max(a)) - 141 > e:
        # clamped from above: only when the row's largest |a| times the layer's largest |w| (>= 2^(f+3)) overflows float32
        assert float(row_max(a)) * 2.0 ** (f + 3) >= 2.0 ** 128
        return
    hi, lo = split_a(a, e)
    assert np.isfinite(hi).all() and np.isfinite(lo).all()
    if np.abs(a).max() > 0 and e > max(-116, -115 - f):
        assert np.abs(hi.astype(np.float64)).max() >= 2.0 ** 14          # the row's largest element uses FP16's range
    got = (hi.astype(np.float64) + lo.astype(np.float64) * 2.0 ** -11) * 2.0 ** e
    a64 = a.astype(np.float64)
    assert (np.abs(got - a64) <= 2.0 ** -22 * np.abs(a64) + 2.0 ** -35 * 2.0 ** e).all()


@pytest.mark.parametrize("scale", [1e-30, 1e-5, 1.0, 1e4, 1e20])
def test_weight_split(scale):
    """W_A, W_B, W_C of a layer: W_A below 2^15, all finite, and 2^f (W_A + W_B) 2^-11 within 2^-22 |w| + 2^-36 2^f of w."""
    r = np.random.default_rng(11)
    w = (r.standard_normal(4096) * scale * 10.0 ** r.uniform(-6, 0, 4096)).astype(F32)
    f = wexp(np.abs(w).max())
    WA, WB, WC = pack_f16(w, f)
    assert np.isfinite(WA).all() and np.isfinite(WB).all() and np.abs(WA.astype(np.float64)).max() <= 2.0 ** 15
    assert 8 <= np.abs(w.astype(np.float64)).max() * 2.0 ** -f < 16 or f in (-100, 100)
    assert (WA.astype(np.float64) == 2048.0 * WC.astype(np.float64)).all()
    got = (WA.astype(np.float64) + WB.astype(np.float64)) * 2.0 ** (f - 11)
    w64 = w.astype(np.float64)
    assert (np.abs(got - w64) <= 2.0 ** -22 * np.abs(w64) + 2.0 ** -36 * 2.0 ** f).all()


@pytest.mark.parametrize("name", sorted(ROWS))
@pytest.mark.parametrize("wscale", [1e-3, 1.0, 1e4])
def test_step_dot(name, wscale):
    """One K step's three products, scaled back, within 2^-20 sum |a w| of the exact dot product (the dropped lo' * w_lo term
    and the two splits), plus the FP16 floor of the row and of the weights."""
    r = np.random.default_rng(13)
    a = ROWS[name]
    w = (r.standard_normal(32) * wscale).astype(F32)
    got = step_dot(a, w)
    f = wexp(np.abs(w).max())
    e = row_exp(row_max(a), f)
    a64, w64 = a.astype(np.float64), w.astype(np.float64)
    want = (a64 * w64).sum()
    bound = 2.0 ** -20 * (np.abs(a64) * np.abs(w64)).sum() + 2.0 ** -34 * (2.0 ** e * np.abs(w64).sum() + 2.0 ** f * np.abs(a64).sum())
    assert abs(got - want) <= bound, (got, want, bound)


def test_non_finite_rows():
    """A row with an infinity takes e = 0; its products are not finite.  A NaN does not decide e (fmaxf skips it) and stays
    NaN through the split."""
    w = np.linspace(-1, 1, 32).astype(F32)
    a = np.ones(32, F32) * 1e-10
    a[3] = np.inf
    assert row_exp(row_max(a), 0) == 0
    assert not np.isfinite(step_dot(a, w))
    b = np.ones(32, F32) * 1e-10
    b[5] = np.nan
    assert row_exp(row_max(b), 0) == exp_bits(F32(1e-10)) - 141
    hi, lo = split_a(b, row_exp(row_max(b), 0))
    assert np.isnan(hi[5]) and np.isnan(step_dot(b, w))
    assert row_exp(np.float32(np.nan), 0) == 0
    assert wexp(np.inf) == 0 and wexp(np.nan) == 0 and wexp(0.0) == -100


def test_channel_order_is_a_permutation():
    """K slots -> channels: a permutation of the 32 channels; thread t's slots of half h are the 16-byte chunk 2t + h."""
    assert sorted(channel(s) for s in range(32)) == list(range(32))
    for h in range(2):
        for t in range(4):
            got = sorted(channel(16 * h + j) for j in (2 * t, 2 * t + 1, 2 * t + 8, 2 * t + 9))
            assert got == [8 * t + 4 * h + i for i in range(4)]
