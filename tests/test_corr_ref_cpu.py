"""tests/corr_ref.py (the float64 shift-and-sum correlation reference) pinned to the oracle (oracle.correlation_fwd /
correlation_bwd, which restate the reference's CorrelateData and its backward kernels over zero-padded copies), on torch's CPU
device.

The oracle returns float32.  With small-integer inputs and a power-of-two channel count every product, every partial sum and
the division by C are exact in float32 as in float64, so the two must agree to 1e-12 relative (in practice bit for bit) in any
summation order: what is compared is the geometry -- top-channel order, displacement signs, stride_2 sampling, zero fill at
the borders.  A second set of cases draws N(0, 1) inputs and checks the oracle's float32 results against the reference within
the float32 error of their sums.
"""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import corr_ref
from tests.util import rng

# (N, C, H, W, md, s2): odd H and W, s2 of 1 and 2, md 4 and 20
CASES = [
    (2, 8, 9, 13, 4, 1),
    (1, 16, 11, 7, 4, 2),
    (2, 4, 23, 29, 20, 2),
    (1, 8, 25, 21, 20, 1),
    (1, 32, 12, 18, 20, 2),
]
IDS = ["n%d-c%d-%dx%d-md%d-s%d" % c for c in CASES]


def _ints(r, shape, hi):
    return r.integers(-hi, hi + 1, shape).astype(np.float32)


def _rel(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-300))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_forward_matches_oracle_exactly(case):
    N, C, H, W, md, s2 = case
    r = rng(101 + sum(case))
    a, b = _ints(r, (N, C, H, W), 4), _ints(r, (N, C, H, W), 4)
    want = O.correlation_fwd(a, b, md, 1, md, 1, s2, 0, exact_order=True)
    got, absref = corr_ref.forward(torch.from_numpy(a), torch.from_numpy(b), md, s2)
    assert got.shape == want.shape
    assert _rel(got.numpy(), want) <= 1e-12
    assert bool((absref >= got.abs()).all())
    # the border rows and columns meet the zero fill: some outputs are exactly 0 by geometry, and the reference knows which
    assert bool((absref == 0).any()) and bool((got[absref == 0] == 0).all())


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_backward_matches_oracle_exactly(case):
    N, C, H, W, md, s2 = case
    r = rng(202 + sum(case))
    a, b = _ints(r, (N, C, H, W), 3), _ints(r, (N, C, H, W), 3)
    D = 2 * (md // s2) + 1
    td = _ints(r, (N, D * D, H, W), 3)
    w0, w1 = O.correlation_bwd(a, b, td, md, 1, md, 1, s2)
    d0, d1, abs0, abs1 = corr_ref.backward(torch.from_numpy(a), torch.from_numpy(b), torch.from_numpy(td), md, s2)
    assert _rel(d0.numpy(), w0) <= 1e-12 and _rel(d1.numpy(), w1) <= 1e-12
    assert bool((abs0 >= d0.abs()).all()) and bool((abs1 >= d1.abs()).all())


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_random_inputs_within_float32_of_oracle(case):
    N, C, H, W, md, s2 = case
    r = rng(303 + sum(case))
    a, b = (r.standard_normal((N, C, H, W)).astype(np.float32) for _ in range(2))
    D = 2 * (md // s2) + 1
    td = r.standard_normal((N, D * D, H, W)).astype(np.float32)
    u = 2.0 ** -24
    got, absref = corr_ref.forward(torch.from_numpy(a), torch.from_numpy(b), md, s2)
    want = O.correlation_fwd(a, b, md, 1, md, 1, s2, 0, exact_order=True)
    assert bool((np.abs(want - got.numpy()) <= (C + 2) * u * absref.numpy()).all())
    d0, d1, abs0, abs1 = corr_ref.backward(torch.from_numpy(a), torch.from_numpy(b), torch.from_numpy(td), md, s2)
    w0, w1 = O.correlation_bwd(a, b, td, md, 1, md, 1, s2)
    assert bool((np.abs(w0 - d0.numpy()) <= (D * D + 2) * u * abs0.numpy()).all())
    assert bool((np.abs(w1 - d1.numpy()) <= (D * D + 2) * u * abs1.numpy()).all())


def test_nan_propagates_where_it_meets_a_product():
    """A NaN in bottom 1 poisons exactly the forward outputs and bottom-0 gradients whose sums take that element."""
    N, C, H, W, md, s2 = 1, 4, 11, 13, 4, 2
    r = rng(404)
    a, b = (r.standard_normal((N, C, H, W)) for _ in range(2))
    b[0, 1, 5, 6] = np.nan
    out, _ = corr_ref.forward(torch.from_numpy(a), torch.from_numpy(b), md, s2)
    bad = ~torch.isfinite(out[0])
    want = torch.zeros_like(bad)
    for t, (dy, dx) in enumerate(corr_ref.displacements(md, s2)):
        if 0 <= 5 - dy < H and 0 <= 6 - dx < W:
            want[t, 5 - dy, 6 - dx] = True
    assert bool((bad == want).all())
    td = r.standard_normal((N, 25, H, W))
    d0, d1, _, _ = corr_ref.backward(torch.from_numpy(a), torch.from_numpy(b), torch.from_numpy(td), md, s2)
    assert bool((~torch.isfinite(d0[0]) == want.any(0)[None] & (torch.arange(C) == 1)[:, None, None]).all())
    assert bool(torch.isfinite(d1).all())
