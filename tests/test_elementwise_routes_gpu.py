"""Every route of the element-wise ops of fn2_ops.cu (ReLU and its backward, Eltwise SUM, axpby, copy, fill) on every kind of
view the nets pass them, compared exactly (==) with the oracle or with float32 numpy.

The channel-group route runs when every view is channel-fast and pixel-linear (dense channels_last, and channel slices of a
channels_last parent, like a concat child); the strided route runs otherwise (NCHW, a spatial window of a channels_last
map, mixed layouts); copy between NCHW and channels_last with C >= 8 runs the transpose.  `test_elementwise_route_kernels`
checks, with the CUDA profiler, that each case runs its route's kernel.
"""
import zlib

import numpy as np
import pytest

from oracle import oracle as O
from tests.util import kernels_per_case, rng

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

SENTINEL = -7.25
N, H, W = 2, 5, 7

# (kind, C, parent channels, channel offset); "spatial" is a window of a larger channels_last map
LAYOUTS = [
    ("nchw", 5, 0, 0),
    ("nhwc", 2, 0, 0), ("nhwc", 3, 0, 0), ("nhwc", 5, 0, 0), ("nhwc", 64, 0, 0),
    ("slice", 3, 8, 0), ("slice", 3, 8, 2), ("slice", 5, 12, 5),
    ("slice", 8, 12, 4),                                     # whole float4 groups only
    ("slice", 2, 4, 0), ("slice", 2, 4, 2),                  # a 2-channel child of a 4-channel parent: float2 stores
    ("slice", 1026, 1032, 0), ("slice", 1026, 1031, 5),      # a tail group of 2 channels
    ("spatial", 6, 0, 0),
]
# op case -> the functor it runs, as the profiler names it
OPS = {"relu": "ReluOp", "relu_bwd0": "ReluBwdOp", "relu_bwd": "ReluBwdOp", "relu_bwd_acc": "ReluBwdOp",
       "eltwise2": "EltwiseSumOp", "eltwise4": "EltwiseSumOp", "axpby": "AxpbyOp", "axpby_beta0": "AxpbyOp", "copy": "CopyOp",
       "fill": "FillOp"}
CASES = [(op, lay, lay) for op in OPS for lay in LAYOUTS] + [
    ("relu", ("nchw", 5, 0, 0), ("nhwc", 5, 0, 0)),
    ("axpby", ("nhwc", 5, 0, 0), ("nchw", 5, 0, 0)),
    ("copy", ("nchw", 3, 0, 0), ("nhwc", 3, 0, 0)),
    ("copy", ("nhwc", 3, 0, 0), ("nchw", 3, 0, 0)),
    ("copy", ("nchw", 40, 0, 0), ("nhwc", 40, 0, 0)),        # transpose
    ("copy", ("nhwc", 40, 0, 0), ("nchw", 40, 0, 0)),        # transpose
]
PARAMS = [pytest.param(op, li, lo, id="%s-%s-%s" % (op, "-".join(map(str, li)), "-".join(map(str, lo)))) for op, li, lo in CASES]
LAYOUT_PARAMS = [pytest.param(lay, id="-".join(map(str, lay))) for lay in LAYOUTS]
AXPBY = [(1.0, 1.0), (-1.0, 0.5), (2.0, -1.0), (0.5, 2.0)]    # exact products: numpy's a*x + b*y rounds like fmaf(a, x, b*y)


@pytest.fixture(scope="module")
def ops(fn2):
    from flownet2_b200 import ops as _ops
    return _ops


def host(t):
    return t.contiguous().cpu().numpy()


def place(a, lay):
    """a (N, C, H, W) on the device in layout lay -> (view, parent, index of the view in the parent).  The parent's elements
    outside the view hold SENTINEL."""
    kind, Cc, pc, off = lay
    cl = torch.channels_last
    if kind == "nchw":
        p, idx = torch.empty(a.shape, device="cuda"), (slice(None),)
    elif kind == "nhwc":
        p, idx = torch.empty(a.shape, device="cuda").contiguous(memory_format=cl), (slice(None),)
    elif kind == "slice":
        p, idx = torch.full((N, pc, H, W), SENTINEL, device="cuda").contiguous(memory_format=cl), (slice(None), slice(off, off + Cc))
    else:
        p = torch.full((N, Cc, H + 3, W + 2), SENTINEL, device="cuda").contiguous(memory_format=cl)
        idx = (slice(None), slice(None), slice(1, 1 + H), slice(2, 2 + W))
    v = p[idx]
    v.copy_(torch.from_numpy(np.ascontiguousarray(a, np.float32)))
    return v, p, idx


def outside_kept(p, idx):
    keep = np.ones(p.shape, bool)
    keep[idx] = False
    return bool((host(p)[keep] == SENTINEL).all())


def route(op, li, lo):
    if op == "copy" and li[0] != lo[0] and li[1] >= 8:
        return "transpose"
    return "group" if li[0] in ("nhwc", "slice") and lo[0] in ("nhwc", "slice") else "strided"


def setup(ops, op, li, lo):
    """-> (run, want, (out view, out parent, out index)): run() launches the op once and returns the output view."""
    r = rng(zlib.crc32(repr((op, li, lo)).encode()))
    shape = (N, li[1], H, W)

    def arr():
        a = r.standard_normal(shape).astype(np.float32)
        a.reshape(-1)[::7] = 0.0
        return a

    nan = np.full(shape, np.nan, np.float32)
    if op == "relu":
        x = arr()
        vx, out = place(x, li)[0], place(nan, lo)
        return (lambda: ops.relu(vx, 0.1, out=out[0])), O.relu(x, 0.1), out
    if op.startswith("relu_bwd"):
        slope, acc = (0.0 if op == "relu_bwd0" else 0.1), op == "relu_bwd_acc"
        t, d = arr(), arr()
        want = O.relu_bwd(t, d, slope)
        prior = nan
        if acc:
            # a prior that nearly cancels the product exposes the product's rounding: the inputs must tell a fused
            # multiply-add from the rounded product added to the prior
            prior = (-want * (1 + 2.0 ** -8 * r.standard_normal(shape))).astype(np.float32)
            g64 = d.astype(np.float64) * np.where(t > 0, 1.0, np.float64(np.float32(slope)))
            assert ((g64 + prior).astype(np.float32) != want + prior).any()
            want = want + prior
        vt, vd, out = place(t, li)[0], place(d, li)[0], place(prior, lo)
        return (lambda: ops.relu_backward(vt, vd, slope, out=out[0], accumulate=acc)), want, out
    if op.startswith("eltwise"):
        coeffs = [1.0, -1.0] if op == "eltwise2" else [0.5, -1.0, 2.0, 0.00392156862745]
        bs = [arr() for _ in coeffs]
        vbs, out = [place(b, li)[0] for b in bs], place(nan, lo)
        return (lambda: ops.eltwise_sum(vbs, coeffs, out=out[0])), O.eltwise_sum(bs, coeffs), out
    if op == "axpby":
        x, y = arr(), arr()
        vx, out = place(x, li)[0], place(y, lo)
        return (lambda: ops.axpby(vx, 0.5, out[0], 2.0)), np.float32(0.5) * x + np.float32(2.0) * y, out
    if op == "axpby_beta0":                             # beta == 0 must not read y (NaN here)
        x = arr()
        vx, out = place(x, li)[0], place(nan, lo)
        return (lambda: ops.axpby(vx, -1.0, out[0], 0.0)), -x, out
    if op == "copy":
        x = arr()
        vx, out = place(x, li)[0], place(nan, lo)
        return (lambda: ops.copy(vx, out[0])), x, out
    out = place(nan, lo)
    return (lambda: ops.fill(out[0], 3.5)), np.full(shape, 3.5, np.float32), out


@pytest.mark.parametrize("op,li,lo", PARAMS)
def test_elementwise_route(ops, op, li, lo):
    run, want, (_, parent, idx) = setup(ops, op, li, lo)
    got = host(run())
    assert np.array_equal(got, want), (op, int((got != want).sum()))
    assert outside_kept(parent, idx)


@pytest.mark.parametrize("li", LAYOUT_PARAMS)
def test_axpby_every_coefficient(ops, li):
    """alpha and beta over {1, -1, 0.5, 2} on every layout."""
    for alpha, beta in AXPBY:
        r = rng(zlib.crc32(repr((alpha, beta, li)).encode()))
        x, y = (r.standard_normal((N, li[1], H, W)).astype(np.float32) for _ in range(2))
        vx, (vy, parent, idx) = place(x, li)[0], place(y, li)
        got = host(ops.axpby(vx, alpha, vy, beta))
        assert np.array_equal(got, np.float32(alpha) * x + np.float32(beta) * y), (alpha, beta)
        assert outside_kept(parent, idx)


def test_elementwise_route_kernels(ops):
    """Every case runs its route's kernel with its op's functor, and no other route's kernel."""
    names = kernels_per_case([setup(ops, op, li, lo)[0] for op, li, lo in CASES])
    bad = []
    for (op, li, lo), got in zip(CASES, names):
        ran = {rt for rt, k in (("group", "ew_group_kernel"), ("strided", "ew_strided_kernel"), ("transpose", "copy_transpose_kernel"))
               if any(k in n for n in got)}
        if ran != {route(op, li, lo)} or (ran != {"transpose"} and not any(OPS[op] + ">" in n for n in got)):
            bad.append((op, li, lo, sorted(got)))
    assert not bad, bad
