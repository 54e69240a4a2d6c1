"""Every route of the FP32 SIMT convolution engine (fn2_conv.cu) against the float64-accumulated oracle.

Each case is built to reach one kernel with engine=1 (the exact-FP32 engine), and `test_simt_route_kernel` checks, with the
CUDA profiler, that it does.  Layouts: "nchw" dense, "nhwc" channels_last, "nhwc4" channels_last with the pixel stride
rounded up to a multiple of 4 channels (the blob layout of the nets: a 2-channel flow is read as one float4 per pixel).
"""
import zlib

import numpy as np
import pytest

from oracle import oracle as O
from tests.conv_ref import ROUTE_KERNEL
from tests.util import kernels_per_case, maxabs, rng

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def ops(fn2):
    from flownet2_b200 import ops as _ops
    return _ops


def dev(a, layout="nchw"):
    t = torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    if layout == "nchw":
        return t
    if layout == "nhwc":
        return t.contiguous(memory_format=torch.channels_last)
    n, c, h, w = t.shape
    padded = torch.zeros((n, (c + 3) // 4 * 4, h, w), device="cuda").contiguous(memory_format=torch.channels_last)
    padded[:, :c] = t
    return padded[:, :c]


ROUTE_CASES = [
    # route, (N, Ci, H, W, Co, k, stride, pad, deconv), layouts
    *[("pf3_tile", (2, ci, 13, 37, 2, 3, 1, pad, False), ("nhwc4",)) for ci in (2, 16, 32) for pad in (0, 1, 2)],
    ("pf_thread", (2, 2, 14, 18, 2, 4, 2, 1, False), ("nhwc4",)),     # backward data of a 2 -> 2 4x4/s2 upsampler
    ("pf_thread", (1, 20, 9, 11, 2, 5, 1, 2, False), ("nhwc4",)),
    ("pf3_warp", (1, 194, 12, 16, 2, 3, 1, 1, False), ("nhwc4",)),    # predict_flow2
    ("pf3_warp", (1, 1024, 6, 8, 2, 3, 1, 1, False), ("nhwc4",)),     # more than 48 KB of weights in shared memory
    ("pf_warp", (1, 64, 10, 12, 2, 5, 1, 2, False), ("nhwc4",)),
    ("pf_warp", (1, 1026, 6, 8, 2, 4, 2, 1, False), ("nhwc4",)),      # more than 48 KB
    ("tiny_deconv", (2, 2, 5, 7, 2, 4, 2, 1, True), ("nchw", "nhwc")),  # upsample_flow (2 -> 2)
    ("tiny_deconv", (1, 3, 6, 5, 4, 3, 1, 1, True), ("nchw", "nhwc")),
    ("tiny_deconv", (1, 4, 5, 6, 3, 5, 3, 2, True), ("nchw", "nhwc")),
    ("tiny_deconv", (1, 3, 4, 5, 2, 2, 3, 0, True), ("nchw",)),         # fewer taps than the stride: bias-only pixels
    ("tiny_conv", (2, 8, 11, 13, 3, 3, 2, 1, False), ("nchw", "nhwc")),
    ("smallco_conv", (1, 48, 9, 10, 2, 3, 1, 1, False), ("nchw",)),
    ("smallco_deconv", (1, 40, 5, 6, 3, 4, 2, 1, True), ("nchw", "nhwc")),
    ("fewci", (2, 3, 12, 20, 40, 3, 1, 1, False), ("nhwc",)),
    ("nhwc", (1, 24, 9, 11, 16, 3, 1, 1, False), ("nhwc",)),
    ("nhwc", (1, 16, 5, 6, 8, 4, 2, 1, True), ("nhwc",)),
    ("igemm_conv", (1, 24, 9, 11, 16, 3, 2, 1, False), ("nchw",)),
    ("igemm_deconv", (1, 16, 5, 6, 8, 4, 2, 1, True), ("nchw",)),
]
ROUTE_PARAMS = [pytest.param(route, case, layout, id="%s-%s-%s" % (route, layout, "-".join(map(str, case))))
                for route, case, layouts in ROUTE_CASES for layout in layouts]


def layer(case):
    N, Ci, H, W, Co, k, s, p, deconv = case
    r = rng(zlib.crc32(repr(case).encode()))
    x = r.standard_normal((N, Ci, H, W)).astype(np.float32)
    w = (r.standard_normal((Ci, Co, k, k) if deconv else (Co, Ci, k, k)) * np.sqrt(2.0 / (Ci * k * k))).astype(np.float32)
    b = r.standard_normal(Co).astype(np.float32)
    return x, w, b


@pytest.mark.parametrize("route,case,layout", ROUTE_PARAMS)
def test_simt_route(ops, route, case, layout):
    N, Ci, H, W, Co, k, s, p, deconv = case
    x, w, b = layer(case)
    fn = O.deconv_fwd if deconv else O.conv_fwd
    want = O.relu(fn(x, w, b, s, p, f64acc=True), 0.1)
    got = ops.conv2d(dev(x, layout), dev(w), torch.from_numpy(b).cuda(), s, p, deconv, 0.1, engine=1).contiguous().cpu().numpy()
    assert maxabs(got, want) <= 1e-5 * max(1.0, np.abs(want).max())
    want = fn(x, w, None, s, p, f64acc=True)
    got = ops.conv2d(dev(x, layout), dev(w), None, s, p, deconv, None, engine=1).contiguous().cpu().numpy()
    assert maxabs(got, want) <= 1e-5 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("route,case,layout", ROUTE_PARAMS)
def test_simt_route_kernel(ops, route, case, layout):
    """The case runs the kernel of its route."""
    N, Ci, H, W, Co, k, s, p, deconv = case
    x, w, b = layer(case)
    xd, wd, bd = dev(x, layout), dev(w), torch.from_numpy(b).cuda()
    names = kernels_per_case([lambda: ops.conv2d(xd, wd, bd, s, p, deconv, 0.1, engine=1)])[0]
    assert any(ROUTE_KERNEL[route] in n for n in names), sorted(names)


@pytest.mark.parametrize("ci", [2, 16, 32])
def test_pf3_tile_padding_is_zero_input(ops, ci):
    """The 3x3 predictor kernel takes any padding: pad 2 equals, bit for bit, pad 1 on the input zero-padded by one pixel."""
    x, w, b = layer((2, ci, 13, 37, 2, 3, 1, 2, False))
    xp = np.pad(x, ((0, 0), (0, 0), (1, 1), (1, 1)))
    wd, bd = dev(w), torch.from_numpy(b).cuda()
    for bias, slope in ((bd, 0.1), (None, None)):
        got = ops.conv2d(dev(x, "nhwc4"), wd, bias, 1, 2, False, slope, engine=1).contiguous().cpu().numpy()
        want = ops.conv2d(dev(xp, "nhwc4"), wd, bias, 1, 1, False, slope, engine=1).contiguous().cpu().numpy()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
