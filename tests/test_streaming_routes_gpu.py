"""Both routes of FlowWarp, ChannelNorm and the warp block of fn2_ops.cu, and both routes of Downsample (fn2_loss.cu).

FlowWarp, ChannelNorm and the warp block take the F4 route when every image pixel is one 16-byte float4 group (C <= 4 in a
channel-fast view with a 16-byte aligned pixel stride: the nets' padded NHWC blobs and the concat children at a multiple of 4
channels), and the strided route otherwise (NCHW, a child at offset 2, C = 5).  FlowWarp and ChannelNorm are compared exactly
(==) with the oracle, the warp block's five tops with the layer chain it replaces; outputs go into channel slices of
sentinel-filled parents, whose other channels must keep their sentinels.  Downsample runs one thread per output, or a block
per output for windows of 256 taps or more (the 1/64 level of a 448x320 crop), and is compared with the oracle at the
training tolerance.  `test_streaming_route_kernels` checks, with the CUDA profiler, that each case runs its route's kernel.
"""
import zlib

import numpy as np
import pytest

from oracle import oracle as O
from tests.refcheck import TRAIN_TOL
from tests.util import kernels_per_case, maxabs, rng

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

SENTINEL = -7.25
N, H, W = 2, 13, 17
# (kind, C, parent channels, channel offset): "nchw" is dense NCHW, "nhwc" dense channels_last, "slice" a channel range of a
# channels_last parent (C = 3 of 4: the nets' padded NHWC images)
F4_LAYOUTS = [("slice", 3, 4, 0), ("slice", 3, 8, 0), ("slice", 3, 8, 4)]
STRIDED_LAYOUTS = [("nchw", 3, 0, 0), ("slice", 3, 8, 2), ("nhwc", 5, 0, 0)]
LAYOUTS = [(lay, True) for lay in F4_LAYOUTS] + [(lay, False) for lay in STRIDED_LAYOUTS]
LAYOUT_PARAMS = [pytest.param(lay, f4, id="-".join(map(str, lay))) for lay, f4 in LAYOUTS]


@pytest.fixture(scope="module")
def ops(fn2):
    from flownet2_b200 import ops as _ops
    return _ops


def host(t):
    return t.contiguous().cpu().numpy()


def place(a, lay):
    """a (N, C, h, w) on the device in layout lay -> (view, parent, index of the view in the parent); the parent's elements
    outside the view hold SENTINEL."""
    kind, Cc, pc, off = lay
    n, _, h, w = a.shape
    if kind == "nchw":
        p, idx = torch.empty(a.shape, device="cuda"), (slice(None),)
    elif kind == "nhwc":
        p, idx = torch.empty(a.shape, device="cuda").contiguous(memory_format=torch.channels_last), (slice(None),)
    else:
        p = torch.full((n, pc, h, w), SENTINEL, device="cuda").contiguous(memory_format=torch.channels_last)
        idx = (slice(None), slice(off, off + Cc))
    v = p[idx]
    v.copy_(torch.from_numpy(np.ascontiguousarray(a, np.float32)))
    return v, p, idx


def out_slice(c, h, w, channels_last):
    """An output of c channels at channel 1 of a sentinel-filled parent -> (view, parent, index)."""
    p = torch.full((N, c + 2, h, w), SENTINEL, device="cuda")
    if channels_last:
        p = p.contiguous(memory_format=torch.channels_last)
    idx = (slice(None), slice(1, 1 + c))
    return p[idx], p, idx


def outside_kept(p, idx):
    keep = np.ones(p.shape, bool)
    keep[idx] = False
    return bool((host(p)[keep] == SENTINEL).all())


def same(got, want):
    return np.array_equal(got, want, equal_nan=True)


def warp_inputs(lay, seed):
    """An image in layout lay and a flow with the edge cases of test_flow_warp_forward_bit_exact."""
    r = rng(seed)
    img = r.standard_normal((N, lay[1], H, W)).astype(np.float32)
    flow = r.uniform(-6, 6, (N, 2, H, W)).astype(np.float32)
    flow[0, :, 5, 7] = 1000.0            # far out of range
    flow[1, 0, 3, 3] = np.nan            # NaN flow -> fill
    flow[0, :, 0, 0] = 0.0               # exact grid point
    flow[0, 0, 10, W - 1] = 0.0          # right edge: R tap clamped to W - 1
    return img, flow


def flow_warp_case(ops, lay, fill_nan):
    img, flow = warp_inputs(lay, zlib.crc32(repr(("warp", lay, fill_nan)).encode()))
    vimg = place(img, lay)[0]
    vflow = place(flow, ("nchw" if lay[0] == "nchw" else "nhwc", 2, 0, 0))[0]
    out = out_slice(lay[1], H, W, lay[0] != "nchw")
    return (lambda: ops.flow_warp(vimg, vflow, fill_nan, out=out[0])), O.flow_warp_fwd(img, flow, fill_nan), out


def channel_norm_case(ops, lay):
    x = rng(zlib.crc32(repr(("norm", lay)).encode())).standard_normal((N, lay[1], H, W)).astype(np.float32)
    vx = place(x, lay)[0]
    out = out_slice(1, H, W, lay[0] != "nchw")
    return (lambda: ops.channel_norm(vx, out=out[0])), O.channel_norm(x), out


@pytest.mark.parametrize("fill_nan", [False, True])
@pytest.mark.parametrize("lay,f4", LAYOUT_PARAMS)
def test_flow_warp_route(ops, lay, f4, fill_nan):
    run, want, (_, parent, idx) = flow_warp_case(ops, lay, fill_nan)
    assert same(host(run()), want)
    assert outside_kept(parent, idx)


@pytest.mark.parametrize("lay,f4", LAYOUT_PARAMS)
def test_channel_norm_route(ops, lay, f4):
    run, want, (_, parent, idx) = channel_norm_case(ops, lay)
    assert same(host(run()), want)
    assert outside_kept(parent, idx)


# ---- warp block ------------------------------------------------------------------------------------------------------------
# (name, image layout, image1 layout, flow (h, w), images (H, W), F4 route)
WARP_BLOCK_CASES = [
    ("net", ("slice", 3, 4, 0), ("slice", 3, 4, 0), (7, 9), (28, 36), True),             # x4, the nets' layout
    ("nchw", ("nchw", 3, 0, 0), ("nchw", 3, 0, 0), (7, 9), (28, 36), False),
    ("misaligned", ("slice", 3, 4, 0), ("slice", 3, 8, 2), (7, 9), (28, 36), False),
    ("ratio", ("slice", 3, 4, 0), ("slice", 3, 4, 0), (27, 49), (109, 197), True),      # a non-integer ratio
    ("ratio_nchw", ("nchw", 3, 0, 0), ("nchw", 3, 0, 0), (27, 49), (109, 197), False),
]
WARP_BLOCK_PARAMS = [pytest.param(c, fill, id="%s-%s" % (c[0], "nan" if fill else "zero")) for c in WARP_BLOCK_CASES
                     for fill in (False, True)]
COEFF = 0.05


def warp_block_case(ops, case, fill_nan):
    """-> (run, chain, parent, idx): run() runs the fused block; chain() runs the five layers it replaces; parent / idx: the
    concat parent the outputs are channel ranges of and their index in it (None for separate outputs)."""
    name, l0, l1, (fh, fw), (ih, iw) = case[:5]
    r = rng(zlib.crc32(repr((case, fill_nan)).encode()))
    flow = r.uniform(-0.2 * fw, 0.2 * fw, (N, 2, fh, fw)).astype(np.float32)
    flow[0, :, 1, 1] = 1000.0                                         # out of the image
    img0 = r.standard_normal((N, 3, ih, iw)).astype(np.float32)
    img1 = r.standard_normal((N, 3, ih, iw)).astype(np.float32)
    cl = l0[0] != "nchw"
    vflow = place(flow, ("slice", 2, 4, 0) if cl else ("nchw", 2, 0, 0))[0]
    v0, v1 = place(img0, l0)[0], place(img1, l1)[0]
    if cl:
        # warped / err / flow_scaled / err_norm as channel ranges of one concat parent
        cat = torch.full((N, 12, ih, iw), SENTINEL, device="cuda").contiguous(memory_format=torch.channels_last)
        full = torch.empty((N, 2, ih, iw), device="cuda").contiguous(memory_format=torch.channels_last)
        outs = (full, cat[:, 0:3], cat[:, 3:6], cat[:, 8:9], cat[:, 6:8])
        parent, idx = cat, (slice(None), slice(0, 9))
    else:
        outs = (torch.empty((N, 2, ih, iw), device="cuda"), torch.empty((N, 3, ih, iw), device="cuda"),
                torch.empty((N, 3, ih, iw), device="cuda"), torch.empty((N, 1, ih, iw), device="cuda"),
                torch.empty((N, 2, ih, iw), device="cuda"))
        parent = idx = None

    def run():
        return ops.warp_block(vflow, v0, v1, COEFF, fill_nan, out=outs)

    def chain():
        full = ops.resample(vflow, ih, iw, 2)
        warped = ops.flow_warp(v1, full, fill_nan)
        err = ops.eltwise_sum([v0, warped], [1.0, -1.0])
        return full, warped, err, ops.channel_norm(err), ops.eltwise_sum([full], [COEFF])

    return run, chain, parent, idx


@pytest.mark.parametrize("case,fill_nan", WARP_BLOCK_PARAMS)
def test_warp_block_matches_layer_chain(ops, case, fill_nan):
    run, chain, parent, idx = warp_block_case(ops, case, fill_nan)
    got = [host(t) for t in run()]
    want = [host(t) for t in chain()]
    for name, g, w in zip(("flow_full", "warped", "err", "err_norm", "flow_scaled"), got, want):
        assert same(g, w), name
    if fill_nan:
        assert np.isnan(got[1]).any()                                # the out-of-image flow reached the fill
    if parent is not None:
        assert outside_kept(parent, idx)


def test_warp_block_rejects(ops):
    r = rng(11)
    img = torch.from_numpy(r.standard_normal((N, 3, 8, 8)).astype(np.float32)).cuda()
    with pytest.raises(Exception, match="up-sampled"):
        ops.warp_block(torch.zeros((N, 2, 16, 16), device="cuda"), img, img, COEFF)
    img5 = torch.from_numpy(r.standard_normal((N, 5, 8, 8)).astype(np.float32)).cuda()
    with pytest.raises(Exception, match="channel counts"):
        ops.warp_block(torch.zeros((N, 2, 4, 4), device="cuda"), img5, img5, COEFF)


# ---- Downsample ------------------------------------------------------------------------------------------------------------
# (name, N, C, H, W, top h, top w, wide route)
DOWNSAMPLE_CASES = [
    ("wide_1_64", 2, 2, 320, 448, 5, 7, True),      # the 1/64 level of a 448x320 crop: 161 x 151 taps per output
    ("narrow_nan", 2, 2, 40, 56, 20, 28, False),
    ("narrow_1_4", 2, 2, 320, 448, 80, 112, False),
]


def downsample_case(ops, case):
    name, n, c, h, w, th, tw = case[:7]
    r = rng(zlib.crc32(name.encode()))
    x = r.standard_normal((n, c, h, w)).astype(np.float32)
    x[r.random(x.shape) < (0.05 if case[7] else 0.45)] = np.nan        # narrow: some outputs are NaN (over half the weight)
    vx = torch.from_numpy(x).cuda().contiguous(memory_format=torch.channels_last)
    out = torch.empty((n, c, th, tw), device="cuda")
    return (lambda: ops.downsample(vx, th, tw, out=out)), O.downsample_fwd(x, th, tw)


@pytest.mark.parametrize("case", DOWNSAMPLE_CASES, ids=[c[0] for c in DOWNSAMPLE_CASES])
def test_downsample_route(ops, case):
    run, want = downsample_case(ops, case)
    got = host(run())
    assert case[7] or (np.isnan(want).any() and not np.isnan(want).all())
    # the tolerance of the training-layer tests (test_train_gpu.py): the oracle does not contract multiply-adds
    assert maxabs(got, want) <= 5 * TRAIN_TOL["downsample"] * max(float(np.nanmax(np.abs(want))), 1e-6)


def test_streaming_route_kernels(ops):
    """Every case runs its route's instantiation and no other."""
    cases = []
    for lay, f4 in LAYOUTS:
        cases.append((flow_warp_case(ops, lay, False)[0], "flow_warp_fwd_kernel<%s>" % ("true" if f4 else "false"),
                      "flow_warp_fwd_kernel<"))
        cases.append((channel_norm_case(ops, lay)[0], "channel_norm_kernel<%s>" % ("true" if f4 else "false"),
                      "channel_norm_kernel<"))
    for case in WARP_BLOCK_CASES:
        cases.append((warp_block_case(ops, case, False)[0], "warp_block_kernel<%s>" % ("true" if case[5] else "false"),
                      "warp_block_kernel<"))
    for case in DOWNSAMPLE_CASES:
        cases.append((downsample_case(ops, case)[0], "downsample_wide_kernel(" if case[7] else "downsample_kernel(",
                      "downsample"))
    names = kernels_per_case([run for run, _, _ in cases])
    bad = []
    for (_, want, family), got in zip(cases, names):
        ran = {n for n in got if family in n}
        if not ran or not all(want in n for n in ran):
            bad.append((want, sorted(got)))
    assert not bad, bad
