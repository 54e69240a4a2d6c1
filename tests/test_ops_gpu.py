"""GPU parity: every hot-path op called through the C-ABI vs the CPU oracle on seeded inputs.

Tolerances: streaming layers (FlowWarp, Resample, SpatialAugmentation, Eltwise, ReLU, ChannelNorm,
mean) are compared BIT-EXACT (same expression order, no FMA contraction on either side).
Correlation and conv/deconv reduce in a different order than the oracle -> 1e-5 relative to the
magnitude of the result (the reference's own conv tests use 1e-4, test_convolution_layer.cpp:256).
"""
import numpy as np
import pytest

from oracle import oracle as O
from tests.util import maxabs, rng

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def dev(a, channels_last=False):
    t = torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    return t.contiguous(memory_format=torch.channels_last) if channels_last else t


def host(t):
    return t.contiguous().cpu().numpy()


@pytest.fixture(scope="module")
def ops(fn2):
    from flownet2_b200 import ops as _ops
    return _ops


CORR_CASES = [
    # N, C, H, W, pad, k, md, s1, s2, type
    (2, 32, 12, 14, 4, 1, 4, 1, 2, 0),       # FlowNetC parameter class, small
    (1, 256, 10, 12, 20, 1, 20, 1, 2, 0),    # FlowNetC parameters (d=21 -> 441 channels)
    (2, 16, 11, 13, 3, 1, 3, 1, 1, 0),       # stride_2 = 1
    (1, 8, 13, 15, 4, 3, 3, 1, 1, 0),        # kernel_size 3
    (1, 8, 16, 18, 4, 3, 2, 2, 2, 0),        # stride_1 = 2
    (1, 8, 12, 12, 2, 1, 4, 1, 2, 0),        # pad < max_displacement (top smaller than bottom)
    (2, 16, 9, 10, 3, 1, 3, 1, 1, 1),        # SUBTRACT
    (1, 8, 12, 13, 4, 3, 2, 1, 2, 1),        # SUBTRACT, k=3
]


@pytest.mark.parametrize("case", CORR_CASES)
@pytest.mark.parametrize("channels_last", [False, True])
def test_correlation_forward(ops, case, channels_last):
    N, C, H, W, pad, k, md, s1, s2, typ = case
    r = rng(hash(case) % 2**31)
    a = r.standard_normal((N, C, H, W)).astype(np.float32)
    b = r.standard_normal((N, C, H, W)).astype(np.float32)
    want = O.correlation_fwd(a, b, pad, k, md, s1, s2, typ, exact_order=False)
    got = host(ops.correlation(dev(a, channels_last), dev(b, channels_last), pad, k, md, s1, s2, typ))
    assert maxabs(got, want) <= 1e-5 * max(1.0, np.abs(want).max())


def test_correlation_index_mapping(ops):
    # shifted copy -> the peak sits in exactly the displacement channel the reference's mapping
    # (tc % D -> x offset, tc / D -> y offset, correlation_layer.cu:81-82) predicts
    r = rng(7)
    a = r.standard_normal((1, 64, 24, 24)).astype(np.float32)
    dx, dy = 4, -2                      # b(x+dx, y+dy) == a(x, y)
    b = np.roll(a, (dy, dx), axis=(2, 3))
    got = host(ops.correlation(dev(a), dev(b), 4, 1, 4, 1, 2))
    D, rr = 5, 2
    tc = (dy // 2 + rr) * D + (dx // 2 + rr)
    inner = got[0, :, 6:-6, 6:-6]
    assert (inner.argmax(0) == tc).all()


@pytest.mark.parametrize("case", [(2, 8, 9, 10, 3, 1, 3, 1, 1), (1, 16, 10, 12, 4, 1, 4, 1, 2), (1, 4, 11, 12, 4, 3, 2, 2, 2)])
def test_correlation_backward(ops, case):
    N, C, H, W, pad, k, md, s1, s2 = case
    r = rng(11)
    a = r.standard_normal((N, C, H, W)).astype(np.float32)
    b = r.standard_normal((N, C, H, W)).astype(np.float32)
    tc, th, tw, _, _ = O.correlation_shape(H, W, pad, k, md, s1, s2)
    td = r.standard_normal((N, tc, th, tw)).astype(np.float32)
    w0, w1 = O.correlation_bwd(a, b, td, pad, k, md, s1, s2)
    g0, g1 = ops.correlation_backward(dev(a), dev(b), dev(td), pad, k, md, s1, s2)
    assert maxabs(host(g0), w0) <= 2e-5 * max(1.0, np.abs(w0).max())
    assert maxabs(host(g1), w1) <= 2e-5 * max(1.0, np.abs(w1).max())


@pytest.mark.parametrize("case", [(2, 64, 24, 40, 2), (1, 32, 37, 21, 2), (1, 32, 19, 45, 1)])
def test_correlation_backward_fast_path(ops, case):
    """FlowNet2-C's layer (MULTIPLY, k = 1, pad = md, 21 x 21 displacements, C % 32 == 0, channel-fast maps): the parity-plane
    kernel of fn2_corr_bwd.cu, including plane / tile tails (odd sizes) and stride_2 = 1."""
    N, C, H, W, s2 = case
    md = 10 * s2
    r = rng(N * 100 + H)
    a = r.standard_normal((N, C, H, W)).astype(np.float32)
    b = r.standard_normal((N, C, H, W)).astype(np.float32)
    td = r.standard_normal((N, 441, H, W)).astype(np.float32)
    w0, w1 = O.correlation_bwd(a, b, td, md, 1, md, 1, s2)
    g0, g1 = ops.correlation_backward(dev(a, True), dev(b, True), dev(td, True), md, 1, md, 1, s2)
    assert maxabs(host(g0), w0) <= 1e-5 * max(1.0, np.abs(w0).max())
    assert maxabs(host(g1), w1) <= 1e-5 * max(1.0, np.abs(w1).max())


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("fill_nan", [False, True])
def test_flow_warp_forward_bit_exact(ops, channels_last, fill_nan):
    r = rng(3)
    N, C, H, W = 2, 3, 37, 53
    img = r.standard_normal((N, C, H, W)).astype(np.float32)
    flow = r.uniform(-20, 20, (N, 2, H, W)).astype(np.float32)
    flow[0, :, 5, 7] = 1000.0            # far out of range
    flow[1, 0, 3, 3] = np.nan            # NaN flow -> fill (comparisons false)
    flow[0, :, 0, 0] = 0.0               # exact grid point
    flow[0, 0, 10, W - 1] = 0.0          # right edge: R tap clamped to W-1
    want = O.flow_warp_fwd(img, flow, fill_nan)
    got = host(ops.flow_warp(dev(img, channels_last), dev(flow, channels_last), fill_nan))
    assert maxabs(got, want) == 0.0


def test_flow_warp_backward(ops):
    r = rng(4)
    N, C, H, W = 2, 3, 17, 19
    img = r.standard_normal((N, C, H, W)).astype(np.float32)
    flow = r.uniform(-5, 5, (N, 2, H, W)).astype(np.float32)
    wd = r.standard_normal((N, C, H, W)).astype(np.float32)
    wi, wf = O.flow_warp_bwd(img, flow, wd)
    gi, gf = ops.flow_warp_backward(dev(img), dev(flow), dev(wd))
    assert maxabs(host(gf), wf) <= 1e-5           # different accumulation order only
    assert maxabs(host(gi), wi) <= 1e-5           # atomics: order-nondeterministic last ulp


RESAMPLE_CASES = [
    (2, 3, 109, 256, 436, 1024, 2, True),     # flow x4 upsample (config 4 shapes, quartered)
    (1, 3, 436, 1024, 448, 1024, 2, True),    # image 436 -> 448 rows
    (1, 2, 112, 256, 436, 1024, 2, True),     # adapted/4 -> target
    (2, 3, 64, 96, 23, 31, 2, True),          # downsample with antialias
    (2, 3, 64, 96, 23, 31, 2, False),         # downsample without
    (1, 2, 20, 30, 45, 77, 3, True),          # cubic up
    (1, 2, 45, 77, 20, 30, 3, True),          # cubic down
    (1, 3, 20, 30, 41, 59, 1, True),          # nearest
    (1, 3, 33, 47, 33, 47, 2, True),          # same size = identity
]


@pytest.mark.parametrize("case", RESAMPLE_CASES)
@pytest.mark.parametrize("channels_last", [False, True])
def test_resample_bit_exact(ops, case, channels_last):
    N, C, H, W, oh, ow, typ, aa = case
    x = rng(5).standard_normal((N, C, H, W)).astype(np.float32)
    want = O.resample_fwd(x, oh, ow, typ, aa)
    got = host(ops.resample(dev(x, channels_last), oh, ow, typ, aa))
    assert maxabs(got, want) == 0.0


@pytest.mark.parametrize("channels_last", [False, True])
def test_spatial_augmentation_bit_exact(ops, channels_last):
    r = rng(6)
    N, C, H, W = 3, 3, 40, 56
    x = r.uniform(0, 1, (N, C, H, W)).astype(np.float32)
    mats = np.stack([O.transmat_from_coeff(W, H, W, H),                                        # deploy: identity
                     O.transmat_from_coeff(48, 32, W, H, mirror=1, angle=0.2, dx=0.05, dy=-0.03, zoom_x=1.2, zoom_y=0.9),
                     O.transmat_from_coeff(48, 32, W, H, angle=-0.4, zoom_x=0.8, zoom_y=0.8)])
    want = O.spatial_augmentation(x, mats, H, W)
    got = host(ops.spatial_augmentation(dev(x, channels_last), dev(mats.reshape(1, 1, N, 6)).reshape(N, 6), H, W))
    assert maxabs(got, want) == 0.0
    want = O.spatial_augmentation(x, mats, 32, 48)
    got = host(ops.spatial_augmentation(dev(x, channels_last), torch.from_numpy(mats).cuda(), 32, 48))
    assert maxabs(got, want) == 0.0


def test_color_contrast(ops):
    r = rng(8)
    x = r.uniform(0, 1, (2, 3, 20, 24)).astype(np.float32)
    chroma = np.array([[1.2, 0.05, 1.1, 0.9, 1.0, 1.1], [0.8, -0.05, 0.9, 1.1, 1.05, 0.95]], np.float32)
    want = O.color_contrast_augmentation(x, chroma, 1.0)
    got = host(ops.color_contrast_augmentation(dev(x), torch.from_numpy(chroma).cuda(), 1.0))
    assert maxabs(got, want) <= 2e-6          # powf: CUDA vs glibc differ by ulps


def test_mean_update_and_subtract(ops):
    r = rng(9)
    N, C, H, W = 4, 3, 12, 14
    top = r.uniform(0, 1, (N, C, H, W)).astype(np.float32)
    mpp = r.uniform(0.3, 0.5, (C, H, W)).astype(np.float32)
    for per_pixel in (False, True):
        want, wpp, wpc = O.mean_subtract(top, 0, num_iter=5.0, recompute_mean=1000, mean_per_pixel=per_pixel, mean_pp=mpp)
        t, m = dev(top), dev(mpp[None])
        pc = torch.zeros(C, device="cuda")
        ops.mean_update(t, m, pc, 5.0)
        ops.mean_subtract(t, m, pc, per_pixel)
        assert maxabs(host(m)[0], wpp) == 0.0
        assert maxabs(host(pc.reshape(1, C, 1, 1)).reshape(-1), wpc) <= 1e-7
        assert maxabs(host(t), want) <= 1e-7
    want, _, _ = O.mean_subtract(top, 1, mean_pc=np.array([0.4, 0.42, 0.44], np.float32))
    t = dev(top)
    ops.mean_subtract(t, None, torch.tensor([0.4, 0.42, 0.44], device="cuda"), False)
    assert maxabs(host(t), want) == 0.0


CONV_CASES = [
    # N, Ci, H, W, Co, k, stride, pad, deconv
    (2, 3, 20, 28, 64, 7, 2, 3, False),       # conv1 of FlowNetC
    (2, 6, 20, 28, 64, 7, 2, 3, False),       # conv1 of FlowNetS
    (1, 64, 16, 20, 128, 5, 2, 2, False),     # conv2
    (2, 473, 10, 14, 256, 3, 1, 1, False),    # conv3_1 (after concat with the cost volume)
    (1, 256, 10, 14, 32, 1, 1, 0, False),     # conv_redir 1x1
    (1, 194, 12, 16, 2, 3, 1, 1, False),      # predict_flow2 (Co = 2)
    (1, 1024, 3, 4, 512, 4, 2, 1, True),      # deconv5
    (2, 2, 5, 7, 2, 4, 2, 1, True),           # upsample_flow (2 -> 2)
    (1, 130, 9, 11, 67, 3, 2, 1, False),      # odd sizes everywhere
]


@pytest.mark.parametrize("case", CONV_CASES)
@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("engine", [1, 0])
def test_conv_forward(ops, case, channels_last, engine):
    N, Ci, H, W, Co, k, s, p, deconv = case
    r = rng(hash(case) % 2**31)
    x = r.standard_normal((N, Ci, H, W)).astype(np.float32)
    wshape = (Ci, Co, k, k) if deconv else (Co, Ci, k, k)
    w = (r.standard_normal(wshape) * np.sqrt(2.0 / (Ci * k * k))).astype(np.float32)
    b = r.standard_normal(Co).astype(np.float32)
    fn = O.deconv_fwd if deconv else O.conv_fwd
    want = O.relu(fn(x, w, b, s, p, f64acc=True), 0.1)
    got = host(ops.conv2d(dev(x, channels_last), dev(w), torch.from_numpy(b).cuda(), s, p, deconv, 0.1, engine))
    tol = 1e-5 if engine == 1 else 2e-5
    assert maxabs(got, want) <= tol * max(1.0, np.abs(want).max())
    want = fn(x, w, None, s, p, f64acc=True)
    got = host(ops.conv2d(dev(x, channels_last), dev(w), None, s, p, deconv, None, engine))
    assert maxabs(got, want) <= tol * max(1.0, np.abs(want).max())


TC_CASES = [
    # N, Ci, H, W, Co, k, stride, pad, deconv    (tensor-core engine: NHWC views with the engine's padded pixel stride)
    (1, 32, 8, 16, 64, 1, 1, 0, False),
    (2, 96, 9, 13, 128, 3, 1, 1, False),
    (1, 64, 16, 20, 128, 5, 2, 2, False),      # stride 2 through TMA element strides
    (2, 473, 10, 14, 256, 3, 1, 1, False),     # channel tail 473 -> zero-filled by TMA
    (1, 256, 6, 7, 64, 4, 2, 1, True),         # deconv: 4 parity classes in one launch
    (1, 1024, 3, 4, 512, 4, 2, 1, True),
    (2, 3, 20, 28, 64, 7, 2, 3, False),        # Ci = 3
    (1, 12, 20, 28, 64, 7, 2, 3, False),
    (1, 82, 16, 24, 16, 3, 1, 1, False),       # Co = 16
    (1, 162, 9, 12, 32, 3, 1, 1, False),       # Co = 32
    (1, 162, 9, 11, 16, 4, 2, 1, True),
    (1, 64, 96, 208, 128, 3, 1, 1, False),     # 192 tiles of 1 x 128 pixels: more than one wave, no split
    (1, 64, 16, 64, 128, 3, 1, 1, False),      # 8 tiles, fewer than the SMs: every tile's K loop split in 2 (tail split)
    (1, 96, 50, 200, 16, 3, 1, 1, False),      # Co = 16 at a larger size: taps-on-N engine
]


@pytest.mark.parametrize("case", TC_CASES)
def test_conv_tensor_core_engine(ops, case):
    """3xTF32 tensor-core engine (engine=2 fails loudly if the shape is not eligible): same tolerance as the FP32
    SIMT engine, and no systematic shrink (the tensor core's round-toward-zero accumulation is drained/compensated)."""
    N, Ci, H, W, Co, k, s, p, deconv = case
    r = rng(hash(case) % 2**31)
    x = r.standard_normal((N, Ci, H, W)).astype(np.float32)
    wshape = (Ci, Co, k, k) if deconv else (Co, Ci, k, k)
    w = (r.standard_normal(wshape) * np.sqrt(2.0 / (Ci * k * k))).astype(np.float32)
    b = r.standard_normal(Co).astype(np.float32)
    want = O.relu((O.deconv_fwd if deconv else O.conv_fwd)(x, w, b, s, p, f64acc=True), 0.1)
    cp = (Ci + 31) // 32 * 32 if Ci >= 32 else (Ci + 3) // 4 * 4          # Blob::compute_cstride
    buf = torch.zeros((N, cp, H, W), device="cuda").contiguous(memory_format=torch.channels_last)
    buf[:, :Ci] = torch.from_numpy(x).cuda()
    got = host(ops.conv2d(buf[:, :Ci], dev(w), torch.from_numpy(b).cuda(), s, p, deconv, 0.1, 2))
    scale = max(1.0, np.abs(want).max())
    assert maxabs(got, want) <= 1e-6 * scale
    shrink = float(((got - want) * np.sign(want)).mean() / np.abs(want).mean())
    assert abs(shrink) < 1e-7, shrink


TN_CASES = [
    # N, Ci, H, W, Co, k, stride, pad, deconv, bias+relu      ("taps on N" engine, fn2_conv_tn.cu: Co in {16, 32}, Ci > 16)
    (1, 82, 16, 24, 16, 3, 1, 1, False, True),        # fuse_interconv0's channels: one strip, two passes of 80 accumulator columns
    (2, 82, 37, 70, 16, 3, 1, 1, False, True),        # odd size: 3 strips, partial last strip / tile, two samples
    (1, 162, 21, 45, 32, 3, 1, 1, False, True),       # fuse_interconv1: three passes of 3 taps, 6 K blocks
    (1, 40, 9, 33, 16, 3, 1, 1, False, False),        # channel tail (40 of 64), no bias / ReLU, strip boundary at column 30
    (1, 162, 9, 11, 16, 4, 2, 1, True, True),         # fuse_deconv0: 16 taps, three passes of <= 6
    (2, 128, 13, 37, 32, 4, 2, 1, True, True),        # fuse_deconv1: six passes, two strips
    (1, 64, 150, 40, 16, 3, 1, 1, False, True),       # tall: several vertical segments per strip
    (1, 96, 70, 33, 16, 4, 2, 1, True, False),        # tall deconvolution
    (1, 48, 20, 40, 32, 2, 1, 0, False, True),        # 2x2 kernel, no padding (output smaller than input)
]


@pytest.mark.parametrize("case", TN_CASES)
def test_conv_taps_on_n_engine(ops, case):
    """Few output channels at high resolution: GEMM over K = Ci with (tap, co) on the MMA's N side, scatter-add ("col2im") through
    a shared-memory ring of output rows.  Same tolerance as the per-tap tensor-core engine; the output goes into a channel slice of a
    wider NHWC buffer (zero-copy concat child) whose other channels must stay untouched."""
    N, Ci, H, W, Co, k, s, p, deconv, act = case
    r = rng(hash(case) % 2**31)
    x = r.standard_normal((N, Ci, H, W)).astype(np.float32)
    wshape = (Ci, Co, k, k) if deconv else (Co, Ci, k, k)
    w = (r.standard_normal(wshape) * np.sqrt(2.0 / (Ci * k * k))).astype(np.float32)
    b = r.standard_normal(Co).astype(np.float32) if act else None
    want = (O.deconv_fwd if deconv else O.conv_fwd)(x, w, b, s, p, f64acc=True)
    if act:
        want = O.relu(want, 0.1)
    cp = (Ci + 31) // 32 * 32
    buf = torch.zeros((N, cp, H, W), device="cuda").contiguous(memory_format=torch.channels_last)
    buf[:, :Ci] = torch.from_numpy(x).cuda()
    plan = ops.conv_plan(Ci, Co, k, s, p, deconv, N, H, W, cp)
    assert plan[3] == 3, plan                                               # taps-on-N mode chosen
    Ho, Wo = want.shape[2], want.shape[3]
    wide = torch.full((N, Co + 32, Ho, Wo), 7.0, device="cuda").contiguous(memory_format=torch.channels_last)
    out = wide[:, 16:16 + Co]
    got = ops.conv2d(buf[:, :Ci], dev(w), torch.from_numpy(b).cuda() if act else None, s, p, deconv, 0.1 if act else None, 2, out=out)
    scale = max(1.0, np.abs(want).max())
    assert maxabs(host(got), want) <= 1e-6 * scale, maxabs(host(got), want)
    assert float((wide[:, :16] - 7.0).abs().max()) == 0.0 and float((wide[:, 16 + Co:] - 7.0).abs().max()) == 0.0
    shrink = float(((host(got) - want) * np.sign(want)).mean() / np.abs(want).mean())
    print("taps-on-N case", case, "max err %.3g shrink %.3g" % (maxabs(host(got), want) / scale, shrink))
    assert abs(shrink) < 1e-7, shrink
    again = ops.conv2d(buf[:, :Ci], dev(w), torch.from_numpy(b).cuda() if act else None, s, p, deconv, 0.1 if act else None, 2, out=out)
    assert torch.equal(again, got)                                          # fixed summation order


ROW_CASES = [
    # N, Ci, H, W, Co, k, stride, pad   (dense small-Ci input + guard band -> kernel-row packing of the tensor-core engine)
    (2, 3, 20, 28, 64, 7, 2, 3),        # FlowNetC conv1: one 32-float K block per kernel row
    (1, 3, 23, 37, 64, 7, 2, 3),        # odd sizes: masked taps on both image edges, partial tiles
    (1, 12, 20, 28, 64, 7, 2, 3),       # stacked FlowNetS conv1: three K blocks per kernel row
    (1, 6, 18, 22, 64, 3, 1, 1),        # FlowNet-SD conv0: stride 1
    (2, 4, 9, 150, 32, 5, 1, 2),        # a row wider than one tile
]


@pytest.mark.parametrize("case", ROW_CASES)
def test_conv_tensor_core_row_mode(ops, case):
    """The guard band is filled with NaN: the row runs of edge pixels reach into it (and into the neighbouring image
    rows), and none of that may leak into the result."""
    N, Ci, H, W, Co, k, s, p = case
    r = rng(hash(case) % 2**31)
    x = r.standard_normal((N, Ci, H, W)).astype(np.float32)
    w = (r.standard_normal((Co, Ci, k, k)) * np.sqrt(2.0 / (Ci * k * k))).astype(np.float32)
    b = r.standard_normal(Co).astype(np.float32)
    want = O.relu(O.conv_fwd(x, w, b, s, p, f64acc=True), 0.1)
    cp = (Ci + 3) // 4 * 4
    guard = 256                                                       # floats, == Blob::kGuardFloats
    flat = torch.full((guard + N * H * W * cp + guard,), float("nan"), device="cuda")
    body = flat[guard:guard + N * H * W * cp].view(N, H, W, cp)
    body.zero_()
    body[..., :Ci] = torch.from_numpy(x).cuda().permute(0, 2, 3, 1)
    xv = body.permute(0, 3, 1, 2)[:, :Ci]                             # NCHW view of the NHWC storage
    got = host(ops.conv2d(xv, dev(w), torch.from_numpy(b).cuda(), s, p, False, 0.1, 2, input_guard_bytes=4 * guard))
    assert np.isfinite(got).all()
    scale = max(1.0, np.abs(want).max())
    assert maxabs(got, want) <= 1e-6 * scale
    ungarded = host(ops.conv2d(xv, dev(w), torch.from_numpy(b).cuda(), s, p, False, 0.1, 2))
    assert maxabs(ungarded, want) <= 1e-6 * scale                     # tap-group packing (no guard promised)


EIGVEC = [0.51, 0.56, 0.65, 0.79, 0.01, -0.62, 0.35, -0.83, 0.44]       # the published FlowNet chromatic eigenvectors


@pytest.mark.parametrize("cl", [False, True])
def test_chromatic_eigen_and_effects(ops, cl):
    """Training-time colour augmentations: parity unpinned by the reference (no test, no CPU path); checked against the
    oracle restatement.  powf/cosf differ by a few ulp between libm and the device."""
    r = rng(77)
    N, H, W = 3, 20, 28
    x = r.uniform(0, 1, (N, 3, H, W)).astype(np.float32)
    space_want = O.chromatic_eigenspace(x, EIGVEC)
    space = ops.chromatic_eigenspace(dev(x, cl), EIGVEC)
    assert maxabs(space[:25].cpu().numpy(), space_want) <= 2e-6
    coeffs = np.tile(np.array([1, 1, 1, 0, 0, 0, 1, 1, 1, 1, 1, 1, 0, 0, 0, 1, 1, 1, 1, 0, 1, 0], np.float32), (N, 1))
    coeffs += (r.uniform(-0.2, 0.2, coeffs.shape)).astype(np.float32)
    want = O.chromatic_eigen_augmentation(x, coeffs, space_want, 1.0)
    got = host(ops.chromatic_eigen_augmentation(dev(x, cl), torch.from_numpy(coeffs).cuda(), space, 1.0))
    assert maxabs(got, want) <= 1e-5
    eff = np.zeros((N, 9), np.float32)
    ang = r.uniform(0, 6.28, N)
    eff[:, 4], eff[:, 5] = np.cos(ang), np.sin(ang)
    eff[:, 6] = r.uniform(-3, 3, N)
    eff[:, 7] = r.uniform(0.1, 0.4, N)
    want = O.apply_effects(x, eff, 1.0)
    got = host(ops.apply_effects(dev(x, cl), torch.from_numpy(eff).cuda(), 1.0))
    assert maxabs(got, want) == 0.0
    # additive noise: own counter-based generator; only the distribution is specified (sigma per sample)
    eff[:, 8] = [0.0, 0.05, 0.2]
    eff[:, 7] = 0.0
    base = np.full((N, 3, 64, 64), 0.5, np.float32)
    noisy = host(ops.apply_effects(dev(base, cl), torch.from_numpy(eff).cuda(), 10.0, noise_seed=1234, add_noise=True))
    d = noisy - base
    assert np.abs(d[0]).max() == 0.0
    for n in (1, 2):
        assert abs(d[n].std() - eff[n, 8]) < 0.03 * eff[n, 8] + 1e-4 and abs(d[n].mean()) < 0.05 * eff[n, 8]


def test_training_augmentations_against_golden_fixture(ops):
    """CUDA kernels vs the committed fixture tests/golden/aug_golden.npz (oracle outputs; generator: make_golden.py)."""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "aug_golden.npz"))
    x = g["x"]
    space = ops.chromatic_eigenspace(dev(x, True), g["eigvec"])
    assert maxabs(space[:25].cpu().numpy(), g["space"]) <= 2e-6
    got = host(ops.chromatic_eigen_augmentation(dev(x, True), torch.from_numpy(g["eigen_coeffs"]).cuda(), space, 1.0))
    assert maxabs(got, g["eigen_out"]) <= 1e-5
    got = host(ops.apply_effects(dev(x, True), torch.from_numpy(g["effects"]).cuda(), 1.0))
    assert maxabs(got, g["effects_out"]) == 0.0
    got = host(ops.color_contrast_augmentation(dev(x, True), torch.from_numpy(g["chroma"]).cuda(), 1.0))
    assert maxabs(got, g["chroma_out"]) <= 1e-5


def test_deconv_known_answer(ops):
    # the reference's TestSimpleDeconvolution (test_deconvolution_layer.cpp:91-137): input and
    # weights all ones, bias 0.1, 3 in / 4 out channels, kernel 3 stride 2: 3.1 / 6.1 / 12.1
    x = np.ones((2, 3, 6, 4), np.float32)
    w = np.ones((3, 4, 3, 3), np.float32)
    b = np.full(4, 0.1, np.float32)
    got = host(ops.conv2d(dev(x), dev(w), torch.from_numpy(b).cuda(), 2, 0, True, None, 1))
    for n in range(2):
        for c in range(4):
            for h in range(got.shape[2]):
                for ww in range(got.shape[3]):
                    expected = 3.1
                    h_overlap = h % 2 == 0 and h > 0 and h < got.shape[2] - 1
                    w_overlap = ww % 2 == 0 and ww > 0 and ww < got.shape[3] - 1
                    if h_overlap and w_overlap: expected += 9
                    elif h_overlap or w_overlap: expected += 3
                    assert abs(got[n, c, h, ww] - expected) < 1e-4


def test_glue_bit_exact(ops):
    r = rng(12)
    a = r.standard_normal((2, 3, 10, 12)).astype(np.float32)
    b = r.standard_normal((2, 3, 10, 12)).astype(np.float32)
    for cl in (False, True):
        assert maxabs(host(ops.relu(dev(a, cl), 0.1)), O.relu(a, 0.1)) == 0.0
        assert maxabs(host(ops.eltwise_sum([dev(a, cl), dev(b, cl)], [1.0, -1.0])), O.eltwise_sum([a, b], [1.0, -1.0])) == 0.0
        assert maxabs(host(ops.eltwise_sum([dev(a, cl)], [0.00392156862745])), O.eltwise_sum([a], [0.00392156862745])) == 0.0
        assert maxabs(host(ops.channel_norm(dev(a, cl))), O.channel_norm(a)) == 0.0
    # strided copy both ways incl. the tiled-transpose path
    x = r.standard_normal((2, 40, 9, 11)).astype(np.float32)
    src = dev(x)
    dst = torch.empty_like(src).contiguous(memory_format=torch.channels_last)
    ops.copy(src, dst)
    assert maxabs(host(dst), x) == 0.0
    back = torch.empty_like(src)
    ops.copy(dst, back)
    assert maxabs(host(back), x) == 0.0
    cat = torch.zeros((2, 48, 9, 11), device="cuda").contiguous(memory_format=torch.channels_last)
    ops.copy(src, cat[:, 5:45])
    assert maxabs(host(cat)[:, 5:45], x) == 0.0 and host(cat)[:, :5].max() == 0.0


def test_error_paths(fn2, ops):
    a = torch.zeros((1, 4, 8, 8), device="cuda")
    with pytest.raises(fn2.Fn2Error, match="Odd kernel size"):
        ops.correlation(a, a, 2, 2, 2, 1, 1)
    with pytest.raises(fn2.Fn2Error, match="Neighborhood and kernel don't fit"):
        ops.correlation_shape(4, 4, 0, 1, 8, 1, 1)
    with pytest.raises(fn2.Fn2Error, match="2 channels"):
        ops.flow_warp(a, a)

