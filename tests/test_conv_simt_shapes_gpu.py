"""The SIMT convolution engine (fn2_conv.cu) at the shapes and in the layouts the nets run it, against float64, element by
element.

Cases (SHAPE_CASES): every convolution of the deploy templates at 1024 x 436 (batch 4) and of the training templates at
448 x 320 (batch 8) whose plan is 0 -- the layers the default engine gives to SIMT: every predict_flow (pf3_warp, pf3_tile),
every upsample_flow (tiny deconvolution), FlowNet2's scale_conv1 (pf_thread) -- and the data-gradient operators of the
training graphs whose plan is 0 (the upsamplers' 2 -> 2, 4 x 4, stride-2 convolutions: pf_thread), one per distinct shape and
layout (tests/conv_ref.py, simt_layers); plus odd maps a drop-in caller produces (2 x 55 x 127, 2 x 41 x 57), with a ragged
last tile and last 4-pixel group.  At these shapes every persistent or grid-stride kernel takes several tiles, groups or
pixels per CTA (test_simt_shapes_iterate), which the small maps of test_conv_simt_routes_gpu.py never reach.

Layouts as the nets give them: the bottom is the layer's own blob (the nets' pixel stride, zero padding channels,
input_guard_bytes = 1024 as ConvolutionLayer sets it, 256 NaN floats before and after the storage) or, for a data-gradient
operator that reads an upsampler's top diff, that concat child at its channel offset and the concat's pixel stride (the
concat's other channels hold 1e30: finite, as the guard promise asks, and far off any sum they would stray into).  The top is the view the net writes: an upsampler writes channels [c0, c0 + 2) of its concat
(Net::AliasConcats, offsets from the prototxt walk); every other layer writes channels [16, 16 + Co) of a wider parent.  The
parent's other channels and its guard bands hold a sentinel that must come out bit-identical.

Inputs are drawn like the nets': leaky-ReLU(0.1) of N(0, 1) activations, mixed-sign weights N(0, 1) sqrt(2 / fan-in), N(0, 1)
bias.  Bound, per element: |got - ref| <= gamma(n + 3) absref, where absref is the same operator applied to |x|, |w| and |b|,
n = (kernel taps that reach the output) x Ci, u = 2^-24 and gamma(k) = k u / (1 - k u).  Every SIMT kernel computes an
output as FP32 FMA chains over its n products (pf3_warp and pf_warp: per-lane chains and a 5-level shuffle tree; the NHWC
engine's split-K: per-range chains and a fixed-order sum), so no product passes through more than n roundings; the bias
addition and the leaky ReLU's product add two more.  That bound holds for any summation order and needs no measured constant:
a dropped, doubled or misplaced tap fails it at any pixel.  The reference evaluates every output pixel, except on the large
maps of the other SIMT routes (ENGINE1_CASES), where it takes every edge row and column and SAMPLE seeded random pixels.
"""
import ctypes as C
import zlib
from collections import namedtuple

import pytest

from tests.conv_ref import (GUARD, SimtLayer, _check, _lib, bottom, case, conv_desc, cstride, guard_bytes, layout_of,
                            op_weights, reference, ROUTE_KERNEL, simt_layers, simt_route, simt_work, taps_at, weight_shape)
from tests.util import deploy_convs, kernels_per_case

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

U = 2.0 ** -24
SLOPE = 0.1
SENTINEL = -7.25
SAMPLE = 2048


@pytest.fixture(scope="module")
def ops(fn2):
    from flownet2_b200 import ops as _ops
    return _ops


# ---- cases ----------------------------------------------------------------------------------------------------------------
def _odd_cases():
    out = []
    for N, H, W in ((2, 55, 127), (2, 41, 57)):
        tag = "odd%dx%d-" % (H, W)
        for ci in (16, 32, 194):
            out.append(SimtLayer(case(tag + "pf3_ci%d" % ci, N, ci, H, W, 2, 3, 1, 1, layout="pad", engine=0), "pad", None))
        out.append(SimtLayer(case(tag + "upsample", N, 2, H, W, 2, 4, 2, 1, True, layout="pad", engine=0), "pad", None))
    return out


SHAPE_CASES = simt_layers() + _odd_cases()
SHAPE_IDS = [L.case.name for L in SHAPE_CASES]


def _engine1_cases():
    """One deploy-shape layer of FlowNet2 per route and regime of the other SIMT kernels, run with engine = 1 (`engine: CAFFE`,
    FN2_CONV_ENGINE=simt): net1_conv1 (fewci), net1_conv2 (NHWC, a large map), net1_conv6 (NHWC split-K on its 7 x 16 map),
    net1_deconv5 (NHWC deconvolution, split-K per parity class)."""
    want = {"net1_conv1": "fewci", "net1_conv2": "nhwc", "net1_conv6": "nhwc-split", "net1_deconv5": "nhwc-split"}
    out = []
    for name, ci, h, w, co, k, s, p, deconv, _ in deploy_convs("FlowNet2", 1024, 436):
        if name in want:
            out.append((SimtLayer(case("engine1-" + name, 4, ci, h, w, co, k, s, p, deconv, layout="pad", engine=1), "pad", None),
                        want[name]))
    return out


ENGINE1_CASES = _engine1_cases()


# ---- device data ------------------------------------------------------------------------------------------------------------
def draw(c):
    """bottom (NCHW, dense), Caffe-layout weights and bias (None without a bias term) on the device"""
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(c.name.encode()))
    x = torch.randn((c.N, c.Ci, c.H, c.W), generator=g, device="cuda")
    x = torch.where(x > 0, x, x * SLOPE)
    ws = weight_shape(c)
    w = torch.randn(ws, generator=g, device="cuda") * (2.0 / (ws[1] * ws[2] * ws[3])) ** 0.5
    b = torch.randn(c.Co, generator=g, device="cuda") if c.bias else None
    return x, w, b


def out_hw(c):
    ho, wo = C.c_int(), C.c_int()
    _check(_lib().fn2_conv_out_shape(C.byref(conv_desc(c)), c.H, c.W, C.byref(ho), C.byref(wo)))
    return ho.value, wo.value


class Top:
    """The top view inside a channels_last parent of `channels` channels at pixel stride `stride`, in one allocation with GUARD
    floats before and after it; the view starts as NaN, everything else holds SENTINEL."""

    def __init__(self, c, c0, channels, stride):
        ho, wo = out_hw(c)
        self.c0, self.co = c0, c.Co
        self.flat = torch.full((2 * GUARD + c.N * ho * wo * stride,), SENTINEL, device="cuda")
        self.body = self.flat[GUARD:GUARD + c.N * ho * wo * stride].view(c.N, ho, wo, stride)
        self.view = self.body.permute(0, 3, 1, 2)[:, c0:c0 + c.Co]
        self.fill_nan()
        self.outside = torch.ones_like(self.flat, dtype=torch.bool)
        self.outside[GUARD:GUARD + self.body.numel()].view(self.body.shape)[..., c0:c0 + c.Co] = False
        self.before = self.flat.clone()

    def fill_nan(self):
        self.view.fill_(float("nan"))

    def bits(self):
        return self.flat.view(torch.int32).clone()

    def outside_intact(self):
        return torch.equal(self.flat.view(torch.int32)[self.outside], self.before.view(torch.int32)[self.outside])


Run = namedtuple("Run", "go top x w b")


def prepare(L, engine=None, relu=None, bottom_layout=None):
    """Pack the weights, lay out the bottom and the top as the case says.  -> Run whose go() enqueues fn2_conv_forward."""
    from flownet2_b200 import ops as _ops
    c = L.case
    bl = bottom_layout or L.bottom
    x, w, b = draw(c)
    xv = bottom(x, bl)
    l, d = _lib(), conv_desc(c, guard_bytes(bl), c.engine if engine is None else engine, relu)
    cis = xv.stride(3)
    nf = C.c_size_t()
    _check(l.fn2_conv_packed_floats(C.byref(d), cis, C.byref(nf)))
    packed = torch.empty(max(nf.value, 1), device="cuda")
    _check(l.fn2_conv_pack_weights(C.byref(d), cis, op_weights(c, w).data_ptr(), packed.data_ptr(),
                                   torch.cuda.current_stream().cuda_stream))
    top = Top(c, L.top[0], L.top[1], cstride(L.top[1])) if L.top else Top(c, 16, c.Co + 32, c.Co + 32)
    nb = C.c_size_t()
    _check(l.fn2_conv_workspace_bytes(C.byref(d), c.N, c.H, c.W, C.byref(nb)))
    ws = torch.empty(max(nb.value // 4, 1), device="cuda")
    dx, dout = _ops.desc(xv), _ops.desc(top.view)

    def go():
        _check(l.fn2_conv_forward(C.byref(d), C.byref(dx), packed.data_ptr(), b.data_ptr() if b is not None else None,
                                  C.byref(dout), ws.data_ptr(), nb.value, torch.cuda.current_stream().cuda_stream))
    go.keep = (xv, packed, ws)
    return Run(go, top, x, w, b)


def route_of(L, bottom_layout=None):
    bl = layout_of(bottom_layout or L.bottom)
    return simt_route(L.case, bl[0], bl[1](L.case.Ci))


# ---- reference and bound ------------------------------------------------------------------------------------------------------
def every_pixel(c):
    ho, wo = out_hw(c)
    m = torch.ones((c.N, ho, wo), dtype=torch.bool, device="cuda")
    return [t.contiguous() for t in m.nonzero().unbind(1)]


def edges_and_sample(c):
    ho, wo = out_hw(c)
    m = torch.zeros((c.N, ho, wo), dtype=torch.bool, device="cuda")
    m[:, [0, ho - 1], :] = True
    m[:, :, [0, wo - 1]] = True
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(c.name.encode()) + 1)
    m.view(-1)[torch.randint(0, m.numel(), (SAMPLE,), generator=g, device="cuda")] = True
    return [t.contiguous() for t in m.nonzero().unbind(1)]


def check_bound(r, c, pixels, relu=None):
    """Every output at `pixels` within gamma(n + 3) absref of the float64 reference.  -> worst |got - ref| / bound"""
    n, oy, ox = pixels
    want = reference(c, r.x, r.w, r.b, n, oy, ox, relu)
    absref = reference(c, r.x.abs(), r.w.abs(), r.b.abs() if r.b is not None else None, n, oy, ox, relu)
    k = taps_at(c, n, oy, ox) * c.Ci + 3
    bound = (k * U / (1 - k * U))[:, None] * absref
    got = r.top.view[n, :, oy, ox].double()
    real = c.fwd[9] if c.fwd else c.Co
    assert bool((got[:, real:] == 0).all()), "padded output channels are not 0"
    got = got[:, :real]
    assert bool(torch.isfinite(got).all()), (c.name, "non-finite output")
    err = (got - want).abs()
    bad = err > bound
    if bool(bad.any()):
        i = int(bad.any(1).nonzero()[0])
        pytest.fail("%s: %d outputs off the bound; first at (n, y, x) = (%d, %d, %d): got %s, want %s, bound %s" % (
            c.name, int(bad.sum()), int(n[i]), int(oy[i]), int(ox[i]), got[i].tolist(), want[i].tolist(), bound[i].tolist()))
    return float((err / bound.clamp_min(1e-300)).max())


def run_checked(L, engine=None, relu=None, pixels=every_pixel):
    """Three runs -- into a NaN top, again unchanged, again after refilling the top with NaN -- with the same bits; nothing
    outside the top's view written; every output within the bound."""
    r = prepare(L, engine, relu)
    r.go()
    first = r.top.bits()
    assert r.top.outside_intact(), (L.case.name, "write outside the top's view")
    r.go()
    assert torch.equal(first, r.top.bits()), (L.case.name, "second run differs")
    r.top.fill_nan()
    r.go()
    assert torch.equal(first, r.top.bits()), (L.case.name, "run into a NaN top differs")
    return check_bound(r, L.case, pixels(L.case), relu)


# ---- the nets' shapes ---------------------------------------------------------------------------------------------------------
def test_simt_shapes_cover_the_routes(ops):
    """The cases reach the four kernels the nets run on SIMT, and every one of them is a layer the default engine does not give
    to the tensor cores."""
    routes = {route_of(L) for L in SHAPE_CASES}
    assert routes == {"pf3_tile", "pf3_warp", "pf_thread", "tiny_deconv"}, routes


def test_simt_shapes_iterate(ops):
    """On this card, for each route at least one case has more work than its grid has CTAs, so some CTA takes a second tile,
    group or pixel (grid rules: simt_route in fn2_conv.cu -- pf3_tile min(4 SMs, tiles), pf3_warp min(per_sm SMs, groups / 8),
    pf_thread min(8 SMs, pixels / 256) -- and ew_grid in fn2_common.cuh for tiny)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    most = {}
    for L in SHAPE_CASES:
        route = route_of(L)
        units, ctas = simt_work(L.case, route.replace("tiny_deconv", "tiny"), *out_hw(L.case), sms)
        most[route] = max(most.get(route, 0), units / ctas)
    assert all(v > 1 for v in most.values()) and len(most) == 4, most


def test_simt_shapes_route_kernels(ops):
    """Each case runs the kernel of its route (one profiler session over all cases)."""
    runs = [prepare(L) for L in SHAPE_CASES]
    names = kernels_per_case([r.go for r in runs])
    for L, got in zip(SHAPE_CASES, names):
        want = ROUTE_KERNEL[route_of(L)]
        assert any(want in k for k in got), (L.case.name, want, sorted(got))
        assert not any("conv_tc_kernel" in k or "conv_tn_kernel" in k for k in got), (L.case.name, sorted(got))


@pytest.mark.parametrize("L", SHAPE_CASES, ids=SHAPE_IDS)
def test_simt_shape(ops, L):
    ratio = run_checked(L)
    print("%s route %s worst err / bound %.3g" % (L.case.name, route_of(L), ratio))


# ---- the lanes beyond Ci --------------------------------------------------------------------------------------------------------
LANE_CASES = [
    SimtLayer(case("pf3_tile_ci2", 2, 2, 23, 45, 2, 3, 1, 1, layout="pad", engine=0), "pad", None),
    SimtLayer(case("pf3_tile_ci18", 2, 18, 23, 45, 2, 3, 1, 1, layout="pad", engine=0), "pad", None),
    SimtLayer(case("pf_thread_ci2", 2, 2, 23, 45, 2, 4, 2, 1, layout="pad", engine=0), "pad", None),
    SimtLayer(case("pf3_warp_ci194", 2, 194, 23, 45, 2, 3, 1, 1, layout="pad", engine=0), "pad", None),
    SimtLayer(case("pf_warp_ci66", 2, 66, 23, 45, 2, 5, 1, 2, layout="pad", engine=0), "pad", None),
]
LANE_LAYOUTS = ("pad", "padjunk", "padnan", "nhwc", "slice")


@pytest.mark.parametrize("L", LANE_CASES, ids=[L.case.name for L in LANE_CASES])
def test_simt_predictor_lanes_beyond_ci(ops, L):
    """Ci % 4 != 0: the last float4 group of a pixel holds lanes beyond Ci -- blob padding (zero, or finite garbage under the
    guard promise), NaN without it, or a neighbouring view's channels.  Under the guard promise the kernel reads them against
    zero weights; without it, its MASK instance (conv_pf3_tile_kernel<C4, true>, conv_pf_thread_kernel<C4, true>, or the
    overload of conv_pf3_warp_kernel / conv_pf_warp_kernel that takes a MaskLanes argument) selects 0 for them, since
    0 * NaN is NaN.  Every predictor route gives the same bits under all five layouts, within the bound of the reference."""
    runs = {bl: prepare(L, bottom_layout=bl) for bl in LANE_LAYOUTS}
    names = kernels_per_case([r.go for r in runs.values()])
    bits = {}
    for (bl, r), got in zip(runs.items(), names):
        route = route_of(L, bl)
        assert route == L.case.name.rsplit("_", 1)[0], (bl, route)
        masked = lambda k: "true>" in k or "MaskLanes" in k
        assert any(ROUTE_KERNEL[route] in k and masked(k) != bool(guard_bytes(bl)) for k in got), (bl, sorted(got))
        r.top.fill_nan()
        r.go()
        if bl == "pad":
            check_bound(r, L.case, every_pixel(L.case))
        bits[bl] = r.top.view.contiguous().view(torch.int32)
    for bl in LANE_LAYOUTS[1:]:
        v = bits[bl].view(torch.float32)
        assert torch.equal(bits[bl], bits["pad"]), (L.case.name, bl, "non-finite outputs: %d" % int((~torch.isfinite(v)).sum()))


# ---- the other SIMT routes at the nets' shapes ---------------------------------------------------------------------------------
@pytest.mark.parametrize("L,regime", ENGINE1_CASES, ids=[L.case.name for L, _ in ENGINE1_CASES])
def test_simt_engine1_layers(ops, L, regime):
    """engine = 1 runs every layer on SIMT: the deploy layers of FlowNet2 that reach fewci and the NHWC engine (unsplit, split-K,
    deconvolution), with leaky ReLU(0.1) as the nets fuse it, within the bound on every edge row and column and SAMPLE seeded
    random pixels; the split-K regimes run the fixed-order reduction, the others do not."""
    assert route_of(L) == regime.split("-")[0]
    got, = kernels_per_case([prepare(L, relu=SLOPE).go])
    assert any(ROUTE_KERNEL[route_of(L)] in k for k in got), sorted(got)
    assert any("conv_nhwc_reduce_kernel" in k for k in got) == regime.endswith("split"), sorted(got)
    ratio = run_checked(L, relu=SLOPE, pixels=edges_and_sample)
    print("%s worst err / bound %.3g" % (L.case.name, ratio))
