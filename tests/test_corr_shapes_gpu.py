"""FlowNet2's correlation (pad 20, kernel 1, max displacement 20, stride_1 1, stride_2 2, 441 displacements) at the shapes the
nets run it, on every forward route (tc, fast10, generic) and both backward routes (fast, tiled), against the float64
reference of tests/corr_ref.py, element by element; and the layer as FlowNet2-C's training graph wires it.

Shapes: 256 channels at the conv3 maps of bench.py's deploy workload (4 x 56 x 128: 1024 x 436 adapted to 1024 x 448), of
FlowNet2-CSS at 768 x 384 (4 x 48 x 96) and of the training step at 448 x 320 (8 x 40 x 56), and two odd maps a drop-in caller
produces (2 x 55 x 127, 2 x 41 x 57).  These reach what small maps do not: every CTA loops over 8 channel chunks, the tc route
has several 16-row tiles per parity plane, the persistent fast backward runs many waves over its 1536 units, and the TMA boxes
are element-strided reads of large maps.  Inputs are drawn like the nets' conv3 tops: leaky-ReLU(0.1) of N(0, 1).

Calls go through the C ABI with workspaces that are never cleared: each bottom sits in an allocation with 256 NaN floats
before and after it (Blob::kGuardFloats), outputs and workspaces start as NaN, the forward top and the backward top diff are
channels [32, 473) of an (N, 480, H, W) channels_last parent -- the place of `corr` in FlowNet2-C's `blob_corr`, after the 32
channels of conv_redir, pixel stride 473 rounded up to 32 --, and a second and third run (stale workspace, then workspace
filled with 1e30) must give the first run's bits.

Tolerance: |got - ref| <= tau * absref per element, absref the same operation on |inputs|.  u = 2^-24.

  * FP32 FMA chain of n products (fast10, generic forward; both backward routes): the chain rounds n - 1 times, each rounding
    at most u of the partial sum, which is at most the sum of the magnitudes; the division by C (or the product with 1 / C)
    adds one more rounding, exact for C = 256.  tau = (n + 2) u with n = C forward (the generic route's per-lane chains and
    5-step shuffle tree round fewer times) and n = 441 backward (tiled: a fresh chain per 8-channel chunk; fast: one chain per
    output over the 21 x 21 displacement grid).

  * tc (3xTF32 on wgmma).  Bottom 1 is split once by corr_split_kernel, bottom 0 in the MMA warpgroups; both with to_tf32, which
    rounds half away from zero to 11 significant bits: x = x_hi + x_lo + e, |x - x_hi| <= 2^-11 |x|, x - x_hi is exact in FP32,
    |e| <= 2^-11 |x - x_hi| <= 2^-22 |x|.  The engine forms a_hi b_hi + a_hi b_lo + a_lo b_hi (each TF32 product exact in FP32)
    and drops a_lo b_lo, so per product
        |ab - computed| <= |a_lo b_lo| + |e_a| |b_hi + b_lo| + |e_b| |a_hi + a_lo| + |e_a e_b|
                        <= ((2^-11 + 2^-22)^2 + 2 * 2^-22 (1 + 2^-22) + 2^-44) |ab|  ~= 12 u |ab|          (TAU_SPLIT)
    Each 32-channel step chains 12 wgmma k8 instructions into one accumulator, which starts at 0 per step (kd = 1 for the
    correlation's 128-row tiles): the 8 cross-term MMAs first, then the 4 a_hi b_hi MMAs.  A wgmma adds its 8 exact products
    to the accumulator by aligning to the largest addend and truncating, then truncates the sum to FP32.  Allowing two such
    alignment-and-normalisation steps per instruction (the k8 reduction may run as two halves), one instruction loses at most
    (8 + 2) 2^-23 (|accumulator| + sum of |its products|).  The accumulator before instruction j is at most the magnitudes of
    the products of instructions 1 .. j-1, so the chain loses at most 20 u sum_i (13 - i) |P_i|: weight <= 4 on the a_hi b_hi
    products (<= (1 + 2^-11)^2 |ab|), <= 12 on the cross terms (<= 2 (2^-11 + 2^-22)(1 + 2^-11) |ab|).            (TAU_MMA)
    The engine drains each step's chain into an FP32 register with acc += fmaf(c, comp, c), comp = TRUNC_LOSS_PER_MMA * 4 =
    5.2e-8 (a mean correction for the truncation, here bounded as an error of at most comp |c|)          (TAU_COMP)
    and the FP32 drain is a chain of C / 32 terms plus the fmaf and the scaling by 1 / C: tau_fp32(C / 32).
        tau_tc = tau_fp32(C / 32) + TAU_SPLIT + TAU_MMA + TAU_COMP  ~= 103.2 u ~= 6.2e-6  (C = 256)
    Second-order terms (errors of errors) are below 1e-4 of the bound; TAU_SLACK = 1 + 2^-10 covers them.
    tau_fp32(C / 32) alone is the FP32 drain's share; the split and the truncating chains are what tau_tc adds to it.
    Negative control (test_tc_bound_rejects_tf32_only): the float64 correlation of the inputs rounded to TF32 -- a 3xTF32 whose
    compensation was lost -- must violate tau_tc, so the bound tells FP32-faithful results from TF32-only ones.

Where absref is 0 (displacements that leave the image) the result must be exactly 0, so a stray halo read cannot hide.  NaNs
of four bit patterns (nan_probes) -- torch's, the device's own 0x7fffffff, a negative one and one with the smallest payload --
in both bottoms, inside a tile and at a tile corner of the route's own tiling, must make exactly the outputs non-finite that
the reference makes non-finite, on every route: the TF32 split must not round a NaN's payload into -0 or Inf, and the
generic route must multiply a non-finite bottom-0 value by the zero fill as the reference does.  Each case records its worst
|got - ref| / (tau absref) as the junit property `ratio`.
"""
import ctypes as C
import zlib

import numpy as np
import pytest

from tests import corr_ref
from tests.util import kernels_per_case

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

CH, PAD, KS, MD, S1, S2 = 256, 20, 1, 20, 1, 2
D = (2 * (MD // S2) + 1) ** 2                   # 441 top channels
PARENT, OFF = 480, 32                           # blob_corr's pixel stride; corr's first channel in it (after conv_redir)
GUARD = 256                                     # floats before and after every allocation (Blob::kGuardFloats)
SENTINEL = -7.25
SLOPE = 0.1

U = 2.0 ** -24


def tau_fp32(n):
    return (n + 2) * U


TAU_SPLIT = (2.0 ** -11 + 2.0 ** -22) ** 2 + 2 * 2.0 ** -22 * (1 + 2.0 ** -22) + 2.0 ** -44
TAU_MMA = 20 * U * (4 * (1 + 2.0 ** -11) ** 2 + 12 * 2 * (2.0 ** -11 + 2.0 ** -22) * (1 + 2.0 ** -11))
TAU_COMP = 1.3e-8 * 4                           # TRUNC_LOSS_PER_MMA (fn2_tc_ptx.cuh) x 4 a_hi b_hi MMAs per step
TAU_SLACK = 1 + 2.0 ** -10
TAU = {
    "tc": TAU_SLACK * (tau_fp32(CH // 32) + TAU_SPLIT + TAU_MMA + TAU_COMP),
    "fast10": TAU_SLACK * tau_fp32(CH),
    "generic": TAU_SLACK * tau_fp32(CH),
    "fast": TAU_SLACK * tau_fp32(D),
    "tiled": TAU_SLACK * tau_fp32(D),
}

# conv_redir's data gradient in the block test: the adjoint 1 x 1 convolution, 32 -> 256 channels, runs on the per-tap
# tensor-core engine in one 32-channel K step, so it has the tc bound with C / 32 = 1, plus 4 u: the two extra additions of
# the engine's drain at NT <= 64, the FP32 product of the top diff with the negative slope, and the scratch-diff addition that
# sums it with corr's bottom-0 gradient.
TAU_CONV_DGRAD = TAU_SLACK * (tau_fp32(1) + TAU_SPLIT + TAU_MMA + TAU_COMP) + 4 * U

# the kernels of each route, as the profiler names them (test_corr_routes_gpu.py)
FWD_KERNELS = {"tc": ["conv_tc_kernel<128, 3>", "corr_split_kernel("], "fast10": ["corr_fast_kernel<10>"],
               "generic": ["corr_generic_kernel("]}
BWD_KERNELS = {"fast": ["corr_bwd_fast_kernel<1>", "corr_bwd_fast_kernel<-1>", "corr_shift_kernel("],
               "tiled": ["corr_apply_kernel<0>", "corr_apply_kernel<1>"]}

DEPLOY, CSS, TRAIN, ODD1, ODD2 = (4, 56, 128), (4, 48, 96), (8, 40, 56), (2, 55, 127), (2, 41, 57)
SHAPES = {"deploy": DEPLOY, "css": CSS, "train": TRAIN, "odd55x127": ODD1, "odd41x57": ODD2}
FWD_CASES = ([("tc", s) for s in SHAPES] + [("fast10", s) for s in SHAPES] + [("generic", "deploy"), ("generic", "odd41x57")])
BWD_CASES = [(r, s) for r in ("fast", "tiled") for s in ("train", "odd55x127", "odd41x57")]

# NaN probes: (bottom, (y, x, channel), bit pattern).  Bottom 1 gets torch's NaN (0x7fc00000) at pixel (13, 11) -- sub-grid
# (6, 5) of parity plane (1, 1), inside the first tile of every tiling below -- and the device's own NaN (0x7fffffff, what
# arithmetic on the GPU produces) at a tile corner: the first pixel of the second tile row and column of the route's own tiling
# (sub-grid tiles of tc 16 x 8, fast10 10 x 8, fast backward 8 x 16; full-resolution 8 x 8 tiles of the tiled backward).
# Bottom 0 gets a negative NaN (0xffffffff) inside the map and a NaN with the smallest payload (0x7f800001) next to its corner,
# where most displacements leave the image: the reference multiplies it by the zero fill there, which is NaN too.
NAN_INTERIOR = (13, 11, 37)
NAN_CORNER = {"tc": (32, 16, 200), "fast10": (20, 16, 200), "generic": (20, 16, 200), "fast": (16, 32, 200),
              "tiled": (16, 16, 200)}


def nan_probes(route):
    return [(1, NAN_INTERIOR, 0x7fc00000), (1, NAN_CORNER[route], 0x7fffffff), (0, (25, 41, 5), 0xffffffff),
            (0, (1, 2, 130), 0x7f800001)]


@pytest.fixture(scope="module")
def ops(fn2):
    from flownet2_b200 import ops as _ops
    return _ops


def _lib():
    from flownet2_b200 import lib
    return lib()


def _check(rc):
    from flownet2_b200 import check
    check(rc)


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---- guarded device tensors ---------------------------------------------------------------------------------------------
class Guarded:
    """An (n, c, h, w) float32 view inside one allocation with GUARD floats of `guard` before and after it."""

    def __init__(self, shape, layout, fill, guard):
        n, c, h, w = shape
        self.guard = guard
        self.flat = torch.full((2 * GUARD + n * c * h * w,), fill, dtype=torch.float32, device="cuda")
        self.flat[:GUARD] = guard
        self.flat[-GUARD:] = guard
        body = self.flat[GUARD:GUARD + n * c * h * w]
        self.t = body.view(n, h, w, c).permute(0, 3, 1, 2) if layout == "nhwc" else body.view(n, c, h, w)

    def guards_intact(self):
        g = torch.cat([self.flat[:GUARD], self.flat[-GUARD:]])
        return bool(torch.isnan(g).all()) if self.guard != self.guard else bool((g == self.guard).all())


def bottom(x, layout):
    g = Guarded(tuple(x.shape), layout, float("nan"), float("nan"))
    g.t.copy_(x)
    return g


def concat_child(n, h, w, fill, rest):
    """Channels [OFF, OFF + D) of an (n, PARENT, h, w) channels_last parent: the child holds `fill`, the rest `rest`."""
    p = Guarded((n, PARENT, h, w), "nhwc", rest, rest)
    p.t[:, OFF:OFF + D] = fill
    return p, p.t[:, OFF:OFF + D]


def siblings_intact(p, rest):
    out = torch.cat([p.t[:, :OFF].reshape(-1), p.t[:, OFF + D:].reshape(-1)])
    return p.guards_intact() and (bool(torch.isnan(out).all()) if rest != rest else bool((out == rest).all()))


# ---- inputs -------------------------------------------------------------------------------------------------------------
def conv3_like(seed, shape):
    """leaky-ReLU(0.1) of N(0, 1), like the nets' conv3 tops."""
    x = np.random.default_rng(seed).standard_normal(shape).astype(np.float32)
    return torch.from_numpy(np.where(x > 0, x, np.float32(SLOPE) * x)).cuda()


def inputs(route, shape_name, backward=False):
    N, H, W = SHAPES[shape_name]
    seed = zlib.crc32(("%s-%s-%d" % (route, shape_name, backward)).encode())
    a, b = conv3_like(seed, (N, CH, H, W)), conv3_like(seed + 1, (N, CH, H, W))
    td = None
    if backward:
        td = torch.from_numpy(np.random.default_rng(seed + 2).standard_normal((N, D, H, W)).astype(np.float32)).cuda()
    return a, b, td


def with_nans(x, route, which):
    """x with the NaNs of nan_probes(route) for bottom `which` (for the reference: any NaN is NaN in float64)."""
    x = x.clone()
    for k, (y, xx, c), _ in nan_probes(route):
        if k == which:
            x[0, c, y, xx] = float("nan")
    return x


def poke_nans(t, route, which):
    """Writes the probes' NaN bit patterns into the device bottom `which`."""
    bits = t.view(torch.int32)
    for k, (y, x, c), pattern in nan_probes(route):
        if k == which:
            bits[0, c, y, x] = pattern - (1 << 32) if pattern >= 1 << 31 else pattern


# ---- comparison ---------------------------------------------------------------------------------------------------------
def worst_ratio(got, ref, absref, tau, what):
    """max |got - ref| / (tau absref) over the finite reference entries; the non-finite sets must be equal and absref == 0 must
    give exactly 0."""
    got = got.double()
    fin = torch.isfinite(ref)
    assert bool((torch.isfinite(got) == fin).all()), "%s: non-finite outputs differ from the reference's" % what
    zero = fin & (absref == 0)
    assert bool((got[zero] == 0).all()), "%s: nonzero output where every product is 0" % what
    nz = fin & (absref > 0)
    return float(((got - ref).abs()[nz] / (tau * absref[nz])).max())


# ---- the calls ----------------------------------------------------------------------------------------------------------
class FwdRun:
    """One forward case through fn2_correlation_forward: guarded bottoms, NaN-filled top and workspace."""

    def __init__(self, route, a, b, shape_name):
        N, H, W = SHAPES[shape_name]
        self.route = route
        self.layout = "nchw" if route == "fast10" or (route == "generic" and shape_name != "deploy") else "nhwc"
        self.b0, self.b1 = bottom(a, self.layout), bottom(b, self.layout)
        if self.layout == "nhwc":
            self.parent, self.top = concat_child(N, H, W, float("nan"), SENTINEL)
        else:
            self.parent = Guarded((N, D, H, W), "nchw", float("nan"), SENTINEL)
            self.top = self.parent.t
        need = C.c_size_t()
        _check(_lib().fn2_correlation_workspace_bytes(N, CH, H, W, PAD, KS, MD, S1, S2, 0, C.byref(need)))
        self.nbytes = need.value if route != "generic" else 0
        self.ws = torch.full((max(self.nbytes // 4, 1),), float("nan"), device="cuda")

    def go(self):
        from flownet2_b200.ops import desc
        ws = C.c_void_p(self.ws.data_ptr()) if self.nbytes else None
        _check(_lib().fn2_correlation_forward(desc(self.b0.t), desc(self.b1.t), desc(self.top), PAD, KS, MD, S1, S2, 0, ws,
                                              C.c_size_t(self.nbytes), _stream()))

    def outputs(self):
        return [self.top]

    def intact(self):
        ok = self.b0.guards_intact() and self.b1.guards_intact()
        if self.layout == "nhwc":
            return ok and siblings_intact(self.parent, SENTINEL)
        return ok and self.parent.guards_intact()

    def kernels(self):
        return FWD_KERNELS


class BwdRun:
    """One backward case through fn2_correlation_backward: guarded bottoms and top diff, NaN-filled diffs and workspace."""

    def __init__(self, route, a, b, td, shape_name):
        N, H, W = SHAPES[shape_name]
        self.route = route
        self.layout = "nhwc" if route == "fast" else "nchw"
        self.b0, self.b1 = bottom(a, self.layout), bottom(b, self.layout)
        if route == "fast":
            self.tdp, self.td = concat_child(N, H, W, 0.0, float("nan"))
            self.td.copy_(td)
        else:
            self.tdp = bottom(td, "nchw")
            self.td = self.tdp.t
        self.d0 = Guarded((N, CH, H, W), self.layout, float("nan"), SENTINEL)
        self.d1 = Guarded((N, CH, H, W), self.layout, float("nan"), SENTINEL)
        need = C.c_size_t()
        _check(_lib().fn2_correlation_backward_workspace_bytes(N, CH, H, W, PAD, KS, MD, S1, S2, 0, C.byref(need)))
        self.nbytes = need.value
        self.ws = torch.full((max(self.nbytes // 4, 1),), float("nan"), device="cuda")

    def go(self):
        from flownet2_b200.ops import desc
        _check(_lib().fn2_correlation_backward(desc(self.b0.t), desc(self.b1.t), desc(self.td), desc(self.d0.t), desc(self.d1.t),
                                               PAD, KS, MD, S1, S2, 0, C.c_void_p(self.ws.data_ptr()), C.c_size_t(self.nbytes),
                                               _stream()))

    def outputs(self):
        return [self.d0.t, self.d1.t]

    def intact(self):
        ok = all(g.guards_intact() for g in (self.b0, self.b1, self.d0, self.d1))
        if self.route == "fast":
            return ok and siblings_intact(self.tdp, float("nan"))
        return ok and self.tdp.guards_intact()

    def kernels(self):
        return BWD_KERNELS


def run_checked(run):
    """Runs `run` three times -- NaN workspace, the stale workspace of the first run, a workspace of 1e30 -- and requires the
    same bits each time, the guards and sibling channels untouched.  -> the outputs (clones)."""
    runs = []
    run.ws.fill_(float("nan"))
    for fill in (None, "stale", 1e30):
        for o in run.outputs():
            o.fill_(float("nan"))
        if fill == 1e30:
            run.ws.fill_(1e30)
        run.go()
        torch.cuda.synchronize()
        runs.append([o.clone() for o in run.outputs()])
        assert run.intact(), "a guard float or a sibling channel changed"
    for other in runs[1:]:
        for x, y in zip(runs[0], other):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), "results depend on the run or on the workspace"
    return runs[0]


def check_route(run):
    """The case runs its route's kernels and no other route's."""
    names = kernels_per_case([run.go])[0]
    for r, knames in run.kernels().items():
        for k in knames:
            assert any(k in n for n in names) == (r == run.route), (run.route, k, sorted(names))


# ---- forward ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route,shape_name", FWD_CASES, ids=["%s-%s" % c for c in FWD_CASES])
def test_corr_forward_shapes(ops, route, shape_name, record_property):
    a, b, _ = inputs(route, shape_name)
    ref, absref = corr_ref.forward(a, b, MD, S2)
    run = FwdRun(route, a, b, shape_name)
    got, = run_checked(run)
    ratio = worst_ratio(got, ref, absref, TAU[route], route)
    check_route(run)
    # NaN probes: the same non-finite set as the reference, everything else still within the bound
    an, bn = with_nans(a, route, 0), with_nans(b, route, 1)
    poke_nans(run.b0.t, route, 0)
    poke_nans(run.b1.t, route, 1)
    got_n, = run_checked(run)
    ref_n, absref_n = corr_ref.forward(an, bn, MD, S2)
    assert not bool(torch.isfinite(ref_n).all())
    ratio = max(ratio, worst_ratio(got_n, ref_n, absref_n, TAU[route], route + " with NaN"))
    record_property("ratio", ratio)
    assert ratio <= 1, (route, shape_name, ratio)


# ---- backward -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route,shape_name", BWD_CASES, ids=["%s-%s" % c for c in BWD_CASES])
def test_corr_backward_shapes(ops, route, shape_name, record_property):
    a, b, td = inputs(route, shape_name, backward=True)
    d0, d1, abs0, abs1 = corr_ref.backward(a, b, td, MD, S2)
    run = BwdRun(route, a, b, td, shape_name)
    g0, g1 = run_checked(run)
    ratio = max(worst_ratio(g0, d0, abs0, TAU[route], "d bottom0"), worst_ratio(g1, d1, abs1, TAU[route], "d bottom1"))
    check_route(run)
    an, bn = with_nans(a, route, 0), with_nans(b, route, 1)
    poke_nans(run.b0.t, route, 0)
    poke_nans(run.b1.t, route, 1)
    g0n, g1n = run_checked(run)
    d0n, d1n, abs0n, abs1n = corr_ref.backward(an, bn, td, MD, S2)
    assert not bool(torch.isfinite(d0n).all()) and not bool(torch.isfinite(d1n).all())
    ratio = max(ratio, worst_ratio(g0n, d0n, abs0n, TAU[route], "d bottom0 with NaN"),
                worst_ratio(g1n, d1n, abs1n, TAU[route], "d bottom1 with NaN"))
    record_property("ratio", ratio)
    assert ratio <= 1, (route, shape_name, ratio)


# ---- the bound tells FP32-faithful from TF32-only -----------------------------------------------------------------------
def tf32(x):
    """x rounded to TF32 as to_tf32 does (half away from zero to 11 significant bits)."""
    return ((x.view(torch.int32) + 0x1000) & -0x2000).view(torch.float32)


def test_tc_bound_rejects_tf32_only(ops, record_property):
    """The float64 correlation of the TF32-rounded bottoms (3xTF32 without its compensation terms) violates tau_tc: the bound
    is tight enough to fail a tensor-core route that lost FP32 faithfulness."""
    a, b, _ = inputs("tc", "train")
    ref, absref = corr_ref.forward(a, b, MD, S2)
    lost, _ = corr_ref.forward(tf32(a), tf32(b), MD, S2)
    ratio = worst_ratio(lost, ref, absref, TAU["tc"], "tf32-only")
    record_property("ratio", ratio)
    assert ratio > 1, ratio


# ---- the layer inside FlowNet2-C's concat, at the training shape ---------------------------------------------------------
def block_prototxt(n, h, w):
    """FlowNet2-C's correlation block (models/FlowNet2-C_train.prototxt.template: corr, ReLU_corr, conv_redir and its ReLU,
    Concat_corr) on conv3a / conv3b inputs."""
    return ('force_backward: true\n'
            'layer { name: "in" type: "Input" top: "conv3a" top: "conv3b" input_param { shape { dim: %d dim: %d dim: %d dim: %d } } }\n'
            'layer { name: "corr" type: "Correlation" bottom: "conv3a" bottom: "conv3b" top: "corr" correlation_param { pad: 20 '
            'kernel_size: 1 max_displacement: 20 stride_1: 1 stride_2: 2 } }\n'
            'layer { name: "ReLU_corr" type: "ReLU" bottom: "corr" top: "corr" relu_param { negative_slope: 0.1 } }\n'
            'layer { name: "conv_redir" type: "Convolution" bottom: "conv3a" top: "conv_redir" param { lr_mult: 1 decay_mult: 1 } '
            'param { lr_mult: 1 decay_mult: 0 } convolution_param { num_output: 32 pad: 0 kernel_size: 1 stride: 1 '
            'weight_filler { type: "msra" } bias_filler { type: "constant" value: 0 } engine: CUDNN } }\n'
            'layer { name: "ReLU_conv_redir" type: "ReLU" bottom: "conv_redir" top: "conv_redir" relu_param { negative_slope: 0.1 } }\n'
            'layer { name: "Concat_corr" type: "Concat" bottom: "conv_redir" bottom: "corr" top: "blob_corr" concat_param { axis: 1 } }\n'
            % (n, CH, h, w))


def run_block(fn2, a, b, seed_diff, bias):
    N, _, H, W = a.shape
    net = fn2.Net(block_prototxt(N, H, W), None, fn2.TEST)
    net.fill_params(11)
    from oracle.net import write_caffemodel
    net.copy_from(write_caffemodel([("conv_redir", "Convolution", [net.param("conv_redir", 0), bias])]))
    net.forward(conv3a=a, conv3b=b)
    net.clear_param_diffs()
    net.backward(blob_corr=seed_diff)
    return {"blob_corr": net.blobs["blob_corr"].data, "conv3a": net.get_diff("conv3a"), "conv3b": net.get_diff("conv3b"),
            "w": net.param("conv_redir", 0, diff=True), "b": net.param("conv_redir", 1, diff=True),
            "weights": net.param("conv_redir", 0)}


def test_corr_block_in_training_graph(fn2, monkeypatch, record_property):
    """blob_corr, the diffs of conv3a (corr's bottom-0 gradient plus conv_redir's data gradient, summed through the layer's
    scratch diff) and conv3b, and conv_redir's parameter diffs, at 8 x 256 x 40 x 56, against float64; then the same block with
    FN2_NO_ALIAS and FN2_NO_FUSE (plain, unfused layout) must give the same bits.  The correlation parts are held to the
    bounds of the kernel tests above (tc forward, fast backward: the net's blobs are channels_last), conv_redir's share of the
    conv3a diff element by element to TAU_CONV_DGRAD; conv_redir's top and parameter diffs to the 1e-5 of the largest entry
    the convolution gradient tests use."""
    N, H, W = TRAIN
    a, b = conv3_like(901, (N, CH, H, W)).cpu().numpy(), conv3_like(902, (N, CH, H, W)).cpu().numpy()
    rng = np.random.default_rng(903)
    seed_diff = rng.standard_normal((N, OFF + D, H, W)).astype(np.float32)
    bias = (0.1 * rng.standard_normal(32)).astype(np.float32)
    got = run_block(fn2, a, b, seed_diff, bias)

    # float64 reference, differentiated at the engine's activations (a ReLU input within rounding of 0 must not pick
    # different sides of the kink in the two computations)
    A, B = torch.from_numpy(a).cuda().double(), torch.from_numpy(b).cuda().double()
    Wt, Bs = torch.from_numpy(got["weights"]).cuda().double(), torch.from_numpy(bias).cuda().double()
    G = torch.from_numpy(seed_diff).cuda().double()
    corr, corr_abs = corr_ref.forward(A, B, MD, S2)
    redir_pre = torch.nn.functional.conv2d(A, Wt, Bs)
    top = torch.from_numpy(got["blob_corr"]).cuda().double()
    u_tc = TAU["tc"] + 2 * U                        # + the rounding of the negative slope's product
    mask = torch.where(top > 0, 1.0, SLOPE)
    r_corr = worst_ratio(top[:, OFF:], mask[:, OFF:] * corr, mask[:, OFF:] * corr_abs, u_tc, "corr")
    redir = mask[:, :OFF] * redir_pre
    e_redir = float((top[:, :OFF] - redir).abs().max() / redir.abs().max())
    assert e_redir <= 1e-5, e_redir

    g_redir = G[:, :OFF] * mask[:, :OFF]
    g_corr = G[:, OFF:] * mask[:, OFF:]
    # the bound of the fast backward on the slope-scaled diff (the product with 0.1 is rounded in FP32 first)
    d0, d1, abs0, abs1 = corr_ref.backward(A, B, g_corr, MD, S2)
    da_redir = torch.nn.functional.conv_transpose2d(g_redir, Wt)
    ga, gb = torch.from_numpy(got["conv3a"]).cuda().double(), torch.from_numpy(got["conv3b"]).cuda().double()
    tb = TAU["fast"] + 2 * U
    r_b = worst_ratio(gb, d1, abs1, tb, "conv3b diff")
    # conv3a, element by element: corr's part within the fast backward's bound plus conv_redir's data gradient within the
    # bound of its own 3xTF32 sum (TAU_CONV_DGRAD) against |g| * |W|
    abs_redir = torch.nn.functional.conv_transpose2d(g_redir.abs(), Wt.abs())
    r_a = float(((ga - d0 - da_redir).abs() / (tb * abs0 + TAU_CONV_DGRAD * abs_redir)).max())
    dw = torch.einsum("nohw,nchw->oc", g_redir, A).reshape(32, CH, 1, 1)
    db = g_redir.sum((0, 2, 3))
    e_w = float((torch.from_numpy(got["w"]).cuda() - dw).abs().max() / dw.abs().max())
    e_b = float((torch.from_numpy(got["b"]).cuda().reshape(-1) - db).abs().max() / db.abs().max())
    assert e_w <= 1e-5 and e_b <= 1e-5, (e_w, e_b)
    record_property("ratio", max(r_corr, r_a, r_b))
    assert r_corr <= 1 and r_a <= 1 and r_b <= 1, (r_corr, r_a, r_b)

    monkeypatch.setenv("FN2_NO_FUSE", "1")
    monkeypatch.setenv("FN2_NO_ALIAS", "1")
    plain = run_block(fn2, a, b, seed_diff, bias)
    for k in got:
        assert np.array_equal(got[k].view(np.int32), plain[k].view(np.int32)), k
