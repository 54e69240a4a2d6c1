"""Weight and bias gradients (fn2_conv_backward_params) on both engines against a float64 reference, plan by plan.

The tensor-core route (fn2_conv_tc.cu, conv_tc_wgrad) takes every layer with at most 49 taps and a stride of at most 8; the
SIMT route (fn2_train.cu, weight_grad_kernel) takes the rest and `engine: CAFFE`.  The cases of PLAN_CASES are built so that,
together, they reach every value of the tensor-core plan (fn2_conv_wgrad_plan: small channels per tile NT, big-map rows per
tap G, big / small channel tiles BT / ST with a tail, K ranges S, column delays, bias blocks over several column tiles) and
both pixel-split regimes of the SIMT route; `test_wgrad_plan_coverage` checks that they do on the card the suite runs on (S
depends on its SM count), `test_wgrad_route_kernels` that each case runs the kernels of its route.  TRAIN_CASES are the
trainable layers of the training graphs at 448x320 with inputs drawn like the nets' (post-ReLU bottom, top diff of non-zero
mean), where every product of a reduction has the same sign.

Reference: per kernel tap one float64 BLAS product of the small map with the strided window of the zero-padded big map
(`ref_grads`), pinned to oracle.conv_bwd (itself pinned to the reference's ConvolutionLayer::Backward by train_golden.npz).
Tolerance: 1e-5 of each tensor's largest entry, as in test_train_gpu.py.
"""
import zlib

import numpy as np
import pytest

from oracle import oracle as O
from tests.util import device_view, kernels_per_case, maxabs, rng, train_convs

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

TOL = 1e-5


@pytest.fixture(scope="module")
def ops(fn2):
    from flownet2_b200 import ops as _ops
    return _ops


# ---- cases ----------------------------------------------------------------------------------------------------------------
def case(name, N, Ci, H, W, Co, k, s, p, deconv=False, engine=0):
    """-> (name, N, Ci, H, W, Co, (kh, kw), s, (ph, pw), deconv, engine)"""
    k = (k, k) if isinstance(k, int) else tuple(k)
    p = (p, p) if isinstance(p, int) else tuple(p)
    return (name, N, Ci, H, W, Co, k, s, p, deconv, engine)


def out_hw(c):
    _, N, Ci, H, W, Co, (kh, kw), s, (ph, pw), deconv, _ = c
    if deconv:
        return s * (H - 1) + kh - 2 * ph, s * (W - 1) + kw - 2 * pw
    return (H + 2 * ph - kh) // s + 1, (W + 2 * pw - kw) // s + 1


def small_big(c):
    """(Cs, Hs, Ws, Cb, Hb, Wb): the small map is the top diff of a convolution and the bottom of a deconvolution."""
    _, N, Ci, H, W, Co, k, s, p, deconv, _ = c
    Ho, Wo = out_hw(c)
    return (Ci, H, W, Co, Ho, Wo) if deconv else (Co, Ho, Wo, Ci, H, W)


PLAN_CASES = [
    # tensor cores; comments: small channels -> NT, big channels -> G (rows per tap), taps per 128-row tile, what else it reaches
    case("nt16_g8_k7s2", 2, 3, 23, 70, 16, 7, 2, 3),              # NT 16, G 8: 49 taps in 4 groups of 16 (last: 1); delays 0-3
    case("nt32_g16_k3", 1, 12, 20, 37, 32, 3, 1, 1),              # NT 32, G 16: 9 taps in groups of 8; 37 columns: 2 segments
    case("nt64_g32_k3", 1, 24, 13, 29, 64, 3, 1, 1),              # NT 64, G 32: 9 taps in groups of 4
    case("nt128_g64_k5s2", 1, 48, 21, 33, 128, 5, 2, 2),          # NT 128, G 64: 25 taps in groups of 2
    case("g128_bt2_tail", 1, 130, 9, 17, 64, 3, 1, 1),            # two big-channel tiles, the second with 2 rows
    case("st2_tail", 2, 32, 15, 19, 144, 3, 2, 1),                # two small-channel tiles, the second with 16 channels
    case("bt2_st2", 1, 200, 6, 10, 160, 3, 1, 1),                 # both
    case("s3", 1, 16, 25, 40, 32, 5, 3, 2),
    case("s4", 1, 8, 30, 45, 16, 6, 4, 1),
    case("s8", 1, 4, 40, 70, 16, 5, 8, 2),
    case("aniso_k3x5", 1, 20, 17, 31, 48, (3, 5), 2, (0, 2)),     # kh != kw, pad_h != pad_w
    case("small_1x1", 2, 64, 3, 3, 128, 3, 1, 0),                 # 1x1 small map: one K segment per sample, S = 1
    case("s1_many_tiles", 1, 1024, 3, 4, 512, 3, 1, 1),           # 9 x 8 x 4 tile units fill the GPU: S = 1
    case("bias_cols_conv", 1, 8, 5, 150, 32, 3, 1, 1),            # top diff 150 wide: bias blocks over 2 column tiles
    case("d_s2", 2, 64, 7, 12, 32, 4, 2, 1, True),
    case("d_s3", 1, 16, 6, 9, 8, 5, 3, 1, True),
    case("d_bias_cols", 1, 32, 4, 130, 16, 4, 2, 1, True),        # top diff 260 wide: parity planes of 133 columns
    case("d_g16_tail", 1, 144, 5, 6, 12, 3, 1, 1, True),          # deconv: small map 144 channels, big map 12
    # SIMT
    case("simt_9x9", 1, 16, 12, 20, 32, 9, 1, 4),                 # 81 taps: one pixel range
    case("simt_9x9_split", 1, 16, 24, 40, 32, 9, 1, 4),           # ... several pixel ranges
    case("simt_s9", 1, 8, 30, 50, 16, 3, 9, 1),                   # stride 9
    case("simt_d9x9", 1, 8, 6, 9, 16, 9, 2, 4, True),
    case("simt_engine1", 2, 32, 20, 30, 64, 3, 2, 1, engine=1),
    case("simt_engine1_d", 1, 32, 7, 12, 16, 4, 2, 1, True, engine=1),
    case("simt_co300", 1, 8, 10, 14, 300, 3, 1, 1, engine=1),     # bias over 300 channels: two passes of 256
]
PLAN_IDS = [c[0] for c in PLAN_CASES]


def is_simt(c):
    return c[10] == 1 or c[6][0] * c[6][1] > 49 or c[7] > 8


# ---- reference --------------------------------------------------------------------------------------------------------------
def ref_grads(x, dy, k, s, p, deconv):
    """float64 (dW in Caffe layout, db): per tap, dW[:, :, ky, kx] = small . window(ky, kx) of the padded big map, on BLAS."""
    (kh, kw), (ph, pw) = k, p
    x, dy = np.asarray(x, np.float64), np.asarray(dy, np.float64)
    small, big = (x, dy) if deconv else (dy, x)
    N, Cs, Hs, Ws = small.shape
    _, Cb, Hb, Wb = big.shape
    eh, ew = max(0, (Hs - 1) * s + kh - ph - Hb), max(0, (Ws - 1) * s + kw - pw - Wb)
    bp = np.zeros((Cb, N, ph + Hb + eh, pw + Wb + ew))
    bp[:, :, ph:ph + Hb, pw:pw + Wb] = big.transpose(1, 0, 2, 3)
    sm = small.transpose(1, 0, 2, 3).reshape(Cs, -1)
    dw = np.empty((Cs, Cb, kh, kw))
    for ky in range(kh):
        for kx in range(kw):
            win = bp[:, :, ky:ky + s * (Hs - 1) + 1:s, kx:kx + s * (Ws - 1) + 1:s].reshape(Cb, -1)
            dw[:, :, ky, kx] = sm @ win.T
    return dw, dy.sum(axis=(0, 2, 3))


def inputs(c, seed, same_sign=False):
    """bottom and top diff; same_sign: drawn like the nets' (bottom >= 0 after a ReLU, top diff of mean 1)."""
    _, N, Ci, H, W, Co, k, s, p, deconv, _ = c
    Ho, Wo = out_hw(c)
    r = rng(seed)
    x = r.standard_normal((N, Ci, H, W))
    dy = r.standard_normal((N, Co, Ho, Wo))
    if same_sign:
        x, dy = np.maximum(x, 0.0), dy + 1.0
    return x.astype(np.float32), dy.astype(np.float32)


def seed_of(c):
    return zlib.crc32(repr(c).encode())


dev = device_view


def weight_shape(c):
    _, N, Ci, H, W, Co, (kh, kw), s, p, deconv, _ = c
    return (Ci, Co, kh, kw) if deconv else (Co, Ci, kh, kw)


def run(ops, c, x, dy, layout="nhwc", **kw):
    """-> (dW, db or None) as torch tensors (no data gradient)."""
    _, N, Ci, H, W, Co, k, s, p, deconv, engine = c
    w = torch.zeros(weight_shape(c), device="cuda")
    _, gw, gb = ops.conv2d_backward(dev(x, layout), w, dev(dy, layout), s, p, deconv, need_input_grad=False, engine=engine, **kw)
    return gw, gb


def rel(got, want):
    return maxabs(got, want) / max(float(np.abs(want).max()), 1e-30)


def shrink(got, want):
    """mean signed error relative to mean |want|: < 0 when the engine's sums come out systematically too small in magnitude"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return float(((got - want) * np.sign(want)).mean() / np.abs(want).mean())


def check(ops, c, layout="nhwc", same_sign=False, seed=None):
    x, dy = inputs(c, seed_of(c) if seed is None else seed, same_sign)
    gw, gb = run(ops, c, x, dy, layout)
    ww, wb = ref_grads(x, dy, c[6], c[7], c[8], c[9])
    gw, gb = gw.cpu().numpy(), gb.cpu().numpy()
    assert np.isfinite(gw).all() and np.isfinite(gb).all()
    ew, eb = rel(gw, ww), rel(gb, wb)
    assert ew <= TOL and eb <= TOL, (c[0], layout, ew, eb)
    return ew, eb, shrink(gw, ww)


# ---- the reference itself ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", [case("c", 2, 5, 9, 11, 7, 3, 1, 1), case("c_s2", 1, 6, 10, 13, 4, 5, 2, 2),
                               case("c_k3x5", 1, 3, 8, 12, 5, (3, 5), 2, (0, 2)), case("d_s2", 2, 4, 4, 5, 3, 4, 2, 1, True),
                               case("d_s3", 1, 3, 3, 4, 5, 5, 3, 1, True)], ids=lambda c: c[0])
def test_reference_matches_oracle(c):
    """ref_grads against oracle.conv_bwd (float64 einsum, no BLAS, result rounded to float32) on small cases: every entry is the
    oracle's to within the float32 rounding of the oracle's result."""
    x, dy = inputs(c, 3)
    _, ow, ob = O.conv_bwd(x, np.zeros(weight_shape(c), np.float32), dy, c[7], c[8], c[9])
    ww, wb = ref_grads(x, dy, c[6], c[7], c[8], c[9])
    for got, want in ((ow, ww), (ob, wb)):
        assert (np.abs(got - want) <= 2 ** -24 * np.abs(want) + 1e-12 * np.abs(want).max()).all()


# ---- plan coverage and routes -------------------------------------------------------------------------------------------------
def plan_of(ops, c, bias=True):
    _, N, Ci, H, W, Co, k, s, p, deconv, engine = c
    return ops.wgrad_plan(Ci, Co, k, s, p, deconv, N, H, W, engine, bias)


def delays(c):
    """column delays (copies of the big map) the taps of a tensor-core case read: (-floor((kx - pad_w) / s)) mod 4"""
    kw, pw, s = c[6][1], c[8][1], c[7]
    return {(-((kx - pw) // s)) % 4 for kx in range(kw)}


def test_wgrad_plan_coverage(ops):
    """The table reaches every plan value listed in the module docstring on this card."""
    tc, simt = [], []
    for c in PLAN_CASES:
        pl = plan_of(ops, c)
        assert pl[0] == (1 if is_simt(c) else 2), (c[0], pl)
        (simt if is_simt(c) else tc).append((c, pl))
    assert {pl[1] for _, pl in tc} >= {16, 32, 64, 128}
    assert {pl[2] for _, pl in tc} >= {8, 16, 32, 64, 128}
    taps = lambda c: c[6][0] * c[6][1]
    for G in (8, 16, 32, 64):           # a partial last tap group at every G with several taps per tile
        assert any(pl[2] == G and taps(c) % (128 // G) for c, pl in tc), G
    assert any(pl[4] > 1 and small_big(c)[3] % 128 for c, pl in tc)
    assert any(pl[5] > 1 and small_big(c)[0] % pl[1] for c, pl in tc)
    assert {c[7] for c, _ in tc if not c[9]} >= {1, 2, 3, 4, 8} and {c[7] for c, _ in tc if c[9]} >= {2, 3}
    assert set().union(*(delays(c) for c, _ in tc)) == {0, 1, 2, 3}
    assert any(c[6][0] != c[6][1] and c[8][0] != c[8][1] for c, _ in tc)
    assert {min(pl[6], 2) for _, pl in tc} == {1, 2}
    assert any(small_big(c)[2] > 32 and small_big(c)[2] % 32 for c, _ in tc)
    assert any(small_big(c)[1:3] == (1, 1) for c, _ in tc)
    # bias blocks over more than one 128-column tile: one block per row of the top diff and column tile; the top diff is the
    # small map of a convolution and the big map, as s parity planes per row, of a deconvolution
    assert any(pl[7] > c[1] * small_big(c)[1] for c, pl in tc if not c[9])
    assert any(pl[7] > c[1] * small_big(c)[4] * c[7] for c, pl in tc if c[9])
    assert {min(pl[6], 2) for _, pl in simt} == {1, 2}
    assert any(c[5] > 256 for c, _ in simt) and any(c[9] for c, _ in simt) and any(not c[9] for c, _ in simt)
    assert plan_of(ops, PLAN_CASES[0], bias=False)[7] == 0


@pytest.mark.parametrize("c", PLAN_CASES, ids=PLAN_IDS)
def test_wgrad_plan_case(ops, c):
    check(ops, c)


@pytest.mark.parametrize("c", PLAN_CASES, ids=PLAN_IDS)
def test_wgrad_route_kernels(ops, c):
    """The case runs the kernels of its plan: the tensor-core kernel with the planned NT, its bias reduction exactly when a bias
    gradient is asked for; the SIMT weight and bias kernels for the others."""
    x, dy = inputs(c, 1)
    xd, dd, wd = dev(x), dev(dy), torch.zeros(weight_shape(c), device="cuda")
    pl = plan_of(ops, c)
    runs = [lambda bias=bias: ops.conv2d_backward(xd, wd, dd, c[7], c[8], c[9], bias=bias, need_input_grad=False, engine=c[10])
            for bias in (True, False)]
    for bias, got in zip((True, False), kernels_per_case(runs)):
        has = lambda k: any(k in n for n in got)
        if pl[0] == 2:
            assert has("conv_tc_kernel<%d, 4>" % pl[1]) and has("wg_reduce_kernel") and not has("weight_grad_kernel("), sorted(got)
            assert has("wg_bias_final_kernel") == bias and not has("bias_grad_partial_kernel"), (bias, sorted(got))
        else:
            assert has("weight_grad_kernel(") and not has("conv_tc_kernel<"), sorted(got)
            assert has("bias_grad_partial_kernel") == bias and not has("wg_bias_final_kernel"), (bias, sorted(got))


# ---- layouts, accumulation, determinism, workspace ----------------------------------------------------------------------------
LAYOUT_CASES = [PLAN_CASES[1], PLAN_CASES[14], PLAN_CASES[22], PLAN_CASES[23]]


@pytest.mark.parametrize("layout", ["nchw", "nhwc", "pad", "slice"])
@pytest.mark.parametrize("c", LAYOUT_CASES, ids=[c[0] for c in LAYOUT_CASES])
def test_wgrad_layouts(ops, c, layout):
    """Bottom and top diff as NCHW, channels_last, with the nets' padded pixel stride, and as a channel slice of a wider parent
    whose other channels hold NaN."""
    check(ops, c, layout)


ACC_CASES = [PLAN_CASES[0], PLAN_CASES[14], PLAN_CASES[22], PLAN_CASES[23]]


@pytest.mark.parametrize("c", ACC_CASES, ids=[c[0] for c in ACC_CASES])
def test_wgrad_accumulate_and_bias_pointer(ops, c):
    """accumulate = 1 adds dW and db to non-zero priors; has_bias = 0 leaves the bias diff alone; a null bias pointer with
    has_bias = 1 computes dW only."""
    x, dy = inputs(c, seed_of(c) + 1)
    ww, wb = ref_grads(x, dy, c[6], c[7], c[8], c[9])
    r = rng(seed_of(c) + 2)
    pw = r.standard_normal(ww.shape).astype(np.float32)
    pb = r.standard_normal(wb.shape).astype(np.float32)
    gw, gb = torch.from_numpy(pw).cuda(), torch.from_numpy(pb).cuda()
    run(ops, c, x, dy, accumulate=True, out=(gw, gb))
    assert rel(gw.cpu().numpy(), pw + ww) <= TOL and rel(gb.cpu().numpy(), pb + wb) <= TOL
    gw, gb = torch.from_numpy(pw).cuda(), torch.from_numpy(pb).cuda()
    run(ops, c, x, dy, bias=False, out=(gw, gb))
    assert rel(gw.cpu().numpy(), ww) <= TOL and np.array_equal(gb.cpu().numpy(), pb)
    gw = torch.from_numpy(pw).cuda()
    run(ops, c, x, dy, bias=True, out=(gw, None))
    torch.cuda.synchronize()
    assert rel(gw.cpu().numpy(), ww) <= TOL


@pytest.mark.parametrize("c", [PLAN_CASES[0], PLAN_CASES[16], PLAN_CASES[19], PLAN_CASES[22]],
                         ids=lambda c: c[0])
def test_wgrad_deterministic(ops, c):
    """Fixed-order reductions: two calls give bit-identical gradients."""
    x, dy = inputs(c, 5, same_sign=True)
    a = [t.cpu().numpy() for t in run(ops, c, x, dy)]
    b = [t.cpu().numpy() for t in run(ops, c, x, dy)]
    assert all(np.array_equal(u.view(np.uint32), v.view(np.uint32)) for u, v in zip(a, b))


def _ws_bytes(ops, c):
    import ctypes as C
    from flownet2_b200 import check as fcheck, lib
    _, N, Ci, H, W, Co, k, s, p, deconv, engine = c
    d = ops._conv_desc(torch.zeros(weight_shape(c)), s, p, deconv, True, engine)
    nb = C.c_size_t()
    fcheck(lib().fn2_conv_backward_params_workspace_bytes(C.byref(d), N, H, W, C.byref(nb)))
    return nb.value


@pytest.mark.parametrize("c", [PLAN_CASES[0], PLAN_CASES[14], PLAN_CASES[16], PLAN_CASES[19], PLAN_CASES[22]],
                         ids=lambda c: c[0])
def test_wgrad_workspace_contract(ops, fn2, c):
    """Exactly the reported bytes, 4 bytes past a 256-byte boundary, suffice and nothing after them is written; one float fewer
    is FN2_ERR_WORKSPACE."""
    nb = _ws_bytes(ops, c)
    guard = 1 << 16
    buf = torch.empty(nb + 512 + guard, dtype=torch.uint8, device="cuda")
    off = (-buf.data_ptr()) % 256 + 4
    buf.fill_(0xA5)
    ws = buf[off:off + nb]
    x, dy = inputs(c, 7)
    ww, wb = ref_grads(x, dy, c[6], c[7], c[8], c[9])
    gw, gb = run(ops, c, x, dy, workspace=ws)
    assert rel(gw.cpu().numpy(), ww) <= TOL and rel(gb.cpu().numpy(), wb) <= TOL
    assert bool((buf[off + nb:] == 0xA5).all()), "write past the end of the workspace"
    with pytest.raises(fn2.Fn2Error, match="fn2 error -5"):
        run(ops, c, x, dy, workspace=buf[off:off + nb - 4])


def test_wgrad_argument_errors(ops, fn2):
    """An anisotropic stride and a bottom whose channels do not match the descriptor are FN2_ERR_INVALID."""
    x = dev(np.ones((1, 8, 12, 14), np.float32))
    with pytest.raises(fn2.Fn2Error, match="fn2 error -1.*anisotropic"):
        ops.conv2d_backward(x, torch.zeros((16, 8, 3, 3), device="cuda"), dev(np.ones((1, 16, 12, 7), np.float32)), (1, 2), 1,
                            need_input_grad=False)
    with pytest.raises(fn2.Fn2Error, match="fn2 error -1.*channel"):
        ops.conv2d_backward(x, torch.zeros((16, 9, 3, 3), device="cuda"), dev(np.ones((1, 16, 12, 14), np.float32)), 1, 1,
                            need_input_grad=False)


# ---- training shapes ------------------------------------------------------------------------------------------------------------
def _train_cases():
    from flownet2_b200 import ops as _ops
    cases, seen, keys = [], set(), set()

    def key(c):
        pl = _ops.wgrad_plan(c[2], c[5], c[6], c[7], c[8], c[9], c[1], c[3], c[4])
        return (pl[0], pl[1], pl[2], pl[4] > 1, pl[5] > 1, c[7], c[9])

    for model in ("FlowNet2-C", "FlowNet2-SD", "FlowNet2"):
        for name, ci, h, w, co, k, s, p, deconv, trainable in train_convs(model):
            c = case("%s-%s" % (model[9:] or "fusion", name), 1, ci, h, w, co, k, s, p, deconv)
            shape = c[2:]
            if not trainable or shape in seen:
                continue
            if model != "FlowNet2-C" and key(c) in keys:
                continue                  # the SD and fusion stages add the layers whose plan the C graph does not reach
            seen.add(shape)
            keys.add(key(c))
            cases.append(c)
            if model == "FlowNet2-C" and name == "conv1":
                cases.append(case("C-conv1-b8", 8, ci, h, w, co, k, s, p, deconv))
    return cases


TRAIN_CASES = _train_cases()


def reduction_len(c):
    Cs, Hs, Ws, Cb, Hb, Wb = small_big(c)
    return c[1] * Hs * Ws


# Bound on |shrink| of dW per training case.  The tensor-core chains truncate, and with same-sign products every chunk loses
# magnitude; the kernel adds back TRUNC_LOSS_PER_MMA per chained MMA (calibrated on forward cases with products of either sign).
# Measured on an H100 80GB HBM3 (700 W power limit) over 4 seeds, with that library and with one built with the constant set to
# 0: the compensation takes back about 60 % (NT <= 64, 4-step chunks: -3.4e-7 -> -1.3e-7 at K >= 35,840) to 75 % (NT = 128,
# 1-step chunks: -8e-8 -> -2e-8) of the loss, and the residual does not grow with K (conv1: -1.3e-7 at batch 1 and 8).  Each
# bound lies between max |shrink| + 3 x spread of the compensating library and half the smallest |shrink| without it, so it
# fails when the compensation is lost.  The cases not listed keep only the 1e-5 bound: the two libraries' shrinks are not that
# far apart there (K of 35-140 pixels, mostly zero-filled K segments, over-compensated by up to +2.6e-8; or a 2-channel small
# map with too few entries for a stable mean; or SD conv0, whose spread over seeds is 1.8e-8).
SHRINK_BOUND = {
    "C-conv1": 1.6e-07, "C-conv1-b8": 1.6e-07, "C-conv2": 3.1e-08, "C-conv3": 2.9e-08, "C-conv_redir": 1.2e-07,
    "C-conv3_1": 2.9e-08, "C-conv4": 3.3e-08, "C-conv4_1": 3.4e-08, "C-conv5": 2.1e-08, "C-conv5_1": 2e-08, "C-deconv4": 2e-08,
    "C-deconv3": 3.4e-08, "C-predict_flow3": 1.3e-07, "C-deconv2": 2.9e-08, "C-predict_flow2": 1.2e-07, "SD-conv1": 1.4e-07,
    "SD-conv1_1": 3.5e-08, "SD-conv2": 3e-08, "SD-conv2_1": 3.1e-08, "SD-interconv3": 2.8e-08, "SD-predict_flow3": 1.2e-07,
    "SD-interconv2": 1.1e-07, "SD-predict_flow2": 1.3e-07, "fusion-fuse_conv0": 1.5e-07, "fusion-fuse_deconv1": 3.1e-08,
    "fusion-fuse_deconv0": 3.8e-08,
}


def test_shrink_bounds_name_training_cases():
    assert set(SHRINK_BOUND) <= {c[0] for c in TRAIN_CASES}


@pytest.mark.parametrize("c", TRAIN_CASES, ids=[c[0] for c in TRAIN_CASES])
def test_wgrad_training_shapes(ops, c):
    """Post-ReLU bottom, top diff of mean 1: dW and db within 1e-5, and dW without the systematic shrink of uncompensated
    truncating chains (SHRINK_BOUND)."""
    ew, eb, sh = check(ops, c, same_sign=True)
    print("%s K=%d maxerr dW %.3g db %.3g shrink %.3g" % (c[0], reduction_len(c), ew, eb, sh))
    if c[0] in SHRINK_BOUND:
        assert abs(sh) <= SHRINK_BOUND[c[0]], (c[0], sh)
