"""Float64 reference of the convolution layer, the operators its data gradient runs, the bottom layouts the engines are tested
under and the route table of the SIMT engine: shared by the tests of both convolution engines.

`ref_at` evaluates a convolution or deconvolution at chosen output pixels, per kernel tap one float64 product of the tap's
weights with the input pixels it reads there, in torch on any device; tests/test_conv_ref_cpu.py pins it to
oracle.conv_fwd / deconv_fwd.  `adjoint` builds the forward operator that computes a layer's data gradient exactly as
BaseConvolutionLayer::BackwardData does (fn2_conv_backward_data_desc, padded output channels), and `reference` evaluates a
case -- a layer or such an operator -- with bias and leaky ReLU.
"""
import ctypes as C
from collections import namedtuple

import torch

GUARD = 256                 # floats of NaN before and after every bottom's storage (Blob::kGuardFloats)


def _lib():
    from flownet2_b200 import lib
    return lib()


def _check(rc):
    from flownet2_b200 import check
    check(rc)


# ---- cases ----------------------------------------------------------------------------------------------------------------
# fwd: None, or the layer whose data gradient the case is: (Ci, Co, k, s, p, deconv, H, W, needs_flip, real output channels)
Case = namedtuple("Case", "name N Ci H W Co k s p deconv op bias layout engine fwd")


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def case(name, N, Ci, H, W, Co, k, s=1, p=0, deconv=False, bias=True, layout="nhwc", engine=2):
    return Case(name, N, Ci, H, W, Co, _pair(k), _pair(s), _pair(p), deconv, (0, 0), bias, layout, engine, None)


def cstride(c):
    """Blob::compute_cstride: the nets' pixel stride (channels rounded up to 4 below 32, else to 32)."""
    return (c + 3) // 4 * 4 if c < 32 else (c + 31) // 32 * 32


def padded_co(co):
    """The output channels BaseConvolutionLayer::BackwardData gives a convolution adjoint (layers.cpp, BackwardData: a
    multiple of 128 when that costs at most 1/8 more channels, else of 64; of 16 up to 64 channels)."""
    if co <= 16 or co % 16 == 0:
        return co
    c128, c64 = (co + 127) // 128 * 128, (co + 63) // 64 * 64
    return (co + 15) // 16 * 16 if co <= 64 else (c128 if (c128 - co) * 8 <= co else c64)


def adjoint(name, N, Ci, H, W, Co, k, s=1, p=0, deconv=False, layout="pad", engine=2):
    """The forward operator that computes the data gradient of a layer (fn2_conv_backward_data_desc) on its top diff, with
    BackwardData's padded output channels."""
    from flownet2_b200 import fn2_conv_desc
    (kh, kw), (sh, sw), (ph, pw) = _pair(k), _pair(s), _pair(p)
    d = fn2_conv_desc(Ci, Co, kh, kw, sh, sw, ph, pw, int(deconv), 1, 0, 0.0, 0, 0)
    bd, flip, ho, wo = fn2_conv_desc(), C.c_int(), C.c_int(), C.c_int()
    _check(_lib().fn2_conv_backward_data_desc(C.byref(d), H, W, C.byref(bd), C.byref(flip)))
    _check(_lib().fn2_conv_out_shape(C.byref(d), H, W, C.byref(ho), C.byref(wo)))
    co = padded_co(bd.co) if not bd.deconv else bd.co
    return Case(name, N, bd.ci, ho.value, wo.value, co, (bd.kh, bd.kw), (bd.stride_h, bd.stride_w), (bd.pad_h, bd.pad_w),
                bool(bd.deconv), (bd.out_pad_h, bd.out_pad_w), False, layout, engine,
                (Ci, Co, (kh, kw), (sh, sw), (ph, pw), deconv, H, W, bool(flip.value), bd.co))


def weight_shape(c):
    """Caffe layout of the weights the reference uses: those of the case, or of the layer it is the data gradient of."""
    if c.fwd:
        Ci, Co, (kh, kw), _, _, deconv, _, _, _, _ = c.fwd
        return (Ci, Co, kh, kw) if deconv else (Co, Ci, kh, kw)
    return (c.Ci, c.Co) + c.k if c.deconv else (c.Co, c.Ci) + c.k


def op_weights(c, w):
    """The Caffe-layout weights of the operator: the case's own, or for a data gradient the layer's, flipped and transposed
    when fn2_conv_backward_data_desc asks for it, with BackwardData's zero rows for padded output channels."""
    if not c.fwd:
        return w
    Ci, Co, k, s, p, deconv, H, W, flip, co_real = c.fwd
    if flip:
        from flownet2_b200 import fn2_conv_desc
        d = fn2_conv_desc(Ci, Co, k[0], k[1], s[0], s[1], p[0], p[1], int(deconv), 1, 0, 0.0, 0, 0)
        w2 = torch.empty((Ci, Co) + tuple(k), device="cuda")
        _check(_lib().fn2_conv_flip_transpose_weights(C.byref(d), w.data_ptr(), w2.data_ptr(), torch.cuda.current_stream().cuda_stream))
        w = w2
    if c.Co > co_real:
        w = torch.cat([w, torch.zeros((c.Co - co_real,) + tuple(w.shape[1:]), device="cuda")])
    return w.contiguous()


# ---- bottom layouts ---------------------------------------------------------------------------------------------------------
# layout -> (first channel, pixel stride, padding channels, guard promise)
LAYOUTS = {
    "nhwc": (0, lambda c: (c + 3) // 4 * 4, "nan", False),      # channels_last, 16-byte pixels
    "pad": (0, cstride, "zero", True),                          # the nets' blobs
    "padjunk": (0, cstride, "junk", True),                      # ... with finite garbage in the padding channels
    "padnan": (0, cstride, "nan", False),                       # ... with NaN there, and no guard promise
    "slice": (4, lambda c: (c + 3) // 4 * 4 + 8, "nan", False),  # a zero-copy concat child
    "misaligned": (1, lambda c: c + 4, "nan", False),           # first channel not on a 16-byte boundary
}


def concat_child(c0, channels):
    """The layout of a zero-copy concat child (Net::AliasConcats): channels [c0, c0 + C) of a concat of `channels` channels,
    at the concat's pixel stride, inside the concat's allocation with its guard band.  The other channels hold finite garbage
    (1e30): the guard promise lets a kernel read those of the child's last float4 group against zero weights (fn2.h,
    input_guard_bytes), and any other read shows in the sum."""
    return (c0, lambda c: cstride(channels), "junk", True)


def layout_of(layout):
    return LAYOUTS[layout] if isinstance(layout, str) else layout


def bottom(x, layout):
    """A view of x in one of LAYOUTS (or a concat_child).  The storage has GUARD floats of NaN before and after it; the
    channels outside the view hold NaN, zero or finite garbage (1e30)."""
    n, c, h, w = x.shape
    off, cs, fill, _ = layout_of(layout)
    cs = cs(c)
    flat = torch.full((2 * GUARD + n * h * w * cs,), float("nan"), device="cuda")
    body = flat[GUARD:GUARD + n * h * w * cs].view(n, h, w, cs)
    if fill != "nan":
        body.fill_(0.0 if fill == "zero" else 1e30)
    body[..., off:off + c] = x.permute(0, 2, 3, 1)
    return body.permute(0, 3, 1, 2)[:, off:off + c]


def guard_bytes(layout):
    return 4 * GUARD if layout_of(layout)[3] else 0


# ---- reference ----------------------------------------------------------------------------------------------------------------
def ref_at(x, w, deconv, s, p, n, oy, ox):
    """float64 (P, Co) outputs at the pixels (n, oy, ox) without bias: per kernel tap one BLAS product of the tap's weights with
    the input pixels it reads there.  x (N, Ci, H, W); w in Caffe layout; a deconvolution's tap (ky, kx) reads input pixel
    ((oy + ph - ky) / sh, (ox + pw - kx) / sw) where both divide exactly."""
    (sh, sw), (ph, pw) = s, p
    x, w = x.double(), w.double()
    N, Ci, H, W = x.shape
    kh, kw = w.shape[2:]
    out = torch.zeros((len(n), w.shape[1] if deconv else w.shape[0]), dtype=torch.float64, device=x.device)

    def coord(o, st, pd, kk, size):
        if deconv:
            t = o + pd - kk
            i = torch.div(t, st, rounding_mode="floor")
            ok = (i * st == t)
        else:
            i = o * st + kk - pd
            ok = torch.ones_like(i, dtype=torch.bool)
        return i, ok & (i >= 0) & (i < size)

    for ky in range(kh):
        iy, oky = coord(oy, sh, ph, ky, H)
        for kx in range(kw):
            ix, okx = coord(ox, sw, pw, kx, W)
            sel = (oky & okx).nonzero().squeeze(1)
            if len(sel):
                wt = w[:, :, ky, kx] if deconv else w[:, :, ky, kx].T             # (Ci, Co)
                out.index_add_(0, sel, x[n[sel], :, iy[sel], ix[sel]] @ wt)
    return out


def operator_geometry(c):
    """(stride, pad, deconv) of the operator the reference evaluates for case c: a data-gradient operator is computed as the
    transpose of its layer."""
    if c.fwd:
        _, _, _, s, p, deconv, _, _, _, _ = c.fwd
        return s, p, not deconv
    return c.s, c.p, c.deconv


def reference(c, x, w, b, n, oy, ox, slope=0.1):
    """The case's outputs at (n, oy, ox) in float64, in chunks that keep the gathered inputs small; a data-gradient operator
    is computed as the transpose of its layer, from the layer's weights.  b: None, or the bias, added with a leaky ReLU of
    `slope` after it (None: no ReLU)."""
    s, p, deconv = operator_geometry(c)
    step = max(256, (1 << 25) // c.Ci)
    out = torch.cat([ref_at(x, w, deconv, s, p, n[i:i + step], oy[i:i + step], ox[i:i + step]) for i in range(0, len(n), step)])
    if b is not None:
        out = out + b.double()
        if slope is not None:
            out = torch.where(out > 0, out, out * slope)
    return out


def taps_at(c, n, oy, ox):
    """How many kernel taps reach each output pixel (n, oy, ox) of case c inside the input (as a float64 tensor)."""
    s, p, deconv = operator_geometry(c)
    kh, kw = (c.fwd[2] if c.fwd else c.k)
    return reference(c._replace(Ci=1), torch.ones((c.N, 1, c.H, c.W), dtype=torch.float64, device=n.device),
                     torch.ones((1, 1, kh, kw), dtype=torch.float64, device=n.device), None, n, oy, ox)[:, 0]


# ---- the SIMT engine's routes (fn2_conv.cu, simt_route) ----------------------------------------------------------------------
# the kernel each route launches, as the profiler names it
ROUTE_KERNEL = {
    "pf3_tile": "conv_pf3_tile_kernel<", "pf_thread": "conv_pf_thread_kernel<", "pf3_warp": "conv_pf3_warp_kernel(",
    "pf_warp": "conv_pf_warp_kernel(", "tiny_deconv": "conv_tiny_kernel<true>", "tiny_conv": "conv_tiny_kernel<false>",
    "smallco_deconv": "conv_smallco_kernel<true", "smallco_conv": "conv_smallco_kernel<false", "fewci": "conv_fewci_kernel(",
    "nhwc": "conv_nhwc_kernel<", "igemm_deconv": "conv_igemm_kernel<true>", "igemm_conv": "conv_igemm_kernel<false>",
}


def simt_route(c, in_off, in_stride):
    """The route simt_route (fn2_conv.cu) gives case c on a channels_last bottom view at channel in_off of a 16-byte aligned
    allocation with pixel stride in_stride, into a channels_last top."""
    taps, c4 = c.k[0] * c.k[1], (c.Ci + 3) // 4
    if not c.deconv and c.Ci <= 4 and c.Co >= 32 and taps * c.Ci <= 200:
        return "fewci"
    if c.Co % 4 == 0 and c.Co >= 8 and taps <= 49 and (not c.deconv or c.s[0] * c.s[1] <= 16):
        return "nhwc"
    float4_groups = in_off % 4 == 0 and in_stride % 4 == 0 and in_stride >= 4 * c4        # T4::px_float4_groups
    if not c.deconv and c.Co == 2 and float4_groups and taps * c4 * 4 * 8 <= 200 * 1024:
        k3 = c.k == (3, 3) and c.s == (1, 1)
        if c4 <= 8:
            return "pf3_tile" if k3 else "pf_thread"
        return "pf3_warp" if k3 else "pf_warp"
    kind = "deconv" if c.deconv else "conv"
    if c.Co <= 4:
        return ("tiny_" if c.Ci <= 32 else "smallco_") + kind
    return "igemm_" + kind


def simt_work(c, route, Ho, Wo, sms):
    """(work units, CTAs) of a persistent or grid-stride SIMT launch on a card with `sms` SMs (simt_route, fn2_conv.cu; ew_grid,
    fn2_common.cuh): pf3_tile loops over 32 x 8 output tiles on min(4 SMs, tiles) CTAs; pf3_warp over groups of 4 outputs of a
    row, 8 warps per CTA, on min(per_sm SMs, groups / 8) CTAs, per_sm = max(1, min(8, 220 KB / (weights + 1 KB))); pf_thread
    and tiny over pixels, 256 per CTA, on min(8 SMs, pixels / 256) CTAs."""
    M = c.N * Ho * Wo
    if route == "pf3_tile":
        tiles = c.N * -(-Wo // 32) * -(-Ho // 8)
        return tiles, min(4 * sms, tiles)
    if route == "pf3_warp":
        warps = c.N * Ho * -(-Wo // 4)
        groups = -(-warps // 8)
        per_sm = max(1, min(8, 220 * 1024 // (c.k[0] * c.k[1] * -(-c.Ci // 4) * 32 + 1024)))
        return groups, min(sms * per_sm, groups)
    blocks = -(-M // 256)
    return blocks, min(8 * sms, blocks)


# ---- the layers of the nets that the default engine runs on SIMT -------------------------------------------------------------
DEPLOY_MODELS = ("FlowNet2", "FlowNet2-C", "FlowNet2-S", "FlowNet2-SD", "FlowNet2-CSS")
TRAIN_MODELS = ("FlowNet2-C", "FlowNet2-CS", "FlowNet2-CSS", "FlowNet2-SD", "FlowNet2")

# bottom: a LAYOUTS key or a concat_child layout; top: None (the layer's own blob), or (first channel, channels) of the concat
# the layer's top is a zero-copy child of
SimtLayer = namedtuple("SimtLayer", "case bottom top")


def conv_desc(c, guard=0, engine=0, relu_slope=None):
    from flownet2_b200 import fn2_conv_desc
    (kh, kw), (sh, sw), (ph, pw) = c.k, c.s, c.p
    d = fn2_conv_desc(c.Ci, c.Co, kh, kw, sh, sw, ph, pw, int(c.deconv), int(c.bias), int(relu_slope is not None),
                      float(relu_slope or 0.0), engine, guard)
    d.out_pad_h, d.out_pad_w = c.op
    return d


def plan(c, ci_stride):
    out = (C.c_int32 * 8)()
    _check(_lib().fn2_conv_plan(C.byref(conv_desc(c, 4 * GUARD)), c.N, c.H, c.W, ci_stride, out))
    return list(out)


def aliased(text):
    """{blob: (first channel, channels) of the concat Net::AliasConcats makes it a zero-copy child of}, from the prototxt walk:
    every bottom of a Concat of two or more bottoms, the first such Concat of each blob, except the nets' input blobs and the
    bottoms of a convolution with at most 16 input channels (which stay dense)."""
    from tests.util import net_walk
    convs, _, concats, io = net_walk(text)
    small = {io[l[0]][0][0] for l in convs if l[1] <= 16 and not l[8]}
    produced = {t for bots, tops in io.values() for t in tops}
    return {b: (c0, ch) for b, (_, c0, ch) in concats.items() if b in produced and b not in small}


def net_simt_layers(text, N, tag, grads):
    """SimtLayer of every convolution of a filled prototxt whose plan is 0 (fn2_conv_plan: the tensor-core engines do not take
    it), and with grads of every data-gradient operator (adjoint) whose plan is 0, of the layers that propagate a gradient to
    their bottom: all but the convolutions on at most 16 channels (the layers on the input images).  A
    layer's bottom is its own blob (the nets' pixel stride, zero padding, guard band) or, when aliased, its concat child; its
    top is its own blob or its concat child.  The data-gradient operator reads the top's diff, laid out like the top."""
    from tests.util import net_walk
    convs, _, _, io = net_walk(text)
    alias = aliased(text)
    out = []

    def layout(blob):
        return concat_child(*alias[blob]) if blob in alias else "pad"

    for name, ci, h, w, co, k, s, p, deconv, _ in convs:
        bots, tops = io[name]
        c = case(tag + name, N, ci, h, w, co, k, s, p, deconv, bias=True, layout="pad", engine=0)
        bl = layout(bots[0])
        if plan(c, layout_of(bl)[1](ci))[0] == 0:
            out.append(SimtLayer(c._replace(layout=bl), bl, alias.get(tops[0])))
        if grads and (ci > 16 or deconv):
            a = adjoint("dgrad-" + tag + name, N, ci, h, w, co, k, s, p, deconv, engine=0)
            tl = layout(tops[0])
            if plan(a, layout_of(tl)[1](a.Ci))[0] == 0:
                out.append(SimtLayer(a._replace(layout=tl), tl, None))
    return out


def simt_layers():
    """net_simt_layers of every deploy template at 1024 x 436, batch 4, and of every training template at 448 x 320, batch 8,
    with their data-gradient operators; one per distinct shape and layout, named after its first layer."""
    from flownet2_b200 import fill_template, fill_train_template, model_template, train_template
    layers, seen = [], set()
    for m in DEPLOY_MODELS:
        layers += net_simt_layers(fill_template(model_template(m), 1024, 436), 4, "deploy-%s-" % m, False)
    for m in TRAIN_MODELS:
        layers += net_simt_layers(fill_train_template(train_template(m), 448, 320, 512, 384, 1), 8, "train-%s-" % m, True)
    out = []
    for L in layers:
        bl = layout_of(L.bottom)
        key = L.case[1:10] + L.case[10:11] + L.case[14:] + (bl[0], bl[1](L.case.Ci), L.top)
        if key not in seen:
            seen.add(key)
            out.append(L)
    return out
