"""Per-op wrappers of the fn2_* C-ABI over torch CUDA tensors.

torch is used for device memory and streams only: every function builds fn2_tensor descriptors
from ``data_ptr()`` / ``stride()`` (so NCHW-contiguous, channels_last and channel-sliced tensors all
work) and calls straight into libfn2.so.  No PyTorch arithmetic happens here and there is no
fallback path.
"""
import ctypes as C

import torch

from . import check, fn2_conv_desc, fn2_tensor, lib


def desc(t):
    assert t.is_cuda and t.dtype == torch.float32 and t.dim() == 4, "need a 4-D float32 CUDA tensor"
    n, c, h, w = t.shape
    sn, sc, sh, sw = t.stride()
    return fn2_tensor(C.c_void_p(t.data_ptr()), n, c, h, w, sn, sc, sh, sw)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _empty(shape, like, channels_last=None):
    if channels_last is None:
        channels_last = like.stride(1) == 1 and like.shape[1] > 1
    t = torch.empty(shape, device=like.device, dtype=torch.float32)
    return t.contiguous(memory_format=torch.channels_last) if channels_last else t


def correlation_shape(H, W, pad, kernel_size, max_displacement, stride1, stride2):
    tc, th, tw = C.c_int(), C.c_int(), C.c_int()
    check(lib().fn2_correlation_shape(H, W, pad, kernel_size, max_displacement, stride1, stride2,
                                      C.byref(tc), C.byref(th), C.byref(tw)))
    return tc.value, th.value, tw.value


def correlation(b0, b1, pad, kernel_size, max_displacement, stride1, stride2, corr_type=0, out=None,
                use_workspace=True):
    N, Cc, H, W = b0.shape
    tc, th, tw = correlation_shape(H, W, pad, kernel_size, max_displacement, stride1, stride2)
    if out is None:
        out = _empty((N, tc, th, tw), b0)
    ws, nbytes = None, C.c_size_t(0)
    if use_workspace:
        check(lib().fn2_correlation_workspace_bytes(N, Cc, H, W, pad, kernel_size, max_displacement, stride1,
                                                    stride2, corr_type, C.byref(nbytes)))
        if nbytes.value:
            ws = torch.zeros(nbytes.value, dtype=torch.uint8, device=b0.device)
    d0, d1, dt = desc(b0), desc(b1), desc(out)
    check(lib().fn2_correlation_forward(C.byref(d0), C.byref(d1), C.byref(dt), pad, kernel_size, max_displacement,
                                        stride1, stride2, corr_type,
                                        C.c_void_p(ws.data_ptr()) if ws is not None else None,
                                        nbytes.value if ws is not None else 0, _stream()))
    return out


def _ws(nbytes, dev):
    return torch.zeros(max(int(nbytes), 4), dtype=torch.uint8, device=dev)


def correlation_backward(b0, b1, top_diff, pad, kernel_size, max_displacement, stride1, stride2, corr_type=0):
    g0, g1 = torch.empty_like(b0), torch.empty_like(b1)
    N, Cc, H, W = b0.shape
    nb = C.c_size_t(0)
    check(lib().fn2_correlation_backward_workspace_bytes(N, Cc, H, W, pad, kernel_size, max_displacement, stride1, stride2, corr_type,
                                                         C.byref(nb)))
    ws = _ws(nb.value, b0.device)
    d0, d1, dt, dg0, dg1 = desc(b0), desc(b1), desc(top_diff), desc(g0), desc(g1)
    check(lib().fn2_correlation_backward(C.byref(d0), C.byref(d1), C.byref(dt), C.byref(dg0), C.byref(dg1), pad,
                                         kernel_size, max_displacement, stride1, stride2, corr_type,
                                         C.c_void_p(ws.data_ptr()), C.c_size_t(nb.value), _stream()))
    return g0, g1


def correlation1d_shape(H, W, pad, kernel_size, max_displacement, stride1, stride2, single_direction=0):
    tc, th, tw = C.c_int(), C.c_int(), C.c_int()
    check(lib().fn2_correlation1d_shape(H, W, pad, kernel_size, max_displacement, stride1, stride2, single_direction,
                                        C.byref(tc), C.byref(th), C.byref(tw)))
    return tc.value, th.value, tw.value


def correlation1d(b0, b1, pad, kernel_size, max_displacement, stride1, stride2, single_direction=0, corr_type=0):
    N, Cc, H, W = b0.shape
    tc, th, tw = correlation1d_shape(H, W, pad, kernel_size, max_displacement, stride1, stride2, single_direction)
    out = _empty((N, tc, th, tw), b0)
    d0, d1, dt = desc(b0), desc(b1), desc(out)
    check(lib().fn2_correlation1d_forward(C.byref(d0), C.byref(d1), C.byref(dt), pad, kernel_size, max_displacement, stride1,
                                          stride2, single_direction, corr_type, _stream()))
    return out


def correlation1d_backward(b0, b1, top_diff, pad, kernel_size, max_displacement, stride1, stride2, single_direction=0, corr_type=0):
    g0, g1 = torch.empty_like(b0), torch.empty_like(b1)
    N, Cc, H, W = b0.shape
    nb = C.c_size_t(0)
    check(lib().fn2_correlation1d_backward_workspace_bytes(N, Cc, H, W, pad, kernel_size, max_displacement, stride1, stride2,
                                                           single_direction, corr_type, C.byref(nb)))
    ws = _ws(nb.value, b0.device)
    d0, d1, dt, dg0, dg1 = desc(b0), desc(b1), desc(top_diff), desc(g0), desc(g1)
    check(lib().fn2_correlation1d_backward(C.byref(d0), C.byref(d1), C.byref(dt), C.byref(dg0), C.byref(dg1), pad, kernel_size,
                                           max_displacement, stride1, stride2, single_direction, corr_type,
                                           C.c_void_p(ws.data_ptr()), C.c_size_t(nb.value), _stream()))
    return g0, g1


def flow_warp(image, flow, fill_nan=False, out=None):
    if out is None:
        out = torch.empty_like(image)
    di, df, do = desc(image), desc(flow), desc(out)
    check(lib().fn2_flow_warp_forward(C.byref(di), C.byref(df), C.byref(do), 1 if fill_nan else 0, _stream()))
    return out


def flow_warp_backward(image, flow, warped_diff):
    gi, gf = torch.empty_like(image), torch.empty_like(flow)
    di, df, dw, dgi, dgf = desc(image), desc(flow), desc(warped_diff), desc(gi), desc(gf)
    check(lib().fn2_flow_warp_backward(C.byref(di), C.byref(df), C.byref(dw), C.byref(dgi), C.byref(dgf), _stream()))
    return gi, gf


def resample(x, out_h, out_w, rtype=2, antialias=True):
    out = _empty((x.shape[0], x.shape[1], out_h, out_w), x)
    dx, do = desc(x), desc(out)
    check(lib().fn2_resample_forward(C.byref(dx), C.byref(do), rtype, 1 if antialias else 0, _stream()))
    return out


def spatial_augmentation(x, mats, out_h, out_w):
    out = _empty((x.shape[0], x.shape[1], out_h, out_w), x)
    mats = mats.contiguous()
    dx, do = desc(x), desc(out)
    check(lib().fn2_spatial_augmentation(C.byref(dx), C.byref(do), C.c_void_p(mats.data_ptr()), _stream()))
    return out


def color_contrast_augmentation(x, chroma, max_multiplier=1.0):
    out = x.clone(memory_format=torch.preserve_format)
    chroma = chroma.contiguous()
    do = desc(out)
    check(lib().fn2_color_contrast_augmentation(C.byref(do), C.c_void_p(chroma.data_ptr()), max_multiplier, _stream()))
    return out


def chromatic_eigenspace(x, eigvec9):
    """-> 25 floats (tChromaticEigenSpace) as a device tensor of 32 (the tail is scratch)."""
    ev = torch.as_tensor(eigvec9, dtype=torch.float32, device=x.device).reshape(9).contiguous()
    space = torch.zeros(32, dtype=torch.float32, device=x.device)
    dx = desc(x)
    check(lib().fn2_chromatic_eigenspace(C.byref(dx), C.c_void_p(ev.data_ptr()), C.c_void_p(space.data_ptr()), _stream()))
    return space


def chromatic_eigen_augmentation(x, coeffs, space, max_multiplier=1.0):
    out = x.clone(memory_format=torch.preserve_format)
    coeffs = coeffs.contiguous()
    do = desc(out)
    check(lib().fn2_chromatic_eigen_augmentation(C.byref(do), C.c_void_p(coeffs.data_ptr()), C.c_void_p(space.data_ptr()),
                                                 C.c_float(max_multiplier), _stream()))
    return out


def apply_effects(x, effects, max_multiplier=1.0, noise_seed=0, add_noise=False):
    out = x.clone(memory_format=torch.preserve_format)
    effects = effects.contiguous()
    do = desc(out)
    check(lib().fn2_apply_effects(C.byref(do), C.c_void_p(effects.data_ptr()), C.c_float(max_multiplier),
                                  C.c_ulonglong(noise_seed), 1 if add_noise else 0, _stream()))
    return out


def mean_update(top, mean_pp, mean_pc, num_iter):
    dt, dm = desc(top), desc(mean_pp)
    check(lib().fn2_mean_update(C.byref(dt), C.byref(dm), C.c_void_p(mean_pc.data_ptr()), float(num_iter), _stream()))


def mean_subtract(top, mean_pp=None, mean_pc=None, per_pixel=False):
    dt = desc(top)
    dm = desc(mean_pp) if mean_pp is not None else None
    check(lib().fn2_mean_subtract(C.byref(dt), C.byref(dm) if dm is not None else None,
                                  C.c_void_p(mean_pc.data_ptr()) if mean_pc is not None else None,
                                  1 if per_pixel else 0, _stream()))
    return top


def conv_plan(ci, co, k, stride, pad, deconv, n, h, w, ci_stride):
    """fn2_conv_plan: the tensor-core engines' host-side plan for a layer shape (8 ints, see include/fn2.h): NT, tile units,
    K steps per tile, mode, first split tile, K ranges per split tile."""
    d = fn2_conv_desc(ci, co, k, k, stride, stride, pad, pad, 1 if deconv else 0, 1, 0, 0.0, 0, 0)
    plan = (C.c_int32 * 8)()
    check(lib().fn2_conv_plan(C.byref(d), n, h, w, ci_stride, plan))
    return list(plan)


def conv2d(x, weight, bias=None, stride=1, pad=0, deconv=False, relu_slope=None, engine=0, channels_last_out=None,
           use_workspace=True, input_guard_bytes=0, out=None):
    """weight in Caffe layout: conv [co,ci,kh,kw], deconv [ci,co,kh,kw]."""
    l = lib()
    if deconv:
        ci, co, kh, kw = weight.shape
    else:
        co, ci, kh, kw = weight.shape
    sh, sw = (stride, stride) if isinstance(stride, int) else stride
    ph, pw = (pad, pad) if isinstance(pad, int) else pad
    d = fn2_conv_desc(ci, co, kh, kw, sh, sw, ph, pw, 1 if deconv else 0, 1 if bias is not None else 0,
                      1 if relu_slope is not None else 0, float(relu_slope or 0.0), engine, input_guard_bytes)
    ho, wo = C.c_int(), C.c_int()
    check(l.fn2_conv_out_shape(C.byref(d), x.shape[2], x.shape[3], C.byref(ho), C.byref(wo)))
    cis = x.stride(3) if x.stride(1) == 1 else ci
    nf = C.c_size_t()
    check(l.fn2_conv_packed_floats(C.byref(d), cis, C.byref(nf)))
    packed = torch.empty(max(nf.value, 1), dtype=torch.float32, device=x.device)
    weight = weight.contiguous()
    check(l.fn2_conv_pack_weights(C.byref(d), cis, C.c_void_p(weight.data_ptr()), C.c_void_p(packed.data_ptr()), _stream()))
    if out is None:
        out = _empty((x.shape[0], co, ho.value, wo.value), x, channels_last_out)
    dx, do = desc(x), desc(out)
    wsb = C.c_size_t()
    check(l.fn2_conv_workspace_bytes(C.byref(d), x.shape[0], x.shape[2], x.shape[3], C.byref(wsb)))
    ws = torch.empty(max(wsb.value, 4), dtype=torch.uint8, device=x.device) if use_workspace else None
    check(l.fn2_conv_forward(C.byref(d), C.byref(dx), C.c_void_p(packed.data_ptr()),
                             C.c_void_p(bias.data_ptr()) if bias is not None else None, C.byref(do),
                             C.c_void_p(ws.data_ptr()) if ws is not None else None, wsb.value if ws is not None else 0, _stream()))
    return out


def _conv_desc(weight, stride, pad, deconv, bias, engine=0):
    if deconv:
        ci, co, kh, kw = weight.shape
    else:
        co, ci, kh, kw = weight.shape
    sh, sw = (stride, stride) if isinstance(stride, int) else stride
    ph, pw = (pad, pad) if isinstance(pad, int) else pad
    return fn2_conv_desc(ci, co, kh, kw, sh, sw, ph, pw, 1 if deconv else 0, 1 if bias else 0, 0, 0.0, engine, 0)


def wgrad_plan(ci, co, k, stride, pad, deconv, n, h, w, engine=0, bias=True):
    """fn2_conv_wgrad_plan: the weight-gradient route a layer shape takes (8 ints, see include/fn2.h): route (1 SIMT, 2 tensor
    cores), NT, G, TG, BT, ST, S (SIMT: pixel splits), bias blocks.  k, stride, pad: an int or (h, w)."""
    kh, kw = (k, k) if isinstance(k, int) else k
    sh, sw = (stride, stride) if isinstance(stride, int) else stride
    ph, pw = (pad, pad) if isinstance(pad, int) else pad
    d = fn2_conv_desc(ci, co, kh, kw, sh, sw, ph, pw, 1 if deconv else 0, 1 if bias else 0, 0, 0.0, engine, 0)
    plan = (C.c_int32 * 8)()
    check(lib().fn2_conv_wgrad_plan(C.byref(d), n, h, w, plan))
    return list(plan)


def conv2d_backward(x, weight, top_diff, stride=1, pad=0, deconv=False, bias=True, need_input_grad=True, engine=0,
                    accumulate=False, out=None, workspace=None):
    """ConvolutionLayer / DeconvolutionLayer::Backward_gpu (conv_layer.cu:26-58, deconv_layer.cu:26-55) through the C-ABI:
    -> (bottom_diff or None, weight_diff, bias_diff or None).
    out=(weight_diff, bias_diff): write (accumulate: add) the parameter gradients there; a None bias_diff passes a null bias
    pointer.  workspace: a uint8 CUDA tensor whose bytes are the workspace (default: one of the reported size)."""
    l = lib()
    d = _conv_desc(weight, stride, pad, deconv, bias, engine)
    weight = weight.contiguous()
    if out is None:
        wd = torch.zeros_like(weight)
        bd = torch.zeros(d.co, dtype=torch.float32, device=x.device) if bias else None
    else:
        wd, bd = out
        assert wd.is_contiguous() and wd.shape == weight.shape and (bd is None or bd.is_contiguous())
    if workspace is None:
        nb = C.c_size_t()
        check(l.fn2_conv_backward_params_workspace_bytes(C.byref(d), x.shape[0], x.shape[2], x.shape[3], C.byref(nb)))
        workspace = _ws(max(nb.value, 4), x.device)
    assert workspace.dtype == torch.uint8 and workspace.is_contiguous()
    tx, tdy = desc(x), desc(top_diff)
    check(l.fn2_conv_backward_params(C.byref(d), C.byref(tx), C.byref(tdy), C.c_void_p(wd.data_ptr()),
                                     C.c_void_p(bd.data_ptr()) if bd is not None else None, 1 if accumulate else 0,
                                     C.c_void_p(workspace.data_ptr()), workspace.numel(), _stream()))
    dx = None
    if need_input_grad:
        bdsc, flip = fn2_conv_desc(), C.c_int()
        check(l.fn2_conv_backward_data_desc(C.byref(d), x.shape[2], x.shape[3], C.byref(bdsc), C.byref(flip)))
        w2 = weight
        if flip.value:
            w2 = torch.empty_like(weight)
            check(l.fn2_conv_flip_transpose_weights(C.byref(d), C.c_void_p(weight.data_ptr()), C.c_void_p(w2.data_ptr()), _stream()))
        cis = top_diff.stride(3) if top_diff.stride(1) == 1 else bdsc.ci
        nf = C.c_size_t()
        check(l.fn2_conv_packed_floats(C.byref(bdsc), cis, C.byref(nf)))
        packed = torch.empty(max(nf.value, 1), dtype=torch.float32, device=x.device)
        check(l.fn2_conv_pack_weights(C.byref(bdsc), cis, C.c_void_p(w2.data_ptr()), C.c_void_p(packed.data_ptr()), _stream()))
        ho, wo = C.c_int(), C.c_int()
        check(l.fn2_conv_out_shape(C.byref(bdsc), top_diff.shape[2], top_diff.shape[3], C.byref(ho), C.byref(wo)))
        assert ho.value == x.shape[2] and wo.value == x.shape[3]
        dx = torch.empty_like(x)
        tv = desc(dx)
        wsb = C.c_size_t()
        check(l.fn2_conv_workspace_bytes(C.byref(bdsc), top_diff.shape[0], top_diff.shape[2], top_diff.shape[3], C.byref(wsb)))
        ws2 = torch.empty(max(wsb.value, 4), dtype=torch.uint8, device=x.device)
        check(l.fn2_conv_forward(C.byref(bdsc), C.byref(tdy), C.c_void_p(packed.data_ptr()), None, C.byref(tv),
                                 C.c_void_p(ws2.data_ptr()), wsb.value, _stream()))
    return dx, wd, bd


def relu_backward(top_data, top_diff, negative_slope=0.0, out=None, accumulate=False):
    """-> out (a new tensor if None) = top_diff * (top_data > 0 ? 1 : negative_slope), added to out's values if accumulate."""
    if out is None:
        out = torch.empty_like(top_diff)
    a, b, c = desc(top_data), desc(top_diff), desc(out)
    check(lib().fn2_relu_backward(C.byref(a), C.byref(b), C.byref(c), negative_slope, 1 if accumulate else 0, _stream()))
    return out


def axpby(x, alpha, y, beta):
    a, b = desc(x), desc(y)
    check(lib().fn2_axpby(C.byref(a), alpha, C.byref(b), beta, _stream()))
    return y


def relu(x, negative_slope=0.0, out=None):
    if out is None:
        out = torch.empty_like(x)
    dx, do = desc(x), desc(out)
    check(lib().fn2_relu_forward(C.byref(dx), C.byref(do), negative_slope, _stream()))
    return out


def eltwise_sum(bottoms, coeffs=None, out=None):
    if out is None:
        out = torch.empty_like(bottoms[0])
    ds = [desc(b) for b in bottoms]
    arr = (C.POINTER(fn2_tensor) * len(ds))(*[C.pointer(d) for d in ds])
    cf = (C.c_float * len(ds))(*(coeffs if coeffs else [1.0] * len(ds)))
    do = desc(out)
    check(lib().fn2_eltwise_sum(arr, cf, len(ds), C.byref(do), _stream()))
    return out


def channel_norm(x, out=None):
    if out is None:
        out = torch.empty((x.shape[0], 1, x.shape[2], x.shape[3]), device=x.device, dtype=torch.float32)
    dx, do = desc(x), desc(out)
    check(lib().fn2_channel_norm_forward(C.byref(dx), C.byref(do), _stream()))
    return out


def warp_block(flow, image0, image1, scale_coeff, fill_nan=False, out=None):
    """The warp block between stacked networks in one pass: flow (N, 2, h, w) up-sampled to the images' size (LINEAR),
    image1 warped by it, the error image0 - warped, its channel norm and the up-sampled flow times scale_coeff.
    -> out = (flow_full, warped, err, err_norm, flow_scaled), new tensors if None."""
    if out is None:
        N, Cc, H, W = image0.shape
        out = (_empty((N, 2, H, W), image0), torch.empty_like(image1), torch.empty_like(image0),
               _empty((N, 1, H, W), image0, False), _empty((N, 2, H, W), image0))
    ds = [desc(t) for t in (flow, image0, image1) + tuple(out)]
    check(lib().fn2_warp_block_forward(*[C.byref(d) for d in ds], scale_coeff, 1 if fill_nan else 0, _stream()))
    return out


def downsample(x, top_h, top_w, out=None):
    if out is None:
        out = _empty((x.shape[0], x.shape[1], top_h, top_w), x)
    dx, do = desc(x), desc(out)
    check(lib().fn2_downsample_forward(C.byref(dx), C.byref(do), _stream()))
    return out


def copy(src, dst):
    ds, dd = desc(src), desc(dst)
    check(lib().fn2_copy(C.byref(ds), C.byref(dd), _stream()))
    return dst


def fill(dst, value):
    dd = desc(dst)
    check(lib().fn2_fill(C.byref(dd), value, _stream()))
    return dst
