"""Per-op wrappers of the fn2_* C-ABI over torch CUDA tensors.

torch is used for device memory and streams only: every function builds fn2_tensor descriptors
from ``data_ptr()`` / ``stride()`` (so NCHW-contiguous, channels_last and channel-sliced tensors all
work) and calls straight into libfn2.so.  No PyTorch arithmetic happens here and there is no
fallback path.  The prototypes come from include/fn2.h: descriptors are passed as they are (ctypes
takes their address), device pointers as ints or None, scalars as Python numbers.
"""
import ctypes as C

import torch

from . import FLOW_ERROR_FIELDS, FLOW_REGION_FIELDS, LPQLOSS_STATE_FLOATS, MASK_CONFUSION_FIELDS, check, fn2_conv_desc, fn2_l1loss_desc, fn2_lpqloss_desc, fn2_tensor, lib


def desc(t):
    assert t.is_cuda and t.dtype == torch.float32 and t.dim() == 4, "need a 4-D float32 CUDA tensor"
    n, c, h, w = t.shape
    sn, sc, sh, sw = t.stride()
    return fn2_tensor(t.data_ptr(), n, c, h, w, sn, sc, sh, sw)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _empty(shape, like, channels_last=None):
    if channels_last is None:
        channels_last = like.stride(1) == 1 and like.shape[1] > 1
    t = torch.empty(shape, device=like.device, dtype=torch.float32)
    return t.contiguous(memory_format=torch.channels_last) if channels_last else t


def _ws(nbytes, dev):
    return torch.zeros(max(int(nbytes), 4), dtype=torch.uint8, device=dev)


def _size(fn, *args):
    """fn(*args, &n) -> n: the workspace and packed-weight size queries."""
    n = C.c_size_t()
    check(fn(*args, C.byref(n)))
    return n.value


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
    ws, nbytes = None, 0
    if use_workspace:
        nbytes = _size(lib().fn2_correlation_workspace_bytes, N, Cc, H, W, pad, kernel_size, max_displacement, stride1,
                       stride2, corr_type)
        if nbytes:
            ws = torch.zeros(nbytes, dtype=torch.uint8, device=b0.device)
    check(lib().fn2_correlation_forward(desc(b0), desc(b1), desc(out), pad, kernel_size, max_displacement, stride1, stride2,
                                        corr_type, _ptr(ws), nbytes if ws is not None else 0, _stream()))
    return out


def correlation_backward(b0, b1, top_diff, pad, kernel_size, max_displacement, stride1, stride2, corr_type=0):
    g0, g1 = torch.empty_like(b0), torch.empty_like(b1)
    N, Cc, H, W = b0.shape
    nb = _size(lib().fn2_correlation_backward_workspace_bytes, N, Cc, H, W, pad, kernel_size, max_displacement, stride1, stride2,
               corr_type)
    ws = _ws(nb, b0.device)
    check(lib().fn2_correlation_backward(desc(b0), desc(b1), desc(top_diff), desc(g0), desc(g1), pad, kernel_size,
                                         max_displacement, stride1, stride2, corr_type, _ptr(ws), nb, _stream()))
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
    check(lib().fn2_correlation1d_forward(desc(b0), desc(b1), desc(out), pad, kernel_size, max_displacement, stride1, stride2,
                                          single_direction, corr_type, _stream()))
    return out


def correlation1d_backward(b0, b1, top_diff, pad, kernel_size, max_displacement, stride1, stride2, single_direction=0, corr_type=0):
    g0, g1 = torch.empty_like(b0), torch.empty_like(b1)
    N, Cc, H, W = b0.shape
    nb = _size(lib().fn2_correlation1d_backward_workspace_bytes, N, Cc, H, W, pad, kernel_size, max_displacement, stride1, stride2,
               single_direction, corr_type)
    ws = _ws(nb, b0.device)
    check(lib().fn2_correlation1d_backward(desc(b0), desc(b1), desc(top_diff), desc(g0), desc(g1), pad, kernel_size,
                                           max_displacement, stride1, stride2, single_direction, corr_type, _ptr(ws), nb,
                                           _stream()))
    return g0, g1


def flow_warp(image, flow, fill_nan=False, out=None):
    if out is None:
        out = torch.empty_like(image)
    check(lib().fn2_flow_warp_forward(desc(image), desc(flow), desc(out), 1 if fill_nan else 0, _stream()))
    return out


def flow_warp_backward(image, flow, warped_diff, out=None):
    """-> (image_diff, flow_diff), into out = (image_diff, flow_diff) if given."""
    gi, gf = out if out is not None else (torch.empty_like(image), torch.empty_like(flow))
    check(lib().fn2_flow_warp_backward(desc(image), desc(flow), desc(warped_diff), desc(gi), desc(gf), _stream()))
    return gi, gf


def resample(x, out_h, out_w, rtype=2, antialias=True):
    out = _empty((x.shape[0], x.shape[1], out_h, out_w), x)
    check(lib().fn2_resample_forward(desc(x), desc(out), rtype, 1 if antialias else 0, _stream()))
    return out


def spatial_augmentation(x, mats, out_h, out_w, out=None):
    if out is None:
        out = _empty((x.shape[0], x.shape[1], out_h, out_w), x)
    mats = mats.contiguous()
    check(lib().fn2_spatial_augmentation(desc(x), desc(out), _ptr(mats), _stream()))
    return out


def color_contrast_augmentation(x, chroma, max_multiplier=1.0):
    out = x.clone(memory_format=torch.preserve_format)
    chroma = chroma.contiguous()
    check(lib().fn2_color_contrast_augmentation(desc(out), _ptr(chroma), max_multiplier, _stream()))
    return out


def chromatic_eigenspace(x, eigvec9):
    """-> 25 floats (tChromaticEigenSpace) as a device tensor of 32 (the tail is scratch)."""
    ev = torch.as_tensor(eigvec9, dtype=torch.float32, device=x.device).reshape(9).contiguous()
    space = torch.zeros(32, dtype=torch.float32, device=x.device)
    check(lib().fn2_chromatic_eigenspace(desc(x), _ptr(ev), _ptr(space), _stream()))
    return space


def chromatic_eigen_augmentation(x, coeffs, space, max_multiplier=1.0):
    out = x.clone(memory_format=torch.preserve_format)
    coeffs = coeffs.contiguous()
    check(lib().fn2_chromatic_eigen_augmentation(desc(out), _ptr(coeffs), _ptr(space), max_multiplier, _stream()))
    return out


def apply_effects(x, effects, max_multiplier=1.0, noise_seed=0, add_noise=False):
    out = x.clone(memory_format=torch.preserve_format)
    effects = effects.contiguous()
    check(lib().fn2_apply_effects(desc(out), _ptr(effects), max_multiplier, noise_seed, 1 if add_noise else 0, _stream()))
    return out


def mean_update(top, mean_pp, mean_pc, num_iter):
    check(lib().fn2_mean_update(desc(top), desc(mean_pp), _ptr(mean_pc), float(num_iter), _stream()))


def mean_subtract(top, mean_pp=None, mean_pc=None, per_pixel=False):
    check(lib().fn2_mean_subtract(desc(top), desc(mean_pp) if mean_pp is not None else None, _ptr(mean_pc),
                                  1 if per_pixel else 0, _stream()))
    return top


def _pair(v):
    return (v, v) if isinstance(v, int) else v


def _layer_desc(ci, co, k, stride, pad, deconv, bias, engine=0, relu_slope=None, input_guard_bytes=0):
    """fn2_conv_desc of a layer; k, stride, pad: an int or (h, w).  relu_slope None: no fused ReLU."""
    (kh, kw), (sh, sw), (ph, pw) = _pair(k), _pair(stride), _pair(pad)
    return fn2_conv_desc(ci, co, kh, kw, sh, sw, ph, pw, 1 if deconv else 0, 1 if bias else 0, 1 if relu_slope is not None else 0,
                         float(relu_slope or 0.0), engine, input_guard_bytes)


def _conv_desc(weight, stride, pad, deconv, bias, engine=0, relu_slope=None, input_guard_bytes=0):
    """The same from a weight blob in Caffe layout: conv [co,ci,kh,kw], deconv [ci,co,kh,kw]."""
    a, b, kh, kw = weight.shape
    ci, co = (a, b) if deconv else (b, a)
    return _layer_desc(ci, co, (kh, kw), stride, pad, deconv, bias, engine, relu_slope, input_guard_bytes)


def _out_shape(d, x):
    ho, wo = C.c_int(), C.c_int()
    check(lib().fn2_conv_out_shape(d, x.shape[2], x.shape[3], C.byref(ho), C.byref(wo)))
    return ho.value, wo.value


def _pack_and_forward(d, x, weight, bias, out, use_workspace=True):
    """Pack the Caffe-layout weight for d and x's channel stride, then run fn2_conv_forward of x into out."""
    l = lib()
    cis = x.stride(3) if x.stride(1) == 1 else d.ci
    packed = torch.empty(max(_size(l.fn2_conv_packed_floats, d, cis), 1), dtype=torch.float32, device=x.device)
    check(l.fn2_conv_pack_weights(d, cis, _ptr(weight), _ptr(packed), _stream()))
    wsb = _size(l.fn2_conv_workspace_bytes, d, x.shape[0], x.shape[2], x.shape[3])
    ws = torch.empty(max(wsb, 4), dtype=torch.uint8, device=x.device) if use_workspace else None
    check(l.fn2_conv_forward(d, desc(x), _ptr(packed), _ptr(bias), desc(out), _ptr(ws), wsb if ws is not None else 0, _stream()))
    return out


def conv_plan(ci, co, k, stride, pad, deconv, n, h, w, ci_stride):
    """fn2_conv_plan: the tensor-core engines' host-side plan for a layer shape (8 ints, see include/fn2.h): NT, tile units,
    K steps per tile, mode, first split tile, K ranges per split tile."""
    plan = (C.c_int32 * 8)()
    check(lib().fn2_conv_plan(_layer_desc(ci, co, k, stride, pad, deconv, True), n, h, w, ci_stride, plan))
    return list(plan)


def conv2d(x, weight, bias=None, stride=1, pad=0, deconv=False, relu_slope=None, engine=0, channels_last_out=None,
           use_workspace=True, input_guard_bytes=0, out=None):
    """weight in Caffe layout: conv [co,ci,kh,kw], deconv [ci,co,kh,kw]."""
    d = _conv_desc(weight, stride, pad, deconv, bias is not None, engine, relu_slope, input_guard_bytes)
    ho, wo = _out_shape(d, x)
    if out is None:
        out = _empty((x.shape[0], d.co, ho, wo), x, channels_last_out)
    return _pack_and_forward(d, x, weight.contiguous(), bias, out, use_workspace)


def wgrad_plan(ci, co, k, stride, pad, deconv, n, h, w, engine=0, bias=True):
    """fn2_conv_wgrad_plan: the weight-gradient route a layer shape takes (8 ints, see include/fn2.h): route (1 SIMT, 2 tensor
    cores), NT, G, TG, BT, ST, S (SIMT: pixel splits), bias blocks.  k, stride, pad: an int or (h, w)."""
    plan = (C.c_int32 * 8)()
    check(lib().fn2_conv_wgrad_plan(_layer_desc(ci, co, k, stride, pad, deconv, bias, engine), n, h, w, plan))
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
        workspace = _ws(_size(l.fn2_conv_backward_params_workspace_bytes, d, x.shape[0], x.shape[2], x.shape[3]), x.device)
    assert workspace.dtype == torch.uint8 and workspace.is_contiguous()
    check(l.fn2_conv_backward_params(d, desc(x), desc(top_diff), _ptr(wd), _ptr(bd), 1 if accumulate else 0, _ptr(workspace),
                                     workspace.numel(), _stream()))
    dx = None
    if need_input_grad:
        bdsc, flip = fn2_conv_desc(), C.c_int()
        check(l.fn2_conv_backward_data_desc(d, x.shape[2], x.shape[3], bdsc, C.byref(flip)))
        w2 = weight
        if flip.value:
            w2 = torch.empty_like(weight)
            check(l.fn2_conv_flip_transpose_weights(d, _ptr(weight), _ptr(w2), _stream()))
        assert _out_shape(bdsc, top_diff) == (x.shape[2], x.shape[3])
        dx = _pack_and_forward(bdsc, top_diff, w2, None, torch.empty_like(x))
    return dx, wd, bd


def relu_backward(top_data, top_diff, negative_slope=0.0, out=None, accumulate=False):
    """-> out (a new tensor if None) = top_diff * (top_data > 0 ? 1 : negative_slope), added to out's values if accumulate."""
    if out is None:
        out = torch.empty_like(top_diff)
    check(lib().fn2_relu_backward(desc(top_data), desc(top_diff), desc(out), negative_slope, 1 if accumulate else 0, _stream()))
    return out


def axpby(x, alpha, y, beta):
    check(lib().fn2_axpby(desc(x), alpha, desc(y), beta, _stream()))
    return y


def relu(x, negative_slope=0.0, out=None):
    if out is None:
        out = torch.empty_like(x)
    check(lib().fn2_relu_forward(desc(x), desc(out), negative_slope, _stream()))
    return out


def eltwise_sum(bottoms, coeffs=None, out=None):
    if out is None:
        out = torch.empty_like(bottoms[0])
    ds = [desc(b) for b in bottoms]
    arr = (C.POINTER(fn2_tensor) * len(ds))(*[C.pointer(d) for d in ds])
    cf = (C.c_float * len(ds))(*(coeffs if coeffs else [1.0] * len(ds)))
    check(lib().fn2_eltwise_sum(arr, cf, len(ds), desc(out), _stream()))
    return out


def channel_norm(x, out=None):
    if out is None:
        out = torch.empty((x.shape[0], 1, x.shape[2], x.shape[3]), device=x.device, dtype=torch.float32)
    check(lib().fn2_channel_norm_forward(desc(x), desc(out), _stream()))
    return out


def warp_block(flow, image0, image1, scale_coeff, fill_nan=False, out=None):
    """The warp block between stacked networks in one pass: flow (N, 2, h, w) up-sampled to the images' size (LINEAR),
    image1 warped by it, the error image0 - warped, its channel norm and the up-sampled flow times scale_coeff.
    -> out = (flow_full, warped, err, err_norm, flow_scaled), new tensors if None."""
    if out is None:
        N, Cc, H, W = image0.shape
        out = (_empty((N, 2, H, W), image0), torch.empty_like(image1), torch.empty_like(image0),
               _empty((N, 1, H, W), image0, False), _empty((N, 2, H, W), image0))
    check(lib().fn2_warp_block_forward(*[desc(t) for t in (flow, image0, image1) + tuple(out)], scale_coeff,
                                       1 if fill_nan else 0, _stream()))
    return out


def downsample(x, top_h, top_w, out=None):
    if out is None:
        out = _empty((x.shape[0], x.shape[1], top_h, top_w), x)
    check(lib().fn2_downsample_forward(desc(x), desc(out), _stream()))
    return out


def _l1_desc(l2_per_location, l2_prescale_by_channels, normalize_by_num_entries, epsilon, plateau):
    return fn2_l1loss_desc(1 if l2_per_location else 0, 1 if l2_prescale_by_channels else 0, 1 if normalize_by_num_entries else 0,
                           float(epsilon), float(plateau))


def l1loss(b0, b1=None, *, l2_per_location=False, l2_prescale_by_channels=False, normalize_by_num_entries=False, epsilon=1e-2,
           plateau=0.0, workspace=None):
    """L1LossLayer::Forward_gpu through the C-ABI -> (loss, state): two device float tensors, the loss (1 float) and the state
    {loss, normalize_coeff, masked sum, not-NaN count} the backward reads.  workspace: a uint8 CUDA tensor whose bytes are the
    workspace (default: one of the reported size)."""
    l = lib()
    d = _l1_desc(l2_per_location, l2_prescale_by_channels, normalize_by_num_entries, epsilon, plateau)
    if workspace is None:
        workspace = _ws(_size(l.fn2_l1loss_workspace_bytes, b0.shape[0], b0.shape[2], b0.shape[3]), b0.device)
    assert workspace.dtype == torch.uint8 and workspace.is_contiguous()
    loss = torch.empty(1, dtype=torch.float32, device=b0.device)
    state = torch.empty(4, dtype=torch.float32, device=b0.device)
    check(l.fn2_l1loss_forward(desc(b0), desc(b1) if b1 is not None else None, d, _ptr(state), _ptr(loss), _ptr(workspace),
                               workspace.numel(), _stream()))
    return loss, state


def l1loss_backward(b0, b1=None, *, l2_per_location=False, l2_prescale_by_channels=False, normalize_by_num_entries=False,
                    epsilon=1e-2, plateau=0.0, state, top_diff, out0=None, out1=None, accumulate0=False, accumulate1=False):
    """L1LossLayer::Backward_gpu: writes (accumulate: adds) the gradient of each bottom into out0 / out1; None: do not
    propagate to that bottom.  state: from l1loss(); top_diff: the loss weight as a device float tensor.  -> (out0, out1)"""
    d = _l1_desc(l2_per_location, l2_prescale_by_channels, normalize_by_num_entries, epsilon, plateau)
    check(lib().fn2_l1loss_backward(desc(b0), desc(b1) if b1 is not None else None, d, _ptr(state), _ptr(top_diff),
                                    desc(out0) if out0 is not None else None, desc(out1) if out1 is not None else None,
                                    1 if accumulate0 else 0, 1 if accumulate1 else 0, _stream()))
    return out0, out1


def _lpq_desc(p_epsilon, q_epsilon, l2_prescale_by_channels, normalize_by_num_entries):
    return fn2_lpqloss_desc(float(p_epsilon), float(q_epsilon), 1 if l2_prescale_by_channels else 0, 1 if normalize_by_num_entries else 0)


def lpqloss(b0, b1=None, *, p, q, p_epsilon=0.0, q_epsilon=1e-2, l2_prescale_by_channels=False, normalize_by_num_entries=False,
            state=None, workspace=None):
    """LpqLossLayer::Forward_gpu through the C-ABI (include/fn2_lpq.h) -> (loss, state): the loss (1 float) and the state
    {loss, normalize_coeff, loss sum, not-NaN count, p, q} the backward reads, both device float tensors.  p and q are written
    into the state on the current stream first; p = None / q = None keep the ones a given state holds."""
    l = lib()
    d = _lpq_desc(p_epsilon, q_epsilon, l2_prescale_by_channels, normalize_by_num_entries)
    if workspace is None:
        workspace = _ws(_size(l.fn2_lpqloss_workspace_bytes, b0.shape[0], b0.shape[2], b0.shape[3]), b0.device)
    assert workspace.dtype == torch.uint8 and workspace.is_contiguous()
    if state is None:
        state = torch.zeros(LPQLOSS_STATE_FLOATS, dtype=torch.float32, device=b0.device)
    if p is not None:
        state[4] = float(p)
    if q is not None:
        state[5] = float(q)
    loss = torch.empty(1, dtype=torch.float32, device=b0.device)
    check(l.fn2_lpqloss_forward(desc(b0), desc(b1) if b1 is not None else None, d, _ptr(state), _ptr(loss), _ptr(workspace),
                                workspace.numel(), _stream()))
    return loss, state


def lpqloss_backward(b0, b1=None, *, p_epsilon=0.0, q_epsilon=1e-2, l2_prescale_by_channels=False, normalize_by_num_entries=False,
                     state, top_diff, out0=None, out1=None, accumulate0=False, accumulate1=False):
    """LpqLossLayer::Backward_gpu: writes (accumulate: adds) the gradient of each bottom into out0 / out1; None: do not
    propagate to that bottom.  state: from lpqloss() (it holds p and q); top_diff: the loss weight as a device float tensor.
    -> (out0, out1)"""
    d = _lpq_desc(p_epsilon, q_epsilon, l2_prescale_by_channels, normalize_by_num_entries)
    check(lib().fn2_lpqloss_backward(desc(b0), desc(b1) if b1 is not None else None, d, _ptr(state), _ptr(top_diff),
                                     desc(out0) if out0 is not None else None, desc(out1) if out1 is not None else None,
                                     1 if accumulate0 else 0, 1 if accumulate1 else 0, _stream()))
    return out0, out1


def flow_augmentation(flow, mats1, mats2_inverse, out_h, out_w, out=None):
    """FlowAugmentation: the flow (N, 2, H, W) of the pair augmented by mats1 / the inverse of mats2 (N x 6 floats each, NAME
    order t0..t5, device tensors) -> out (N, 2, out_h, out_w), a new tensor if None."""
    if out is None:
        out = _empty((flow.shape[0], 2, out_h, out_w), flow)
    mats1, mats2_inverse = mats1.contiguous(), mats2_inverse.contiguous()
    check(lib().fn2_flow_augmentation(desc(flow), desc(out), _ptr(mats1), _ptr(mats2_inverse), _stream()))
    return out


def copy(src, dst):
    check(lib().fn2_copy(desc(src), desc(dst), _stream()))
    return dst


def fill(dst, value):
    check(lib().fn2_fill(desc(dst), value, _stream()))
    return dst


def frames_to_tensor(frames, dst):
    """uint8 CUDA frames (N, H, W, K), K = 1, 3 or 4, dense -> dst, a float32 (N, 3, H, W) view, as BGR 0..255."""
    assert frames.is_cuda and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.is_contiguous(), \
        "need dense uint8 CUDA frames (N, H, W, K)"
    assert tuple(frames.shape[:3]) == (dst.shape[0], dst.shape[2], dst.shape[3]), (tuple(frames.shape), tuple(dst.shape))
    check(lib().fn2_frames_to_tensor(frames.data_ptr(), frames.shape[3], desc(dst), _stream()))
    return dst


def flow_to_tensor(payload, format, flags, dst):
    """Dense CUDA flow-file payloads (any dtype; .flo [N][H][W][2] or PFM [N][H][W][3] floats, format FLOW_FLO, FLOW_PFM or
    FLOW_PFM_BE; a KITTI PNG's unfiltered [N][H][W][3] big-endian uint16 samples, FLOW_KITTI, NaN at invalid pixels) -> dst, a
    float32 (N, 2, H, W) view; flags FLOW_UINT16FLOW quantises as the reference's training data."""
    assert payload.is_cuda and payload.is_contiguous(), "need a dense CUDA payload"
    check(lib().fn2_flow_to_tensor(payload.data_ptr(), int(format), int(flags), desc(dst), _stream()))
    return dst


def flow_to_kitti_png_rows(flow, out=None):
    """A float32 (N, 2, H, W) CUDA view of any strides -> out, N*H Paeth-filtered KITTI PNG scanlines of 1 + 6 W bytes (a dense
    uint8 CUDA tensor of at least N*H*(1 + 6 W) bytes; a new (N, H, 1 + 6 W) one if None)."""
    N, _, H, W = flow.shape
    if out is None:
        out = torch.empty((N, H, 1 + 6 * W), dtype=torch.uint8, device=flow.device)
    assert out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and out.numel() >= N * H * (1 + 6 * W)
    check(lib().fn2_flow_to_kitti_png_rows(desc(flow), out.data_ptr(), _stream()))
    return out


def flow_max_radius(flow, out=None):
    """A float32 (N, 2, H, W) CUDA view of any strides -> out, N float32 on the device (a new tensor if None): each image's
    largest sqrt(u^2 + v^2) over its known pixels (include/fn2_flow.h), -1 for an image without one.  No host sync."""
    if out is None:
        out = torch.empty(flow.shape[0], dtype=torch.float32, device=flow.device)
    assert out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.numel() == flow.shape[0]
    check(lib().fn2_flow_max_radius(desc(flow), out.data_ptr(), _stream()))
    return out


def _colour_scale(flow, max_flow, max_radius, fallback):
    """-> (max, fallback, max_flow) arguments of the colour entry points: a fixed max_flow, or per-image radii (max_radius, the
    flow's own when None)."""
    if max_flow is not None:
        return None, None, float(max_flow)
    if max_radius is None:
        max_radius = flow_max_radius(flow)
    for t in (max_radius, fallback):
        assert t is None or (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.numel() == flow.shape[0])
    return max_radius.data_ptr(), _ptr(fallback), 0.0


def flow_to_color(flow, max_flow=None, out=None, max_radius=None, fallback=None):
    """A float32 (N, 2, H, W) CUDA view of any strides -> out, a dense uint8 (N, H, W, 3) CUDA tensor (a new one if None) of
    Middlebury colour-coded RGB (include/fn2_flow.h).  Scale: max_flow (> 0) for every image, else per image max_radius (N
    device floats, flow_max_radius(flow) when None), fallback's where max_radius is negative, and 1 where the result is not
    positive."""
    N, _, H, W = flow.shape
    if out is None:
        out = torch.empty((N, H, W, 3), dtype=torch.uint8, device=flow.device)
    assert out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and out.numel() >= N * H * W * 3
    m, fb, mf = _colour_scale(flow, max_flow, max_radius, fallback)
    check(lib().fn2_flow_to_color(desc(flow), m, fb, mf, out.data_ptr(), _stream()))
    return out


def flow_to_color_png_rows(flow, out=None, max_flow=None, max_radius=None, fallback=None):
    """As flow_to_color, written as N*H Paeth-filtered 8-bit RGB PNG scanlines of 1 + 3 W bytes -> out, a dense uint8 CUDA
    tensor of at least N*H*(1 + 3 W) bytes (a new (N, H, 1 + 3 W) one if None)."""
    N, _, H, W = flow.shape
    if out is None:
        out = torch.empty((N, H, 1 + 3 * W), dtype=torch.uint8, device=flow.device)
    assert out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and out.numel() >= N * H * (1 + 3 * W)
    m, fb, mf = _colour_scale(flow, max_flow, max_radius, fallback)
    check(lib().fn2_flow_to_color_png_rows(desc(flow), m, fb, mf, out.data_ptr(), _stream()))
    return out


def flow_fb_occlusion(fwd, bwd, alpha1=0.01, alpha2=0.5, out=None, row_stride=None, pair_stride=None):
    """Frame 0's occlusion mask by the forward-backward check (include/fn2_flow.h): fwd and bwd are float32 (N, 2, H, W) CUDA
    views of any strides -> out, a uint8 CUDA tensor (a new dense (N, H, W) one if None), 255 where occluded and 0 where
    visible.  With row_stride / pair_stride, pixel (n, y, x) goes to byte n * pair_stride + y * row_stride + x of out (a dense
    uint8 buffer), and no other byte is written."""
    N, _, H, W = fwd.shape
    if out is None:
        out = torch.empty((N, H, W), dtype=torch.uint8, device=fwd.device)
    rs = W if row_stride is None else row_stride
    ps = H * rs if pair_stride is None else pair_stride
    assert out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and out.numel() >= (N - 1) * ps + (H - 1) * rs + W
    check(lib().fn2_flow_fb_occlusion(desc(fwd), desc(bwd), float(alpha1), float(alpha2), out.data_ptr(), rs, ps, _stream()))
    return out


def mask_confusion(pred, gt, out=None):
    """Per-pair confusion counts of predicted against ground-truth occlusion masks (include/fn2_eval.h): pred and gt are dense
    uint8 (N, H, W) CUDA tensors, nonzero meaning occluded -> out, an (N, len(MASK_CONFUSION_FIELDS)) float64 CUDA tensor (a
    new one if None) with the fields of MASK_CONFUSION_FIELDS (tp, fp, fn, tn)."""
    N, H, W = pred.shape
    assert tuple(gt.shape) == (N, H, W), (tuple(pred.shape), tuple(gt.shape))
    if out is None:
        out = torch.empty((N, len(MASK_CONFUSION_FIELDS)), dtype=torch.float64, device=pred.device)
    assert out.is_cuda and out.dtype == torch.float64 and out.is_contiguous() and out.numel() == N * len(MASK_CONFUSION_FIELDS)
    check(lib().fn2_mask_confusion(_planes(pred, N, H, W, H * W), _planes(gt, N, H, W, H * W), H * W, N, H, W,
                                   C.cast(out.data_ptr(), C.POINTER(C.c_double)), _stream()))
    return out


def flow_error_workspace_bytes(N, H, W):
    return _size(lib().fn2_flow_error_workspace_bytes, N, H, W)


def flow_error(pred, gt, out=None, workspace=None):
    """Per-pair scores of a predicted flow against ground truth (include/fn2_eval.h): pred and gt are float32 (N, 2, H, W) CUDA
    views of any strides -> out, an (N, len(FLOW_ERROR_FIELDS)) float64 CUDA tensor (a new one if None) with the fields of
    FLOW_ERROR_FIELDS.  workspace: a uint8 CUDA tensor whose bytes are the workspace (default: one of the reported size)."""
    N, _, H, W = pred.shape
    if workspace is None:
        workspace = _ws(flow_error_workspace_bytes(N, H, W), pred.device)
    assert workspace.dtype == torch.uint8 and workspace.is_contiguous()
    if out is None:
        out = torch.empty((N, len(FLOW_ERROR_FIELDS)), dtype=torch.float64, device=pred.device)
    assert out.dtype == torch.float64 and out.is_contiguous() and out.numel() == N * len(FLOW_ERROR_FIELDS)
    check(lib().fn2_flow_error(desc(pred), desc(gt), C.cast(out.data_ptr(), C.POINTER(C.c_double)), _ptr(workspace),
                               workspace.numel(), _stream()))
    return out


def _planes(masks, N, H, W, pair_stride):
    """A dense uint8 CUDA tensor holding N mask planes [H][W], pair i's at byte i * pair_stride -> its device address."""
    assert masks.is_cuda and masks.dtype == torch.uint8 and masks.is_contiguous(), "need dense uint8 CUDA masks"
    assert pair_stride >= H * W and masks.numel() >= (N - 1) * pair_stride + H * W, (tuple(masks.shape), pair_stride)
    return masks.data_ptr()


def occlusion_boundary_dist2(masks, out=None, pair_stride=None):
    """Squared distance of every pixel to the nearest occlusion boundary (include/fn2_eval.h): masks is a dense uint8 CUDA
    tensor, (N, H, W) occlusion masks, or any buffer holding them at pair_stride bytes with out given -> out, a dense int32
    (N, H, W) CUDA tensor (a new one if None), DIST2_NONE throughout a pair without a boundary."""
    if out is None:
        out = torch.empty(masks.shape, dtype=torch.int32, device=masks.device)
    assert out.is_cuda and out.dtype == torch.int32 and out.dim() == 3 and out.is_contiguous()
    N, H, W = out.shape
    pair_stride = H * W if pair_stride is None else pair_stride
    check(lib().fn2_occlusion_boundary_dist2(_planes(masks, N, H, W, pair_stride), pair_stride, N, H, W,
                                             C.cast(out.data_ptr(), C.POINTER(C.c_int32)), _stream()))
    return out


def flow_error_regions_workspace_bytes(N, H, W):
    return _size(lib().fn2_flow_error_regions_workspace_bytes, N, H, W)


def flow_error_regions(pred, gt, occ=None, obj=None, dist2=None, mask_pair_stride=None, out=None, workspace=None):
    """Per-pair scores by region (include/fn2_eval.h): pred and gt as for flow_error; occ and obj are dense uint8 CUDA tensors
    of (N, H, W) occlusion masks and object maps, or buffers holding them at mask_pair_stride bytes, each may be None; dist2 is
    occlusion_boundary_dist2(occ), required with occ -> out, an (N, len(FLOW_REGION_FIELDS)) float64 CUDA tensor (a new one if
    None).  workspace as for flow_error."""
    N, _, H, W = pred.shape
    stride = H * W if mask_pair_stride is None else mask_pair_stride
    if workspace is None:
        workspace = _ws(flow_error_regions_workspace_bytes(N, H, W), pred.device)
    assert workspace.dtype == torch.uint8 and workspace.is_contiguous()
    if out is None:
        out = torch.empty((N, len(FLOW_REGION_FIELDS)), dtype=torch.float64, device=pred.device)
    assert out.dtype == torch.float64 and out.is_contiguous() and out.numel() == N * len(FLOW_REGION_FIELDS)
    if dist2 is not None:
        assert dist2.is_cuda and dist2.dtype == torch.int32 and dist2.is_contiguous() and tuple(dist2.shape) == (N, H, W)
    check(lib().fn2_flow_error_regions(desc(pred), desc(gt), None if occ is None else _planes(occ, N, H, W, stride),
                                       None if obj is None else _planes(obj, N, H, W, stride), stride,
                                       None if dist2 is None else C.cast(dist2.data_ptr(), C.POINTER(C.c_int32)),
                                       C.cast(out.data_ptr(), C.POINTER(C.c_double)), _ptr(workspace), workspace.numel(),
                                       _stream()))
    return out
