"""Shared helpers for the parity tests (seeded synthetic inputs, comparison)."""
import time

import numpy as np


def rng(seed=1701):     # seed mirrors the reference's GradientChecker (test_gradient_check_util.hpp:25)
    return np.random.default_rng(seed)


def smooth_images(r, n, h, w, shift=(1.7, -2.3)):
    """Two BGR frames with integer values 0..255 as scripts/run-flownet.py:30-35 feeds them: low-pass noise,
    second frame = first shifted by a sub-pixel offset plus noise."""
    import scipy.ndimage as ndi
    base = r.standard_normal((n, 3, h + 16, w + 16))
    base = ndi.gaussian_filter(base, sigma=(0, 0, 3, 3))
    base = (base - base.min()) / (base.max() - base.min())
    a = base[:, :, 8:8 + h, 8:8 + w]
    b = ndi.shift(base, (0, 0, shift[1], shift[0]), order=1, mode="nearest")[:, :, 8:8 + h, 8:8 + w]
    b = b + 0.01 * r.standard_normal(b.shape)
    to8 = lambda x: np.clip(np.round(x * 255), 0, 255).astype(np.float32)
    return to8(a), to8(b)


def maxabs(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    nan_a, nan_b = np.isnan(a), np.isnan(b)
    assert (nan_a == nan_b).all(), "NaN pattern differs"
    d = np.abs(np.where(nan_a, 0, a) - np.where(nan_b, 0, b))
    return float(d.max()) if d.size else 0.0


def device_view(a, layout="nhwc"):
    """a (N, C, H, W) on the device: "nchw" / "nhwc" dense; "pad": the nets' pixel stride (Blob::compute_cstride: channels
    rounded up to 4 below 32, else to 32); "slice": channels [5, 5 + C) of a wider channels_last parent (a zero-copy concat
    child).  Channels outside the view hold NaN, so a stray read shows in any sum and a stray write replaces a NaN."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    if layout == "nchw":
        return t
    if layout == "nhwc":
        return t.contiguous(memory_format=torch.channels_last)
    n, c, h, w = t.shape
    if layout == "pad":
        align = 4 if c < 32 else 32
        off, width = 0, (c + align - 1) // align * align
    else:
        off, width = 5, c + 8
    parent = torch.full((n, width, h, w), float("nan"), device="cuda").contiguous(memory_format=torch.channels_last)
    parent[:, off:off + c] = t
    return parent[:, off:off + c]


def net_convs(text):
    """The Convolution / Deconvolution layers of a filled prototxt: (name, Ci, H, W, Co, (kh, kw), s, (ph, pw), deconv,
    trainable), from the oracle's prototxt parser and a walk over the blob shapes.  A layer with two bottoms (the deploy nets'
    conv1 on both images) is listed once; its bottoms have the same shape."""
    return net_walk(text)[0]


def net_losses(text):
    """The L1Loss layers of a filled prototxt: (name, (C, H, W) of its first bottom), by the walk of net_convs."""
    return net_walk(text)[1]


def net_walk(text):
    """-> (net_convs, net_losses, concats, io) of a filled prototxt.  concats: {bottom blob of a Concat of two or more bottoms:
    (the concat's top, the bottom's first channel in it, the top's channels)}; io: {layer name: (bottom blobs, top blobs)}."""
    from flownet2_b200 import ops as _ops
    from oracle import net as onet
    get, getall = onet.get, onet.getall
    net = onet.parse_prototxt(text)
    shp, out, losses, concats, io = {}, [], [], {}, {}
    for t, s in zip(getall(net, "input"), getall(net, "input_shape")):            # legacy deploy inputs
        shp[t] = tuple(int(d) for d in getall(s, "dim"))[1:]
    for l in getall(net, "layer"):
        ty, bots, tops = get(l, "type"), getall(l, "bottom"), getall(l, "top")
        b = [shp.get(n) for n in bots]
        io[get(l, "name")] = (bots, tops)
        if ty == "Input":
            for t, s in zip(tops, getall(get(l, "input_param"), "shape")):
                shp[t] = tuple(int(d) for d in getall(s, "dim"))[1:]
        elif ty in ("Convolution", "Deconvolution"):
            cp = get(l, "convolution_param")
            kh, kw = onet._hw(cp, "kernel_size", "kernel_h", "kernel_w", 0)
            sh, sw = onet._hw(cp, "stride", "stride_h", "stride_w", 1)
            ph, pw = onet._hw(cp, "pad", "pad_h", "pad_w", 0)
            assert sh == sw and all(x == b[0] for x in b)
            ci, h, w = b[0]
            co = int(get(cp, "num_output"))
            if ty == "Deconvolution":
                ho, wo = sh * (h - 1) + kh - 2 * ph, sw * (w - 1) + kw - 2 * pw
            else:
                ho, wo = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
            for t in tops:
                shp[t] = (co, ho, wo)
            lr = [float(get(pp, "lr_mult", 1)) for pp in getall(l, "param")]
            out.append((get(l, "name"), ci, h, w, co, (kh, kw), sh, (ph, pw), ty == "Deconvolution", any(lr) or not lr))
        elif ty == "DataAugmentation":
            ap = get(l, "augmentation_param")
            shp[tops[0]] = (b[0][0], int(get(ap, "crop_height")), int(get(ap, "crop_width")))
            for t in tops[1:]:
                shp[t] = (1, 1, 1)
        elif ty == "GenerateAugmentationParameters":
            shp[tops[0]] = (1, 1, 1)
        elif ty == "FlowAugmentation":
            ap = get(l, "augmentation_param")
            shp[tops[0]] = (b[0][0], int(get(ap, "crop_height")), int(get(ap, "crop_width")))
        elif ty == "Correlation":
            cp = get(l, "correlation_param")
            shp[tops[0]] = _ops.correlation_shape(b[0][1], b[0][2], int(get(cp, "pad", 0)), int(get(cp, "kernel_size")),
                                                  int(get(cp, "max_displacement")), int(get(cp, "stride_1", 1)),
                                                  int(get(cp, "stride_2", 1)))
        elif ty == "Concat":
            shp[tops[0]] = (sum(x[0] for x in b),) + b[0][1:]
            c0 = 0
            for n_, x in zip(bots, b):
                if len(bots) > 1:
                    concats.setdefault(n_, (tops[0], c0, shp[tops[0]][0]))
                c0 += x[0]
        elif ty in ("Downsample", "Resample"):
            # the size of the second bottom, else the layer's own (the deploy nets' 436 -> 448 adaptation)
            rp = get(l, "resample_param", [])
            hw = b[1][1:] if len(b) > 1 else (int(get(rp, "height", get(get(l, "downsample_param", []), "top_height"))),
                                               int(get(rp, "width", get(get(l, "downsample_param", []), "top_width"))))
            shp[tops[0]] = (b[0][0],) + tuple(hw)
        elif ty == "ChannelNorm":
            shp[tops[0]] = (1,) + b[0][1:]
        elif ty in ("ReLU", "Eltwise", "FlowWarp"):
            shp[tops[0]] = b[0]
        elif ty == "L1Loss":
            losses.append((get(l, "name"), b[0]))
        else:
            assert ty == "Silence", ty
    return out, losses, concats, io


def train_convs(model, width=448, height=320):
    """net_convs of models/<model>_train.prototxt.template at a width x height crop."""
    from flownet2_b200 import fill_train_template, train_template
    return net_convs(fill_train_template(train_template(model), width, height, width + 64, height + 64, 1))


def deploy_convs(model, width=1024, height=436):
    """net_convs of models/<model>_deploy.prototxt.template for width x height frames (adapted to multiples of 64 inside)."""
    from flownet2_b200 import fill_template, model_template
    return net_convs(fill_template(model_template(model), width, height))


def kernels_per_case(runs):
    """Names of the kernels each of runs launches, from one profiler session.  Every run sits in a window of its own between
    synchronisations, 2 ms from the next.  A kernel belongs to the window of its launch call (the profiler gives both the
    same correlation id), else to the window its start falls in or is nearest to (a warm-up run of the first case before
    the windows lands in that case's).  A session in which some window has no kernel at all (the profiler now and then
    drops device activity) is taken again; the windows' own annotations on the device timeline do not count as kernels."""
    import torch
    cpu, cuda = torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA
    for _ in range(3):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[cpu, cuda]) as prof:
            runs[0]()                                   # the session's first kernels can go unrecorded
            torch.cuda.synchronize()
            time.sleep(0.002)
            for i, run in enumerate(runs):
                with torch.profiler.record_function("ew_case_%d" % i):
                    run()
                    torch.cuda.synchronize()
                time.sleep(0.002)
        events = prof.events()
        win = {int(e.name[8:]): e.time_range for e in events if e.name.startswith("ew_case_")}

        def window(t):
            return min(win, key=lambda i: max(win[i].start - t, t - win[i].end, 0))

        launch = {e.id: window(e.time_range.start) for e in events
                  if e.device_type == torch.autograd.DeviceType.CPU and "LaunchKernel" in e.name}
        names = [set() for _ in runs]
        for e in events:     # the device timeline also carries the ew_case_ ranges: not kernels, so a window with one only is empty
            if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith("ew_case_"):
                names[launch.get(e.id, window(e.time_range.start))].add(e.name)
        if all(names):
            break
    return names
