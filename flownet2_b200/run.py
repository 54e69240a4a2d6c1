"""Optical flow of image files: the command line of the reference's scripts/run-flownet.py and run-flownet-many.py.

    python -m flownet2_b200.run weights.caffemodel models/FlowNet2_deploy.prototxt.template img0.png img1.png out.flo
    python -m flownet2_b200.run weights.caffemodel models/FlowNet2_deploy.prototxt.template pairs.txt [--batch 4] [--kitti]

The list file holds one ``img0 img1 out.flo`` line per pair; blank lines are skipped.  The weights (.caffemodel or
.caffemodel.h5) are read once.  Pairs are grouped by frame size in order of first appearance, and each size gets one
Net(fill_template(template, W, H), weights, TEST, batch=B); at most one net is alive at a time.  Every forward runs B pairs;
the last batch of a size is padded by repeating its last pair, and the extra outputs are dropped.

Frames are PPM / PGM (P6 / P5, maxval 255, read here) or anything Pillow reads, converted the way scipy.misc.imread hands
them to the reference (palette to RGB or RGBA, LA to L).  The 8-bit frames are copied to the device as they are and
converted there (fn2_net_set_input_frames_device), and the flow comes back as (H, W, 2), the payload order of .flo
(fn2_net_get_blob_nhwc_device).  While batch k runs, batch k+1 is decoded on a thread pool into one of two pinned buffers and
copied to the device on a copy stream, and batch k-1's flow is copied back on another and written by a writer thread.

--kitti writes every output as a KITTI flow PNG (flownet2_b200.kitti, the format the KITTI benchmark takes) instead of a
.flo: the flow becomes Paeth-filtered PNG scanlines on the net's stream (fn2_flow_to_kitti_png_rows, 6 bytes a pixel instead
of 8), and the writer thread deflates them.  A pixel whose flow is not finite is stored as invalid.

There is no NaN-retry loop (the reference retries for a race in its Caffe build that this engine does not have): a pair whose
flow is not finite is named on stderr and the exit status is 1.  Under torchrun (WORLD_SIZE, RANK, LOCAL_RANK), rank r takes
the lines i with i % WORLD_SIZE == r on device LOCAL_RANK; no collective is needed.

Two limits on what the outputs promise:
  * Bit identity only at --batch 1.  The tensor-core convolution engines split K by the tile count, which depends on the
    batch, so a pair's flow at B > 1 can differ from its flow at B = 1 in the last bits.  At --batch 1 every file equals the
    single-pair run's bit for bit; batched outputs are held to the project's 1e-4 bound against the float64 oracle.
  * Order and batching matter while the augmentation mean is still updating: weights whose DataAugmentation iteration
    counter is at or below recompute_mean keep updating the running mean with the pairs they see.  Released caffemodels
    and Net.fill_params are past that counter.
"""
import argparse
import gc
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np


class RunError(Exception):
    """A refused input: the message names the file, and the list line where there is one."""


# ------------------------------------------------------------------------------------------------
# Frames
# ------------------------------------------------------------------------------------------------
def _pnm_header(f, path):
    """-> (magic, width, height, maxval, raster offset) of a binary PGM / PPM; header comments are allowed."""
    data = f.read(4096)
    if data[:2] not in (b"P5", b"P6"):
        return None
    fields, i = [], 2
    while len(fields) < 3:
        while i < len(data) and data[i:i + 1].isspace():
            i += 1
        if data[i:i + 1] == b"#":
            while i < len(data) and data[i:i + 1] not in (b"\n", b"\r"):
                i += 1
            continue
        j = i
        while j < len(data) and data[j:j + 1].isdigit():
            j += 1
        if j == i:
            raise RunError("%s: malformed %s header" % (path, data[:2].decode()))
        fields.append(int(data[i:j]))
        i = j
    if not data[i:i + 1].isspace():
        raise RunError("%s: malformed %s header" % (path, data[:2].decode()))
    return data[:2], fields[0], fields[1], fields[2], i + 1


def _pil():
    try:
        from PIL import Image
        return Image
    except ImportError:
        return None


# Pillow modes -> the mode scipy.misc.imread hands over (palette with transparency -> RGBA, else RGB; LA -> L; bilevel -> L)
_PIL_MODES = {"L": "L", "RGB": "RGB", "RGBA": "RGBA", "1": "L", "LA": "L", "P": "RGB"}


def _pil_mode(im):
    if im.mode == "P" and "transparency" in im.info:
        return "RGBA"
    return _PIL_MODES.get(im.mode)


def probe_image(path):
    """-> (width, height, channels) of an image file without decoding its pixels; refuses what read_image would refuse."""
    if not os.path.isfile(path):
        raise RunError("%s: no such file" % path)
    with open(path, "rb") as f:
        hdr = _pnm_header(f, path)
    if hdr is not None:
        magic, w, h, maxval, _ = hdr
        if maxval != 255:
            raise RunError("%s: maxval %d, only 8-bit frames (maxval 255) are supported" % (path, maxval))
        return w, h, 1 if magic == b"P5" else 3
    Image = _pil()
    if Image is None:
        raise RunError("%s: not a binary PGM/PPM, and Pillow is not installed to read other formats" % path)
    try:
        with Image.open(path) as im:
            mode, (w, h) = _pil_mode(im), im.size
            src = im.mode
    except Exception as e:
        raise RunError("%s: cannot read the image: %s" % (path, e))
    if mode is None:
        raise RunError("%s: image mode %s is not an 8-bit gray, RGB or RGBA image" % (path, src))
    return w, h, {"L": 1, "RGB": 3, "RGBA": 4}[mode]


def read_image(path):
    """-> uint8 (H, W) gray, (H, W, 3) RGB or (H, W, 4) RGBA frame, as scipy.misc.imread returns it."""
    with open(path, "rb") as f:
        hdr = _pnm_header(f, path)
        if hdr is not None:
            magic, w, h, maxval, off = hdr
            if maxval != 255:
                raise RunError("%s: maxval %d, only 8-bit frames (maxval 255) are supported" % (path, maxval))
            k = 1 if magic == b"P5" else 3
            f.seek(off)
            raw = f.read(w * h * k)
            if len(raw) != w * h * k:
                raise RunError("%s: truncated raster (%d of %d bytes)" % (path, len(raw), w * h * k))
            a = np.frombuffer(raw, np.uint8).reshape((h, w, k) if k == 3 else (h, w))
            return a
    Image = _pil()
    if Image is None:
        raise RunError("%s: not a binary PGM/PPM, and Pillow is not installed to read other formats" % path)
    with Image.open(path) as im:
        mode = _pil_mode(im)
        if mode is None:
            raise RunError("%s: image mode %s is not an 8-bit gray, RGB or RGBA image" % (path, im.mode))
        a = np.asarray(im if im.mode == mode else im.convert(mode))
    return check_frame(a, path)


def check_frame(a, path):
    """Refuses a frame that is not 8-bit or has two channels (the reference's [2, 1, 0] cannot index it)."""
    if a.dtype != np.uint8:
        raise RunError("%s: %s pixels, only 8-bit frames are supported" % (path, a.dtype))
    if not (a.ndim == 2 or a.ndim == 3 and a.shape[2] in (3, 4)):
        raise RunError("%s: frames of shape %s; gray, RGB or RGBA frames are supported" % (path, a.shape))
    return a


def frame_as(a, k):
    """Frame a (H, W[, K]) as (H, W, k) bytes: k = its own channel count, or 3 (gray repeated, alpha dropped), all exact."""
    a = a[:, :, np.newaxis] if a.ndim == 2 else a
    if a.shape[2] == k:
        return a
    return np.repeat(a, 3, axis=2) if a.shape[2] == 1 else a[:, :, :3]


# ------------------------------------------------------------------------------------------------
# Lists, sizes, shards
# ------------------------------------------------------------------------------------------------
class Pair(object):
    def __init__(self, where, img0, img1, out):
        self.where, self.img0, self.img1, self.out = where, img0, img1, out
        self.size = self.channels = None


def read_list(path):
    """-> [Pair] of a list file: one ``img0 img1 out.flo`` line per pair, blank lines skipped."""
    if not os.path.isfile(path):
        raise RunError("%s: no such list file" % path)
    pairs = []
    with open(path) as f:
        for no, line in enumerate(f, 1):
            fields = line.split()
            if not fields:
                continue
            if len(fields) != 3:
                raise RunError("%s:%d: %d fields, expected 'img0 img1 out.flo'" % (path, no, len(fields)))
            pairs.append(Pair("%s:%d" % (path, no), *fields))
    return pairs


def shard(items, world, rank):
    """The items i with i % world == rank: frame-pair sharding over the ranks."""
    return [p for i, p in enumerate(items) if i % world == rank]


def probe_pairs(pairs):
    """Sets each pair's (width, height) and frame channel counts; refuses missing, unreadable or mismatched frames."""
    for p in pairs:
        try:
            w0, h0, k0 = probe_image(p.img0)
            w1, h1, k1 = probe_image(p.img1)
        except RunError as e:
            raise RunError("%s: %s" % (p.where, e))
        if (w0, h0) != (w1, h1):
            raise RunError("%s: %s is %dx%d but %s is %dx%d" % (p.where, p.img0, w0, h0, p.img1, w1, h1))
        p.size, p.channels = (w0, h0), (k0, k1)


def group_by_size(pairs):
    """-> [((width, height), [Pair])] in order of each size's first appearance."""
    groups = {}
    for p in pairs:
        groups.setdefault(p.size, []).append(p)
    return list(groups.items())


def batches(pairs, batch):
    """Consecutive batches of `batch` pairs; the last is padded with its last pair -> [(pairs, number of real pairs)]."""
    out = []
    for i in range(0, len(pairs), batch):
        b = pairs[i:i + batch]
        out.append((b + [b[-1]] * (batch - len(b)), len(b)))
    return out


def write_pnm(path, a):
    """Binary PGM (H, W) or PPM (H, W, 3) frame, maxval 255 -> path."""
    with open(path, "wb") as f:
        f.write(b"%s\n%d %d\n255\n" % (b"P5" if a.ndim == 2 else b"P6", a.shape[1], a.shape[0]))
        f.write(np.ascontiguousarray(a, np.uint8).tobytes())
    return str(path)


def write_flo(path, flow_hw2):
    """.flo file (src/caffe/util/output.cpp:16-64): 'PIEH', width, height (int32), then (H, W, 2) float32."""
    h, w = flow_hw2.shape[:2]
    with open(path, "wb") as f:
        f.write(b"PIEH")
        f.write(np.array([w, h], np.int32).tobytes())
        f.write(np.ascontiguousarray(flow_hw2, np.float32).tobytes())


# ------------------------------------------------------------------------------------------------
# The pipeline
# ------------------------------------------------------------------------------------------------
def _align(n, a=16):
    return (n + a - 1) // a * a


class FlowFiles(object):
    """run's per-batch sink: each pair's flow goes to the host and into its .flo file; a pair whose flow is not finite is named
    on stderr and kept in `bad`.

    The sink interface of _group_batches: payload_bytes(batch, H, W) pinned bytes per slot beyond the frames, read_payload(p,
    out) the host read of one pair's part of them (on the pool), stage(...) the net stream's use of them before the forward;
    bind(...) allocates dev[s] / host[s] for one frame size, score(s) runs on the net's stream after the flow is in
    flow_dev[s] and fills dev[s], which then goes to host[s] on the copy-back stream, and take(pairs, s, n_real)
    consumes host[s] on the writer thread."""

    def __init__(self):
        self.bad = []
        self.stats = {"write": 0.0}

    def payload_bytes(self, batch, H, W):
        return 0

    read_payload = stage = None

    def bind(self, torch, batch, H, W, flow_dev):
        self.dev = flow_dev
        self.host = [torch.empty((batch, H, W, 2)).pin_memory() for _ in range(2)]

    def score(self, s):
        pass

    def take(self, pairs, s, n_real):
        t0 = time.perf_counter()
        flows = self.host[s].numpy()
        for i, p in enumerate(pairs[:n_real]):
            if not np.isfinite(flows[i]).all():
                self.bad.append(p)
                sys.stderr.write("%s: the flow of %s %s is not finite\n" % (p.where, p.img0, p.img1))
            write_flo(p.out, flows[i])
        self.stats["write"] += time.perf_counter() - t0


class KittiFiles(FlowFiles):
    """run --kitti's sink: on the net's stream each batch's flow becomes KITTI PNG scanlines (fn2_flow_to_kitti_png_rows) and
    fn2_flow_error against a zero flow counts each pair's non-finite pixels; both come back in one copy, and the writer
    thread deflates each pair's rows into its file.  A pair with a non-finite pixel is named on stderr and kept in `bad`."""

    def bind(self, torch, batch, H, W, flow_dev):
        from . import FLOW_ERROR_FIELDS, kitti, ops
        self.ops, self.kitti, self.size = ops, kitti, (W, H)
        self.nonfinite, fields = FLOW_ERROR_FIELDS.index("nonfinite"), len(FLOW_ERROR_FIELDS)
        self.row_bytes = H * (1 + kitti.BPP * W)                          # one pair's scanlines
        self.rec_off = _align(batch * self.row_bytes, 8)                  # then the pairs' float64 records
        nb = self.rec_off + batch * fields * 8
        self.pred = [f.permute(0, 3, 1, 2) for f in flow_dev]             # (B, 2, H, W) views of the NHWC flow
        self.dev = [torch.empty(nb, dtype=torch.uint8, device="cuda") for _ in range(2)]
        self.host = [torch.empty(nb, dtype=torch.uint8).pin_memory() for _ in range(2)]
        self.records = [d[self.rec_off:].view(torch.float64).view(batch, fields) for d in self.dev]
        self.zero = torch.zeros((batch, 2, H, W), device="cuda")
        self.workspace = torch.empty(max(ops.flow_error_workspace_bytes(batch, H, W), 8), dtype=torch.uint8, device="cuda")

    def score(self, s):
        self.ops.flow_to_kitti_png_rows(self.pred[s], self.dev[s])
        self.ops.flow_error(self.pred[s], self.zero, out=self.records[s], workspace=self.workspace)

    def take(self, pairs, s, n_real):
        t0 = time.perf_counter()
        buf = self.host[s].numpy()
        rec = buf[self.rec_off:].view(np.float64).reshape(len(pairs), -1)
        n = self.row_bytes
        for i, p in enumerate(pairs[:n_real]):
            if rec[i, self.nonfinite] > 0:
                self.bad.append(p)
                sys.stderr.write("%s: the flow of %s %s is not finite\n" % (p.where, p.img0, p.img1))
            self.kitti.write_png_rows(p.out, buf[i * n:(i + 1) * n], *self.size)
        self.stats["write"] += time.perf_counter() - t0


def _group_batches(torch, net, size, pairs, batch, pool, stats, sink):
    """Runs one size's pairs through `net`, B per forward, with decode, copies, forward and the sink's work overlapped."""
    W, H = size
    in0, in1 = net.inputs[:2]
    todo = batches(pairs, batch)
    px = batch * H * W                                             # pixels of one input's frames; bytes: px * K, K <= 4
    pay_off = _align(2 * px * 4)                                   # the sink's payload follows the frames
    pay_bytes = sink.payload_bytes(batch, H, W)
    pay_one = pay_bytes // batch
    pin = [torch.empty(pay_off + pay_bytes, dtype=torch.uint8).pin_memory() for _ in range(2)]
    dev = [torch.empty(pay_off + pay_bytes, dtype=torch.uint8, device="cuda") for _ in range(2)]
    flow_dev = [torch.empty((batch, H, W, 2), device="cuda") for _ in range(2)]
    sink.bind(torch, batch, H, W, flow_dev)
    net_stream = torch.cuda.ExternalStream(net.stream)
    h2d_stream, d2h_stream = torch.cuda.Stream(), torch.cuda.Stream()
    ev = lambda: torch.cuda.Event(enable_timing=True)
    ev_h2d = [torch.cuda.Event() for _ in range(2)]                # pin[s] copied to dev[s]
    ev_used = [torch.cuda.Event() for _ in range(2)]               # the net has converted dev[s]
    ev_flow = [torch.cuda.Event() for _ in range(2)]               # sink.dev[s] holds the batch's result
    ev_d2h = [torch.cuda.Event() for _ in range(2)]                # sink.host[s] holds it
    timing = []                                                    # per batch: (h2d, forward, d2h) event pairs
    takes = [None, None]
    kinds = [None] * len(todo)

    def channels_of(b):
        ks = set(k for p in b for k in p.channels)
        return ks.pop() if len(ks) == 1 else 3

    def decode_one(p, j, s, i, k):
        t0 = time.perf_counter()
        path = (p.img0, p.img1)[j]
        a = frame_as(read_image(path), k)
        if a.shape[:2] != (H, W):
            raise RunError("%s: %s decodes to %dx%d, its header says %dx%d" % (p.where, path, a.shape[1], a.shape[0], W, H))
        o = j * px * k + i * H * W * k                             # frames of img0, then of img1, each [B][H][W][k]
        pin[s][o:o + H * W * k].numpy()[:] = a.reshape(-1)
        return time.perf_counter() - t0

    def read_one(p, s, i):
        t0 = time.perf_counter()
        o = pay_off + i * pay_one
        sink.read_payload(p, pin[s][o:o + pay_one].numpy())
        return time.perf_counter() - t0

    def decode(k_batch):
        s = k_batch & 1
        b = todo[k_batch][0]
        kinds[k_batch] = channels_of(b)
        ev_h2d[s].synchronize()                                    # the copy out of pin[s] two batches ago is done
        futs = [pool.submit(decode_one, p, j, s, i, kinds[k_batch]) for i, p in enumerate(b) for j in (0, 1)]
        if pay_bytes:
            futs += [pool.submit(read_one, p, s, i) for i, p in enumerate(b)]
        return futs

    def take(k_batch, s, n_real):
        ev_d2h[s].synchronize()
        sink.take(todo[k_batch][0], s, n_real)

    decoding = decode(0)
    with ThreadPoolExecutor(max_workers=1) as taker:
        for kb, (b, n_real) in enumerate(todo):
            s, k = kb & 1, kinds[kb]
            stats["decode"] += sum(f.result() for f in decoding)
            t = [ev() for _ in range(6)]
            with torch.cuda.stream(h2d_stream):
                h2d_stream.wait_event(ev_used[s])                  # dev[s] was converted two batches ago
                t[0].record(h2d_stream)
                dev[s][:2 * px * k].copy_(pin[s][:2 * px * k], non_blocking=True)
                if pay_bytes:
                    dev[s][pay_off:].copy_(pin[s][pay_off:], non_blocking=True)
                t[1].record(h2d_stream)
                ev_h2d[s].record(h2d_stream)
            if kb + 1 < len(todo):
                decoding = decode(kb + 1)                          # batch k+1 decodes while batch k runs
            with torch.cuda.stream(net_stream):
                net_stream.wait_event(ev_h2d[s])
                t[2].record(net_stream)
                net.set_input_image_device(in0, dev[s].data_ptr(), k)
                net.set_input_image_device(in1, dev[s].data_ptr() + px * k, k)
                if pay_bytes:
                    sink.stage(b, s, dev[s][pay_off:], pay_one)
                ev_used[s].record(net_stream)
                net.forward_async()
                net_stream.wait_event(ev_d2h[s])                   # sink.dev[s] has left for the host two batches ago
                net.get_blob_nhwc_device("predict_flow_final", flow_dev[s].data_ptr())
                sink.score(s)
                t[3].record(net_stream)
                ev_flow[s].record(net_stream)
            if takes[s] is not None:
                takes[s].result()                                  # sink.host[s] taken two batches ago
            with torch.cuda.stream(d2h_stream):
                d2h_stream.wait_event(ev_flow[s])
                t[4].record(d2h_stream)
                sink.host[s].copy_(sink.dev[s], non_blocking=True)
                t[5].record(d2h_stream)
                ev_d2h[s].record(d2h_stream)
            timing.append(t)
            takes[s] = taker.submit(take, kb, s, n_real)
        for w in takes:
            if w is not None:
                w.result()
    torch.cuda.synchronize()
    for t in timing:
        stats["h2d"] += t[0].elapsed_time(t[1]) * 1e-3
        stats["forward"] += t[2].elapsed_time(t[3]) * 1e-3
        stats["d2h"] += t[4].elapsed_time(t[5]) * 1e-3


def check_inputs(caffemodel, template, batch):
    """Refuses a batch below 1 and a missing caffemodel or template, before anything is read."""
    if batch < 1:
        raise RunError("--batch must be at least 1, got %d" % batch)
    for path, what in ((caffemodel, "caffemodel"), (template, "deploy prototxt template")):
        if not os.path.isfile(path):
            raise RunError("%s: no such %s" % (path, what))


def run_groups(caffemodel, template, pairs, batch, device, threads, sink, t0):
    """The pipeline of run and evaluate over probed pairs (probe_pairs): one net per frame size, the weights read once, each
    size's batches through _group_batches into `sink` -> (per-stage busy seconds, number of sizes).  The build time counts
    from t0, when the caller started checking its inputs."""
    import torch
    import flownet2_b200 as F
    torch.cuda.set_device(device)
    stats = {k: 0.0 for k in ("build", "decode", "h2d", "forward", "d2h")}
    stats.update(sink.stats)
    with open(template) as f:
        text = f.read()
    with open(caffemodel, "rb") as f:
        weights = f.read()
    stats["build"] += time.perf_counter() - t0
    groups = group_by_size(pairs)
    with ThreadPoolExecutor(max_workers=threads or min(16, os.cpu_count() or 4)) as pool:
        for size, group in groups:
            tb = time.perf_counter()
            net = F.Net(F.fill_template(text, size[0], size[1]), weights, F.TEST, batch=batch)
            stats["build"] += time.perf_counter() - tb
            try:
                _group_batches(torch, net, size, group, batch, pool, stats, sink)
            finally:
                del net
                gc.collect()                                       # the net's blob views refer back to it: free it now
                torch.cuda.empty_cache()
    stats.update(sink.stats)
    return stats, len(groups)


def run(caffemodel, template, pairs, batch=1, device=0, threads=None, kitti=False):
    """Flow of every Pair into its .flo file (kitti: its KITTI flow PNG) -> summary dict: pairs, sizes, nets, wall (s),
    per-stage busy seconds (build: checking the inputs, reading the weights and constructing the nets; decode: host, summed
    over the pool's threads; h2d / forward / d2h: device; write: host) and the pairs whose flow is not finite."""
    t0 = time.perf_counter()
    check_inputs(caffemodel, template, batch)
    probe_pairs(pairs)
    sink = KittiFiles() if kitti else FlowFiles()
    stats, sizes = run_groups(caffemodel, template, pairs, batch, device, threads, sink, t0)
    return {"pairs": len(pairs), "sizes": sizes, "nets": sizes, "batch": batch, "wall": time.perf_counter() - t0,
            "busy": stats, "not_finite": [p.where for p in sink.bad]}


def parse_args(argv):
    ap = argparse.ArgumentParser(prog="python -m flownet2_b200.run", description=__doc__.split("\n\n")[0])
    ap.add_argument("caffemodel", help="weights: .caffemodel or .caffemodel.h5")
    ap.add_argument("deployproto", help="deploy prototxt template, e.g. models/FlowNet2_deploy.prototxt.template")
    ap.add_argument("files", nargs="+", metavar="img0 img1 out | listfile",
                    help="one pair (img0 img1 out.flo) or a list file of such lines")
    ap.add_argument("--gpu", type=int, default=0, help="device to use without torchrun")
    ap.add_argument("--verbose", action="store_true", help="accepted for compatibility; the engine does not log")
    ap.add_argument("--batch", type=int, default=1, help="pairs per forward (outputs bit-identical to single pairs only at 1)")
    ap.add_argument("--kitti", action="store_true", help="write each output as a KITTI 16-bit flow PNG instead of a .flo")
    a = ap.parse_args(argv)
    if len(a.files) not in (1, 3):
        ap.error("expected img0 img1 out, or one list file; got %d paths" % len(a.files))
    return a


def main(argv=None):
    a = parse_args(sys.argv[1:] if argv is None else argv)
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    device = int(os.environ.get("LOCAL_RANK", a.gpu)) if "WORLD_SIZE" in os.environ else a.gpu
    try:
        pairs = read_list(a.files[0]) if len(a.files) == 1 else [Pair("command line", *a.files)]
        s = run(a.caffemodel, a.deployproto, shard(pairs, world, rank), batch=a.batch, device=device, kitti=a.kitti)
    except RunError as e:
        sys.stderr.write("error: %s\n" % e)
        return 2
    tag = "rank %d/%d: " % (rank, world) if world > 1 else ""
    print("%s%d pairs, %d sizes, %d nets built, %.2f s" % (tag, s["pairs"], s["sizes"], s["nets"], s["wall"]), flush=True)
    return 1 if s["not_finite"] else 0


if __name__ == "__main__":
    sys.exit(main())
