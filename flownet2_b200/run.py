"""Optical flow of image files: the command line of the reference's scripts/run-flownet.py and run-flownet-many.py.

    python -m flownet2_b200.run weights.caffemodel models/FlowNet2_deploy.prototxt.template img0.png img1.png out.flo
    python -m flownet2_b200.run weights.caffemodel models/FlowNet2_deploy.prototxt.template pairs.txt [--batch 4] [--kitti]
                                [--visualize [--max-flow F]] [--backward [--fb-alpha1 A] [--fb-alpha2 B]]

The list file holds one ``img0 img1 out.flo`` line per pair; blank lines are skipped.  The weights (.caffemodel or
.caffemodel.h5) are read once.  Pairs are grouped by frame size in order of first appearance, and each size gets one
Net(fill_template(template, W, H), weights, TEST, batch=B); at most one net is alive at a time.  Every forward runs B pairs;
the last batch of a size is padded by repeating its last pair, and the extra outputs are dropped.

Frames are PPM / PGM (P6 / P5, maxval 255) or anything Pillow reads, converted the way scipy.misc.imread hands them to the
reference (palette to RGB or RGBA, LA to L; flownet2_b200.files, which probes every frame before a net is built).  The
8-bit frames are copied to the device as they are and converted there (fn2_net_set_input_frames_device), and the flow comes
back as (H, W, 2), the payload order of .flo (fn2_net_get_blob_nhwc_device).  The batches ahead are read on a thread pool
into two pinned slots and copied to the device on a copy stream (flownet2_b200.feed) while batch k runs, and batch k-1's flow
is copied back on another stream and written by a writer thread.

--visualize also writes, beside each output, <output without its extension>.vis.png: the flow colour-coded on the net's stream
(fn2_flow_to_color_png_rows, the Middlebury colour wheel scaled by the pair's largest known flow, or by --max-flow F), coming
back in the same copy as the flow and deflated by the writer thread (flownet2_b200.viz).  It shows the net's float prediction,
also under --kitti; a pixel whose flow is not finite is black.  A list in which two outputs map to one .vis.png, or a
.vis.png is another line's output, is refused.

--backward also runs the net on every pair with its frames exchanged, at the same batch on the same net (the feeder converts
each batch's frames a second time, flownet2_b200.feed), and writes two more files beside each output:
<output without its extension>.bwd<extension>, the backward flow in the output's format, and <output without its
extension>.occ.png, frame 0's occlusion mask as an 8-bit grey PNG (255 occluded, 0 visible; Sintel's convention).  The mask
is the forward-backward consistency check of Sundaram, Brox and Keutzer (ECCV 2010) on the two flows, computed on the net's
stream (fn2_flow_fb_occlusion, include/fn2_flow.h, which states the arithmetic), with alpha1 = --fb-alpha1 (0.01) and
alpha2 = --fb-alpha2 (0.5).  Its scanlines come back in the batch's one copy with the flows and the writer thread deflates
them.  The forward outputs are the files run writes without the flag, and each .bwd file is the output run writes for the
pair with its frames exchanged, bit for bit at the same --batch.  Every derived path (.vis.png, .bwd, .occ.png) is checked
against every output and every other derived path before a net is built.

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
import functools
import gc
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .feed import Feeder, _align
from .files import Pair, RunError, probe, read_list, write_flo
# the frame helpers this module held before flownet2_b200.files, still importable from here
from .files import check_frame, frame_as, probe_image, read_image, write_pnm  # noqa: F401


# ------------------------------------------------------------------------------------------------
# Sizes, batches, shards
# ------------------------------------------------------------------------------------------------
def shard(items, world, rank):
    """The items i with i % world == rank: frame-pair sharding over the ranks."""
    return [p for i, p in enumerate(items) if i % world == rank]


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


# ------------------------------------------------------------------------------------------------
# The sinks
# ------------------------------------------------------------------------------------------------
class FlowFiles(object):
    """run's per-batch sink: each pair's flow goes to the host and into its .flo file; a pair whose flow is not finite is named
    on stderr and kept in `bad`.

    The sink interface of _run_size: item_bytes(H, W) the pinned payload bytes per pair the feeder reads (each pair's
    flow file, flownet2_b200.feed), stage(pairs, s, payload, stride) the net stream's use of them before the forward (None
    without a payload); bind(...) allocates dev[s] / host[s] for one frame size (and may replace flow_dev[s] by a view into
    dev[s]), score(s) runs on the net's stream after the flow is in flow_dev[s] and fills dev[s], which then goes to host[s]
    on the copy-back stream, and take(pairs, s, n_real) consumes host[s] on the writer thread.

    visualize: each batch's flow is also colour-coded into PNG scanlines at the end of dev[s] (fn2_flow_to_color_png_rows, at
    the fixed scale max_flow, else at each pair's own largest radius), and take() writes each pair's vis_path(flow).

    backward (alphas: alpha1, alpha2): _run_size also fills bwd_dev[s] with the flow of the exchanged frames; score() turns the
    two flows into frame 0's occlusion mask as 8-bit grey PNG scanlines in dev[s] (fn2_flow_fb_occlusion), and take() writes
    each pair's bwd_path(flow) and occ_path(flow)."""

    def __init__(self, visualize=False, max_flow=None, backward=False, alphas=(0.01, 0.5)):
        self.bad = []
        self.stats = {"write": 0.0}
        self.visualize, self.max_flow = visualize, max_flow
        self.backward, self.alphas = backward, alphas

    def item_bytes(self, H, W):
        return 0

    stage = None

    def bind(self, torch, batch, H, W, flow_dev, bwd_dev=None):
        if not (self.visualize or self.backward):
            self.dev = flow_dev
            self.host = [torch.empty((batch, H, W, 2)).pin_memory() for _ in range(2)]
            return
        self.flow_bytes = batch * H * W * 8                               # the flow, then with backward the backward flow
        nb = self.flow_bytes * (2 if self.backward else 1)
        if self.backward:
            nb = self._bind_occ(batch, H, W, nb)
        if self.visualize:
            nb = self._bind_vis(torch, batch, H, W, flow_dev, nb)
        self.dev = [torch.empty(nb, dtype=torch.uint8, device="cuda") for _ in range(2)]
        self.host = [torch.empty(nb, dtype=torch.uint8).pin_memory() for _ in range(2)]
        flows = lambda s, k: self.dev[s][k * self.flow_bytes:(k + 1) * self.flow_bytes].view(torch.float32).view(batch, H, W, 2)
        for s in range(2):                                                # the net writes its flows straight into dev[s]
            flow_dev[s] = flows(s, 0)
            if self.backward:
                bwd_dev[s] = flows(s, 1)
        self.pred = [f.permute(0, 3, 1, 2) for f in flow_dev]
        if self.backward:
            self._zero_occ(bwd_dev)

    def _bind_occ(self, batch, H, W, offset):
        """The mask rows' place in dev[s], from `offset` on -> the offset after them."""
        from . import ops
        self.ops, self.size, self.occ_off, self.occ_bytes = ops, (W, H), offset, H * (1 + W)
        return offset + batch * self.occ_bytes

    def _zero_occ(self, bwd_dev):
        """Zeroes the mask rows of both dev[s] once: the check writes each row from byte 1 on, so every filter byte stays 0
        (None)."""
        self.bwd = [b.permute(0, 3, 1, 2) for b in bwd_dev]               # (B, 2, H, W) views of the NHWC backward flow
        for d in self.dev:
            d[self.occ_off:self.occ_off + len(bwd_dev[0]) * self.occ_bytes].zero_()

    def _score_occ(self, s):
        W, H = self.size
        self.ops.flow_fb_occlusion(self.pred[s], self.bwd[s], *self.alphas, out=self.dev[s][self.occ_off + 1:],
                                   row_stride=1 + W, pair_stride=self.occ_bytes)

    def _take_occ(self, buf, i, p):
        from . import kitti
        n, o = self.occ_bytes, self.occ_off
        kitti.write_png_rows(occ_path(p.flow), buf[o + i * n:o + (i + 1) * n], *self.size, 8, 1)

    def _bind_vis(self, torch, batch, H, W, flow_dev, offset):
        """The colour rows' place in dev[s], from `offset` on -> dev[s]'s size."""
        from . import ops
        self.ops, self.size = ops, (W, H)
        self.pred = [f.permute(0, 3, 1, 2) for f in flow_dev]             # (B, 2, H, W) views of the NHWC flow
        self.vis_off, self.vis_bytes = _align(offset, 16), H * (1 + 3 * W)
        self.radius = [torch.empty(batch, device="cuda") for _ in range(2)]
        return self.vis_off + batch * self.vis_bytes

    def _score_vis(self, s):
        radius = None if self.max_flow is not None else self.ops.flow_max_radius(self.pred[s], self.radius[s])
        self.ops.flow_to_color_png_rows(self.pred[s], self.dev[s][self.vis_off:], self.max_flow, max_radius=radius)

    def _take_vis(self, buf, i, p):
        from . import kitti
        n, o = self.vis_bytes, self.vis_off
        kitti.write_png_rows(vis_path(p.flow), buf[o + i * n:o + (i + 1) * n], *self.size, 8)

    def score(self, s):
        if self.backward:
            self._score_occ(s)
        if self.visualize:
            self._score_vis(s)

    def take(self, pairs, s, n_real):
        t0 = time.perf_counter()
        buf = self.host[s].numpy()
        if self.visualize or self.backward:
            flows = buf[:self.flow_bytes * (2 if self.backward else 1)].view(np.float32).reshape(-1, len(pairs), self.size[1],
                                                                                                  self.size[0], 2)
        else:
            flows = buf[None]
        for i, p in enumerate(pairs[:n_real]):
            if not np.isfinite(flows[0, i]).all():
                self.bad.append(p)
                sys.stderr.write("%s: the flow of %s %s is not finite\n" % (p.where, p.img0, p.img1))
            write_flo(p.flow, flows[0, i])
            if self.backward:
                write_flo(bwd_path(p.flow), flows[1, i])
                self._take_occ(buf, i, p)
            if self.visualize:
                self._take_vis(buf, i, p)
        self.stats["write"] += time.perf_counter() - t0


class KittiFiles(FlowFiles):
    """run --kitti's sink: on the net's stream each batch's flow becomes KITTI PNG scanlines (fn2_flow_to_kitti_png_rows) and
    fn2_flow_error against a zero flow counts each pair's non-finite pixels; both come back in one copy, and the writer
    thread deflates each pair's rows into its file.  A pair with a non-finite pixel is named on stderr and kept in `bad`.
    With backward the backward flow's scanlines follow the flow's, and the mask rows the records."""

    def bind(self, torch, batch, H, W, flow_dev, bwd_dev=None):
        from . import FLOW_ERROR_FIELDS, kitti, ops
        self.ops, self.kitti, self.size = ops, kitti, (W, H)
        self.nonfinite, fields = FLOW_ERROR_FIELDS.index("nonfinite"), len(FLOW_ERROR_FIELDS)
        self.row_bytes = H * (1 + kitti.BPP * W)                          # one pair's scanlines
        self.rec_off = _align(batch * self.row_bytes * (2 if self.backward else 1), 8)   # then the pairs' float64 records
        nb = self.rec_off + batch * fields * 8
        if self.backward:                                                 # then the mask rows
            nb = self._bind_occ(batch, H, W, nb)
        if self.visualize:                                                # then the colour rows
            nb = self._bind_vis(torch, batch, H, W, flow_dev, nb)
        self.pred = [f.permute(0, 3, 1, 2) for f in flow_dev]             # (B, 2, H, W) views of the NHWC flow
        self.dev = [torch.empty(nb, dtype=torch.uint8, device="cuda") for _ in range(2)]
        if self.backward:
            self._zero_occ(bwd_dev)
        self.host = [torch.empty(nb, dtype=torch.uint8).pin_memory() for _ in range(2)]
        self.records = [d[self.rec_off:self.rec_off + batch * fields * 8].view(torch.float64).view(batch, fields)
                        for d in self.dev]
        self.zero = torch.zeros((batch, 2, H, W), device="cuda")
        self.workspace = torch.empty(max(ops.flow_error_workspace_bytes(batch, H, W), 8), dtype=torch.uint8, device="cuda")

    def score(self, s):
        self.ops.flow_to_kitti_png_rows(self.pred[s], self.dev[s])
        self.ops.flow_error(self.pred[s], self.zero, out=self.records[s], workspace=self.workspace)
        if self.backward:
            B = len(self.zero)
            self.ops.flow_to_kitti_png_rows(self.bwd[s], self.dev[s][B * self.row_bytes:2 * B * self.row_bytes])
            self._score_occ(s)
        if self.visualize:
            self._score_vis(s)

    def take(self, pairs, s, n_real):
        t0 = time.perf_counter()
        buf = self.host[s].numpy()
        rec = buf[self.rec_off:self.rec_off + len(pairs) * len(self.records[s][0]) * 8].view(np.float64).reshape(len(pairs), -1)
        n = self.row_bytes
        for i, p in enumerate(pairs[:n_real]):
            if rec[i, self.nonfinite] > 0:
                self.bad.append(p)
                sys.stderr.write("%s: the flow of %s %s is not finite\n" % (p.where, p.img0, p.img1))
            self.kitti.write_png_rows(p.flow, buf[i * n:(i + 1) * n], *self.size)
            if self.backward:
                b = len(pairs) * n
                self.kitti.write_png_rows(bwd_path(p.flow), buf[b + i * n:b + (i + 1) * n], *self.size)
                self._take_occ(buf, i, p)
            if self.visualize:
                self._take_vis(buf, i, p)
        self.stats["write"] += time.perf_counter() - t0


def vis_path(out):
    """The colour-coded image run --visualize writes beside the output `out`: out without its extension, then .vis.png."""
    return os.path.splitext(out)[0] + ".vis.png"


def bwd_path(out):
    """The backward flow run --backward writes beside the output `out`: out without its extension, .bwd, then the extension."""
    root, ext = os.path.splitext(out)
    return root + ".bwd" + ext


def occ_path(out):
    """Frame 0's occlusion mask run --backward writes beside the output `out`: out without its extension, then .occ.png."""
    return os.path.splitext(out)[0] + ".occ.png"


# what each derived path is, in the refusals of check_vis_paths
DERIVED = {vis_path: ("visualisation", "visualise to"), bwd_path: ("backward flow", "have the backward flow"),
           occ_path: ("occlusion mask", "have the occlusion mask")}


def check_vis_paths(pairs, derived=(vis_path,)):
    """Refuses a list in which two different outputs have one derived path (each function of `derived` maps an output to one
    of the files written beside it), or a derived path is an output, naming the lines."""
    outs = {os.path.normpath(p.flow): p for p in pairs}
    seen = {}
    for p in pairs:
        out = os.path.normpath(p.flow)
        for f in derived:
            what, verb = DERIVED[f]
            v = os.path.normpath(f(p.flow))
            if v in seen and os.path.normpath(seen[v].flow) != out:
                raise RunError("%s: the outputs %s and %s (%s) both %s %s" % (p.where, p.flow, seen[v].flow, seen[v].where, verb,
                                                                          f(p.flow)))
            if v in outs:
                raise RunError("%s: the %s %s of %s is the output of %s" % (p.where, what, f(p.flow), p.flow, outs[v].where))
            seen[v] = p


def derived_paths(visualize, backward):
    """The functions of the files run writes beside each output, for check_vis_paths."""
    return ((vis_path,) if visualize else ()) + ((bwd_path, occ_path) if backward else ())


def check_fb_alphas(alpha1, alpha2):
    """Refuses forward-backward thresholds that are negative or not finite."""
    for name, a in (("--fb-alpha1", alpha1), ("--fb-alpha2", alpha2)):
        if not (np.isfinite(a) and a >= 0):
            raise RunError("%s must be a finite non-negative number, got %r" % (name, a))


def check_max_flow(max_flow):
    """Refuses a --max-flow that is not a finite positive number; None passes."""
    if max_flow is not None and not (max_flow > 0 and np.isfinite(max_flow)):
        raise RunError("--max-flow must be a finite positive number, got %r" % max_flow)


def _run_size(torch, net, size, pairs, batch, threads, stats, sink):
    """Runs one size's pairs through `net`, B per forward, with reads, copies, forward and the sink's work overlapped."""
    W, H = size
    todo = batches(pairs, batch)
    both = sink.backward                                           # also the flow of the exchanged frames, into bwd_dev[s]
    flow_dev = [torch.empty((batch, H, W, 2), device="cuda") for _ in range(2)]
    bwd_dev = [torch.empty((batch, H, W, 2), device="cuda") for _ in range(2)] if both else None
    sink.bind(torch, batch, H, W, flow_dev, bwd_dev)
    feed = Feeder(net, batch, size, sink.item_bytes(H, W), lambda k: todo[k][0] if k < len(todo) else None, 2, threads,
                  swap=both)
    net_stream, d2h_stream = feed.stream, torch.cuda.Stream()
    ev = lambda: torch.cuda.Event(enable_timing=True)
    ev_flow = [torch.cuda.Event() for _ in range(2)]               # sink.dev[s] holds the batch's result
    ev_d2h = [torch.cuda.Event() for _ in range(2)]                # sink.host[s] holds it
    timing = []                                                    # per batch: (forward, d2h) event pairs
    takes = [None, None]

    def take(k_batch, s, n_real):
        ev_d2h[s].synchronize()
        sink.take(todo[k_batch][0], s, n_real)

    try:
        feed.seek(0)
        with ThreadPoolExecutor(max_workers=1) as taker:
            for kb, (b, n_real) in enumerate(todo):
                s = kb & 1
                feed(functools.partial(sink.stage, b, s) if sink.stage else None)     # batch kb + 2 starts reading
                t = [ev() for _ in range(4)]
                with torch.cuda.stream(net_stream):
                    t[0].record(net_stream)
                    net.forward_async()
                    net_stream.wait_event(ev_d2h[s])               # sink.dev[s] has left for the host two batches ago
                    net.get_blob_nhwc_device("predict_flow_final", flow_dev[s].data_ptr())
                    if both:
                        feed.swap()                                # the same frames, img1 first; frees the feeder's slot
                        net.forward_async()
                        net.get_blob_nhwc_device("predict_flow_final", bwd_dev[s].data_ptr())
                    sink.score(s)
                    t[1].record(net_stream)
                    ev_flow[s].record(net_stream)
                if takes[s] is not None:
                    takes[s].result()                              # sink.host[s] taken two batches ago
                with torch.cuda.stream(d2h_stream):
                    d2h_stream.wait_event(ev_flow[s])
                    t[2].record(d2h_stream)
                    sink.host[s].copy_(sink.dev[s], non_blocking=True)
                    t[3].record(d2h_stream)
                    ev_d2h[s].record(d2h_stream)
                timing.append(t)
                takes[s] = taker.submit(take, kb, s, n_real)
            for w in takes:
                if w is not None:
                    w.result()
        busy = feed.busy()
    finally:
        feed.close()
    torch.cuda.synchronize()
    stats["decode"] += busy["read"]
    stats["h2d"] += busy["h2d"]
    stats["forward"] += busy["convert"]                            # the frames' conversion and the sink's stage
    for t in timing:
        stats["forward"] += t[0].elapsed_time(t[1]) * 1e-3
        stats["d2h"] += t[2].elapsed_time(t[3]) * 1e-3


def check_inputs(caffemodel, template, batch):
    """Refuses a batch below 1 and a missing caffemodel or template, before anything is read."""
    if batch < 1:
        raise RunError("--batch must be at least 1, got %d" % batch)
    for path, what in ((caffemodel, "caffemodel"), (template, "deploy prototxt template")):
        if not os.path.isfile(path):
            raise RunError("%s: no such %s" % (path, what))


STAGES = ("build", "decode", "h2d", "forward", "d2h")                 # the busy seconds of run_groups, in this order


def run_groups(caffemodel, template, pairs, batch, device, threads, sink, t0):
    """The pipeline of run and evaluate over probed pairs (files.probe): one net per frame size, the weights read once, each
    size's batches through _run_size into `sink` -> (per-stage busy seconds, number of sizes).  The build time counts
    from t0, when the caller started checking its inputs."""
    import torch
    import flownet2_b200 as F
    torch.cuda.set_device(device)
    stats = dict.fromkeys(STAGES, 0.0)
    stats.update(sink.stats)
    with open(template) as f:
        text = f.read()
    with open(caffemodel, "rb") as f:
        weights = f.read()
    stats["build"] += time.perf_counter() - t0
    groups = group_by_size(pairs)
    for size, group in groups:
        tb = time.perf_counter()
        net = F.Net(F.fill_template(text, size[0], size[1]), weights, F.TEST, batch=batch)
        stats["build"] += time.perf_counter() - tb
        try:
            _run_size(torch, net, size, group, batch, threads, stats, sink)
        finally:
            del net
            gc.collect()                                           # the net's blob views refer back to it: free it now
            torch.cuda.empty_cache()
    stats.update(sink.stats)
    return stats, len(groups)


def run(caffemodel, template, pairs, batch=1, device=0, threads=None, kitti=False, visualize=False, max_flow=None,
        backward=False, fb_alpha1=0.01, fb_alpha2=0.5):
    """Flow of every files.Pair into its flow file, a .flo (kitti: a KITTI flow PNG) -> summary dict: pairs, sizes, nets, wall (s),
    per-stage busy seconds (build: checking the inputs, reading the weights and constructing the nets; decode: host, summed
    over the pool's threads; h2d / forward / d2h: device; write: host) and the pairs whose flow is not finite.  visualize:
    also each flow colour-coded into vis_path(flow), at the fixed scale max_flow if given.  backward: also the flow of the
    exchanged frames into bwd_path(flow) and frame 0's forward-backward occlusion mask (thresholds fb_alpha1, fb_alpha2)
    into occ_path(flow)."""
    t0 = time.perf_counter()
    check_fb_alphas(fb_alpha1, fb_alpha2)
    check_inputs(caffemodel, template, batch)
    check_max_flow(max_flow)
    probe(pairs)
    if visualize or backward:
        check_vis_paths(pairs, derived_paths(visualize, backward))
    sink = (KittiFiles if kitti else FlowFiles)(visualize, max_flow, backward, (fb_alpha1, fb_alpha2))
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
    ap.add_argument("--visualize", action="store_true", help="also write each flow colour-coded, as <output>.vis.png")
    ap.add_argument("--max-flow", type=float, metavar="F", help="with --visualize: colour every flow at this scale (pixels) "
                                                                "instead of each pair's largest flow")
    ap.add_argument("--backward", action="store_true", help="also write the backward flow, as <output>.bwd<ext>, and frame 0's "
                                                            "forward-backward occlusion mask, as <output>.occ.png")
    ap.add_argument("--fb-alpha1", type=float, default=0.01, metavar="A", help="with --backward: the check's relative term "
                                                                               "(default 0.01)")
    ap.add_argument("--fb-alpha2", type=float, default=0.5, metavar="B", help="with --backward: the check's constant term, in "
                                                                              "squared pixels (default 0.5)")
    a = ap.parse_args(argv)
    if len(a.files) not in (1, 3):
        ap.error("expected img0 img1 out, or one list file; got %d paths" % len(a.files))
    return a


def main(argv=None):
    a = parse_args(sys.argv[1:] if argv is None else argv)
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    device = int(os.environ.get("LOCAL_RANK", a.gpu)) if "WORLD_SIZE" in os.environ else a.gpu
    try:
        check_max_flow(a.max_flow)
        check_fb_alphas(a.fb_alpha1, a.fb_alpha2)
        pairs = read_list(a.files[0], ground_truth=False) if len(a.files) == 1 else [Pair("command line", *a.files)]
        if a.visualize or a.backward:
            check_vis_paths(pairs, derived_paths(a.visualize, a.backward))     # the whole list: ranks must not collide either
        s = run(a.caffemodel, a.deployproto, shard(pairs, world, rank), batch=a.batch, device=device, kitti=a.kitti,
                visualize=a.visualize, max_flow=a.max_flow, backward=a.backward, fb_alpha1=a.fb_alpha1,
                fb_alpha2=a.fb_alpha2)
    except RunError as e:
        sys.stderr.write("error: %s\n" % e)
        return 2
    tag = "rank %d/%d: " % (rank, world) if world > 1 else ""
    print("%s%d pairs, %d sizes, %d nets built, %.2f s" % (tag, s["pairs"], s["sizes"], s["nets"], s["wall"]), flush=True)
    return 1 if s["not_finite"] else 0


if __name__ == "__main__":
    sys.exit(main())
