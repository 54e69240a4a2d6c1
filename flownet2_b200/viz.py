"""Flow as a picture: the Middlebury colour code (include/fn2_flow.h) drawn on the device and written as 8-bit RGB PNGs.

    python -m flownet2_b200.viz FLOW OUT.png [--max-flow F] [--kitti]
    python -m flownet2_b200.viz LIST [--max-flow F] [--kitti] [--batch N]

    write_flow_png(path, flow_hw2, max_flow=None)          # a float (H, W, 2) numpy flow -> one PNG

The hue is the flow's direction, the saturation its length over the scale: each image's largest flow over its known pixels
(both components finite and at most 1e9), or --max-flow F for every image (a constant scale across a video).  Unknown pixels
are black.  run --visualize and evaluate --visualize draw the same images from their own pipelines.

A LIST holds one ``flow out.png`` line per image, blank lines skipped.  Flows are .flo or 'PF' PFM of either byte order, or,
with --kitti, KITTI 16-bit PNGs; every flow is probed before any device work.  The flows are grouped by size in order of
first appearance and run N at a time through the pinned-slot feeder (flownet2_b200.feed, without a net): the reader pool
reads each payload into a slot, the copy stream moves it to the device, and on the feeder's stream fn2_flow_to_tensor
decodes it, fn2_flow_max_radius finds each image's scale and fn2_flow_to_color_png_rows draws Paeth-filtered scanlines.  The
scanlines come back in one copy per batch and a writer thread deflates them (flownet2_b200.kitti.write_png_rows).  A refused
input is named on stderr with exit status 2.
"""
import argparse
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .feed import Feeder, _align, mask_offset
from .files import Pair, RunError, flow_header
from .run import batches, check_max_flow, group_by_size


def write_flow_png(path, flow_hw2, max_flow=None):
    """A float (H, W, 2) flow (numpy) colour-coded on the device into an 8-bit RGB PNG at `path`: scaled by max_flow, else by its
    largest known flow."""
    import torch
    from . import kitti, ops
    f = np.asarray(flow_hw2, np.float32)
    assert f.ndim == 3 and f.shape[2] == 2, f.shape
    check_max_flow(max_flow)
    dev = torch.from_numpy(np.ascontiguousarray(f)).cuda()[None].permute(0, 3, 1, 2)
    rows = ops.flow_to_color_png_rows(dev, max_flow=max_flow).cpu().numpy()
    return kitti.write_png_rows(path, rows, f.shape[1], f.shape[0], 8)


def read_viz_list(path):
    """-> [Pair] of a LIST file: one ``flow out.png`` line per image (the Pair's flow is the input, `out` the PNG)."""
    if not os.path.isfile(path):
        raise RunError("%s: no such list file" % path)
    out = []
    with open(path) as f:
        for no, line in enumerate(f, 1):
            fields = line.split()
            if not fields:
                continue
            if len(fields) != 2:
                raise RunError("%s:%d: %d fields, expected 'flow out.png'" % (path, no, len(fields)))
            p = Pair("%s:%d" % (path, no), None, None, fields[0])
            p.out = fields[1]
            out.append(p)
    return out


def probe_flows(items, kitti=False):
    """Reads every flow's header (kitti: as a KITTI PNG) into flow_header and its size; a refusal names the line."""
    if kitti:
        from . import kitti as kitti_png
    for p in items:
        try:
            p.flow_header = kitti_png.probe(p.flow) if kitti else flow_header(p.flow)
        except RunError as e:
            raise RunError("%s: %s" % (p.where, e))
        p.size = (p.flow_header.width, p.flow_header.height)


def _colour_size(torch, size, items, batch, max_flow, threads, stats):
    """One size's flows through the feeder, `batch` per step, into their PNGs."""
    from . import kitti, ops
    W, H = size
    todo = batches(items, batch)
    stride = _align(mask_offset(H, W))                               # holds a payload of any format
    flow = [torch.empty((batch, 2, H, W), device="cuda") for _ in range(2)]
    radius = [torch.empty(batch, device="cuda") for _ in range(2)]
    row_bytes = H * (1 + 3 * W)
    dev = [torch.empty(batch * row_bytes, dtype=torch.uint8, device="cuda") for _ in range(2)]
    host = [torch.empty(batch * row_bytes, dtype=torch.uint8).pin_memory() for _ in range(2)]
    ev_rows = [torch.cuda.Event() for _ in range(2)]                 # dev[s] holds the batch's scanlines
    ev_d2h = [torch.cuda.Event() for _ in range(2)]                  # host[s] holds them
    takes = [None, None]

    def stage(pairs, s, payload, item_bytes):
        torch.cuda.current_stream().wait_event(ev_d2h[s])            # dev[s] has left for the host two batches ago
        for i, p in enumerate(pairs):
            fh = p.flow_header
            ops.flow_to_tensor(payload[i * item_bytes:i * item_bytes + fh.nbytes], fh.format, 0, flow[s][i:i + 1])
        r = None if max_flow is not None else ops.flow_max_radius(flow[s], radius[s])
        ops.flow_to_color_png_rows(flow[s], dev[s], max_flow, max_radius=r)

    def take(kb, s, n_real):
        ev_d2h[s].synchronize()
        t0 = time.perf_counter()
        buf = host[s].numpy()
        for i, p in enumerate(todo[kb][0][:n_real]):
            kitti.write_png_rows(p.out, buf[i * row_bytes:(i + 1) * row_bytes], W, H, 8)
        stats["write"] += time.perf_counter() - t0

    feed = Feeder(None, batch, size, stride, lambda k: todo[k][0] if k < len(todo) else None, 2, threads)
    d2h = torch.cuda.Stream()
    try:
        feed.seek(0)
        with ThreadPoolExecutor(max_workers=1) as taker:
            for kb, (b, n_real) in enumerate(todo):
                s = kb & 1
                feed(lambda payload, item_bytes, b=b, s=s: stage(b, s, payload, item_bytes))
                ev_rows[s].record(feed.stream)
                if takes[s] is not None:
                    takes[s].result()                                # host[s] written out two batches ago
                with torch.cuda.stream(d2h):
                    d2h.wait_event(ev_rows[s])
                    host[s].copy_(dev[s], non_blocking=True)
                    ev_d2h[s].record(d2h)
                takes[s] = taker.submit(take, kb, s, n_real)
            for t in takes:
                if t is not None:
                    t.result()
        busy = feed.busy()
    finally:
        feed.close()
    torch.cuda.synchronize()
    stats["read"] += busy["read"]
    stats["device"] += busy["h2d"] + busy["convert"]


def colour_files(items, batch=8, max_flow=None, kitti=False, device=0, threads=None):
    """Every item (a files.Pair whose flow is the input and `out` the PNG to write) colour-coded -> summary dict: images,
    sizes, wall (s) and busy seconds (read: host, summed over the reader threads; device: copies and kernels; write: deflate and
    file writes)."""
    import torch
    t0 = time.perf_counter()
    if batch < 1:
        raise RunError("--batch must be at least 1, got %d" % batch)
    check_max_flow(max_flow)
    probe_flows(items, kitti)
    torch.cuda.set_device(device)
    stats = {"read": 0.0, "device": 0.0, "write": 0.0}
    groups = group_by_size(items)
    for size, group in groups:
        _colour_size(torch, size, group, batch, max_flow, threads, stats)
    return {"images": len(items), "sizes": len(groups), "wall": time.perf_counter() - t0, "busy": stats}


def parse_args(argv):
    ap = argparse.ArgumentParser(prog="python -m flownet2_b200.viz", description=__doc__.split("\n\n")[0])
    ap.add_argument("files", nargs="+", metavar="FLOW OUT.png | LIST", help="one flow and its PNG, or a list of such lines")
    ap.add_argument("--max-flow", type=float, metavar="F", help="colour every flow at this scale (pixels) instead of its own "
                                                                "largest flow")
    ap.add_argument("--kitti", action="store_true", help="the flows are KITTI 16-bit PNGs")
    ap.add_argument("--batch", type=int, default=8, help="flows per device step")
    ap.add_argument("--gpu", type=int, default=0, help="device to use")
    a = ap.parse_args(argv)
    if len(a.files) not in (1, 2):
        ap.error("expected FLOW OUT.png, or one list file; got %d paths" % len(a.files))
    return a


def main(argv=None):
    a = parse_args(sys.argv[1:] if argv is None else argv)
    try:
        check_max_flow(a.max_flow)
        if len(a.files) == 1:
            items = read_viz_list(a.files[0])
        else:
            items = [Pair("command line", None, None, a.files[0])]
            items[0].out = a.files[1]
        s = colour_files(items, batch=a.batch, max_flow=a.max_flow, kitti=a.kitti, device=a.gpu)
    except RunError as e:
        sys.stderr.write("error: %s\n" % e)
        return 2
    print("%d images, %d sizes, %.2f s" % (s["images"], s["sizes"], s["wall"]), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
