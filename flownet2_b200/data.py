"""Training samples from image and flow files: the reference's convert_imageset_and_flow + CustomData path without the LMDB.

    ds = FlowDataset("train.txt", batch=8)              # reads the list, probes every file, fixes the order
    net = Net(fill_train_template(text, 448, 320, *ds.size, 8), None, TRAIN)
    ds.bind(net)                                         # pinned slots, device slots, streams; starts reading ahead
    solver.step(n, ds)                                   # each call enqueues the next batch on the net's stream

The list file holds one ``img0 img1 flow`` line per sample (the converter's format); blank lines are skipped and an occlusion
field is refused.  Frames are whatever flownet2_b200.run reads (PPM / PGM here, anything else through Pillow); flows are .flo
or PFM ('PF' only), one format per list, and every file has one size, as one LMDB has one Datum shape.  With kitti=True every
flow is a KITTI 16-bit PNG (flownet2_b200.kitti): invalid pixels become NaN, which L1Loss, Downsample and LpqLoss leave out.

Order.  CustomData's (custom_data_layer.cpp:28-41, 394-470): the list line i is key i; the keys are optionally permuted with
libstdc++'s std::random_shuffle after std::srand(rand_permute_seed) -- glibc's rand(), restated in Python -- per block of
block_size keys (keeping the reference's off-by-one: a block shuffles [n1, n2 - 1)), before or after the range_start..range_end
cut as rand_permute_order says.  A seed <= 0 uses glibc's initial state (that of srand(1)); the reference uses whatever state
its process has at that point.  The permutation is made once and the item index wraps per item, so a batch can straddle the end
of the sequence.  Rank r of a world of W takes batch k from sequence position (k W + r) B, so world 1 is the reference's own
sequence.  seek(b) moves to batch b of this rank; after Solver.restore the train command seeks to iter * iter_size, so a
resumed run sees what an uninterrupted one would have seen (the reference restarts its sequence at 0 on resume).

Ground truth.  With flow_encoding "uint16" (the default) the flow blob holds what the reference's LMDB hands its net:
trunc(32 v) / 32, NaN for NaN and out-of-range values (include/fn2_flow.h).  "float" passes the file's floats through (for a
KITTI PNG: its exact (R - 32768) / 64).

Pipeline.  Frames and flows are not converted on the host: a thread pool reads the PPM rasters and the flow payloads of the
batches ahead straight into slices of a pinned slot (other image formats decode through Pillow into the slice), the slot goes
to the device on a copy stream, and the net's stream waits for that copy, converts the three inputs on the device
(fn2_net_set_input_frames_device twice, fn2_net_set_input_flow_device once) and records that the slot is free again.  The
step's path never synchronises with the device.  busy() reports the per-stage times.  A KITTI PNG is inflated and unfiltered
by the reader thread into the slot (its raw big-endian samples) and converted by fn2_net_set_input_kitti_flow_device.
"""
import os
import struct
import time
from collections import deque
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import FLOW_FLO, FLOW_PFM, FLOW_PFM_BE, FLOW_UINT16FLOW, image_to_blob, kitti as kitti_png
from .run import RunError, _pnm_header, frame_as, probe_image, read_image

FLO_TAG = 202021.25                        # 'PIEH' read as a little-endian float
ORDERS = ("FIRST_PERMUTE_THEN_RANGE", "FIRST_RANGE_THEN_PERMUTE")
ENCODINGS = ("uint16", "float")


# ------------------------------------------------------------------------------------------------
# The order: glibc rand() and libstdc++ std::random_shuffle
# ------------------------------------------------------------------------------------------------
class GlibcRand(object):
    """glibc's rand() (random_r.c, TYPE_3: x[i] = x[i-3] + x[i-31] mod 2^32, output x >> 1) after srand(seed)."""

    def __init__(self, seed=1):
        seed &= 0xffffffff
        word = seed - (1 << 32) if seed >= 1 << 31 else seed          # srandom_r keeps the seed as an int32_t
        if word == 0:
            word = 1
        r = [word]
        for _ in range(1, 31):
            hi, lo = int(word / 127773), word - int(word / 127773) * 127773     # C division truncates
            word = 16807 * lo - 2836 * hi
            if word < 0:
                word += 2147483647
            r.append(word)
        r = [x & 0xffffffff for x in r]
        self._r = deque(r, maxlen=34)
        for i in range(31, 34):
            self._r.append(r[i - 31])
        for _ in range(310):
            self._next()

    def _next(self):
        v = (self._r[-31] + self._r[-3]) & 0xffffffff
        self._r.append(v)
        return v

    def __call__(self):
        return self._next() >> 1


def random_shuffle(v, lo, hi, rand):
    """std::random_shuffle(v.begin() + lo, v.begin() + hi) of libstdc++: j = rand() % (i + 1) for i = 1 .. n - 1."""
    for i in range(1, hi - lo):
        j = rand() % (i + 1)
        if j != i:
            v[lo + i], v[lo + j] = v[lo + j], v[lo + i]


def permutation(n, rand_permute=False, seed=0, block_size=0, range_start=0, range_end=-1, order=ORDERS[0]):
    """CustomDataLayer's permutation_vector_ over n keys (custom_data_layer.cpp:28-41, 394-470) -> list of keys."""
    if n < 1:
        raise RunError("the list holds no samples")
    if order not in ORDERS:
        raise RunError("rand_permute_order must be one of %s, got %s" % (", ".join(ORDERS), order))
    if block_size < 0:
        raise RunError("block_size must be at least 0, got %d" % block_size)
    rs = min(max(range_start, 0), n - 1)
    re_ = n - 1 if range_end < 0 or range_end >= n else range_end
    if re_ < rs:
        raise RunError("range end %d is before range start %d" % (re_, rs))

    def permute(v):
        s = seed & 0xffffffff
        rand = GlibcRand(s if 0 < s < 1 << 31 else 1)                  # generateRandomPermutation: srand only if seed > 0
        if block_size > 0:
            for b in range((len(v) + block_size - 1) // block_size):
                random_shuffle(v, b * block_size, min((b + 1) * block_size, len(v)) - 1, rand)
        else:
            random_shuffle(v, 0, len(v), rand)

    v = list(range(n))
    if order == ORDERS[1]:
        v = v[rs:re_ + 1]
    if rand_permute:
        permute(v)
    return v if order == ORDERS[1] else v[rs:re_ + 1]


def batch_keys(perm, batch, k, world=1, rank=0):
    """Keys of rank `rank`'s k-th batch: sequence positions (k world + rank) B .. + B - 1, wrapping per item."""
    start = (k * world + rank) * batch
    return [perm[(start + i) % len(perm)] for i in range(batch)]


# ------------------------------------------------------------------------------------------------
# Flow files
# ------------------------------------------------------------------------------------------------
class FlowHeader(object):
    """format (FLOW_FLO / FLOW_PFM / FLOW_PFM_BE), width, height, payload offset and bytes of a flow file."""

    def __init__(self, fmt, w, h, offset, floats_per_pixel):
        self.format, self.width, self.height, self.offset = fmt, w, h, offset
        self.nbytes = w * h * floats_per_pixel * 4


def flow_header(path):
    """Reads a .flo or PFM header without its payload; refuses missing, truncated, mistagged and 'Pf' files."""
    if not os.path.isfile(path):
        raise RunError("%s: no such file" % path)
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        head = f.read(256)
    if path.endswith(".flo"):
        if len(head) < 12:
            raise RunError("%s: truncated .flo header" % path)
        tag, w, h = struct.unpack("<fii", head[:12])
        if tag != FLO_TAG:
            raise RunError("%s: .flo tag is %r, expected 'PIEH' (%.2f)" % (path, head[:4], FLO_TAG))
        if w < 1 or h < 1:
            raise RunError("%s: .flo size %dx%d" % (path, w, h))
        hdr = FlowHeader(FLOW_FLO, w, h, 12, 2)
    elif path.endswith(".pfm"):
        fields, i = [], 0
        while len(fields) < 4:
            while i < len(head) and head[i:i + 1].isspace():
                i += 1
            j = i
            while j < len(head) and not head[j:j + 1].isspace():
                j += 1
            if j == i or j == len(head):
                raise RunError("%s: malformed PFM header" % path)
            fields.append(head[i:j])
            i = j
        if fields[0] == b"Pf":
            raise RunError("%s: a one-channel 'Pf' PFM, a flow needs the three-channel 'PF' kind" % path)
        if fields[0] != b"PF":
            raise RunError("%s: not a PFM file (magic %r)" % (path, fields[0]))
        try:
            w, h, scale = int(fields[1]), int(fields[2]), float(fields[3])
        except ValueError:
            raise RunError("%s: malformed PFM header" % path)
        if w < 1 or h < 1:
            raise RunError("%s: PFM size %dx%d" % (path, w, h))
        # CImg byte-swaps when (scale > 0) differs from a big-endian host: on x86, a positive scale is big-endian
        hdr = FlowHeader(FLOW_PFM_BE if scale > 0 else FLOW_PFM, w, h, i + 1, 3)
    else:
        raise RunError("%s: flows must be .flo or .pfm files" % path)
    if size < hdr.offset + hdr.nbytes:
        raise RunError("%s: truncated payload (%d of %d bytes)" % (path, max(size - hdr.offset, 0), hdr.nbytes))
    return hdr


def read_flow_payload(path, hdr, out):
    """The payload bytes of a flow file, as stored, into the writable buffer `out` (hdr.nbytes long)."""
    with open(path, "rb", buffering=0) as f:
        f.seek(hdr.offset)
        got = f.readinto(out)
    if got != hdr.nbytes:
        raise RunError("%s: truncated payload (%d of %d bytes)" % (path, got, hdr.nbytes))


def read_flow(path):
    """Host reading of a flow file -> float32 (H, W, 2) top-down, as the reference's converter reads it (no quantisation)."""
    hdr = flow_header(path)
    buf = np.empty(hdr.nbytes, np.uint8)
    read_flow_payload(path, hdr, buf)
    if hdr.format == FLOW_FLO:
        return buf.view("<f4").reshape(hdr.height, hdr.width, 2).astype(np.float32)
    a = buf.view(">f4" if hdr.format == FLOW_PFM_BE else "<f4").reshape(hdr.height, hdr.width, 3)
    return a[::-1, :, :2].astype(np.float32)


def write_pfm(path, hw3, big_endian=False):
    """'PF' PFM of a top-down (H, W, 3) float array: rows stored bottom-to-top, scale 1 (big-endian) or -1 (little-endian)."""
    h, w = hw3.shape[:2]
    with open(path, "wb") as f:
        f.write(b"PF\n%d %d\n%s\n" % (w, h, b"1.0" if big_endian else b"-1.0"))
        f.write(np.ascontiguousarray(hw3[::-1], ">f4" if big_endian else "<f4").tobytes())
    return str(path)


# ------------------------------------------------------------------------------------------------
# The list
# ------------------------------------------------------------------------------------------------
class Sample(object):
    def __init__(self, where, img0, img1, flow):
        self.where, self.img0, self.img1, self.flow = where, img0, img1, flow
        self.channels = self.flow_header = None


def read_list(path):
    """-> [Sample] of a list file: one ``img0 img1 flow`` line per sample, blank lines skipped."""
    if not os.path.isfile(path):
        raise RunError("%s: no such list file" % path)
    out = []
    with open(path) as f:
        for no, line in enumerate(f, 1):
            fields = line.split()
            if not fields:
                continue
            if len(fields) == 4:
                raise RunError("%s:%d: an occlusion field (%s); occlusion masks are not supported" % (path, no, fields[3]))
            if len(fields) != 3:
                raise RunError("%s:%d: %d fields, expected 'img0 img1 flow'" % (path, no, len(fields)))
            out.append(Sample("%s:%d" % (path, no), *fields))
    return out


def probe_samples(samples, kitti=False):
    """Probes every frame and flow without decoding pixels -> (width, height, flow format); refuses missing or truncated files,
    bad flow files, mixed flow formats and any file whose size differs from the first sample's.  kitti: every flow is a KITTI
    PNG (kitti.probe)."""
    size = fmt = None
    for s in samples:
        try:
            dims = []
            chans = []
            for p in (s.img0, s.img1):
                w, h, k = probe_image(p)
                with open(p, "rb") as f:
                    hdr = _pnm_header(f, p)
                if hdr is not None and os.path.getsize(p) < hdr[4] + w * h * k:
                    raise RunError("%s: truncated raster (%d of %d bytes)" % (p, os.path.getsize(p) - hdr[4], w * h * k))
                dims.append((p, w, h))
                chans.append(k)
            fh = kitti_png.probe(s.flow) if kitti else flow_header(s.flow)
            dims.append((s.flow, fh.width, fh.height))
        except RunError as e:
            raise RunError("%s: %s" % (s.where, e))
        if size is None:
            size, fmt = (dims[0][1], dims[0][2]), fh.format
        for p, w, h in dims:
            if (w, h) != size:
                raise RunError("%s: %s is %dx%d, the other files are %dx%d" % (s.where, p, w, h, size[0], size[1]))
        if fh.format != fmt:
            raise RunError("%s: %s is a %s flow, the list's first is a %s flow" % (
                s.where, s.flow, _fmt_name(fh.format), _fmt_name(fmt)))
        s.channels, s.flow_header = tuple(chans), fh
    return size[0], size[1], fmt


def _fmt_name(fmt):
    return {FLOW_FLO: ".flo", FLOW_PFM: "little-endian .pfm", FLOW_PFM_BE: "big-endian .pfm",
            kitti_png.KITTI: "KITTI .png"}[fmt]


def read_flow_into(path, hdr, out):
    """The payload of a flow file (flow_header or kitti.probe) into `out`: as stored, or a KITTI PNG's unfiltered samples."""
    if hdr.format == kitti_png.KITTI:
        kitti_png.read_payload(path, hdr, out)
    else:
        read_flow_payload(path, hdr, out)


# ------------------------------------------------------------------------------------------------
# The dataset
# ------------------------------------------------------------------------------------------------
def _align(n, a=16):
    return (n + a - 1) // a * a


class FlowDataset(object):
    """The Solver's ``feed``: each call enqueues the next batch's three inputs on the bound net's stream and returns {}.

    list_file: ``img0 img1 flow`` lines.  batch: samples per call.  rand_permute, rand_permute_seed, block_size, range_start,
    range_end, rand_permute_order: CustomData's data_param fields (the defaults are the train command's: permuted, seed 77).
    flow_encoding: "uint16" (the reference's LMDB values) or "float".  world, rank: data-parallel shard (default: the
    initialised torch.distributed group, else 1, 0).  slots: batches in flight (2 or 3).  threads: reader pool size.
    kitti: the flows are KITTI 16-bit PNGs.
    """

    def __init__(self, list_file, batch, rand_permute=True, rand_permute_seed=77, block_size=0, range_start=0, range_end=-1,
                 rand_permute_order=ORDERS[0], flow_encoding="uint16", world=None, rank=None, slots=3, threads=None, kitti=False):
        if batch < 1:
            raise RunError("batch must be at least 1, got %d" % batch)
        if flow_encoding not in ENCODINGS:
            raise RunError("flow encoding must be uint16 or float, got %s" % flow_encoding)
        if slots not in (2, 3):
            raise RunError("slots must be 2 or 3, got %d" % slots)
        if world is None:
            world, rank = _dist_world()
        self.samples = read_list(list_file)
        w, h, self.flow_format = probe_samples(self.samples, kitti)
        self.size = (w, h)
        self.batch, self.world, self.rank = int(batch), int(world), int(rank)
        self.flow_encoding, self.slots, self.threads = flow_encoding, slots, threads
        self.perm = permutation(len(self.samples), rand_permute, rand_permute_seed, block_size, range_start, range_end,
                                rand_permute_order)
        self.next_batch = 0
        self.net = None

    def __len__(self):
        return len(self.perm)

    def keys(self, k):
        """List lines (keys) of this rank's k-th batch."""
        return batch_keys(self.perm, self.batch, k, self.world, self.rank)

    def channels(self, k):
        """Frame channel count of batch k's pinned slot: the frames' own when they all share it, else 3 (gray repeated, alpha
        dropped -- both exact)."""
        ks = set(c for i in self.keys(k) for c in self.samples[i].channels)
        return ks.pop() if len(ks) == 1 else 3

    def host_batch(self, k):
        """Batch k restated on the host -> (img0, img1, flow) float32 NCHW arrays, the blobs the device path fills."""
        img = [np.stack([image_to_blob(frame_as(read_image(getattr(self.samples[i], n)), 3))[0] for i in self.keys(k)])
               for n in ("img0", "img1")]
        read = kitti_png.read_kitti_flow if self.flow_format == kitti_png.KITTI else read_flow
        flow = np.stack([read(self.samples[i].flow).transpose(2, 0, 1) for i in self.keys(k)])
        if self.flow_encoding == "uint16":
            flow = uint16flow(flow)
        return img[0], img[1], flow

    # ---- the pipeline ----
    def bind(self, net):
        """Allocates the slots for `net` (its first three inputs: (B, 3, H, W) twice, (B, 2, H, W)) and starts reading ahead."""
        import torch
        W, H = self.size
        B = self.batch
        names = list(net.inputs[:3])
        want = [(B, 3, H, W), (B, 3, H, W), (B, 2, H, W)]
        if len(names) < 3 or [net.blobs[n].shape for n in names] != want:
            have = ", ".join("%s %s" % (n, net.blobs[n].shape) for n in names) or "none"
            raise RunError("the net's first three inputs must be img0, img1 (%d, 3, %d, %d) and flow (%d, 2, %d, %d); it has %s"
                           % (B, H, W, B, H, W, have))
        self.close()
        self.net, self.inputs = net, names
        px = B * H * W
        self._flow_off = _align(2 * px * 4)                            # frames of img0, then of img1 ([B][H][W][K] each, K <= 4)
        self._bytes = self._flow_off + px * self._flow_px_bytes()
        S = self.slots
        self._pin = [torch.empty(self._bytes, dtype=torch.uint8).pin_memory() for _ in range(S)]
        self._host = [p.numpy() for p in self._pin]
        self._dev = [torch.empty(self._bytes, dtype=torch.uint8, device="cuda") for _ in range(S)]
        self._net_stream = torch.cuda.ExternalStream(net.stream)
        self._copy_stream = torch.cuda.Stream()
        self._ev_h2d = [torch.cuda.Event() for _ in range(S)]            # pin[s] has reached dev[s]
        self._ev_free = [torch.cuda.Event() for _ in range(S)]           # the net has converted dev[s]
        # the readers wait on CUDA events: on the net's device, so that no thread touches (and creates a context on) another
        self._pool = ThreadPoolExecutor(max_workers=self.threads or min(16, os.cpu_count() or 4),
                                        initializer=torch.cuda.set_device, initargs=(torch.cuda.current_device(),))
        self._reads = {}
        self._timing = deque()
        self._busy = {k: 0.0 for k in ("read", "host_wait", "h2d", "stream_wait", "convert")}
        self._calls = 0
        self.seek(self.next_batch)
        return self

    def seek(self, k):
        """The next call delivers this rank's batch k (after Solver.restore: iter * iter_size)."""
        self.next_batch = int(k)
        if self.net is None:
            return
        for fut in self._reads.values():
            for f in fut[1]:
                f.result()
        self._reads = {}
        for j in range(self.slots):
            self._submit(self.next_batch + j)

    def _submit(self, k):
        s = k % self.slots
        K = self.channels(k)
        self._reads[k] = (K, [self._pool.submit(self._read_one, k, s, K, i, j) for i in range(self.batch) for j in range(3)])

    def _read_one(self, k, s, K, i, j):
        """Item i of batch k, part j (img0, img1, flow) into pinned slot s; waits (in this thread) for the slot's last copy."""
        self._ev_h2d[s].synchronize()
        t0 = time.perf_counter()
        W, H = self.size
        smp = self.samples[self.keys(k)[i]]
        out = self._host[s]
        if j == 2:
            fh = smp.flow_header
            o = self._flow_off + i * fh.nbytes
            try:
                read_flow_into(smp.flow, fh, out[o:o + fh.nbytes])
            except (OSError, RunError) as e:
                raise RunError("%s: %s" % (smp.where, e))
            return time.perf_counter() - t0
        path = (smp.img0, smp.img1)[j]
        n = H * W * K
        o = j * self.batch * n + i * n
        try:
            done = False
            if smp.channels[j] == K:
                with open(path, "rb", buffering=0) as f:
                    hdr = _pnm_header(f, path)
                    if hdr is not None:                                 # the raster as stored: readinto the slot
                        f.seek(hdr[4])
                        if f.readinto(out[o:o + n]) != n:
                            raise RunError("%s: truncated raster" % path)
                        done = True
            if not done:
                a = frame_as(read_image(path), K)
                if a.shape[:2] != (H, W):
                    raise RunError("%s decodes to %dx%d, its header says %dx%d" % (path, a.shape[1], a.shape[0], W, H))
                out[o:o + n] = a.reshape(-1)
        except (OSError, RunError) as e:
            raise RunError("%s: %s" % (smp.where, e))
        return time.perf_counter() - t0

    def __call__(self):
        import torch
        if self.net is None:
            raise RunError("the dataset is not bound to a net: call bind(net) first")
        k, B = self.next_batch, self.batch
        s = k % self.slots
        K, futs = self._reads.pop(k)
        t0 = time.perf_counter()
        self._busy["read"] += sum(f.result() for f in futs)
        self._busy["host_wait"] += time.perf_counter() - t0
        W, H = self.size
        px = B * H * W
        fb = px * self._flow_px_bytes()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._ev_free[s])               # dev[s] was converted `slots` batches ago
            ev[0].record(self._copy_stream)
            self._dev[s][:2 * px * K].copy_(self._pin[s][:2 * px * K], non_blocking=True)
            self._dev[s][self._flow_off:self._flow_off + fb].copy_(self._pin[s][self._flow_off:self._flow_off + fb],
                                                                   non_blocking=True)
            ev[1].record(self._copy_stream)
            self._ev_h2d[s].record(self._copy_stream)
        ns = self._net_stream
        ev[2].record(ns)
        ns.wait_event(self._ev_h2d[s])
        ev[3].record(ns)
        base = self._dev[s].data_ptr()
        self.net.set_input_image_device(self.inputs[0], base, K)
        self.net.set_input_image_device(self.inputs[1], base + px * K, K)
        flags = FLOW_UINT16FLOW if self.flow_encoding == "uint16" else 0
        if self.flow_format == kitti_png.KITTI:
            self.net.set_input_kitti_flow_device(self.inputs[2], base + self._flow_off, flags)
        else:
            self.net.set_input_flow_device(self.inputs[2], base + self._flow_off, self.flow_format, flags)
        ev[4].record(ns)
        self._ev_free[s].record(ns)
        self._timing.append(ev)
        self._harvest(block=False)
        self.next_batch = k + 1
        self._calls += 1
        self._submit(k + self.slots)                                     # reads into pin[s] once its copy is done
        return {}

    def _flow_px_bytes(self):
        return {FLOW_FLO: 8, kitti_png.KITTI: kitti_png.PAYLOAD_PX_BYTES}.get(self.flow_format, 12)

    def _harvest(self, block):
        while self._timing and (block or self._timing[0][4].query()):
            ev = self._timing.popleft()
            ev[4].synchronize()
            self._busy["h2d"] += ev[0].elapsed_time(ev[1]) * 1e-3
            self._busy["stream_wait"] += ev[2].elapsed_time(ev[3]) * 1e-3
            self._busy["convert"] += ev[3].elapsed_time(ev[4]) * 1e-3

    def busy(self):
        """Per-stage busy seconds since bind: read (host, summed over the pool's threads), host_wait (the caller blocked on
        reads), h2d and convert (device), stream_wait (the net's stream stalled on a slot's copy); and calls.  Synchronises."""
        self._harvest(block=True)
        return dict(self._busy, calls=self._calls)

    def close(self):
        """Waits for the reads in flight and releases the pool (the slots go with the object)."""
        if getattr(self, "_pool", None) is not None:
            for fut in self._reads.values():
                for f in fut[1]:
                    f.exception()
            self._pool.shutdown(wait=True)
            self._pool = None
            self._reads = {}
        self.net = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def uint16flow(v):
    """The reference's short(32 v) / 32 round trip on the host (float32 in and out; include/fn2_flow.h)."""
    v = np.asarray(v, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        s = v * np.float32(32)
        ok = (s < 32767) & (s > -32769)
        t = np.where(ok, s, 0).astype(np.float64)
    q = (np.trunc(t).astype(np.int32).astype(np.float32) * np.float32(0.03125)).astype(np.float32)
    return np.where(ok, q, np.float32(np.nan)).astype(np.float32)


def _dist_world():
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return dist.get_world_size(), dist.get_rank()
    except ImportError:
        pass
    return 1, 0
