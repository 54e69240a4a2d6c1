"""Training samples from image and flow files: the reference's convert_imageset_and_flow + CustomData path without the LMDB.

    ds = FlowDataset("train.txt", batch=8)              # reads the list, probes every file, fixes the order
    net = Net(fill_train_template(text, 448, 320, *ds.size, 8), None, TRAIN)
    ds.bind(net)                                         # pinned slots, device slots, streams; starts reading ahead
    solver.step(n, ds)                                   # each call enqueues the next batch on the net's stream

The list file holds one ``img0 img1 flow`` line per sample (the converter's format); blank lines are skipped and an occlusion
field is refused.  Frames and flows are read by flownet2_b200.files (frames PPM / PGM or anything Pillow reads, flows .flo or
'PF' PFM), and the list is probed there before anything runs; a training list has one flow format, and every file has one
size, as one LMDB has one Datum shape.  With kitti=True every flow is a KITTI 16-bit PNG (flownet2_b200.kitti): invalid
pixels become NaN, which L1Loss, Downsample and LpqLoss leave out.

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

Pipeline.  Frames and flows are not converted on the host: bind() sets up a flownet2_b200.feed.Feeder, whose reader pool
reads the batches ahead into pinned slots (the PPM rasters and flow payloads as stored, a KITTI PNG inflated and unfiltered
into its raw samples), and each call enqueues one slot's copy and its conversion on the net's stream: the frames by the
feeder, the flow by fn2_net_set_input_flow_device.  The step's path never synchronises with the device.  busy() reports the
per-stage times.
"""
from collections import deque

import numpy as np

from . import FLOW_FLO, FLOW_KITTI, FLOW_PFM, FLOW_PFM_BE, FLOW_UINT16FLOW, image_to_blob
from .feed import Feeder
from .files import FLOW_PX_BYTES, RunError, frame_as, probe, read_flow, read_image, read_list
# the flow-file helpers this module held before flownet2_b200.files, still importable from here
from .files import FLO_TAG, FlowHeader, flow_header, read_flow_payload, write_pfm  # noqa: F401

FORMAT_NAMES = {FLOW_FLO: ".flo", FLOW_PFM: "little-endian .pfm", FLOW_PFM_BE: "big-endian .pfm", FLOW_KITTI: "KITTI .png"}
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
# The dataset
# ------------------------------------------------------------------------------------------------
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
        probe(self.samples, ground_truth=True, kitti=kitti)
        self.size = self.flow_format = None
        for s in self.samples:                         # one size and one flow format, as one LMDB has one Datum shape
            if self.size is None:
                self.size, self.flow_format = s.size, s.flow_header.format
            if s.size != self.size:
                raise RunError("%s: %s is %dx%d, the other files are %dx%d" % (s.where, s.img0, s.size[0], s.size[1],
                                                                               self.size[0], self.size[1]))
            if s.flow_header.format != self.flow_format:
                raise RunError("%s: %s is a %s flow, the list's first is a %s flow" % (
                    s.where, s.flow, FORMAT_NAMES[s.flow_header.format], FORMAT_NAMES[self.flow_format]))
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

    def host_batch(self, k):
        """Batch k restated on the host -> (img0, img1, flow) float32 NCHW arrays, the blobs the device path fills."""
        img = [np.stack([image_to_blob(frame_as(read_image(getattr(self.samples[i], n)), 3))[0] for i in self.keys(k)])
               for n in ("img0", "img1")]
        flow = np.stack([read_flow(self.samples[i].flow, self.samples[i].flow_header).transpose(2, 0, 1) for i in self.keys(k)])
        if self.flow_encoding == "uint16":
            flow = uint16flow(flow)
        return img[0], img[1], flow

    # ---- the pipeline ----
    def bind(self, net):
        """Allocates the slots for `net` (its first three inputs: (B, 3, H, W) twice, (B, 2, H, W)) and starts reading ahead."""
        W, H = self.size
        B = self.batch
        names = list(net.inputs[:3])
        want = [(B, 3, H, W), (B, 3, H, W), (B, 2, H, W)]
        if len(names) < 3 or [net.blobs[n].shape for n in names] != want:
            have = ", ".join("%s %s" % (n, net.blobs[n].shape) for n in names) or "none"
            raise RunError("the net's first three inputs must be img0, img1 (%d, 3, %d, %d) and flow (%d, 2, %d, %d); it has %s"
                           % (B, H, W, B, H, W, have))
        self.close()
        self.net = net
        self._feed = Feeder(net, B, self.size, W * H * FLOW_PX_BYTES[self.flow_format],
                            lambda k: [self.samples[i] for i in self.keys(k)], self.slots, self.threads)
        flags = FLOW_UINT16FLOW if self.flow_encoding == "uint16" else 0
        self._stage = lambda payload, stride: net.set_input_flow_device(names[2], payload.data_ptr(), self.flow_format, flags)
        self._calls = 0
        self.seek(self.next_batch)
        return self

    def seek(self, k):
        """The next call delivers this rank's batch k (after Solver.restore: iter * iter_size)."""
        self.next_batch = int(k)
        if self.net is not None:
            self._feed.seek(self.next_batch)

    def __call__(self):
        if self.net is None:
            raise RunError("the dataset is not bound to a net: call bind(net) first")
        self._feed(self._stage)
        self.next_batch += 1
        self._calls += 1
        return {}

    def busy(self):
        """Per-stage busy seconds since bind: read (host, summed over the pool's threads), host_wait (the caller blocked on
        reads), h2d and convert (device), stream_wait (the net's stream stalled on a slot's copy); and calls.  Synchronises."""
        return dict(self._feed.busy(), calls=self._calls)

    def close(self):
        """Waits for the reads in flight and releases the pool (the slots go with the object)."""
        if getattr(self, "_feed", None) is not None:
            self._feed.close()
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
