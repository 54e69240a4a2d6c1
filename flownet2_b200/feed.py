"""The pinned-slot ring that brings list items' files to a net's device: run, evaluate and FlowDataset are fed through it.

    feed = Feeder(net, batch, (W, H), item_bytes, items_of, slots)
    feed.seek(k)                  # the next call feeds batch k; reading starts for batches k .. k + slots - 1
    feed(stage)                   # enqueues the next batch on the net's stream and starts reading the one `slots` ahead
    feed.swap()                   # with swap=True, after the first forward: the slot's frames again, the two inputs exchanged
    feed.busy(); feed.close()
    Feeder(None, batch, (W, H), item_bytes, items_of, slots)     # payloads only, on a stream of its own (flownet2_b200.viz)

items_of(k) gives batch k's probed items (flownet2_b200.files.Pair; None past the end).  Each of the S slots is a pinned host
buffer and a device buffer holding [img0 frames][img1 frames][payload]: the frames [B][H][W][K] bytes, K the batch's frame
channel count (batch_channels), and from a 16-byte boundary item i's flow payload at i * item_bytes (none when item_bytes is
0), followed by its masks (files.Pair.masks, H x W bytes each) from mask_offset(H, W) on.  A reader pool on the net's device
reads every part of a batch into its host slot: a PNM frame with K channels as stored, any other frame decoded (a mask as one
channel), a payload through files.read_flow_into.  A call waits for the batch's reads, copies the slot to the
device on a copy stream, and on the net's stream waits for that copy, converts the frames into the net's first two inputs
(fn2_net_set_input_frames_device), runs stage(payload, item_bytes) on the device payload and records the slot free.  A
feeder built with swap=True (run --backward, evaluate --fb-check) leaves the slot in use after the call: swap(), once the
first forward has been enqueued, converts the same frames into the two inputs exchanged (img1 first) and only then records
the slot free.  Without a net (net None) a slot holds the payloads alone, from offset 0, and stage() runs on a stream of the
feeder's own.

Three orderings keep a slot from being overwritten while in use:
  * a reader writes host slot s only after the copy out of s from S batches ago has finished; it waits for that copy itself,
    so the caller's thread never synchronises with the device;
  * the copy into device slot s waits until the net's stream has converted s from S batches ago;
  * slot s is recorded free only after its frames and stage() have been enqueued (with swap, after swap()'s conversion).
"""
import os
import time
from collections import deque
from concurrent.futures import ThreadPoolExecutor

from .files import FLOW_PX_BYTES, RunError, read_flow_into, read_frame_into


def _align(n, a=16):
    return (n + a - 1) // a * a


def batch_channels(items):
    """Frame channel count of a batch's slot: the frames' own when they all share it, else 3 (gray repeated, alpha dropped --
    both exact)."""
    ks = set(k for p in items for k in p.channels)
    return ks.pop() if len(ks) == 1 else 3


def mask_offset(H, W):
    """Offset of an item's first mask plane in its payload stride: after the largest flow payload of an H x W pair."""
    return H * W * max(FLOW_PX_BYTES.values())


def read_part(p, j, size, k, out):
    """Part j of item p -- 0: img0, 1: img1 as (H, W, k) bytes of `size` (W, H); 2: its flow's payload; 3 + m: its mask m as
    (H, W) bytes -- into the start of the writable buffer `out`; a refusal names the list line (a mask's, its mask list's)."""
    where = p.masks[j - 3][0] if j >= 3 else p.where
    try:
        if j >= 3:
            read_frame_into(p.masks[j - 3][1], size, 1, out[:size[0] * size[1]])
        elif j == 2:
            read_flow_into(p.flow, p.flow_header, out[:p.flow_header.nbytes])
        else:
            read_frame_into((p.img0, p.img1)[j], size, k, out[:size[0] * size[1] * k])
    except (OSError, RunError) as e:
        raise RunError("%s: %s" % (where, e))


class Feeder(object):
    def __init__(self, net, batch, size, item_bytes, items_of, slots, threads=None, swap=False):
        import torch
        self.torch, self.net, self.swap_inputs, self._held = torch, net, swap, None
        self.batch, self.size, self.item_bytes, self.items_of, self.slots = batch, size, item_bytes, items_of, slots
        self.frame_bytes = batch * size[0] * size[1] if net is not None else 0    # of one input at K = 1
        self.payload_off = _align(2 * self.frame_bytes * 4)             # after both inputs' frames, K <= 4
        nbytes = self.payload_off + batch * item_bytes
        self._pin = [torch.empty(nbytes, dtype=torch.uint8).pin_memory() for _ in range(slots)]
        self._host = [p.numpy() for p in self._pin]
        self._dev = [torch.empty(nbytes, dtype=torch.uint8, device="cuda") for _ in range(slots)]
        self.stream = torch.cuda.ExternalStream(net.stream) if net is not None else torch.cuda.Stream()
        self._copy_stream = torch.cuda.Stream()
        self._ev_h2d = [torch.cuda.Event() for _ in range(slots)]      # pin[s] has reached dev[s]
        self._ev_free = [torch.cuda.Event() for _ in range(slots)]     # the net has converted dev[s]
        # the readers wait on CUDA events: on the net's device, so that no thread touches (and creates a context on) another
        self._pool = ThreadPoolExecutor(max_workers=threads or min(16, os.cpu_count() or 4),
                                        initializer=torch.cuda.set_device, initargs=(torch.cuda.current_device(),))
        self._reads = {}
        self._timing = deque()
        self._busy = {k: 0.0 for k in ("read", "host_wait", "h2d", "stream_wait", "convert")}
        self.next = 0

    def seek(self, k):
        """The next call feeds batch k: waits for the reads in flight, then starts reading batches k .. k + slots - 1."""
        for _, futs in self._reads.values():
            for f in futs:
                f.result()
        self._reads = {}
        self.next = k
        for j in range(self.slots):
            self._submit(k + j)

    def _submit(self, k):
        items = self.items_of(k)
        if items is None:
            return
        s, K = k % self.slots, batch_channels(items) if self.net is not None else 0
        frames = (0, 1) if self.net is not None else ()
        parts = lambda p: frames + (2,) + tuple(range(3, 3 + len(p.masks))) if self.item_bytes else frames
        self._reads[k] = (K, [self._pool.submit(self._read, s, K, i, j, p) for i, p in enumerate(items) for j in parts(p)])

    def _read(self, s, K, i, j, p):
        self._ev_h2d[s].synchronize()                                  # the copy out of pin[s] `slots` batches ago is done
        t0 = time.perf_counter()
        W, H = self.size
        if j >= 3:
            o = self.payload_off + i * self.item_bytes + mask_offset(H, W) + (j - 3) * H * W
        else:
            o = self.payload_off + i * self.item_bytes if j == 2 else (j * self.batch + i) * W * H * K
        read_part(p, j, self.size, K, self._host[s][o:])
        return time.perf_counter() - t0

    def __call__(self, stage=None):
        """Enqueues the next batch on the net's stream: its frames into the net's first two inputs, then stage(payload,
        item_bytes) with the device payload (a uint8 tensor) and the net's stream current."""
        torch = self.torch
        assert self._held is None, "swap() was not called for the last batch"
        k = self.next
        s = k % self.slots
        K, futs = self._reads.pop(k)
        t0 = time.perf_counter()
        self._busy["read"] += sum(f.result() for f in futs)
        self._busy["host_wait"] += time.perf_counter() - t0
        n, off, pay = 2 * self.frame_bytes * K, self.payload_off, self.batch * self.item_bytes
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._ev_free[s])             # dev[s] was converted `slots` batches ago
            ev[0].record(self._copy_stream)
            if n:
                self._dev[s][:n].copy_(self._pin[s][:n], non_blocking=True)
            if pay:
                self._dev[s][off:off + pay].copy_(self._pin[s][off:off + pay], non_blocking=True)
            ev[1].record(self._copy_stream)
            self._ev_h2d[s].record(self._copy_stream)
        ns = self.stream
        ev[2].record(ns)
        ns.wait_event(self._ev_h2d[s])
        ev[3].record(ns)
        if self.net is not None:
            base, inputs = self._dev[s].data_ptr(), self.net.inputs[:2]
            self.net.set_input_image_device(inputs[0], base, K)
            self.net.set_input_image_device(inputs[1], base + n // 2, K)
        if stage is not None:
            with torch.cuda.stream(ns):
                stage(self._dev[s][off:], self.item_bytes)
        ev[4].record(ns)
        if self.swap_inputs:
            self._held = (s, K)                                        # swap() converts dev[s] again, then frees it
        else:
            self._ev_free[s].record(ns)
        self._timing.append(ev)
        self._harvest(block=False)
        self.next = k + 1
        self._submit(k + self.slots)                                   # reads into pin[s] once its copy is done

    def swap(self):
        """Enqueues the last batch's frames again on the net's stream, into the net's first two inputs exchanged (img1 into the
        first), then records its slot free.  For a feeder built with swap=True, once per call, after that batch's first
        forward."""
        s, K = self._held
        n = 2 * self.frame_bytes * K
        base, inputs = self._dev[s].data_ptr(), self.net.inputs[:2]
        self.net.set_input_image_device(inputs[0], base + n // 2, K)
        self.net.set_input_image_device(inputs[1], base, K)
        self._ev_free[s].record(self.stream)
        self._held = None

    def _harvest(self, block):
        while self._timing and (block or self._timing[0][4].query()):
            ev = self._timing.popleft()
            ev[4].synchronize()
            self._busy["h2d"] += ev[0].elapsed_time(ev[1]) * 1e-3
            self._busy["stream_wait"] += ev[2].elapsed_time(ev[3]) * 1e-3
            self._busy["convert"] += ev[3].elapsed_time(ev[4]) * 1e-3

    def busy(self):
        """Per-stage busy seconds: read (host, summed over the pool's threads), host_wait (the caller blocked on reads), h2d
        and convert (device; convert includes stage()), stream_wait (the net's stream stalled on a slot's copy).
        Synchronises."""
        self._harvest(block=True)
        return dict(self._busy)

    def close(self):
        """Waits for the reads in flight and releases the pool (the slots go with the object)."""
        if self._pool is not None:
            for _, futs in self._reads.values():
                for f in futs:
                    f.exception()
            self._pool.shutdown(wait=True)
            self._pool = None
            self._reads = {}
