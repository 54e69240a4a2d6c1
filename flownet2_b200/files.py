"""Image and flow files on the host: the frame and flow readers and writers, the list file, and the probe that checks a list
before anything runs.  numpy only; the device side is flownet2_b200.feed, the KITTI PNG container flownet2_b200.kitti.

Frames are PPM / PGM (P6 / P5, maxval 255, read here) or anything Pillow reads, converted the way scipy.misc.imread hands
them to the reference (palette to RGB or RGBA, LA to L).  Flows are .flo, 'PF' PFM of either byte order, or (kitti=True)
KITTI 16-bit PNGs; a flow file's payload is the bytes after its header as stored (a PNG: its unfiltered samples), and
FLOW_PX_BYTES gives its bytes per pixel in each format.

A list file holds one ``img0 img1 flow`` line per pair, blank lines skipped.  For run the third column is the flow to write;
for evaluate and train it is the ground truth, and a fourth (occlusion) column is refused.  Masks (evaluate's occlusion masks
and object maps) come in lists of their own, one path per line in the pair list's order (attach_masks).
"""
import os
import struct

import numpy as np

from . import FLOW_FLO, FLOW_KITTI, FLOW_PFM, FLOW_PFM_BE

FLO_TAG = 202021.25                        # 'PIEH' read as a little-endian float
FLOW_PX_BYTES = {FLOW_FLO: 8, FLOW_PFM: 12, FLOW_PFM_BE: 12, FLOW_KITTI: 6}


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


def _pnm_channels(path, magic, maxval):
    if maxval != 255:
        raise RunError("%s: maxval %d, only 8-bit frames (maxval 255) are supported" % (path, maxval))
    return 1 if magic == b"P5" else 3


def probe_image(path):
    """-> (width, height, channels) of an image file without decoding its pixels; refuses what read_image would refuse,
    a PNM whose raster is cut short included."""
    if not os.path.isfile(path):
        raise RunError("%s: no such file" % path)
    with open(path, "rb") as f:
        hdr = _pnm_header(f, path)
    if hdr is not None:
        magic, w, h, maxval, off = hdr
        k = _pnm_channels(path, magic, maxval)
        size = os.path.getsize(path)
        if size < off + w * h * k:
            raise RunError("%s: truncated raster (%d of %d bytes)" % (path, max(size - off, 0), w * h * k))
        return w, h, k
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
            k = _pnm_channels(path, magic, maxval)
            f.seek(off)
            raw = f.read(w * h * k)
            if len(raw) != w * h * k:
                raise RunError("%s: truncated raster (%d of %d bytes)" % (path, len(raw), w * h * k))
            return np.frombuffer(raw, np.uint8).reshape((h, w, k) if k == 3 else (h, w))
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


def read_frame_into(path, size, k, out):
    """The frame at `path`, of `size` (width, height), as (H, W, k) bytes into the writable buffer `out`: a PNM with k channels
    is read into it as stored, any other frame is decoded and converted (frame_as)."""
    W, H = size
    with open(path, "rb", buffering=0) as f:
        hdr = _pnm_header(f, path)
        if hdr is not None and _pnm_channels(path, hdr[0], hdr[3]) == k:
            f.seek(hdr[4])
            if f.readinto(out) != H * W * k:
                raise RunError("%s: truncated raster" % path)
            return
    a = frame_as(read_image(path), k)
    if a.shape[:2] != (H, W):
        raise RunError("%s decodes to %dx%d, its header says %dx%d" % (path, a.shape[1], a.shape[0], W, H))
    out[:] = a.reshape(-1)


def write_pnm(path, a):
    """Binary PGM (H, W) or PPM (H, W, 3) frame, maxval 255 -> path."""
    with open(path, "wb") as f:
        f.write(b"%s\n%d %d\n255\n" % (b"P5" if a.ndim == 2 else b"P6", a.shape[1], a.shape[0]))
        f.write(np.ascontiguousarray(a, np.uint8).tobytes())
    return str(path)


# ------------------------------------------------------------------------------------------------
# Flow files
# ------------------------------------------------------------------------------------------------
class FlowHeader(object):
    """format (FLOW_FLO / FLOW_PFM / FLOW_PFM_BE / FLOW_KITTI), width, height, payload offset and bytes of a flow file."""

    def __init__(self, fmt, w, h, offset):
        self.format, self.width, self.height, self.offset = fmt, w, h, offset
        self.nbytes = w * h * FLOW_PX_BYTES[fmt]


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
        hdr = FlowHeader(FLOW_FLO, w, h, 12)
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
        hdr = FlowHeader(FLOW_PFM_BE if scale > 0 else FLOW_PFM, w, h, i + 1)
    else:
        raise RunError("%s: flows must be .flo or .pfm files" % path)
    if size < hdr.offset + hdr.nbytes:
        raise RunError("%s: truncated payload (%d of %d bytes)" % (path, max(size - hdr.offset, 0), hdr.nbytes))
    return hdr


def read_flow_payload(path, hdr, out):
    """The payload bytes of a .flo or PFM file, as stored, into the writable buffer `out` (hdr.nbytes long)."""
    with open(path, "rb", buffering=0) as f:
        f.seek(hdr.offset)
        got = f.readinto(out)
    if got != hdr.nbytes:
        raise RunError("%s: truncated payload (%d of %d bytes)" % (path, got, hdr.nbytes))


def read_flow_into(path, hdr, out):
    """The payload of a flow file (flow_header or kitti.probe) into `out`: as stored, or a KITTI PNG's unfiltered samples."""
    if hdr.format == FLOW_KITTI:
        from . import kitti
        kitti.read_payload(path, hdr, out)
    else:
        read_flow_payload(path, hdr, out)


def read_flow(path, hdr=None):
    """Host reading of a flow file (its header: flow_header's, read here if not given, or kitti.probe's) -> float32 (H, W, 2)
    top-down, as the reference's converter reads it (no quantisation; NaN at a KITTI PNG's invalid pixels)."""
    hdr = hdr or flow_header(path)
    buf = np.empty(hdr.nbytes, np.uint8)
    read_flow_into(path, hdr, buf)
    if hdr.format == FLOW_KITTI:
        from . import kitti
        return kitti.decode(buf.view(">u2").reshape(hdr.height, hdr.width, 3))
    if hdr.format == FLOW_FLO:
        return buf.view("<f4").reshape(hdr.height, hdr.width, 2).astype(np.float32)
    a = buf.view(">f4" if hdr.format == FLOW_PFM_BE else "<f4").reshape(hdr.height, hdr.width, 3)
    return a[::-1, :, :2].astype(np.float32)


def write_flo(path, flow_hw2):
    """.flo file (src/caffe/util/output.cpp:16-64): 'PIEH', width, height (int32), then (H, W, 2) float32."""
    h, w = flow_hw2.shape[:2]
    with open(path, "wb") as f:
        f.write(b"PIEH")
        f.write(np.array([w, h], np.int32).tobytes())
        f.write(np.ascontiguousarray(flow_hw2, np.float32).tobytes())


def write_pfm(path, hw3, big_endian=False):
    """'PF' PFM of a top-down (H, W, 3) float array: rows stored bottom-to-top, scale 1 (big-endian) or -1 (little-endian)."""
    h, w = hw3.shape[:2]
    with open(path, "wb") as f:
        f.write(b"PF\n%d %d\n%s\n" % (w, h, b"1.0" if big_endian else b"-1.0"))
        f.write(np.ascontiguousarray(hw3[::-1], ">f4" if big_endian else "<f4").tobytes())
    return str(path)


# ------------------------------------------------------------------------------------------------
# The list and its probe
# ------------------------------------------------------------------------------------------------
class Pair(object):
    """One list line: where ('list:line'), the frames img0 and img1, and flow, the flow file (written by run, ground truth
    for evaluate and train).  masks: the pair's 8-bit mask planes, [(where, path)] in the order attach_masks was given their
    lists.  probe() sets size (width, height), channels (img0's, img1's) and, with ground truth, flow_header."""

    def __init__(self, where, img0, img1, flow):
        self.where, self.img0, self.img1, self.flow = where, img0, img1, flow
        self.masks = ()
        self.size = self.channels = self.flow_header = None


def read_list(path, ground_truth=True):
    """-> [Pair] of a list file: one ``img0 img1 flow`` line per pair, blank lines skipped.  ground_truth: the third column is
    a flow to read, and an occlusion column is refused; else it is the flow to write (run's ``img0 img1 out.flo``)."""
    if not os.path.isfile(path):
        raise RunError("%s: no such list file" % path)
    out = []
    with open(path) as f:
        for no, line in enumerate(f, 1):
            fields = line.split()
            if not fields:
                continue
            if ground_truth and len(fields) == 4:
                raise RunError("%s:%d: an occlusion field (%s); occlusion masks are not supported" % (path, no, fields[3]))
            if len(fields) != 3:
                raise RunError("%s:%d: %d fields, expected 'img0 img1 %s'" % (path, no, len(fields),
                                                                              "flow" if ground_truth else "out.flo"))
            out.append(Pair("%s:%d" % (path, no), *fields))
    return out


def read_mask_list(path, n):
    """-> [(where, mask path)] of a mask list: one path per line, blank lines skipped, line k (counting non-blank lines) for
    pair k of a pair list of n lines; refuses any other count, naming both."""
    if not os.path.isfile(path):
        raise RunError("%s: no such mask list" % path)
    out = []
    with open(path) as f:
        for no, line in enumerate(f, 1):
            fields = line.split()
            if not fields:
                continue
            if len(fields) != 1:
                raise RunError("%s:%d: %d fields, expected one mask path" % (path, no, len(fields)))
            out.append(("%s:%d" % (path, no), fields[0]))
    if len(out) != n:
        raise RunError("%s: %d masks for a list of %d pairs" % (path, len(out), n))
    return out


def attach_masks(pairs, lists):
    """Pair k of `pairs` (a whole list, before any sharding) gets line k of each mask list in `lists`, in that order, as its
    masks."""
    masks = [read_mask_list(path, len(pairs)) for path in lists]
    for k, p in enumerate(pairs):
        p.masks = tuple(m[k] for m in masks)


def probe(pairs, ground_truth=False, kitti=False):
    """Checks every pair's frames without decoding them (present, 8-bit, a PNM's raster in full, one size per pair) and sets
    its size and channels; with ground truth also reads the flow's header (flow_header, or kitti.probe under kitti) into
    flow_header and refuses a flow whose size is not its frames'; and checks each of its masks is a one-channel 8-bit image of
    its frames' size.  Every refusal names the list line (a mask's: its mask list's line)."""
    if kitti:
        from . import kitti as kitti_png
    for p in pairs:
        try:
            w0, h0, k0 = probe_image(p.img0)
            w1, h1, k1 = probe_image(p.img1)
            fh = (kitti_png.probe(p.flow) if kitti else flow_header(p.flow)) if ground_truth else None
        except RunError as e:
            raise RunError("%s: %s" % (p.where, e))
        if (w0, h0) != (w1, h1):
            raise RunError("%s: %s is %dx%d but %s is %dx%d" % (p.where, p.img0, w0, h0, p.img1, w1, h1))
        if fh is not None and (fh.width, fh.height) != (w0, h0):
            raise RunError("%s: %s is %dx%d but its frames are %dx%d" % (p.where, p.flow, fh.width, fh.height, w0, h0))
        for where, path in p.masks:
            try:
                w, h, k = probe_image(path)
            except RunError as e:
                raise RunError("%s: %s" % (where, e))
            if k != 1:
                raise RunError("%s: %s has %d channels, a mask is a one-channel 8-bit image" % (where, path, k))
            if (w, h) != (w0, h0):
                raise RunError("%s: %s is %dx%d but the frames of %s are %dx%d" % (where, path, w, h, p.where, w0, h0))
        p.size, p.channels, p.flow_header = (w0, h0), (k0, k1), fh
