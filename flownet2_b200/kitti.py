"""KITTI flow files: the 16-bit RGB PNGs of the KITTI 2012 / 2015 flow benchmarks, read as ground truth and written as
predictions.  This module is the only place that knows the container; the value convention is stated in include/fn2_flow.h.

    info = probe(path)                      # IHDR only: a FlowHeader with width, height, nbytes of the payload
    read_payload(path, info, out)           # inflate + unfilter into `out`: [H][W][3] big-endian uint16, the file's own bytes
    write_png_rows(path, rows, w, h)        # scanlines already filtered (fn2_flow_to_kitti_png_rows) -> a PNG file
    write_png_rows(path, rows, w, h, 8)     # the same for 8-bit RGB (fn2_flow_to_color_png_rows, flownet2_b200.viz)
    write_png_rows(path, rows, w, h, 8, 1)  # 8-bit grey (fn2_flow_fb_occlusion's masks, run --backward)
    read_kitti_flow(path) / write_kitti_flow(path, flow_hw2)     # host helpers in numpy, float32 (H, W, 2) with NaN = invalid

The host only undoes (or makes) the PNG container: the chunks, zlib's deflate and the per-row filters.  The conversion
between the raw samples and the flow runs on the device (fn2_flow_to_tensor with FLOW_KITTI, fn2_flow_to_kitti_png_rows) in
the pipelines of data, evaluate and run; the numpy helpers here restate it for users converting files and for the tests.

Accepted: colour type 2 (RGB), bit depth 16, compression, filter and interlace methods 0, any number of IDAT chunks;
ancillary chunks (and a suggested palette, PLTE) are skipped.  Refused, naming the file: another colour type or depth, an
interlaced file, a bad signature, a CRC mismatch on IHDR or IDAT, a missing IDAT or IEND, an unknown critical chunk, a
truncated file, and a stream that does not inflate to exactly the image's scanlines.
"""
import os
import struct
import zlib

import numpy as np

from . import FLOW_KITTI
from .files import FlowHeader, RunError, read_flow

SIGNATURE = b"\x89PNG\r\n\x1a\n"
BPP = 6                                     # bytes per pixel: three 16-bit samples
LEVEL = 6                                   # zlib's default level, libpng's default
KNOWN_CRITICAL = (b"IHDR", b"PLTE", b"IDAT", b"IEND")


def _ihdr(path, head):
    if len(head) < 8 or head[:8] != SIGNATURE:
        raise RunError("%s: not a PNG file (signature)" % path)
    if len(head) < 33:
        raise RunError("%s: truncated PNG header" % path)
    n, kind = struct.unpack(">I4s", head[8:16])
    if kind != b"IHDR" or n != 13:
        raise RunError("%s: the first PNG chunk is %r of %d bytes, expected IHDR of 13" % (path, kind, n))
    if struct.unpack(">I", head[29:33])[0] != zlib.crc32(head[12:29]):
        raise RunError("%s: CRC mismatch in chunk IHDR" % path)
    w, h, depth, colour, comp, filt, interlace = struct.unpack(">IIBBBBB", head[16:29])
    if colour != 2 or depth != 16:
        raise RunError("%s: PNG colour type %d at bit depth %d; a KITTI flow is 16-bit RGB (colour type 2, depth 16)"
                       % (path, colour, depth))
    if interlace != 0:
        raise RunError("%s: an interlaced PNG; KITTI flows are not interlaced" % path)
    if comp != 0 or filt != 0:
        raise RunError("%s: PNG compression method %d / filter method %d, expected 0 / 0" % (path, comp, filt))
    if w < 1 or h < 1 or w >= 1 << 31 or h >= 1 << 31:
        raise RunError("%s: PNG size %dx%d" % (path, w, h))
    return FlowHeader(FLOW_KITTI, w, h, 0)


def probe(path):
    """-> FlowHeader (format FLOW_KITTI) from the signature and IHDR alone; refuses what _ihdr refuses, naming the file."""
    if not os.path.isfile(path):
        raise RunError("%s: no such file" % path)
    with open(path, "rb") as f:
        return _ihdr(path, f.read(33))


def _idat(path, data):
    """The concatenated IDAT data of a PNG file's bytes, checking every chunk up to IEND."""
    out, pos, seen_end = [], 8, False
    while pos < len(data):
        if pos + 8 > len(data):
            break
        n, kind = struct.unpack(">I4s", data[pos:pos + 8])
        if pos + 12 + n > len(data):
            raise RunError("%s: truncated PNG (chunk %r of %d bytes at offset %d)" % (path, kind, n, pos))
        body = data[pos + 8:pos + 8 + n]
        if kind in (b"IHDR", b"IDAT"):
            if struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0] != zlib.crc32(body, zlib.crc32(kind)):
                raise RunError("%s: CRC mismatch in chunk %s at offset %d" % (path, kind.decode("latin-1"), pos))
        elif not kind[0] & 0x20 and kind not in KNOWN_CRITICAL:        # a lower-case first letter marks an ancillary chunk
            raise RunError("%s: unknown critical PNG chunk %r" % (path, kind))
        if kind == b"IDAT":
            out.append(body)
        pos += 12 + n
        if kind == b"IEND":
            seen_end = True
            break
    if not out:
        raise RunError("%s: no IDAT chunk" % path)
    if not seen_end:
        raise RunError("%s: truncated PNG (no IEND chunk)" % path)
    return b"".join(out)


def read_payload(path, info, out):
    """The payload of a KITTI PNG ([H][W][3] big-endian uint16, info.nbytes bytes) into the writable buffer `out`: the IDAT
    stream inflated by zlib and the filters undone by fn2_png_unfilter (both release the GIL)."""
    import ctypes as C
    from . import check, lib
    with open(path, "rb") as f:
        data = f.read()
    _ihdr(path, data[:33])
    try:
        raw = zlib.decompress(_idat(path, data))
    except zlib.error as e:
        raise RunError("%s: the PNG data does not inflate: %s" % (path, e))
    row = info.width * BPP
    if len(raw) != info.height * (row + 1):
        raise RunError("%s: the PNG data inflates to %d bytes, a %dx%d image has %d" % (
            path, len(raw), info.width, info.height, info.height * (row + 1)))
    dst = np.frombuffer(out, np.uint8) if not isinstance(out, np.ndarray) else out
    assert dst.nbytes >= info.nbytes and dst.flags.c_contiguous and dst.flags.writeable
    src = np.frombuffer(raw, np.uint8)
    try:
        check(lib().fn2_png_unfilter(C.c_void_p(src.ctypes.data), info.height, row, BPP, C.c_void_p(dst.ctypes.data)))
    except Exception as e:
        raise RunError("%s: %s" % (path, str(e).split(": ", 1)[-1]))


def _chunk(kind, body):
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(body, zlib.crc32(kind)))


def png_bytes(rows, w, h, depth=16, channels=3):
    """An RGB PNG (colour type 2) of bit depth 16 (a KITTI flow) or 8 (a colour-coded flow, flownet2_b200.viz), or with
    channels 1 an 8-bit grey one (colour type 0, an occlusion mask), from h filtered scanlines of 1 + channels (depth / 8) w
    bytes: IHDR, one IDAT deflated at level 6, IEND."""
    assert (depth, channels) in ((8, 3), (16, 3), (8, 1)), (depth, channels)
    rows = memoryview(rows).cast("B")
    assert len(rows) == h * (1 + channels * depth // 8 * w), (len(rows), w, h, depth, channels)
    return (SIGNATURE + _chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, 2 if channels == 3 else 0, 0, 0, 0))
            + _chunk(b"IDAT", zlib.compress(rows, LEVEL)) + _chunk(b"IEND", b""))


def write_png_rows(path, rows, w, h, depth=16, channels=3):
    with open(path, "wb") as f:
        f.write(png_bytes(rows, w, h, depth, channels))
    return str(path)


# ------------------------------------------------------------------------------------------------
# The value convention in numpy (include/fn2_flow.h)
# ------------------------------------------------------------------------------------------------
def decode(samples):
    """[..., 3] uint16 samples (R, G, B as numbers) -> float32 [..., 2] flow, NaN in both channels where B = 0."""
    s = np.asarray(samples)
    uv = (s[..., :2].astype(np.int32) - 32768).astype(np.float32) * np.float32(1.0 / 64)
    return np.where(s[..., 2:3] > 0, uv, np.float32(np.nan)).astype(np.float32)


def encode(flow):
    """float32 [..., 2] flow -> [..., 3] uint16 samples: (uint16) max(min(64 v + 32768, 65535), 0) and B = 1 where both
    components are finite, (0, 0, 0) elsewhere."""
    f = np.asarray(flow, np.float32)
    ok = np.isfinite(f).all(axis=-1, keepdims=True)
    with np.errstate(over="ignore", invalid="ignore"):
        q = np.clip(np.where(ok, f, 0) * np.float32(64) + np.float32(32768), 0, 65535).astype(np.float32)
    out = np.concatenate([q.astype(np.uint16), np.ones_like(q[..., :1], np.uint16)], axis=-1)
    return np.where(ok, out, 0).astype(np.uint16)


def paeth_rows(samples):
    """(H, W, 3) uint16 samples -> (H, 1 + 6 W) uint8 scanlines, every row Paeth-filtered (type 4), as the device writes them."""
    raw = np.ascontiguousarray(samples, ">u2").view(np.uint8).reshape(samples.shape[0], -1).astype(np.int16)
    a = np.zeros_like(raw)
    a[:, BPP:] = raw[:, :-BPP]
    b = np.zeros_like(raw)
    b[1:] = raw[:-1]
    c = np.zeros_like(raw)
    c[1:] = a[:-1]
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    pred = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
    rows = ((raw - pred) & 0xff).astype(np.uint8)
    return np.concatenate([np.full((rows.shape[0], 1), 4, np.uint8), rows], axis=1)


def read_kitti_flow(path):
    """Host reading of a KITTI flow PNG -> float32 (H, W, 2), NaN in both channels at invalid pixels (unquantised)."""
    return read_flow(path, probe(path))


def write_kitti_flow(path, flow_hw2):
    """A float (H, W, 2) flow as a KITTI flow PNG, the bytes run --kitti writes for the same flow; NaN / Inf pixels are invalid."""
    f = np.asarray(flow_hw2, np.float32)
    assert f.ndim == 3 and f.shape[2] == 2, f.shape
    return write_png_rows(path, paeth_rows(encode(f)), f.shape[1], f.shape[0])
