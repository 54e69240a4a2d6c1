"""Host side of KITTI flow PNGs (flownet2_b200.kitti): fn2_png_unfilter against a pure-Python restatement, the decoder against
Pillow's 8-bit view of files whose rows use every filter, the module's writer read back by Pillow and by itself, the
container's accepted and refused cases, and the --kitti list handling of evaluate and train.  No GPU needed."""
import re
import struct
import zlib

import numpy as np
import pytest

import flownet2_b200 as F
from flownet2_b200 import data as D, evaluate as E, feed as FD, files as FI, kitti as K, train as T
from flownet2_b200.files import RunError, write_flo
from tests.test_run_flownet_cpu import write_pnm

Image = pytest.importorskip("PIL.Image")


# ---- a test-side PNG encoder: any filter per row, any chunk layout ----
def paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else b if pb <= pc else c


def filter_row(ftype, raw, prev, bpp):
    """PNG's forward filter of one row of raw bytes (lists of ints) against the raw row above."""
    out = []
    for i, x in enumerate(raw):
        a = raw[i - bpp] if i >= bpp else 0
        b = prev[i]
        c = prev[i - bpp] if i >= bpp else 0
        pred = [0, a, b, (a + b) // 2, paeth(a, b, c)][ftype]
        out.append((x - pred) & 0xff)
    return [ftype] + out


def unfilter_ref(data, rows, row_bytes, bpp):
    """Pure-Python restatement of fn2_png_unfilter."""
    out, prev = [], [0] * row_bytes
    for y in range(rows):
        f = data[y * (row_bytes + 1)]
        s = data[y * (row_bytes + 1) + 1:(y + 1) * (row_bytes + 1)]
        cur = []
        for i, x in enumerate(s):
            a = cur[i - bpp] if i >= bpp else 0
            b = prev[i]
            c = prev[i - bpp] if i >= bpp else 0
            cur.append((x + [0, a, b, (a + b) // 2, paeth(a, b, c)][f]) & 0xff)
        out += cur
        prev = cur
    return bytes(out)


def chunk(kind, body, crc=None):
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body) if crc is None else crc)


def ihdr(w, h, depth=16, colour=2, interlace=0):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, colour, 0, 0, interlace))


def encode_png(samples, filters, idat_parts=1, extra=(), ihdr_chunk=None):
    """(H, W, 3) uint16 samples -> PNG bytes whose row y uses filters[y % len(filters)], the stream split over idat_parts
    IDATs, `extra` chunks after IHDR."""
    h, w = samples.shape[:2]
    raw = np.ascontiguousarray(samples, ">u2").view(np.uint8).reshape(h, -1).tolist()
    rows, prev = [], [0] * (6 * w)
    for y in range(h):
        rows += filter_row(filters[y % len(filters)], raw[y], prev, 6)
        prev = raw[y]
    z = zlib.compress(bytes(rows))
    cut = [len(z) * i // idat_parts for i in range(idat_parts + 1)]
    return (K.SIGNATURE + (ihdr_chunk or ihdr(w, h)) + b"".join(extra)
            + b"".join(chunk(b"IDAT", z[cut[i]:cut[i + 1]]) for i in range(idat_parts)) + chunk(b"IEND", b""))


def samples_of(seed, h=9, w=13):
    r = np.random.default_rng(seed)
    s = r.integers(0, 65536, (h, w, 3)).astype(np.uint16)
    s[0, :4] = [[0, 0, 0], [32767, 32768, 1], [65535, 65535, 65535], [32768, 0, 0]]
    return s


def payload_of(path):
    info = K.probe(str(path))
    buf = np.empty(info.nbytes, np.uint8)
    K.read_payload(str(path), info, buf)
    return buf.view(">u2").reshape(info.height, info.width, 3)


# ---- fn2_png_unfilter ----
@pytest.mark.parametrize("filters", [[0], [1], [2], [3], [4], [4, 0, 3, 1, 2, 4, 3]])
@pytest.mark.parametrize("bpp", [1, 3, 6])
def test_unfilter_equals_restatement(fn2, filters, bpp):
    r = np.random.default_rng(bpp * 10 + len(filters))
    rows, row_bytes = 7, 6 * 5
    raw = r.integers(0, 256, (rows, row_bytes)).tolist()
    data, prev = [], [0] * row_bytes
    for y in range(rows):
        data += filter_row(filters[y % len(filters)], raw[y], prev, bpp)
        prev = raw[y]
    data = bytes(data)
    src = np.frombuffer(data, np.uint8)
    dst = np.full(rows * row_bytes, 0xaa, np.uint8)
    assert fn2.lib().fn2_png_unfilter(src.ctypes.data, rows, row_bytes, bpp, dst.ctypes.data) == 0
    assert dst.tobytes() == unfilter_ref(data, rows, row_bytes, bpp) == bytes(np.array(raw, np.uint8).tobytes())


def test_unfilter_refuses_filter_type_5(fn2):
    data = np.frombuffer(bytes([0] + [1] * 6 + [5] + [1] * 6), np.uint8)
    dst = np.zeros(12, np.uint8)
    assert fn2.lib().fn2_png_unfilter(data.ctypes.data, 2, 6, 6, dst.ctypes.data) == -1
    assert fn2.lib().fn2_last_error().decode() == "png_unfilter: row 1 has filter type 5 (PNG defines 0 to 4)"


# ---- the decoder against Pillow ----
@pytest.mark.parametrize("filters", [[0, 1, 2, 3, 4], [4, 3, 2, 1, 0, 4, 4, 3]])
def test_decoder_high_and_low_bytes_equal_pillow(tmp_path, filters):
    s = samples_of(1)
    for name, img, shift in (("hi", s, 8), ("lo", s.byteswap(), 0)):
        p = tmp_path / ("%s.png" % name)
        p.write_bytes(encode_png(img, filters))
        got = payload_of(p)
        assert np.array_equal(got, img)
        with Image.open(str(p)) as im:
            assert im.mode == "RGB" and im.size == (13, 9)
            view8 = np.asarray(im)                                           # Pillow keeps each sample's high byte
        # the twin's high bytes are the image's low bytes
        assert np.array_equal(view8, ((got >> 8) & 0xff).astype(np.uint8))
        assert np.array_equal(view8, ((s >> shift) & 0xff).astype(np.uint8))


def test_writer_round_trip_and_pillow(tmp_path):
    r = np.random.default_rng(3)
    f = (r.standard_normal((21, 34, 2)) * 100).astype(np.float32)
    f[0, :8] = [[600, 0], [-600, 1], [511.99, -512], [np.nan, 0], [0, np.inf], [-np.inf, -np.inf], [1e30, 0], [0.0078, -0.0078]]
    f[5, 5] = [np.nan, np.nan]
    p = K.write_kitti_flow(str(tmp_path / "f.png"), f)
    with Image.open(p) as im:
        assert im.mode == "RGB" and im.size == (34, 21)
        view8 = np.asarray(im)
    s = payload_of(p)
    assert np.array_equal(view8, (s >> 8).astype(np.uint8))
    g = K.read_kitti_flow(p)
    ok = np.isfinite(f).all(axis=2)
    assert np.array_equal(np.isnan(g).all(axis=2), ~ok) and not np.isnan(g[ok]).any()
    with np.errstate(over="ignore"):
        want = np.floor(np.clip(f[ok] * np.float32(64) + np.float32(32768), 0, 65535)).astype(np.float64)
    assert np.array_equal(g[ok].astype(np.float64) * 64 + 32768, want)
    assert np.array_equal(s[~ok], np.zeros((int((~ok).sum()), 3))) and (s[ok][:, 2] == 1).all()
    assert list(s[0, 0]) == [65535, 32768, 1] and list(s[0, 1]) == [0, 32832, 1] and list(s[0, 2, :2]) == [65535, 0]
    rows = np.frombuffer(zlib.decompress(_chunks(open(p, "rb").read())[b"IDAT"]), np.uint8).reshape(21, -1)
    assert (rows[:, 0] == 4).all()                                           # every row Paeth-filtered


def _chunks(data):
    out, pos = {}, 8
    while pos < len(data):
        n, kind = struct.unpack(">I4s", data[pos:pos + 8])
        out[kind] = out.get(kind, b"") + data[pos + 8:pos + 8 + n]
        pos += 12 + n
    return out


# ---- the container ----
def test_accepts_multiple_idats_and_skips_ancillary_chunks(tmp_path):
    s = samples_of(5)
    p = tmp_path / "ok.png"
    extra = (chunk(b"tEXt", b"Comment\0kitti"), chunk(b"gAMA", b"\0\0\xb1\x8f", crc=1), chunk(b"PLTE", b"\0" * 9))
    p.write_bytes(encode_png(s, [4, 1], idat_parts=5, extra=extra))
    assert np.array_equal(payload_of(p), s)
    info = K.probe(str(p))
    assert (info.width, info.height, info.nbytes, info.format) == (13, 9, 13 * 9 * 6, F.FLOW_KITTI)


def refusals():
    """(name, bytes, message) of files the module refuses, and whether the probe alone refuses them."""
    s = samples_of(7)
    good = encode_png(s, [2])
    i_idat = good.index(b"IDAT") - 4
    i_iend = good.index(b"IEND") - 4
    bad_crc_idat = bytearray(good)
    bad_crc_idat[i_iend - 1] ^= 0xff
    bad_crc_ihdr = bytearray(good)
    bad_crc_ihdr[20] ^= 0x01
    garbled = bytearray(good)
    garbled[i_idat + 8:i_idat + 12] = b"\xff\xff\xff\xff"
    garbled[i_iend - 4:i_iend] = struct.pack(">I", zlib.crc32(bytes(garbled[i_idat + 4:i_iend - 4])))
    return [
        ("sig", b"\x89PNX" + good[4:], r"not a PNG file \(signature\)", True),
        ("crc_ihdr", bytes(bad_crc_ihdr), r"CRC mismatch in chunk IHDR", True),
        ("crc_idat", bytes(bad_crc_idat), r"CRC mismatch in chunk IDAT", False),
        ("interlaced", encode_png(s, [0], ihdr_chunk=ihdr(13, 9, interlace=1)), r"an interlaced PNG", True),
        ("rgb8", encode_png(s, [0], ihdr_chunk=ihdr(13, 9, depth=8)), r"PNG colour type 2 at bit depth 8", True),
        ("grey16", encode_png(s, [0], ihdr_chunk=ihdr(13, 9, colour=0)), r"PNG colour type 0 at bit depth 16", True),
        ("palette", encode_png(s, [0], ihdr_chunk=ihdr(13, 9, depth=8, colour=3)), r"PNG colour type 3 at bit depth 8", True),
        ("short", good[:20], r"truncated PNG header", True),
        ("cut", good[:i_idat + 30], r"truncated PNG \(chunk b'IDAT'", False),
        ("no_iend", good[:i_iend], r"truncated PNG \(no IEND chunk\)", False),
        ("no_idat", good[:i_idat] + chunk(b"IEND", b""), r"no IDAT chunk", False),
        ("critical", good[:i_idat] + chunk(b"XYZW", b"1") + good[i_idat:], r"unknown critical PNG chunk b'XYZW'", False),
        ("garbled", bytes(garbled), r"the PNG data does not inflate", False),
        ("small", encode_png(s, [0], ihdr_chunk=ihdr(13, 10)), r"the PNG data inflates to 711 bytes, a 13x10 image has 790", False),
        ("filter", K.SIGNATURE + ihdr(13, 9) + chunk(b"IDAT", zlib.compress(bytes([7] + [0] * 78) * 9)) + chunk(b"IEND", b""),
         r"png_unfilter: row 0 has filter type 7", False),
    ]


def test_refusals_name_the_file(tmp_path):
    for name, data, msg, at_probe in refusals():
        p = tmp_path / ("%s.png" % name)
        p.write_bytes(data)
        with pytest.raises(RunError, match=re.escape(str(p)) + ": " + msg):
            if at_probe:
                K.probe(str(p))
            else:
                payload_of(p)
        if not at_probe:
            K.probe(str(p))                                                  # the header alone is fine


def kitti_list(tmp_path, n=3, size=(13, 9), bad=None):
    """n lines of PPM frames and KITTI flows (plus each flow's .flo twin) -> (list path, [png], [flo])."""
    r = np.random.default_rng(11)
    w, h = size
    lines, pngs, flos = [], [], []
    for i in range(n):
        a = write_pnm(tmp_path / ("a%d.ppm" % i), r.integers(0, 256, (h, w, 3), dtype=np.uint8))
        b = write_pnm(tmp_path / ("b%d.ppm" % i), r.integers(0, 256, (h, w, 3), dtype=np.uint8))
        f = (r.standard_normal((h, w, 2)) * 20).astype(np.float32)
        f[r.random((h, w)) < 0.3] = np.nan
        png = K.write_kitti_flow(str(tmp_path / ("g%d.png" % i)), f)
        flo = str(tmp_path / ("g%d.flo" % i))
        write_flo(flo, K.read_kitti_flow(png))
        lines.append("%s %s %s\n" % (a, b, bad if bad and i == n - 1 else png))
        pngs.append(png)
        flos.append(flo)
    p = tmp_path / "kitti.txt"
    p.write_text("".join(lines))
    return str(p), pngs, flos


def test_refusals_name_the_list_line(tmp_path):
    bad = tmp_path / "interlaced.png"
    bad.write_bytes(encode_png(samples_of(1), [0], ihdr_chunk=ihdr(13, 9, interlace=1)))
    lst, _, _ = kitti_list(tmp_path, bad=str(bad))
    with pytest.raises(RunError, match=r"kitti\.txt:3: .*interlaced\.png: an interlaced PNG"):
        D.FlowDataset(lst, 2, kitti=True)
    samples = FI.read_list(lst)
    with pytest.raises(RunError, match=r"kitti\.txt:3: .*interlaced\.png: an interlaced PNG"):
        FI.probe(samples, ground_truth=True, kitti=True)
    # a file whose header is fine and whose data is not: refused by the read, naming the line
    crc = tmp_path / "crc.png"
    good = bytearray(encode_png(samples_of(1), [4]))
    good[good.index(b"IEND") - 5] ^= 0xff
    crc.write_bytes(bytes(good))
    lst, _, _ = kitti_list(tmp_path, bad=str(crc))
    samples = FI.read_list(lst)
    FI.probe(samples, ground_truth=True, kitti=True)
    with pytest.raises(RunError, match=r"kitti\.txt:3: .*crc\.png: CRC mismatch in chunk IDAT"):
        FD.read_part(samples[2], 2, (13, 9), 3, np.empty(13 * 9 * 12, np.uint8))


def test_evaluate_kitti_list(tmp_path, capsys):
    assert E.parse_args(["w", "t", "l"]).kitti is False and E.parse_args(["w", "t", "l", "--kitti"]).kitti is True
    lst, pngs, flos = kitti_list(tmp_path)
    samples = FI.read_list(lst)
    FI.probe(samples, ground_truth=True, kitti=True)
    assert [s.flow_header.nbytes for s in samples] == [13 * 9 * 6] * 3
    out = np.empty(13 * 9 * 12, np.uint8)
    FD.read_part(samples[0], 2, (13, 9), 3, out)
    assert np.array_equal(out[:13 * 9 * 6], payload_of(pngs[0]).astype(">u2").view(np.uint8).reshape(-1))
    model, proto = tmp_path / "m.caffemodel", tmp_path / "t.template"
    model.write_bytes(b"")
    proto.write_text("")
    # a .flo in a --kitti list, and a KITTI PNG without --kitti, are refused naming the line
    (tmp_path / "mixed.txt").write_text(open(lst).read().replace(pngs[1], flos[1]))
    assert E.main([str(model), str(proto), str(tmp_path / "mixed.txt"), "--kitti"]) == 2
    assert re.search(r"mixed\.txt:2: .*g1\.flo: not a PNG file \(signature\)", capsys.readouterr().err)
    assert E.main([str(model), str(proto), lst]) == 2
    assert re.search(r"kitti\.txt:1: .*g0\.png: flows must be \.flo or \.pfm files", capsys.readouterr().err)


def test_train_kitti_list(tmp_path):
    assert T.parse_args(["--solver", "s", "--model", "m", "--data", "d", "--crop", "8x8", "--batch", "1"]).kitti is False
    a = T.parse_args(["--solver", "s", "--model", "m", "--data", "d", "--crop", "8x8", "--batch", "1", "--kitti"])
    assert a.kitti is True
    lst, pngs, flos = kitti_list(tmp_path, n=4)
    for enc in ("uint16", "float"):
        ds = D.FlowDataset(lst, 2, flow_encoding=enc, kitti=True)
        assert ds.size == (13, 9) and ds.flow_format == F.FLOW_KITTI and FI.FLOW_PX_BYTES[ds.flow_format] == 6
        twin = tmp_path / "twin.txt"
        twin.write_text("".join(l.replace(p, f) for l, p, f in zip(open(lst).readlines(), pngs, flos)))
        ref = D.FlowDataset(str(twin), 2, flow_encoding=enc)
        assert ds.perm == ref.perm
        for k in range(3):
            got, want = ds.host_batch(k)[2], ref.host_batch(k)[2]
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (enc, k)
    with pytest.raises(RunError, match=r"flows must be \.flo or \.pfm files"):
        D.FlowDataset(lst, 2)
    # one size per training list
    (tmp_path / "o").mkdir()
    other, _, _ = kitti_list(tmp_path / "o", n=1, size=(14, 9))
    mixed = tmp_path / "mixed.txt"
    mixed.write_text(open(lst).read() + open(other).read())
    with pytest.raises(RunError, match=r"mixed\.txt:5: .*a0\.ppm is 14x9, the other files are 13x9"):
        D.FlowDataset(str(mixed), 2, kitti=True)
