"""Host side of the image-file driver (flownet2_b200.run): frame readers, list parsing, grouping, sharding, the refusals, and the
C-ABI of include/fn2_frames.h.  No GPU needed."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from flownet2_b200 import files as FI, run as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def write_pnm(path, a, comments=True):
    """Binary PGM (H, W) or PPM (H, W, 3), maxval 255, with comment lines inside the header."""
    magic = b"P5" if a.ndim == 2 else b"P6"
    c = b"# written by the test\n" if comments else b""
    with open(path, "wb") as f:
        f.write(magic + b"\n" + c + b"%d %d\n" % (a.shape[1], a.shape[0]) + c + b"255\n" + np.ascontiguousarray(a, np.uint8).tobytes())
    return str(path)


def frames(seed=0, h=7, w=9):
    r = np.random.default_rng(seed)
    return r.integers(0, 256, (h, w, 3), dtype=np.uint8), r.integers(0, 256, (h, w), dtype=np.uint8)


@pytest.mark.parametrize("gray", [False, True])
def test_pnm_reader_equals_pillow(tmp_path, gray):
    Image = pytest.importorskip("PIL.Image")
    rgb, g = frames(1)
    a = g if gray else rgb
    p = write_pnm(tmp_path / ("f.pgm" if gray else "f.ppm"), a)
    got = FI.read_image(p)
    assert got.dtype == np.uint8 and np.array_equal(got, a)
    assert np.array_equal(got, np.asarray(Image.open(p)))
    assert FI.probe_image(p) == (a.shape[1], a.shape[0], 1 if gray else 3)


def test_pillow_modes_follow_imread(tmp_path):
    Image = pytest.importorskip("PIL.Image")
    rgb, g = frames(2)
    rgba = np.concatenate([rgb, rgb[:, :, :1]], axis=2)
    cases = {"rgb.png": (Image.fromarray(rgb), rgb), "gray.png": (Image.fromarray(g), g), "rgba.png": (Image.fromarray(rgba), rgba),
             "la.png": (Image.fromarray(g).convert("LA"), g),
             "pal.png": (Image.fromarray(rgb).convert("P"), None)}
    for name, (im, want) in cases.items():
        p = str(tmp_path / name)
        im.save(p)
        got = FI.read_image(p)
        if want is None:                                   # palette -> RGB, as the palette maps it
            want = np.asarray(Image.open(p).convert("RGB"))
        assert np.array_equal(got, want), name
        k = 1 if got.ndim == 2 else got.shape[2]
        assert FI.probe_image(p) == (9, 7, k), name


def test_frame_as_is_exact():
    rgb, g = frames(3)
    assert np.array_equal(FI.frame_as(g, 1)[:, :, 0], g)
    assert np.array_equal(FI.frame_as(g, 3), np.stack([g] * 3, axis=2))
    rgba = np.concatenate([rgb, g[:, :, None]], axis=2)
    assert np.array_equal(FI.frame_as(rgba, 3), rgb) and np.array_equal(FI.frame_as(rgba, 4), rgba)


def test_list_parsing(tmp_path):
    p = tmp_path / "list.txt"
    p.write_text("a.ppm b.ppm o1.flo\n\n   \nc.ppm d.ppm o2.flo\n")
    pairs = FI.read_list(str(p), ground_truth=False)
    assert [(x.img0, x.img1, x.flow) for x in pairs] == [("a.ppm", "b.ppm", "o1.flo"), ("c.ppm", "d.ppm", "o2.flo")]
    assert pairs[1].where == "%s:4" % p
    p.write_text("a.ppm b.ppm o1.flo\n\nc.ppm d.ppm\n")
    with pytest.raises(FI.RunError, match=r"list\.txt:3: 2 fields"):
        FI.read_list(str(p), ground_truth=False)
    p.write_text("a b c d\n")
    with pytest.raises(FI.RunError, match=r"list\.txt:1: 4 fields"):
        FI.read_list(str(p), ground_truth=False)


def test_grouping_keeps_first_appearance_order(tmp_path):
    sizes = [(64, 32), (32, 16), (64, 32), (16, 16), (32, 16), (64, 32)]
    pairs = []
    for i, (w, h) in enumerate(sizes):
        rgb = np.zeros((h, w, 3), np.uint8)
        a, b = write_pnm(tmp_path / ("a%d.ppm" % i), rgb), write_pnm(tmp_path / ("b%d.ppm" % i), rgb)
        pairs.append(FI.Pair("l:%d" % i, a, b, "o%d.flo" % i))
    FI.probe(pairs)
    groups = R.group_by_size(pairs)
    assert [s for s, _ in groups] == [(64, 32), (32, 16), (16, 16)]
    assert [[p.where for p in g] for _, g in groups] == [["l:0", "l:2", "l:5"], ["l:1", "l:4"], ["l:3"]]


def test_batches_pad_with_the_last_pair():
    b = R.batches(list("abcde"), 2)
    assert b == [(["a", "b"], 2), (["c", "d"], 2), (["e", "e"], 1)]
    assert R.batches(list("abc"), 1) == [(["a"], 1), (["b"], 1), (["c"], 1)]
    assert R.batches(list("ab"), 4) == [(["a", "b", "b", "b"], 2)]


@pytest.mark.parametrize("world", [1, 2, 3])
def test_sharding_covers_every_line_once(world):
    items = list(range(11))
    shards = [R.shard(items, world, r) for r in range(world)]
    assert sorted(x for s in shards for x in s) == items
    for r, s in enumerate(shards):
        assert all(i % world == r for i in s)


def test_refusals_name_file_and_line(tmp_path, monkeypatch):
    rgb, g = frames(4)
    ok = write_pnm(tmp_path / "ok.ppm", rgb)
    # not 8-bit: a 16-bit PGM
    deep = tmp_path / "deep.pgm"
    deep.write_bytes(b"P5\n9 7\n65535\n" + np.zeros(9 * 7 * 2, np.uint8).tobytes())
    with pytest.raises(FI.RunError, match="deep.pgm: maxval 65535, only 8-bit"):
        FI.read_image(str(deep))
    pairs = [FI.Pair("list.txt:3", str(deep), ok, "o.flo")]
    with pytest.raises(FI.RunError, match=r"list\.txt:3: .*deep\.pgm: maxval 65535"):
        FI.probe(pairs)
    # two channels
    with pytest.raises(FI.RunError, match=r"two\.png: frames of shape \(7, 9, 2\)"):
        FI.check_frame(np.zeros((7, 9, 2), np.uint8), "two.png")
    with pytest.raises(FI.RunError, match=r"f\.png: float32 pixels, only 8-bit"):
        FI.check_frame(np.zeros((7, 9, 3), np.float32), "f.png")
    # sizes differ within a pair
    small = write_pnm(tmp_path / "small.ppm", rgb[:5])
    with pytest.raises(FI.RunError, match=r"list\.txt:7: .*ok\.ppm is 9x7 but .*small\.ppm is 9x5"):
        FI.probe([FI.Pair("list.txt:7", ok, small, "o.flo")])
    # a missing file
    with pytest.raises(FI.RunError, match=r"list\.txt:2: .*nope\.ppm: no such file"):
        FI.probe([FI.Pair("list.txt:2", ok, str(tmp_path / "nope.ppm"), "o.flo")])
    # an unsupported format without Pillow
    png = tmp_path / "x.png"
    png.write_bytes(b"\x89PNG\r\n\x1a\n" + b"\0" * 32)
    monkeypatch.setattr(FI, "_pil", lambda: None)
    with pytest.raises(FI.RunError, match=r"list\.txt:5: .*x\.png: not a binary PGM/PPM, and Pillow is not installed"):
        FI.probe([FI.Pair("list.txt:5", str(png), ok, "o.flo")])
    with pytest.raises(FI.RunError, match=r"x\.png: not a binary PGM/PPM"):
        FI.read_image(str(png))


def test_sixteen_bit_png_is_refused(tmp_path):
    Image = pytest.importorskip("PIL.Image")
    p = str(tmp_path / "deep.png")
    Image.fromarray(np.zeros((7, 9), np.uint16)).save(p)
    with pytest.raises(FI.RunError, match=r"deep\.png: image mode I.* is not an 8-bit"):
        FI.probe_image(p)


def test_main_refuses_before_touching_a_device(tmp_path, capsys):
    rgb, _ = frames(5)
    ok = write_pnm(tmp_path / "ok.ppm", rgb)
    lst = tmp_path / "pairs.txt"
    lst.write_text("%s %s %s\n%s %s\n" % (ok, ok, tmp_path / "o.flo", ok, ok))
    model, proto = tmp_path / "m.caffemodel", tmp_path / "t.template"
    model.write_bytes(b"")
    proto.write_text("")
    assert R.main([str(model), str(proto), str(lst)]) == 2
    assert "pairs.txt:2: 2 fields" in capsys.readouterr().err
    assert R.main([str(tmp_path / "none.caffemodel"), str(proto), ok, ok, "o.flo"]) == 2
    assert "none.caffemodel: no such caffemodel" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        R.parse_args([str(model), str(proto), ok, ok])


def test_truncated_frame_is_refused_before_a_net_is_built(tmp_path, capsys):
    from flownet2_b200 import evaluate as E
    rgb, _ = frames(7)
    ok = write_pnm(tmp_path / "ok.ppm", rgb)
    (tmp_path / "cut.ppm").write_bytes(open(ok, "rb").read()[:-5])
    FI.write_flo(str(tmp_path / "g.flo"), np.zeros((7, 9, 2), np.float32))
    model, proto = tmp_path / "m.caffemodel", tmp_path / "t.template"
    model.write_bytes(b"")
    proto.write_text("")
    lst = tmp_path / "pairs.txt"
    lst.write_text("%s %s %s\n%s %s %s\n" % (ok, ok, tmp_path / "o0.flo", ok, tmp_path / "cut.ppm", tmp_path / "o1.flo"))
    assert R.main([str(model), str(proto), str(lst)]) == 2
    assert re.search(r"pairs\.txt:2: .*cut\.ppm: truncated raster \(184 of 189 bytes\)", capsys.readouterr().err)
    lst.write_text("%s %s %s\n" % (tmp_path / "cut.ppm", ok, tmp_path / "g.flo"))
    assert E.main([str(model), str(proto), str(lst)]) == 2
    assert re.search(r"pairs\.txt:1: .*cut\.ppm: truncated raster", capsys.readouterr().err)


def test_flo_writer_round_trips(fn2, tmp_path):
    flow = np.random.default_rng(6).standard_normal((5, 7, 2)).astype(np.float32)
    p = str(tmp_path / "x.flo")
    FI.write_flo(p, flow)
    raw = open(p, "rb").read()
    assert raw[:4] == b"PIEH" and np.frombuffer(raw[4:12], np.int32).tolist() == [7, 5] and len(raw) == 12 + flow.nbytes
    assert np.array_equal(fn2.read_flo(p), flow.transpose(2, 0, 1))


def test_frames_header_abi(fn2):
    from flownet2_b200 import _abi
    fn2_structs, fn2_h = _abi.read_header(open(os.path.join(ROOT, "include", "fn2.h")).read())
    with pytest.raises(ValueError, match="fn2_tensor"):                 # fn2_tensor comes from fn2.h
        _abi.read_header(open(os.path.join(ROOT, "include", "fn2_frames.h")).read())
    structs, protos = _abi.read_header(open(os.path.join(ROOT, "include", "fn2_frames.h")).read(), {"fn2_tensor": fn2.fn2_tensor})
    assert not structs
    assert sorted(protos) == ["fn2_frames_to_tensor", "fn2_net_get_blob_nhwc", "fn2_net_get_blob_nhwc_device",
                              "fn2_net_set_input_frames", "fn2_net_set_input_frames_device"]
    assert not set(protos) & set(fn2_h) and "fn2_tensor" in fn2_structs
    lib = fn2.lib()
    for name, (restype, argtypes) in protos.items():
        f = getattr(lib, name)                                  # the library exports it
        assert f.restype is restype and f.argtypes == argtypes, name
    T = C.POINTER(fn2.fn2_tensor)
    assert lib.fn2_frames_to_tensor.argtypes == [C.c_void_p, C.c_int, T, C.c_void_p]
    assert lib.fn2_net_set_input_frames.argtypes == [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int]


def test_frames_to_tensor_refusals(fn2):
    """Argument checks run on the host before any launch: they need no device."""
    lib = fn2.lib()
    buf = (C.c_float * 12)()
    t = fn2.fn2_tensor(C.addressof(buf), 1, 3, 2, 2, 12, 4, 2, 1)
    frames = (C.c_uint8 * 16)()
    for k in (0, 2, 5):
        assert lib.fn2_frames_to_tensor(C.addressof(frames), k, t, None) == -1
        assert lib.fn2_last_error().decode() == "frames_to_tensor: channels must be 1, 3 or 4 (gray, RGB, RGBA), got %d" % k
    t4 = fn2.fn2_tensor(C.addressof(buf), 1, 4, 1, 3, 12, 3, 3, 1)
    assert lib.fn2_frames_to_tensor(C.addressof(frames), 3, t4, None) == -1
    assert lib.fn2_last_error().decode() == "frames_to_tensor: dst must have 3 channels (B, G, R), has 4"
    assert lib.fn2_frames_to_tensor(None, 3, t, None) == -1 and "frames is null" in lib.fn2_last_error().decode()
    assert lib.fn2_net_set_input_frames(None, b"img0", C.addressof(frames), 3) == -1
    assert lib.fn2_last_error().decode() == "set_input_frames: null argument"
    assert lib.fn2_net_get_blob_nhwc_device(None, b"x", None) == -1
    assert lib.fn2_last_error().decode() == "get_blob_nhwc_device: null argument"
