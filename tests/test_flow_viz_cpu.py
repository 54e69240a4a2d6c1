"""The flow colour code's restatement (tests/flow_viz_ref.py) at its anchors, its PNG rows through zlib and fn2_png_unfilter,
the 8-bit PNG writer, the KITTI writer's bytes, and the refusals of viz, run --visualize and evaluate --visualize before any
device work."""
import hashlib
import struct
import zlib

import numpy as np
import pytest

from flownet2_b200 import evaluate as E
from flownet2_b200 import kitti as K
from flownet2_b200 import run as R
from flownet2_b200 import viz as V
from tests import flow_viz_ref as ref
from tests.test_run_flownet_cpu import write_pnm


def test_wheel_segments():
    w = ref.wheel()
    assert w.shape == (55, 3)
    starts = np.cumsum([0] + [n for _, n in ref.SEGMENTS])
    first = {"RY": (255, 0, 0), "YG": (255, 255, 0), "GC": (0, 255, 0), "CB": (0, 255, 255), "BM": (0, 0, 255),
             "MR": (255, 0, 255)}
    last = {"RY": (255, 238, 0), "YG": (43, 255, 0), "GC": (0, 255, 191), "CB": (0, 24, 255), "BM": (235, 0, 255),
            "MR": (255, 0, 43)}
    for (name, _), a, b in zip(ref.SEGMENTS, starts[:-1], starts[1:]):
        assert tuple(w[a]) == first[name] and tuple(w[b - 1]) == last[name], name


# (u, v) at scale 1 -> RGB.  (0, -1) is 87, not the 88 a float64 evaluation gives: in float32 1 - (1 - 88/255) rounds to
# just below 88/255.
ANCHORS = [((0, 0), (255, 255, 255)), ((1, 0), (255, 0, 0)), ((-1, 0), (0, 209, 255)), ((0, -1), (87, 0, 255)),
           ((0, 1), (255, 229, 0)), ((0.5, 0), (255, 127, 127)), ((2, 0), (191, 0, 0)), ((np.nan, 0), (0, 0, 0)),
           ((0, np.nan), (0, 0, 0)), ((2e9, 0), (0, 0, 0)), ((0, 2e9), (0, 0, 0)), ((np.inf, 0), (0, 0, 0))]


def test_anchors():
    flow = np.array([a for a, _ in ANCHORS], np.float32)[None]
    got = ref.colour(flow, np.float32(1))[0]
    assert [tuple(int(x) for x in c) for c in got] == [c for _, c in ANCHORS]


def test_scale():
    f = np.zeros((3, 4, 2), np.float32)
    assert ref.max_radius(f) == 0 and ref.scale_of(f) == 1
    f[1, 2] = (3, 4)
    f[0, 0] = (np.nan, 100)
    f[0, 1] = (2e9, 0)
    assert ref.max_radius(f) == 5 and ref.scale_of(f) == 5 and ref.scale_of(f, 2.5) == np.float32(2.5)
    assert ref.max_radius(np.full((2, 2, 2), np.nan, np.float32)) == -1


def test_png_rows_round_trip():
    import flownet2_b200 as F
    r = np.random.default_rng(4)
    flow = (r.standard_normal((17, 29, 2)) * 5).astype(np.float32)
    flow[3, 3] = np.nan
    rgb = ref.flow_to_color(flow)
    rows = ref.paeth_rows(rgb)
    assert rows.shape == (17, 1 + 3 * 29) and (rows[:, 0] == 4).all()
    raw = np.frombuffer(zlib.decompress(zlib.compress(rows.tobytes())), np.uint8).copy()
    out = np.empty(17 * 29 * 3, np.uint8)
    assert F.lib().fn2_png_unfilter(raw.ctypes.data, 17, 29 * 3, 3, out.ctypes.data) == 0
    assert np.array_equal(out.reshape(17, 29, 3), rgb)


def test_8bit_png_writer(tmp_path):
    r = np.random.default_rng(5)
    rgb = r.integers(0, 256, (9, 13, 3), dtype=np.uint8)
    path = K.write_png_rows(str(tmp_path / "c.png"), ref.paeth_rows(rgb), 13, 9, 8)
    data = open(path, "rb").read()
    assert data[:8] == K.SIGNATURE
    n, kind = struct.unpack(">I4s", data[8:16])
    assert (n, kind) == (13, b"IHDR")
    assert struct.unpack(">IIBBBBB", data[16:29]) == (13, 9, 8, 2, 0, 0, 0)
    assert struct.unpack(">I", data[29:33])[0] == zlib.crc32(data[12:29])
    try:
        from PIL import Image
    except ImportError:
        return
    with Image.open(path) as im:
        assert im.mode == "RGB" and np.array_equal(np.asarray(im), rgb)


def test_kitti_png_bytes_unchanged(tmp_path):
    """The 16-bit writer is the 8-bit one's twin; its bytes for this flow were hashed before the two were one function."""
    r = np.random.default_rng(7)
    f = (r.standard_normal((23, 37, 2)) * 40).astype(np.float32)
    f[3, 4] = np.nan
    f[5, 6, 1] = np.inf
    f[0, 0] = 1e6
    path = K.write_kitti_flow(str(tmp_path / "k.png"), f)
    digest = hashlib.sha256(open(path, "rb").read()).hexdigest()
    assert digest == "c510576bfc6af318af37973616a84ffaa08bc8f5b249a1764fd040372ad0187e"


# ---- refusals, before any device work ----
@pytest.fixture
def no_device(monkeypatch):
    """Fails a test that reaches the device."""
    def boom(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(R, "run_groups", boom)
    monkeypatch.setattr(E, "run_groups", boom)
    monkeypatch.setattr(V, "_colour_size", boom)
    import torch
    monkeypatch.setattr(torch.cuda, "set_device", boom)


@pytest.mark.parametrize("value", ["0", "nan", "-1", "inf"])
def test_max_flow_refused(tmp_path, capsys, no_device, value):
    flo = str(tmp_path / "f.flo")
    from flownet2_b200.files import write_flo
    write_flo(flo, np.zeros((4, 5, 2), np.float32))
    assert V.main([flo, str(tmp_path / "o.png"), "--max-flow", value]) == 2
    assert R.main(["w", "t", "a", "b", "o.flo", "--visualize", "--max-flow", value]) == 2
    assert E.main(["w", "t", "l", "--visualize", str(tmp_path), "--max-flow", value]) == 2
    err = capsys.readouterr().err.strip().splitlines()
    assert len(err) == 3 and all("--max-flow must be a finite positive number" in e for e in err)


def test_viz_missing_file_refused(tmp_path, capsys, no_device):
    assert V.main([str(tmp_path / "none.flo"), str(tmp_path / "o.png")]) == 2
    lst = tmp_path / "l.txt"
    lst.write_text("%s %s\n" % (tmp_path / "none.pfm", tmp_path / "o.png"))
    assert V.main([str(lst)]) == 2
    assert V.main([str(tmp_path / "none.txt")]) == 2
    lst.write_text("a b c\n")
    assert V.main([str(lst)]) == 2
    err = capsys.readouterr().err.strip().splitlines()
    assert len(err) == 4
    assert "none.flo: no such file" in err[0] and "l.txt:1: " in err[1] and "none.pfm: no such file" in err[1]
    assert "no such list file" in err[2] and "3 fields, expected 'flow out.png'" in err[3]


def test_run_colliding_vis_paths_refused(tmp_path, capsys, no_device):
    a = write_pnm(tmp_path / "a.ppm", np.zeros((8, 8, 3), np.uint8))
    b = write_pnm(tmp_path / "b.ppm", np.zeros((8, 8, 3), np.uint8))
    w, t = tmp_path / "w.caffemodel", tmp_path / "t.template"
    w.write_bytes(b"")
    t.write_text("")
    lst = tmp_path / "l.txt"
    for outs, what in ((("x.flo", "x.png"), "both visualise to"), (("y.flo", "y.vis.png"), "is the output of")):
        lst.write_text("".join("%s %s %s\n" % (a, b, tmp_path / o) for o in outs))
        assert R.main([str(w), str(t), str(lst), "--visualize"]) == 2
        err = capsys.readouterr().err
        assert what in err and err.count("\n") == 1
        with pytest.raises(R.RunError, match=what):
            R.run(str(w), str(t), R.read_list(str(lst), ground_truth=False), visualize=True)
    lst.write_text("%s %s %s\n%s %s %s\n" % (a, b, tmp_path / "z.flo", a, b, tmp_path / "z.flo"))
    R.check_vis_paths(R.read_list(str(lst), ground_truth=False))          # one output listed twice: one image
