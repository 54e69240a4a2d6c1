"""Flow colour coding on the device (include/fn2_flow.h) against tests/flow_viz_ref.py: fn2_flow_max_radius exactly,
fn2_flow_to_color within one level, fn2_flow_to_color_png_rows against numpy Paeth filtering, and run --visualize,
evaluate --visualize and python -m flownet2_b200.viz end to end."""
import json
import os
import struct
import zlib

import numpy as np
import pytest

from flownet2_b200 import evaluate as E
from flownet2_b200 import files as FI
from flownet2_b200 import kitti as K
from flownet2_b200 import run as R
from flownet2_b200 import viz as V
from tests import flow_viz_ref as ref
from tests.test_kitti_flow_gpu import kitti_scene
from tests.test_run_flownet_gpu import TEMPLATE, chairs_frames, flownet2c, write_list

pytestmark = pytest.mark.gpu


def dev_view(flow_nhw2, layout):
    """(N, H, W, 2) numpy -> a (N, 2, H, W) CUDA view: NCHW, channels_last, or channels 0..1 of a padded NHWC net output."""
    import torch
    f = torch.from_numpy(np.ascontiguousarray(flow_nhw2))
    if layout == "nchw":
        return f.permute(0, 3, 1, 2).contiguous().cuda()
    if layout == "channels_last":
        return f.permute(0, 3, 1, 2).cuda().contiguous(memory_format=torch.channels_last)
    N, H, W, _ = f.shape
    pad = torch.full((N, H, W, 4), float("nan"))
    pad[..., :2] = f
    return pad.cuda().permute(0, 3, 1, 2)[:, :2]


def cases():
    r = np.random.default_rng(11)
    f = (r.standard_normal((4, 19, 33, 2)) * r.choice([0.5, 8.0, 60.0], (4, 1, 1, 1))).astype(np.float32)
    f[1, 2, 3] = (np.nan, 1)
    f[1, 4, 5] = (np.inf, 0)
    f[1, 6, 7] = (0, -np.inf)
    f[1, 8, 9] = (2e9, 1)
    f[1, 9, 9] = (1e9, 0)                                         # exactly at the threshold: known
    f[2] = 0                                                      # all zero: radius 0, scale 1
    f[3] = np.nan                                                 # all unknown: radius -1
    f[3, 0, 0] = (-3e9, 0)
    return f


@pytest.mark.parametrize("layout", ["nchw", "channels_last", "padded"])
def test_max_radius_exact(fn2, layout):
    from flownet2_b200 import ops
    f = cases()
    got = ops.flow_max_radius(dev_view(f, layout)).cpu().numpy()
    want = np.array([ref.max_radius(x) for x in f], np.float32)
    assert np.array_equal(got, want) and got[2] == 0 and got[3] == -1 and got[1] == np.float32(1e9)


def test_max_radius_large_random(fn2):
    from flownet2_b200 import ops
    r = np.random.default_rng(12)
    f = (r.standard_normal((3, 436, 1024, 2)) * 30).astype(np.float32)
    f[1, r.random((436, 1024)) < 0.3] = np.nan
    got = ops.flow_max_radius(dev_view(f, "padded")).cpu().numpy()
    assert np.array_equal(got, np.array([ref.max_radius(x) for x in f], np.float32))


def check_colour(got, want):
    d = np.abs(got.astype(np.int16) - want.astype(np.int16))
    assert d.max() <= 1 and (d == 0).mean() >= 0.999, (d.max(), (d == 0).mean())


@pytest.mark.parametrize("layout", ["nchw", "channels_last", "padded"])
@pytest.mark.parametrize("max_flow", [None, 7.5])
def test_colour_against_restatement(fn2, layout, max_flow):
    from flownet2_b200 import ops
    f = cases()
    got = ops.flow_to_color(dev_view(f, layout), max_flow=max_flow).cpu().numpy()
    want = np.stack([ref.flow_to_color(x, max_flow) for x in f])
    check_colour(got, want)
    unknown = ~ref.known(f)
    assert (got[unknown] == 0).all()
    if max_flow is None:
        assert (got[2] == 255).all()                              # zero flow at scale 1: white
    assert got.shape == (4, 19, 33, 3)


def test_anchors_exact(fn2):
    from flownet2_b200 import ops
    from tests.test_flow_viz_cpu import ANCHORS
    f = np.array([a for a, _ in ANCHORS], np.float32)[None, None]
    got = ops.flow_to_color(dev_view(f, "nchw"), max_flow=1.0).cpu().numpy()[0, 0]
    assert [tuple(int(x) for x in c) for c in got] == [c for _, c in ANCHORS]


def test_rad_one_branch(fn2):
    """Pixels whose float32 radius is exactly 1 at scale 3 take the restatement's rad <= 1 branch: the other branch would scale
    the colour by 0.75, far more than the one level atan2 may move it."""
    from flownet2_b200 import ops
    r = np.random.default_rng(13)
    ang = r.uniform(-np.pi, np.pi, 200000)
    u, v = (3 * np.cos(ang)).astype(np.float32), (3 * np.sin(ang)).astype(np.float32)
    fx, fy = u / np.float32(3), v / np.float32(3)
    at_one = np.sqrt(fx * fx + fy * fy) == np.float32(1)
    assert at_one.sum() > 1000
    f = np.stack([u, v], -1)[at_one][None, None]
    got = ops.flow_to_color(dev_view(f, "nchw"), max_flow=3.0).cpu().numpy()[0, 0]
    want = ref.colour(f[0], np.float32(3))[0]
    check_colour(got, want)


@pytest.mark.parametrize("max_flow", [None, 20.0])
def test_png_rows(fn2, max_flow):
    import flownet2_b200 as F
    from flownet2_b200 import ops
    f = cases()
    dev = dev_view(f, "padded")
    dense = ops.flow_to_color(dev, max_flow=max_flow).cpu().numpy()
    rows = ops.flow_to_color_png_rows(dev, max_flow=max_flow).cpu().numpy()
    N, H, W, _ = dense.shape
    for n in range(N):
        assert np.array_equal(rows[n], ref.paeth_rows(dense[n]))
        out = np.empty(H * W * 3, np.uint8)
        src = np.ascontiguousarray(rows[n])
        assert F.lib().fn2_png_unfilter(src.ctypes.data, H, 3 * W, 3, out.ctypes.data) == 0
        assert np.array_equal(out.reshape(H, W, 3), dense[n])


def test_refusals(fn2):
    import torch
    from flownet2_b200 import ops
    f = torch.zeros((1, 2, 3, 4), device="cuda")
    with pytest.raises(fn2.Fn2Error, match="flow_to_color: max_flow must be 0"):
        ops.flow_to_color(f, max_flow=float("nan"))
    with pytest.raises(fn2.Fn2Error, match="flow_to_color_png_rows: src must have 2 channels"):
        ops.flow_to_color_png_rows(torch.zeros((1, 3, 3, 4), device="cuda"), max_flow=1.0)
    with pytest.raises(fn2.Fn2Error, match="flow_max_radius: src must have 2 channels"):
        ops.flow_max_radius(torch.zeros((1, 1, 3, 4), device="cuda"))
    out = torch.empty(12 * 3, dtype=torch.uint8, device="cuda")
    assert fn2.lib().fn2_flow_to_color(ops.desc(f), None, None, 0.0, out.data_ptr(), None) == -1
    assert "max is null and max_flow is 0" in fn2.lib().fn2_last_error().decode()


# ---- the commands ----
def read_png_rgb(path):
    """An 8-bit RGB PNG written by kitti.png_bytes -> (H, W, 3) uint8, through zlib and the restated Paeth rows."""
    import flownet2_b200 as F
    data = open(path, "rb").read()
    w, h = struct.unpack(">II", data[16:24])
    assert (data[24], data[25]) == (8, 2)                         # bit depth 8, RGB
    raw = np.frombuffer(zlib.decompress(K._idat(path, data)), np.uint8).copy()
    out = np.empty(h * w * 3, np.uint8)
    assert F.lib().fn2_png_unfilter(raw.ctypes.data, int(h), int(3 * w), 3, out.ctypes.data) == 0
    return out.reshape(h, w, 3)


@pytest.fixture(scope="module")
def c_weights(tmp_path_factory, fn2):
    d = tmp_path_factory.mktemp("viz")
    net = flownet2c(fn2, 64, 64, 1)
    path = d / "c.caffemodel"
    path.write_bytes(net.to_caffemodel())
    del net
    return d, str(path)


def frames_list(d, sizes):
    pairs = []
    for i, size in enumerate(sizes):
        f0, f1 = chairs_frames(size, 300 + i)
        pairs.append((size, FI.write_pnm(str(d / ("v%d_0.ppm" % i)), f0), FI.write_pnm(str(d / ("v%d_1.ppm" % i)), f1)))
    return pairs


def test_run_visualize(fn2, c_weights, tmp_path):
    d, weights = c_weights
    pairs = frames_list(tmp_path, [(128, 96), (192, 64), (128, 96), (128, 96), (128, 96), (192, 64)])
    lst = tmp_path / "l.txt"
    for kitti in (False, True):
        outs = write_list(lst, pairs, tmp_path / ("plain%d" % kitti))
        if kitti:
            outs = [o[:-4] + ".png" for o in outs]
            lst.write_text("".join("%s %s %s\n" % (a, b, o) for (_, a, b), o in zip(pairs, outs)))
        flags = ["--kitti"] if kitti else []
        assert R.main([weights, TEMPLATE, str(lst)] + flags) == 0
        plain = [open(o, "rb").read() for o in outs]
        assert not any(os.path.exists(R.vis_path(o)) for o in outs)
        assert R.main([weights, TEMPLATE, str(lst), "--visualize"] + flags) == 0
        assert [open(o, "rb").read() for o in outs] == plain           # the outputs do not change
        for o in outs:
            flow = fn2.read_flo(o).transpose(1, 2, 0) if not kitti else None
            if kitti:                                                 # the float prediction: the .flo run's image
                assert open(R.vis_path(o), "rb").read() == open(R.vis_path(o[:-4].replace("plain1", "plain0") + ".flo"),
                                                                    "rb").read()
                continue
            want = V.write_flow_png(str(tmp_path / "want.png"), flow)
            assert open(R.vis_path(o), "rb").read() == open(want, "rb").read()
            check_colour(read_png_rgb(R.vis_path(o)), ref.flow_to_color(flow))
    # a fixed scale, and batches of 4 with a partial last batch per size: every listed pair gets its image
    outs = write_list(lst, pairs, tmp_path / "b4")
    assert R.main([weights, TEMPLATE, str(lst), "--visualize", "--batch", "4", "--max-flow", "2.5"]) == 0
    for o in outs:
        flow = fn2.read_flo(o).transpose(1, 2, 0)
        assert open(R.vis_path(o), "rb").read() == open(V.write_flow_png(str(tmp_path / "w.png"), flow, 2.5), "rb").read()
    assert sorted(os.listdir(str(tmp_path / "b4"))) == sorted([os.path.basename(o) for o in outs]
                                                               + [os.path.basename(R.vis_path(o)) for o in outs])


def test_evaluate_visualize(fn2, c_weights, tmp_path, capsys):
    d, weights = c_weights
    lists = kitti_scene(tmp_path, [(128, 96), (192, 64), (128, 96)], 700)
    vis = tmp_path / "vis"
    for extra in ([], ["--max-flow", "12"]):
        capsys.readouterr()
        pp0, pp1 = str(tmp_path / "a.tsv"), str(tmp_path / "b.tsv")
        assert E.main([weights, TEMPLATE, lists["flo"], "--per-pair", pp0, "--batch", "2"]) == 0
        assert E.main([weights, TEMPLATE, lists["flo"], "--per-pair", pp1, "--visualize", str(vis), "--batch", "2"] + extra) == 0
        a, b = [json.loads(l) for l in capsys.readouterr().out.strip().splitlines()]
        assert {k: v for k, v in a.items() if k != "wall"} == {k: v for k, v in b.items() if k != "wall"}
        samples = FI.read_list(lists["flo"])
        for k, s in enumerate(samples):
            gt = FI.read_flow(s.flow)
            scale = 12.0 if extra else float(ref.max_radius(gt))
            assert open(str(vis / ("%06d_gt.png" % k)), "rb").read() == \
                open(V.write_flow_png(str(tmp_path / "g.png"), gt, scale), "rb").read()
            pred = read_png_rgb(str(vis / ("%06d_pred.png" % k)))
            assert pred.shape == gt.shape[:2] + (3,)
    assert open(pp0).read() == open(pp1).read()


def test_evaluate_visualize_scale_without_known_truth(fn2, c_weights, tmp_path):
    """Ground truth with no known pixel: both images take the prediction's scale."""
    d, weights = c_weights
    (size, a, b), = frames_list(tmp_path, [(128, 96)])
    gt = str(tmp_path / "g.flo")
    FI.write_flo(gt, np.full((96, 128, 2), np.nan, np.float32))
    lst = tmp_path / "l.txt"
    lst.write_text("%s %s %s\n" % (a, b, gt))
    out = str(tmp_path / "p.flo")
    assert R.main([weights, TEMPLATE, a, b, out]) == 0
    vis = str(tmp_path / "vis")
    with pytest.raises(FI.RunError, match="no ground-truth pixel is valid"):
        E.evaluate(weights, TEMPLATE, FI.read_list(str(lst)), visualize=vis)
    pred = fn2.read_flo(out).transpose(1, 2, 0)
    assert open(os.path.join(vis, "000000_pred.png"), "rb").read() == \
        open(V.write_flow_png(str(tmp_path / "w.png"), pred), "rb").read()
    assert (read_png_rgb(os.path.join(vis, "000000_gt.png")) == 0).all()


def test_viz_command_formats(fn2, tmp_path):
    r = np.random.default_rng(21)
    flow = np.round(r.standard_normal((37, 53, 2)) * 20 * 64) / 64
    flow = flow.astype(np.float32)
    flow[5, 6] = np.nan
    paths = {"flo": str(tmp_path / "f.flo"), "pfm": str(tmp_path / "f.pfm"), "pfm_be": str(tmp_path / "fb.pfm"),
             "kitti": str(tmp_path / "f.png")}
    FI.write_flo(paths["flo"], flow)
    hw3 = np.concatenate([flow, np.zeros_like(flow[..., :1])], -1)
    FI.write_pfm(paths["pfm"], hw3)
    FI.write_pfm(paths["pfm_be"], hw3, big_endian=True)
    K.write_kitti_flow(paths["kitti"], flow)
    want = open(V.write_flow_png(str(tmp_path / "want.png"), flow), "rb").read()
    for k, p in paths.items():
        out = str(tmp_path / ("o_%s.png" % k))
        assert V.main([p, out] + (["--kitti"] if k == "kitti" else [])) == 0
        assert open(out, "rb").read() == want, k
    # a list, two sizes, a partial batch, a fixed scale
    small = flow[:20, :31]
    FI.write_flo(str(tmp_path / "s.flo"), small)
    lst = tmp_path / "l.txt"
    items = [(paths["flo"], "l0.png"), (str(tmp_path / "s.flo"), "l1.png"), (paths["pfm"], "l2.png"), (paths["pfm_be"], "l3.png")]
    lst.write_text("".join("%s %s\n\n" % (f, tmp_path / o) for f, o in items))
    assert V.main([str(lst), "--batch", "2", "--max-flow", "9"]) == 0
    for f, o in items:
        w = open(V.write_flow_png(str(tmp_path / "w.png"), FI.read_flow(f), 9.0), "rb").read()
        assert open(str(tmp_path / o), "rb").read() == w, o
