"""GPU: fn2_occlusion_boundary_dist2 and fn2_flow_error_regions (include/fn2_eval.h, ops) against the numpy restatement in
tests/flow_region_ref.py -- the distance equal everywhere, the region records' counts exact and sums within 1e-12 relative --,
the invariants that tie the region records to fn2_flow_error's, bit-identical repeats, the refusals, and the evaluate command
with --occlusions and --objects end to end."""
import ctypes as C
import json
import os

import numpy as np
import pytest
from scipy import ndimage

from flownet2_b200 import DIST2_NONE, FLOW_ERROR_FIELDS, FLOW_REGION_FIELDS
from flownet2_b200 import evaluate as E
from flownet2_b200 import run as R
from flownet2_b200.files import read_flow, read_list, write_flo
from tests.flow_error_ref import flow_error_ref
from tests.flow_region_ref import assert_region_match, dist2_ref, flow_region_ref
from tests.test_evaluate_gpu import ground_truth
from tests.test_flow_error_gpu import seeded_flows
from tests.test_run_flownet_cpu import write_pnm
from tests.test_run_flownet_gpu import chairs_frames

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELD = {f: i for i, f in enumerate(FLOW_ERROR_FIELDS)}
REGION = {f: i for i, f in enumerate(FLOW_REGION_FIELDS)}


def blobs(n, h, w, seed, sigma=6.0, level=0.4):
    """(n, h, w) uint8 masks of smooth random blobs, the occluded bytes any of 1..255."""
    r = np.random.default_rng(seed)
    out = np.zeros((n, h, w), np.uint8)
    for i in range(n):
        field = ndimage.gaussian_filter(r.standard_normal((h, w)), sigma, mode="wrap")
        on = field > level * field.std()
        out[i][on] = r.integers(1, 256, int(on.sum()))
    return out


def dist2_op(masks, pair_stride=None):
    """The op on (N, H, W) masks, laid out at pair_stride bytes (filler bytes between the planes) when given."""
    import torch
    from flownet2_b200 import ops
    n, h, w = masks.shape
    stride = pair_stride or h * w
    buf = np.full(n * stride, 0xA5, np.uint8)
    for i in range(n):
        buf[i * stride:i * stride + h * w] = masks[i].reshape(-1)
    out = torch.full((n, h, w), -7, dtype=torch.int32, device="cuda")
    ops.occlusion_boundary_dist2(torch.from_numpy(buf).cuda(), out=out, pair_stride=stride)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def checkerboard(h, w):
    return (np.indices((1, h, w)).sum(axis=0) % 2).astype(np.uint8)


def single_pixel():
    m = np.zeros((1, 64, 80), np.uint8)
    m[0, 17, 61] = 1
    return m


def clear_and_occluded():
    return np.stack([np.zeros((20, 30), np.uint8), np.full((20, 30), 200, np.uint8)])


def wide_rows():
    m = np.zeros((3, 16384), np.uint8)
    m[:, 5000:5003] = 1                                                 # the boundary in a few columns: the envelope spans the row
    m[1, 16000:] = 9
    return m[None]


MASKS = {
    "sintel": lambda: blobs(3, 436, 1024, 1),
    "kitti": lambda: blobs(1, 375, 1242, 2, sigma=12.0),
    "row": lambda: blobs(2, 1, 300, 3, sigma=4.0),
    "column": lambda: blobs(2, 300, 1, 4, sigma=4.0),
    "pixel": single_pixel,
    "checker": lambda: checkerboard(33, 47),
    "flat": clear_and_occluded,
    "w16384": wide_rows,
    "h16384": lambda: wide_rows().transpose(0, 2, 1).copy(),
    "sparse": lambda: (np.random.default_rng(5).random((2, 200, 260)) < 0.0005).astype(np.uint8),
}


@pytest.mark.parametrize("case", sorted(MASKS))
def test_dist2_equals_restatement(fn2, case):
    masks = MASKS[case]()
    want = dist2_ref(masks)
    got = dist2_op(masks)
    assert np.array_equal(got, want), (case, np.argwhere(got != want)[:5])
    if case == "flat":
        assert np.all(got == DIST2_NONE)
    if case == "checker":
        assert np.all(got == 0)


def test_dist2_pair_stride(fn2):
    masks = blobs(3, 45, 71, 6)
    want = dist2_ref(masks)
    assert np.array_equal(dist2_op(masks, pair_stride=45 * 71 + 37), want)        # odd, unaligned stride
    assert np.array_equal(dist2_op(masks, pair_stride=2 * 45 * 71), want)


def test_dist2_refusals(fn2):
    import torch
    lib = fn2.lib()
    buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
    out = torch.zeros(64, dtype=torch.int32, device="cuda")
    optr = C.cast(out.data_ptr(), C.POINTER(C.c_int32))
    call = lambda stride, n, h, w: lib.fn2_occlusion_boundary_dist2(buf.data_ptr(), stride, n, h, w, optr, None)
    assert call(8 * 8, 1, 8, 8) == 0
    assert call(16385, 1, 1, 16385) == -1 and "at most 16384" in lib.fn2_last_error().decode()
    assert call(16385, 1, 16385, 1) == -1
    assert call(1, 65536, 1, 1) == -1 and "65535" in lib.fn2_last_error().decode()
    assert call(63, 1, 8, 8) == -1 and "pair stride 63 is below H * W = 64" in lib.fn2_last_error().decode()
    assert lib.fn2_occlusion_boundary_dist2(None, 64, 1, 8, 8, optr, None) == -1
    assert lib.fn2_occlusion_boundary_dist2(buf.data_ptr(), 64, 1, 8, 8, None, None) == -1
    torch.cuda.synchronize()


# ---- region records ----
def regions_op(pred, gt, occ, obj, mask_stride=None):
    """fn2_flow_error_regions and fn2_flow_error on device copies -> (region records, error records)."""
    import torch
    from flownet2_b200 import ops
    n, _, h, w = pred.shape
    p, g = torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda()
    stride = mask_stride or h * w

    def planes(m):
        if m is None:
            return None
        buf = np.full(n * stride, 0x5A, np.uint8)
        for i in range(n):
            buf[i * stride:i * stride + h * w] = m[i].reshape(-1)
        return torch.from_numpy(buf).cuda()

    o, b = planes(occ), planes(obj)
    d2 = None
    if o is not None:
        d2 = ops.occlusion_boundary_dist2(o, out=torch.empty((n, h, w), dtype=torch.int32, device="cuda"), pair_stride=stride)
    reg = ops.flow_error_regions(p, g, occ=o, obj=b, dist2=d2, mask_pair_stride=stride)
    err = ops.flow_error(p, g)
    torch.cuda.synchronize()
    return reg.cpu().numpy(), err.cpu().numpy()


def check_invariants(reg, err, occ=True, obj=True):
    col = lambda f: reg[:, REGION[f]]
    counted = err[:, FIELD["valid"]] - err[:, FIELD["nonfinite"]]
    if occ:
        assert np.array_equal(col("n_matched") + col("n_unmatched"), counted)
        assert np.all(col("n_d0_10") + col("n_d10_60") + col("n_d60_140") <= counted)
        out = col("out_matched") + col("out_unmatched")
        assert np.array_equal(out, err[:, FIELD["outliers"]])
    if obj:
        assert np.array_equal(col("n_bg") + col("n_fg"), counted)
        assert np.array_equal(col("out_bg") + col("out_fg"), err[:, FIELD["outliers"]])


@pytest.mark.parametrize("shape", [(1, 7, 13), (3, 37, 61), (3, 436, 1024), (2, 375, 1242)])
def test_regions_match_restatement(fn2, shape):
    n, h, w = shape
    pred, gt = seeded_flows(n, h, w, seed=h + w)                        # planted NaN / Inf / 1e10 ground truth and predictions
    occ, obj = blobs(n, h, w, 7, sigma=min(6.0, h / 4)), blobs(n, h, w, 8, sigma=min(9.0, h / 4))
    want = flow_region_ref(pred, gt, occ, obj)
    got, err = regions_op(pred, gt, occ, obj)
    assert_region_match(got, want)
    check_invariants(got, err)
    again, _ = regions_op(pred, gt, occ, obj)
    assert np.array_equal(got.view(np.uint64), again.view(np.uint64))              # bit-identical repeat
    strided, _ = regions_op(pred, gt, occ, obj, mask_stride=h * w + 13)
    assert np.array_equal(got.view(np.uint64), strided.view(np.uint64))
    if h > 100:
        assert all(got[:, REGION["n_d10_60"]] > 0) and all(got[:, REGION["n_unmatched"]] > 0)


def test_regions_one_mask_or_none(fn2):
    n, h, w = 2, 40, 90
    pred, gt = seeded_flows(n, h, w, seed=11)
    occ, obj = blobs(n, h, w, 9), blobs(n, h, w, 10)
    only_occ, err = regions_op(pred, gt, occ, None)
    assert_region_match(only_occ, flow_region_ref(pred, gt, occ, None))
    check_invariants(only_occ, err, obj=False)
    assert np.all(only_occ[:, REGION["n_bg"]:] == 0)
    only_obj, _ = regions_op(pred, gt, None, obj)
    assert_region_match(only_obj, flow_region_ref(pred, gt, None, obj))
    assert np.all(only_obj[:, :REGION["n_bg"]] == 0)
    both, _ = regions_op(pred, gt, occ, obj)
    assert np.array_equal(both[:, :REGION["n_bg"]], only_occ[:, :REGION["n_bg"]])
    assert np.array_equal(both[:, REGION["n_bg"]:], only_obj[:, REGION["n_bg"]:])
    nothing, _ = regions_op(pred, gt, None, None)
    assert np.all(nothing == 0)
    flat = np.zeros((n, h, w), np.uint8)                                # no boundary: every pixel matched, in no band
    rec, err = regions_op(pred, gt, flat, None)
    assert np.array_equal(rec[:, REGION["n_matched"]], err[:, FIELD["valid"]] - err[:, FIELD["nonfinite"]])
    assert np.all(rec[:, REGION["n_d0_10"]:REGION["n_bg"]] == 0)


def test_regions_refusals(fn2):
    import torch
    from flownet2_b200 import ops
    lib = fn2.lib()
    p = torch.zeros((2, 2, 5, 7), device="cuda")
    m = torch.zeros(2 * 35, dtype=torch.uint8, device="cuda")
    d2 = torch.zeros((2, 5, 7), dtype=torch.int32, device="cuda")
    d2p = C.cast(d2.data_ptr(), C.POINTER(C.c_int32))
    out = torch.zeros((2, len(FLOW_REGION_FIELDS)), dtype=torch.float64, device="cuda")
    optr = C.cast(out.data_ptr(), C.POINTER(C.c_double))
    n = ops.flow_error_regions_workspace_bytes(2, 5, 7)
    ws = torch.zeros(n + 8, dtype=torch.uint8, device="cuda")
    err = lambda: lib.fn2_last_error().decode()

    def call(a, b, occ=m.data_ptr(), obj=m.data_ptr(), stride=35, dist=d2p, w=ws.data_ptr(), nb=n):
        return lib.fn2_flow_error_regions(ops.desc(a), ops.desc(b), occ, obj, stride, dist, optr, w, nb, None)

    assert call(p, p) == 0
    assert call(p, p, occ=None, dist=None) == 0 and call(p, p, occ=None, obj=None, dist=None) == 0
    assert call(p, p, dist=None) == -1 and "dist2 is required" in err()                    # occ without dist2
    assert call(p, p, occ=None) == -1 and "dist2 is required" in err()                     # dist2 without occ
    assert call(p, p, stride=34) == -1 and "mask pair stride 34 is below H * W = 35" in err()
    assert call(p, torch.zeros((2, 2, 5, 8), device="cuda")) == -1
    assert err() == "flow_error_regions: pred is 2x2x5x7 but gt is 2x2x5x8"
    three = torch.zeros((2, 3, 5, 7), device="cuda")
    assert call(three, three) == -1 and "2 channels, got 3" in err()
    assert call(p, p, w=None) == -5 and "workspace" in err()
    assert call(p, p, nb=n - 8) == -5
    assert call(p, p, w=ws.data_ptr() + 4) == -5 and "8-byte aligned" in err()
    assert lib.fn2_flow_error_regions_workspace_bytes(0, 5, 7, C.byref(C.c_size_t())) == -1
    torch.cuda.synchronize()


# ---- the evaluate command ----
A, B = (128, 96), (160, 64)
SIZES = [A, B, A]


@pytest.fixture(scope="module")
def scene(tmp_path_factory, fn2):
    """Frames, ground truth, occlusion masks (PGM) and object maps (gray PNG) over SIZES, evaluate's and run's lists, and
    FlowNet2-S weights from fill_params."""
    from PIL import Image
    d = tmp_path_factory.mktemp("regions")
    ev, rn, occ, obj = [], [], [], []
    for i, (w, h) in enumerate(SIZES):
        f0, f1 = chairs_frames((w, h), 500 + i)
        a, b = write_pnm(d / ("p%d_0.ppm" % i), f0), write_pnm(d / ("p%d_1.ppm" % i), f1)
        g = str(d / ("g%d.flo" % i))
        write_flo(g, ground_truth((w, h), 600 + i))
        occ.append(write_pnm(d / ("occ%d.pgm" % i), blobs(1, h, w, 700 + i, sigma=5.0)[0]))
        obj.append(str(d / ("obj%d.png" % i)))
        Image.fromarray(blobs(1, h, w, 800 + i, sigma=8.0)[0], "L").save(obj[-1])
        ev.append("%s %s %s\n" % (a, b, g))
        rn.append("%s %s %s\n" % (a, b, d / ("out%d.flo" % i)))
    for name, lines in (("val.txt", ev), ("run.txt", rn), ("occ.txt", [p + "\n" for p in occ]),
                        ("obj.txt", ["\n"] + [p + "\n\n" for p in obj])):
        (d / name).write_text("".join(lines))
    net = fn2.Net(fn2.fill_template(fn2.model_template("FlowNet2-S"), 128, 128), None, fn2.TEST, batch=1)
    net.fill_params(1701)
    (d / "w.caffemodel").write_bytes(net.to_caffemodel())
    del net
    return d


def printed(capsys, argv):
    capsys.readouterr()
    assert E.main(argv) == 0
    lines = capsys.readouterr().out.strip().splitlines()
    assert len(lines) == 1
    return json.loads(lines[0])


@pytest.mark.parametrize("batch", [1, 2])
def test_evaluate_regions_end_to_end(fn2, scene, batch, capsys, tmp_path):
    from PIL import Image
    weights, template = str(scene / "w.caffemodel"), os.path.join(ROOT, "models", "FlowNet2-S_deploy.prototxt.template")
    assert R.main([weights, template, str(scene / "run.txt"), "--batch", str(batch)]) == 0
    samples = read_list(str(scene / "val.txt"))
    want = []
    for i, s in enumerate(samples):
        pred = fn2.read_flo(str(scene / ("out%d.flo" % i)))[None]
        gt = read_flow(s.flow).transpose(2, 0, 1)[None]
        occ = np.asarray(Image.open(str(scene / ("occ%d.pgm" % i))))[None]
        obj = np.asarray(Image.open(str(scene / ("obj%d.png" % i))))[None]
        want.append(np.concatenate([flow_error_ref(pred, gt)[0], flow_region_ref(pred, gt, occ, obj)[0]]))
    want = np.array(want)
    pixels = [w * h for w, h in SIZES]
    expect = E.summarize(want, pixels, "val.txt", occlusions=True, objects=True)

    summary, rec = E.evaluate(weights, template, samples, batch=batch, occlusions=str(scene / "occ.txt"),
                              objects=str(scene / "obj.txt"))
    assert rec.shape == (3, len(FLOW_ERROR_FIELDS) + len(FLOW_REGION_FIELDS))
    assert_region_match(rec[:, len(FLOW_ERROR_FIELDS):], want[:, len(FLOW_ERROR_FIELDS):])
    for k, v in expect.items():
        assert summary[k] == (v if v is None or isinstance(v, int) else pytest.approx(v, rel=1e-12)), k
    assert summary["d0-10"] is not None and summary["epe_unmatched"] is not None and summary["fg_px"] > 0

    base = [str(weights), template, str(scene / "val.txt"), "--batch", str(batch)]
    plain = printed(capsys, base)
    tsv = tmp_path / "pairs.tsv"
    flagged = printed(capsys, base + ["--occlusions", str(scene / "occ.txt"), "--objects", str(scene / "obj.txt"),
                                      "--per-pair", str(tsv)])
    for k in plain:
        if k != "wall":
            assert flagged[k] == plain[k], k
    assert set(flagged) - set(plain) == set(expect) - set(E.summarize(want[:, :len(FLOW_ERROR_FIELDS)], pixels, "val.txt"))
    for k, v in expect.items():
        assert flagged[k] == (v if v is None or isinstance(v, int) else pytest.approx(v, rel=1e-12)), k
    rows = tsv.read_text().splitlines()
    assert len(rows) == 4 and rows[0].split("\t")[7:] == [k for k, _, _ in E.region_keys(True, True)]
    occ_only = printed(capsys, base + ["--occlusions", str(scene / "occ.txt")])
    assert "epe_matched" in occ_only and "fl_bg" not in occ_only and occ_only["epe_matched"] == flagged["epe_matched"]
