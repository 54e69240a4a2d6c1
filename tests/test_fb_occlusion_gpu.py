"""GPU: fn2_flow_fb_occlusion (include/fn2_flow.h) byte for byte against tests/fb_ref.py and against the check applied to the
engine's own FlowWarp output, fn2_mask_confusion against numpy, and run --backward and evaluate --fb-check end to end."""
import json
import os
import re
import zlib

import numpy as np
import pytest
from scipy import ndimage

from flownet2_b200 import FLOW_ERROR_FIELDS, FLOW_REGION_FIELDS, MASK_CONFUSION_FIELDS
from flownet2_b200 import evaluate as E
from flownet2_b200 import files as FI
from flownet2_b200 import kitti as K
from flownet2_b200 import run as R
from tests import fb_ref as ref
from tests.flow_error_ref import flow_error_ref
from tests.flow_region_ref import assert_region_match, flow_region_ref
from tests.test_flow_viz_gpu import dev_view, frames_list
from tests.test_kitti_flow_gpu import kitti_scene
from tests.test_run_flownet_cpu import write_pnm
from tests.test_run_flownet_gpu import TEMPLATE, flownet2c

pytestmark = pytest.mark.gpu


def smooth_flow(r, N, H, W, scale):
    """N smooth random flows (N, H, W, 2) with displacements up to about `scale` pixels."""
    coarse = r.standard_normal((N, 4, 5, 2))
    f = np.stack([ndimage.zoom(c, (H / 4, W / 5, 1), order=3)[:H, :W] for c in coarse])
    return (f * scale).astype(np.float32)


def analytic():
    """The CPU file's analytic cases as one batch of 13 x 17 pairs: (fwd, bwd) each (N, H, W, 2)."""
    H, W = 13, 17
    fw, bw = np.zeros((5, H, W, 2), np.float32), np.zeros((5, H, W, 2), np.float32)
    fw[1, ..., 0], fw[1, ..., 1], bw[1, ..., 0], bw[1, ..., 1] = 3, -2, -3, 2             # a translation
    fw[2, 3:9, 4:10, 0] = 2                                                                # a square moving right
    bw[2, 3:9, 6:12, 0] = -2
    fw[3, 1, 2], fw[3, 2, 3], bw[3, 6, 7], bw[3, 0, 5] = (np.nan, 0), (0, np.inf), (np.nan, 1), (-np.inf, 0)
    fw[3, 0, 0] = (4.5, 0.0)
    bw[4, ..., 0] = 0.6                                                                    # tiny flows near alpha2
    return fw, bw


def cases():
    """(name, fwd, bwd): the analytic batch, and random smooth flows with large displacements, non-finite entries and odd
    sizes, N up to 8."""
    r = np.random.default_rng(31)
    out = [("analytic",) + analytic()]
    for N, H, W, scale in ((8, 37, 53, 20.0), (3, 64, 96, 60.0), (1, 31, 1, 5.0), (2, 1, 45, 8.0)):
        fwd = smooth_flow(r, N, H, W, scale)
        bwd = -fwd + (r.standard_normal(fwd.shape) * r.choice([0.1, 1.0, 3.0], (N, 1, 1, 1))).astype(np.float32)
        for f, k in ((fwd, 0.01), (bwd, 0.01)):
            sel = r.random(f.shape[:3]) < k
            f[sel] = r.choice([np.nan, np.inf, -np.inf], (sel.sum(), 1)).astype(np.float32)
        out.append(("smooth%dx%dx%d" % (N, H, W), fwd, bwd))
    return out


CASES = cases()


def expected(fwd, bwd, a1=0.01, a2=0.5):
    return np.stack([ref.fb_occlusion(f, b, a1, a2) for f, b in zip(fwd, bwd)])


@pytest.mark.parametrize("layout", ["nchw", "channels_last", "padded"])
@pytest.mark.parametrize("case", range(len(CASES)), ids=[c[0] for c in CASES])
def test_kernel_equals_restatement(fn2, layout, case):
    from flownet2_b200 import ops
    _, fwd, bwd = CASES[case]
    got = ops.flow_fb_occlusion(dev_view(fwd, layout), dev_view(bwd, layout)).cpu().numpy()
    want = expected(fwd, bwd)
    assert np.array_equal(got, want), (np.argwhere(got != want)[:5], (got != want).sum())
    if CASES[case][0] == "analytic":
        assert (got[0] == 0).all() and (got[1] == 255).any() and (got[2] == 255).sum() == 6 * 2


@pytest.mark.parametrize("alphas", [(0.0, 0.0), (0.0, 0.36), (0.05, 2.0), (1.0, 0.0)])
def test_kernel_alphas(fn2, alphas):
    from flownet2_b200 import ops
    for _, fwd, bwd in CASES[:2]:
        got = ops.flow_fb_occlusion(dev_view(fwd, "nchw"), dev_view(bwd, "nchw"), *alphas).cpu().numpy()
        assert np.array_equal(got, expected(fwd, bwd, *alphas))


def test_strided_output(fn2):
    """row_stride W + 1 and a padded pair stride: every pixel in its place, no other byte written."""
    import torch
    from flownet2_b200 import ops
    _, fwd, bwd = CASES[1]
    N, H, W, _ = fwd.shape
    rs, ps = W + 1, H * (W + 1) + 5
    buf = torch.full((N * ps,), 77, dtype=torch.uint8, device="cuda")
    ops.flow_fb_occlusion(dev_view(fwd, "padded"), dev_view(bwd, "padded"), out=buf, row_stride=rs, pair_stride=ps)
    b = buf.cpu().numpy().reshape(N, ps)
    want = expected(fwd, bwd)
    assert np.array_equal(b[:, :H * rs].reshape(N, H, rs)[..., :W], want)
    assert (b[:, :H * rs].reshape(N, H, rs)[..., W] == 77).all() and (b[:, H * rs:] == 77).all()


def test_tied_to_flowwarp(fn2):
    """The mask is the check applied to fn2_flow_warp_forward(image = bwd, flow = fwd): the kernel samples as FlowWarp does."""
    from flownet2_b200 import ops
    for _, fwd, bwd in CASES:
        f, b = dev_view(fwd, "nchw"), dev_view(bwd, "nchw")
        warped = ops.flow_warp(b, f).permute(0, 2, 3, 1).cpu().numpy()
        want = np.stack([ref.decide(x, w, ref.landing(x)[2]) for x, w in zip(fwd, warped)])
        assert np.array_equal(ops.flow_fb_occlusion(f, b).cpu().numpy(), want)


def test_refusals(fn2):
    import torch
    from flownet2_b200 import ops
    f = torch.zeros((2, 2, 5, 6), device="cuda")
    out = torch.zeros(2 * 5 * 7, dtype=torch.uint8, device="cuda")

    def call(a, b, a1=0.01, a2=0.5, rs=6, ps=30):
        return fn2.lib().fn2_flow_fb_occlusion(ops.desc(a), ops.desc(b), a1, a2, out.data_ptr(), rs, ps, None)

    assert call(f, f) == 0
    for args, msg in (((f, torch.zeros((2, 2, 5, 7), device="cuda")), "fwd is 2x2x5x6 but bwd is 2x2x5x7"),
                      ((torch.zeros((2, 3, 5, 6), device="cuda"),) * 2, "flows need 2 channels"),
                      ((f, f, -0.1), "alpha1 and alpha2 must be finite and non-negative"),
                      ((f, f, 0.01, float("nan")), "alpha1 and alpha2 must be finite and non-negative"),
                      ((f, f, float("inf")), "alpha1 and alpha2 must be finite and non-negative"),
                      ((f, f, 0.01, 0.5, 5), "row stride 5 is below W = 6"),
                      ((f, f, 0.01, 0.5, 7, 34), "pair stride 34 is below H \\* row stride = 35")):
        assert call(*args) == -1, msg
        assert re.search(msg, fn2.lib().fn2_last_error().decode()), (msg, fn2.lib().fn2_last_error())
    many = torch.zeros((65536, 2, 1, 1), device="cuda")
    big = torch.zeros(65536, dtype=torch.uint8, device="cuda")
    assert fn2.lib().fn2_flow_fb_occlusion(ops.desc(many), ops.desc(many), 0.01, 0.5, big.data_ptr(), 1, 1, None) == -1
    assert "65536 pairs, at most 65535" in fn2.lib().fn2_last_error().decode()


def confusion_ref(pred, gt):
    p, g = np.asarray(pred) != 0, np.asarray(gt) != 0
    return np.stack([np.stack([(a & b).sum(), (a & ~b).sum(), (~a & b).sum(), (~a & ~b).sum()]) for a, b in zip(p, g)]) \
        .astype(np.float64)


@pytest.mark.parametrize("shape", [(5, 37, 53), (3, 436, 1024), (1, 1, 1)])
def test_mask_confusion_exact(fn2, shape):
    import torch
    from flownet2_b200 import ops
    r = np.random.default_rng(41)
    pred = (r.random(shape) < 0.3) * r.choice([1, 7, 255], shape)
    gt = (r.random(shape) < 0.2) * r.choice([1, 128, 255], shape)
    got = ops.mask_confusion(torch.from_numpy(pred.astype(np.uint8)).cuda(), torch.from_numpy(gt.astype(np.uint8)).cuda())
    want = confusion_ref(pred, gt)
    assert MASK_CONFUSION_FIELDS == ("tp", "fp", "fn", "tn")
    assert np.array_equal(got.cpu().numpy(), want) and want.sum() == np.prod(shape)
    again = ops.mask_confusion(torch.from_numpy(pred.astype(np.uint8)).cuda(), torch.from_numpy(gt.astype(np.uint8)).cuda())
    assert np.array_equal(again.cpu().numpy(), want)


# ---- the commands ----
@pytest.fixture(scope="module")
def c_weights(tmp_path_factory, fn2):
    d = tmp_path_factory.mktemp("fb")
    net = flownet2c(fn2, 64, 64, 1)
    path = d / "c.caffemodel"
    path.write_bytes(net.to_caffemodel())
    del net
    return str(path)


def read_grey_png(path):
    data = open(path, "rb").read()
    w, h = int.from_bytes(data[16:20], "big"), int.from_bytes(data[20:24], "big")
    assert (data[24], data[25]) == (8, 0)                                              # 8-bit grey
    raw = np.frombuffer(zlib.decompress(K._idat(path, data)), np.uint8).reshape(h, 1 + w)
    assert (raw[:, 0] == 0).all()                                                      # filter None
    return raw[:, 1:]


def write_pairs(path, pairs, outs):
    path.write_text("".join("%s %s %s\n" % (a, b, o) for (_, a, b), o in zip(pairs, outs)))


def test_run_backward(fn2, c_weights, tmp_path):
    from PIL import Image
    sizes = [(128, 96), (192, 64), (128, 96), (128, 96), (192, 64)]
    pairs = frames_list(tmp_path, sizes)
    swapped = [(s, b, a) for s, a, b in pairs]
    lst, sw = tmp_path / "l.txt", tmp_path / "s.txt"
    for batch in (1, 3):
        masks = {}
        for kitti in (False, True):
            ext, flags = (".png", ["--kitti"]) if kitti else (".flo", [])
            flags += ["--batch", str(batch)]
            d = tmp_path / ("b%d_k%d" % (batch, kitti))
            os.makedirs(str(d))
            outs = [str(d / ("o%d%s" % (i, ext))) for i in range(len(pairs))]
            write_pairs(lst, pairs, outs)
            assert R.main([c_weights, TEMPLATE, str(lst)] + flags) == 0
            plain = [open(o, "rb").read() for o in outs]
            assert not any(os.path.exists(R.bwd_path(o)) or os.path.exists(R.occ_path(o)) for o in outs)
            assert R.main([c_weights, TEMPLATE, str(lst), "--backward"] + flags) == 0
            assert [open(o, "rb").read() for o in outs] == plain, (batch, kitti)             # the forward outputs
            rev = [str(d / ("r%d%s" % (i, ext))) for i in range(len(pairs))]
            write_pairs(sw, swapped, rev)
            assert R.main([c_weights, TEMPLATE, str(sw)] + flags) == 0
            for o, r_ in zip(outs, rev):
                assert open(R.bwd_path(o), "rb").read() == open(r_, "rb").read(), (batch, kitti, o)
            assert sorted(os.listdir(str(d))) == sorted(
                [os.path.basename(p) for o in outs for p in (o, R.bwd_path(o), R.occ_path(o))] +
                [os.path.basename(r_) for r_ in rev])
            for i, o in enumerate(outs):
                got = read_grey_png(R.occ_path(o))
                with Image.open(R.occ_path(o)) as im:
                    assert im.mode == "L" and np.array_equal(np.asarray(im), got)
                if kitti:                                       # the float flows' mask: the .flo run's, bit for bit
                    assert np.array_equal(got, masks[i]), (batch, i)
                    continue
                fwd = FI.read_flow(o)
                bwd = FI.read_flow(R.bwd_path(o))
                want = ref.fb_occlusion(fwd, bwd)
                assert np.array_equal(got, want), (batch, i, (got != want).sum())
                masks[i] = got
        assert any((m == 255).any() for m in masks.values()) and any((m == 0).any() for m in masks.values())
        # the masks are evaluate --occlusions input: the forward flows as ground truth score zero everywhere
        d = tmp_path / ("b%d_k0" % batch)
        val, occ = tmp_path / "val.txt", tmp_path / "occ.txt"
        val.write_text("".join("%s %s %s\n" % (a, b, d / ("o%d.flo" % i)) for i, (_, a, b) in enumerate(pairs)))
        occ.write_text("".join("%s\n" % R.occ_path(str(d / ("o%d.flo" % i))) for i in range(len(pairs))))
        summary, rec = E.evaluate(c_weights, TEMPLATE, FI.read_list(str(val)), batch=batch, occlusions=str(occ))
        assert summary["unmatched_px"] == sum(int((m != 0).sum()) for m in masks.values())
        assert summary["epe"] == 0.0


def occ_masks(d, sizes, seed):
    """Smooth random occlusion masks as PGM files over sizes [(w, h)] -> their list file."""
    r = np.random.default_rng(seed)
    paths = []
    for i, (w, h) in enumerate(sizes):
        m = ndimage.gaussian_filter(r.standard_normal((h, w)), 4.0)
        paths.append(write_pnm(d / ("occ%d.pgm" % i), np.where(m > 0.05, 255, 0).astype(np.uint8)))
    (d / "occ.txt").write_text("".join(p + "\n" for p in paths))
    return str(d / "occ.txt")


def printed(capsys, argv):
    capsys.readouterr()
    assert E.main(argv) == 0
    lines = capsys.readouterr().out.strip().splitlines()
    assert len(lines) == 1
    return json.loads(lines[0])


def close(a, b):
    return a == b if a is None or b is None or isinstance(b, int) else a == pytest.approx(b, rel=1e-12)


@pytest.mark.parametrize("batch", [1, 2])
def test_evaluate_fb_check(fn2, c_weights, tmp_path, capsys, batch):
    from PIL import Image
    sizes = [(128, 96), (192, 64), (128, 96)]
    lists = kitti_scene(tmp_path, sizes, 900)
    occ_list = occ_masks(tmp_path, sizes, 901)
    assert R.main([c_weights, TEMPLATE, lists["run_flo"], "--backward", "--batch", str(batch)]) == 0
    samples = FI.read_list(lists["flo"])
    outs = [l.split()[2] for l in open(lists["run_flo"]).read().splitlines()]
    nf, nr = len(FLOW_ERROR_FIELDS), len(FLOW_REGION_FIELDS)
    want = []
    for s, o, op in zip(samples, outs, open(occ_list).read().split()):
        fwd, bwd = FI.read_flow(o), FI.read_flow(R.bwd_path(o))
        pred, gt = fwd.transpose(2, 0, 1)[None], FI.read_flow(s.flow).transpose(2, 0, 1)[None]
        mask = ref.fb_occlusion(fwd, bwd)[None]
        occ = np.asarray(Image.open(op))[None]
        want.append(np.concatenate([flow_error_ref(pred, gt)[0], flow_region_ref(pred, gt, occ=occ)[0],
                                    flow_region_ref(pred, gt, obj=mask)[0], confusion_ref(mask, occ)[0]]))
    want = np.array(want)
    pixels = [w * h for w, h in sizes]
    base = [c_weights, TEMPLATE, lists["flo"], "--batch", str(batch)]

    # with --occlusions: every new field, the records and the per-pair file
    summary, rec = E.evaluate(c_weights, TEMPLATE, FI.read_list(lists["flo"]), batch=batch, occlusions=occ_list,
                              fb=(0.01, 0.5))
    assert rec.shape == (3, nf + nr + nr + len(MASK_CONFUSION_FIELDS))
    assert np.array_equal(rec[:, :nf], want[:, :nf])
    assert_region_match(rec[:, nf:nf + nr], want[:, nf:nf + nr])
    assert_region_match(rec[:, nf + nr:nf + 2 * nr], want[:, nf + nr:nf + 2 * nr])
    assert np.array_equal(rec[:, -4:], want[:, -4:])
    expect = E.summarize(want, pixels, "val", occlusions=True, fb=True)
    new = {"epe_fb_visible", "epe_fb_flagged", "fb_visible_px", "fb_flagged_px", "occ_tp", "occ_fp", "occ_fn", "occ_precision",
           "occ_recall", "occ_f1"}
    assert new <= set(expect) and expect["fb_flagged_px"] > 0 and expect["occ_tp"] > 0
    for k, v in expect.items():
        assert close(summary[k], v), k
    tp, fp, fn = (int(want[:, -4 + j].sum()) for j in range(3))
    assert summary["occ_f1"] == pytest.approx(2 * tp / (2 * tp + fp + fn), rel=1e-15)

    tsv_plain, tsv_fb = tmp_path / "a.tsv", tmp_path / "b.tsv"
    plain = printed(capsys, base + ["--occlusions", occ_list, "--per-pair", str(tsv_plain)])
    flagged = printed(capsys, base + ["--occlusions", occ_list, "--per-pair", str(tsv_fb), "--fb-check"])
    assert set(flagged) - set(plain) == new
    for k in plain:
        if k != "wall":
            assert flagged[k] == plain[k], k
    for k in new:
        assert close(flagged[k], expect[k]), k
    a, b = tsv_plain.read_text().splitlines(), tsv_fb.read_text().splitlines()
    assert b[0] == a[0] + "\t" + "\t".join(E.fb_keys(True))
    for ra, rb, w in zip(a[1:], b[1:], want):
        assert rb.startswith(ra + "\t")
        extra = [float(x) for x in rb[len(ra) + 1:].split("\t")]
        exp = [np.nan if v is None else v for _, v in E.fb_scores(w[-E.FB_FIELDS:], True)]
        assert np.allclose(extra, exp, rtol=1e-8, equal_nan=True)

    # without --occlusions: the EPE split alone; without the flag: byte-identical per-pair files
    plain = printed(capsys, base + ["--per-pair", str(tsv_plain)])
    flagged = printed(capsys, base + ["--fb-check"])
    assert set(flagged) - set(plain) == {"epe_fb_visible", "epe_fb_flagged", "fb_visible_px", "fb_flagged_px"}
    expect = E.summarize(np.concatenate([want[:, :nf], want[:, nf + nr:]], 1), pixels, "val", fb=True)
    for k in plain:
        if k != "wall":
            assert flagged[k] == plain[k], k
    for k in ("epe_fb_visible", "epe_fb_flagged", "fb_visible_px", "fb_flagged_px"):
        assert close(flagged[k], expect[k]), k
    again = tmp_path / "c.tsv"
    printed(capsys, base + ["--per-pair", str(again)])
    assert again.read_text() == tsv_plain.read_text()
