"""Host side of evaluating by region: mask lists and their refusals, the summary and per-pair columns with and without the mask
flags, the recombination of wider per-rank records, and the numpy restatement (tests/flow_region_ref.py) against hand-worked
masks.  No GPU needed."""
import json
import re

import numpy as np
import pytest

from flownet2_b200 import DIST2_NONE, FLOW_ERROR_FIELDS, FLOW_REGION_FIELDS
from flownet2_b200 import evaluate as E, feed as FD, files as FI
from flownet2_b200.files import RunError, write_flo
from flownet2_b200.run import shard
from tests.flow_region_ref import boundary, dist2_ref, flow_region_ref
from tests.test_evaluate_cpu import synthetic_records
from tests.test_run_flownet_cpu import write_pnm

NF = len(FLOW_ERROR_FIELDS)
REGION = {f: NF + i for i, f in enumerate(FLOW_REGION_FIELDS)}


def test_record_fields():
    assert FLOW_ERROR_FIELDS == ("valid", "epe_sum", "outliers", "nonfinite", "n_s0_10", "sum_s0_10", "n_s10_40", "sum_s10_40",
                                 "n_s40", "sum_s40")
    regions = ("matched", "unmatched", "d0_10", "d10_60", "d60_140", "bg", "fg")
    assert FLOW_REGION_FIELDS == tuple("%s_%s" % (k, r) for r in regions for k in ("n", "sum", "out"))
    assert DIST2_NONE == 2 ** 31 - 1
    assert E.record_width(()) == 10 and E.record_width(("objects",)) == 31


# ---- the restatement on masks worked by hand ----
def test_dist2_restatement_by_hand():
    one = np.zeros((1, 5, 5), np.uint8)
    one[0, 2, 2] = 7                                                   # any nonzero byte is occluded
    assert boundary(one[0]).sum() == 5                                 # the pixel and its four neighbours
    assert dist2_ref(one)[0].tolist() == [[5, 2, 1, 2, 5], [2, 1, 0, 1, 2], [1, 0, 0, 0, 1], [2, 1, 0, 1, 2], [5, 2, 1, 2, 5]]
    row = np.array([[[0, 0, 0, 255, 0, 0, 0, 0]]], np.uint8)
    assert dist2_ref(row)[0, 0].tolist() == [4, 1, 0, 0, 0, 1, 4, 9]
    col = row.transpose(0, 2, 1)
    assert dist2_ref(col)[0, :, 0].tolist() == [4, 1, 0, 0, 0, 1, 4, 9]
    checker = (np.indices((1, 4, 6)).sum(axis=0) % 2).astype(np.uint8)
    assert np.all(dist2_ref(checker) == 0)
    flat = np.stack([np.zeros((3, 4), np.uint8), np.full((3, 4), 9, np.uint8)])
    assert np.all(dist2_ref(flat) == DIST2_NONE)                        # no boundary: all clear, all occluded
    half = np.zeros((1, 3, 200), np.uint8)
    half[0, :, 100:] = 1
    d = dist2_ref(half)[0, 0]
    assert d[99] == d[100] == 0 and d[0] == 99 ** 2 and d[199] == 99 ** 2


def test_region_restatement_by_hand():
    # one 2x3 pair: gt (3, 4) everywhere, pred off by EPE 0, 5, 10 in row 0 and NaN / valid / invalid gt in row 1
    gt = np.zeros((1, 2, 2, 3), np.float32)
    gt[0, 0], gt[0, 1] = 3, 4
    pred = gt.copy()
    pred[0, 0, 0, 1] += 5                                              # EPE 5 > 3 and > 0.25: an outlier
    pred[0, 0, 0, 2] += 10
    pred[0, 0, 1, 0] = np.nan                                          # not counted
    pred[0, 0, 1, 1] += 1                                              # EPE 1
    gt[0, 1, 1, 2] = 1e10                                              # invalid ground truth
    occ = np.array([[[0, 0, 1], [0, 0, 1]]], np.uint8)
    obj = np.array([[[0, 1, 1], [1, 0, 0]]], np.uint8)
    r = dict(zip(FLOW_REGION_FIELDS, flow_region_ref(pred, gt, occ, obj)[0]))
    assert (r["n_matched"], r["sum_matched"], r["out_matched"]) == (3, 6, 1)      # EPE 0, 5, 1
    assert (r["n_unmatched"], r["sum_unmatched"], r["out_unmatched"]) == (1, 10, 1)
    assert r["n_d0_10"] == 4 and r["n_d10_60"] == r["n_d60_140"] == 0              # every pixel is within 1 of the boundary
    assert (r["n_bg"], r["sum_bg"], r["out_bg"]) == (2, 1, 0) and (r["n_fg"], r["sum_fg"], r["out_fg"]) == (2, 15, 2)
    none = flow_region_ref(pred, gt)
    assert np.all(none == 0)


# ---- mask lists ----
@pytest.fixture
def files(tmp_path):
    """A model and template that exist, a 9x7 pair list of two lines, and masks: gray PGM, gray PNG, RGB, wrong size."""
    from PIL import Image
    r = np.random.default_rng(0)
    f = r.integers(0, 256, (7, 9, 3), dtype=np.uint8)
    d = {"model": tmp_path / "m.caffemodel", "proto": tmp_path / "t.template", "dir": tmp_path}
    d["model"].write_bytes(b"")
    d["proto"].write_text("")
    a, b = write_pnm(tmp_path / "a.ppm", f), write_pnm(tmp_path / "b.ppm", f)
    g = str(tmp_path / "g.flo")
    write_flo(g, r.standard_normal((7, 9, 2)).astype(np.float32))
    d["list"] = tmp_path / "val.txt"
    d["list"].write_text("%s %s %s\n\n%s %s %s\n" % (a, b, g, a, b, g))
    d["pgm"] = write_pnm(tmp_path / "m.pgm", (r.random((7, 9)) < 0.3).astype(np.uint8) * 255)
    d["png"] = str(tmp_path / "m.png")
    Image.fromarray(r.integers(0, 3, (7, 9), dtype=np.uint8), "L").save(d["png"])
    d["rgb"] = write_pnm(tmp_path / "rgb.ppm", f)
    d["wide"] = write_pnm(tmp_path / "wide.pgm", np.zeros((7, 10), np.uint8))
    return d


def mask_list(files, name, lines):
    p = files["dir"] / name
    p.write_text("".join(l + "\n" for l in lines))
    return str(p)


def refused(files, capsys, args, match):
    assert E.main([str(files["model"]), str(files["proto"]), str(files["list"])] + args) == 2
    err = capsys.readouterr().err
    assert re.search(match, err), err


def test_mask_lists_attach_before_sharding(files):
    samples = FI.read_list(str(files["list"]))
    occ = mask_list(files, "occ.txt", ["", files["pgm"], "  ", files["png"], ""])           # blank lines skipped
    obj = mask_list(files, "obj.txt", [files["png"], files["pgm"]])
    FI.attach_masks(samples, [occ, obj])
    assert [s.masks for s in samples] == [((occ + ":2", files["pgm"]), (obj + ":1", files["png"])),
                                          ((occ + ":4", files["png"]), (obj + ":2", files["pgm"]))]
    FI.probe(samples, ground_truth=True)                               # a PGM and a gray PNG are one-channel 8-bit frames
    mine = shard(samples, 2, 1)
    assert mine[0].masks[0][1] == files["png"]                         # rank 1 holds line 2 with line 2's masks
    plain = FI.read_list(str(files["list"]))
    assert all(s.masks == () for s in plain)


def test_mask_list_refusals(files, capsys):
    pgm = files["pgm"]
    refused(files, capsys, ["--occlusions", mask_list(files, "occ.txt", [pgm])], r"occ\.txt: 1 masks for a list of 2 pairs")
    refused(files, capsys, ["--objects", mask_list(files, "obj.txt", [pgm] * 3)], r"obj\.txt: 3 masks for a list of 2 pairs")
    refused(files, capsys, ["--occlusions", str(files["dir"] / "none.txt")], r"none\.txt: no such mask list")
    refused(files, capsys, ["--occlusions", mask_list(files, "occ.txt", [pgm, "%s extra" % pgm])],
            r"occ\.txt:2: 2 fields, expected one mask path")
    refused(files, capsys, ["--occlusions", mask_list(files, "occ.txt", [pgm, str(files["dir"] / "gone.png")])],
            r"occ\.txt:2: .*gone\.png: no such file")
    refused(files, capsys, ["--objects", mask_list(files, "obj.txt", [files["wide"], pgm])],
            r"obj\.txt:1: .*wide\.pgm is 10x7 but the frames of .*val\.txt:1 are 9x7")
    refused(files, capsys, ["--occlusions", mask_list(files, "occ.txt", [pgm, files["rgb"]])],
            r"occ\.txt:2: .*rgb\.ppm has 3 channels, a mask is a one-channel 8-bit image")
    refused(files, capsys, ["--occlusions", mask_list(files, "occ.txt", [pgm, pgm]), "--objects",
                            mask_list(files, "obj.txt", [pgm])], r"obj\.txt: 1 masks for a list of 2 pairs")


def test_mask_read_into_its_plane(files):
    """The reader puts a mask as H x W bytes, a gray PNG decoded; a refusal names the mask list's line."""
    from PIL import Image
    samples = FI.read_list(str(files["list"]))
    FI.attach_masks(samples, [mask_list(files, "occ.txt", [files["pgm"], files["png"]])])
    FI.probe(samples, ground_truth=True)
    out = np.full(9 * 7 + 5, 77, np.uint8)
    FD.read_part(samples[1], 3, (9, 7), 3, out)
    assert np.array_equal(out[:63].reshape(7, 9), np.asarray(Image.open(files["png"]))) and np.all(out[63:] == 77)
    FD.read_part(samples[0], 3, (9, 7), 3, out)
    assert np.array_equal(out[:63].reshape(7, 9), FI.read_image(files["pgm"]))
    samples[0].masks = (("occ.txt:1", str(files["dir"] / "gone.pgm")),)
    with pytest.raises(RunError, match=r"^occ\.txt:1: "):
        FD.read_part(samples[0], 3, (9, 7), 3, out)
    sink = E.Scores(2, ("occlusions", "objects"))
    assert sink.item_bytes(7, 9) == FD._align(63 * 12 + 2 * 63) and FD.mask_offset(7, 9) == 63 * 12
    assert sink.records.shape == (2, 31) and E.Scores(2).records.shape == (2, 10)


def test_arguments():
    a = E.parse_args(["w", "t", "l"])
    assert a.occlusions is None and a.objects is None
    a = E.parse_args(["w", "t", "l", "--occlusions", "occ.txt", "--objects", "obj.txt"])
    assert (a.occlusions, a.objects) == ("occ.txt", "obj.txt")


# ---- summary, per-pair rows, ranks ----
def region_records(n, seed):
    """synthetic_records widened by plausible region fields: matched + unmatched = bg + fg = valid - nonfinite."""
    r = np.random.default_rng(seed)
    base = synthetic_records(n, seed)
    rec = np.concatenate([base, np.zeros((n, len(FLOW_REGION_FIELDS)))], axis=1)
    for i in range(n):
        counted = base[i, 0] - base[i, 3]
        for a, b in (("matched", "unmatched"), ("bg", "fg")):
            k = r.integers(0, counted + 1)
            for reg, c in ((a, k), (b, counted - k)):
                rec[i, REGION["n_" + reg]] = c
                rec[i, REGION["sum_" + reg]] = c * r.uniform(0.1, 9.0)
                rec[i, REGION["out_" + reg]] = r.integers(0, c + 1)
        for reg in ("d0_10", "d10_60", "d60_140"):
            c = r.integers(0, counted // 3 + 1)
            rec[i, REGION["n_" + reg]], rec[i, REGION["sum_" + reg]] = c, c * r.uniform(0.1, 9.0)
    return rec


def test_summary_with_and_without_regions():
    rec = region_records(6, 4)
    rec[2, REGION["n_d60_140"]] = 0
    rec[:, REGION["n_d60_140"]] = rec[:, REGION["sum_d60_140"]] = 0          # an empty band
    pixels = np.full(6, 5000)
    plain = E.summarize(rec[:, :NF], pixels, "val.txt")
    assert E.summarize(rec, pixels, "val.txt") == plain                      # no flag: the region fields are not read
    s = E.summarize(rec, pixels, "val.txt", occlusions=True, objects=True)
    assert {k: s[k] for k in plain} == plain
    assert list(s)[len(plain):] == ["epe_matched", "epe_unmatched", "d0-10", "d10-60", "d60-140", "fl_bg", "fl_fg", "epe_bg",
                                    "epe_fg", "matched_px", "unmatched_px", "bg_px", "fg_px"]
    tot = lambda f: rec[:, REGION[f]].sum()
    assert s["epe_matched"] == tot("sum_matched") / tot("n_matched")
    assert s["epe_unmatched"] == tot("sum_unmatched") / tot("n_unmatched")
    assert s["d0-10"] == tot("sum_d0_10") / tot("n_d0_10") and s["d60-140"] is None
    assert s["fl_bg"] == 100.0 * tot("out_bg") / tot("n_bg") and s["fl_fg"] == 100.0 * tot("out_fg") / tot("n_fg")
    assert s["epe_fg"] == tot("sum_fg") / tot("n_fg")
    counted = (rec[:, 0] - rec[:, 3]).sum()
    assert s["matched_px"] + s["unmatched_px"] == s["bg_px"] + s["fg_px"] == counted
    json.dumps(s)
    occ = E.summarize(rec, pixels, "val.txt", occlusions=True)
    assert "epe_matched" in occ and "fl_bg" not in occ and "bg_px" not in occ
    obj = E.summarize(rec, pixels, "val.txt", objects=True)
    assert "fl_fg" in obj and "d0-10" not in obj and "matched_px" not in obj


def test_per_pair_columns(tmp_path):
    rec = region_records(3, 5)
    rec[1, NF:] = 0                                                     # a pair whose regions are empty

    class S(object):
        def __init__(self, i):
            self.where, self.img0, self.img1, self.flow = "val.txt:%d" % (i + 1), "a%d" % i, "b%d" % i, "f%d" % i

    samples = [S(i) for i in range(3)]
    p = tmp_path / "plain.tsv"
    E.write_per_pair(str(p), samples, rec[:, :NF])
    plain = p.read_text()
    E.write_per_pair(str(p), samples, rec)
    assert p.read_text() == plain                                      # no flag: the same file
    E.write_per_pair(str(p), samples, rec, occlusions=True, objects=True)
    rows = [l.split("\t") for l in p.read_text().splitlines()]
    assert rows[0] == ["where", "img0", "img1", "flow", "valid", "epe", "fl_percent", "epe_matched", "epe_unmatched", "d0-10",
                       "d10-60", "d60-140", "fl_bg", "fl_fg", "epe_bg", "epe_fg"]
    assert [r[:7] for r in rows] == [l.split("\t") for l in plain.splitlines()]
    assert float(rows[1][7]) == pytest.approx(rec[0, REGION["sum_matched"]] / rec[0, REGION["n_matched"]], rel=1e-8)
    assert float(rows[1][12]) == pytest.approx(100 * rec[0, REGION["out_bg"]] / rec[0, REGION["n_bg"]], rel=1e-8)
    assert rows[2][7:] == ["nan"] * 9
    E.write_per_pair(str(p), samples, rec, objects=True)
    assert p.read_text().splitlines()[0].split("\t")[7:] == ["fl_bg", "fl_fg", "epe_bg", "epe_fg"]


@pytest.mark.parametrize("n", [1, 5, 13])
def test_rank_recombination_of_wider_records(n):
    rec = np.concatenate([region_records(n, 6), np.full((n, 1), 375.0 * 1242)], axis=1)
    want = E.summarize(rec[:, :-1], rec[:, -1], "val.txt", occlusions=True, objects=True)
    for world in (1, 2, 3, 8):
        shards = [np.array([rec[i] for i in shard(range(n), world, r)]).reshape(-1, rec.shape[1]) for r in range(world)]
        back = E.combine_shards(shards)
        assert np.array_equal(back.view(np.uint64), rec.view(np.uint64)), world
        assert E.summarize(back[:, :-1], back[:, -1], "val.txt", occlusions=True, objects=True) == want, world
