"""The train command's validation without a GPU: the schedule against Caffe's TestAll rule, the printed lines and the log
record, the hand-over check on layer tables, and every refused flag, each refused before a net is built."""
import json
import math
import re

import numpy as np
import pytest

from flownet2_b200 import FLOW_ERROR_FIELDS, FLOW_REGION_FIELDS
from flownet2_b200 import evaluate as E
from flownet2_b200 import train as T
from flownet2_b200.files import RunError, write_flo, write_pnm

CAFFE_TEST = re.compile(r"Test net output #(\d+): (\S+) = (\S+)")


def caffe_tests(start, max_iter, interval, initialization):
    """Solver::Solve / Step (solver.cpp:194-330) with test_interval and test_initialization: the iterations TestAll runs at."""
    out, it = [], start
    while it < max_iter:
        if it % interval == 0 and (it > 0 or initialization):
            out.append(it)
        it += 1                                  # ... ApplyUpdate, ++iter_
    if it % interval == 0:
        out.append(it)
    return out


def test_schedule_follows_caffe():
    for start in range(0, 14):
        for max_iter in range(0, 14):
            for n in range(1, 6):
                for initial in (True, False):
                    assert T.val_iters(start, max_iter, n, initial) == caffe_tests(start, max_iter, n, initial), (
                        start, max_iter, n, initial)
    assert T.val_iters(0, 10, 5) == [0, 5, 10]
    assert T.val_iters(0, 10, 5, initial=False) == [5, 10]
    assert T.val_iters(0, 12, 5) == [0, 5, 10]                       # max_iter not a multiple of N: no validation at the end
    assert T.val_iters(5, 10, 5, initial=False) == [5, 10]           # a resumed run validates at its first iteration
    assert T.val_iters(6, 12, 4) == [8, 12]


def records(rows, masks=False):
    """Per-pair records from {field: value} rows (the other fields 0)."""
    names = list(FLOW_ERROR_FIELDS) + (list(FLOW_REGION_FIELDS) if masks else [])
    out = np.zeros((len(rows), len(names)))
    for i, r in enumerate(rows):
        for k, v in r.items():
            out[i, names.index(k)] = v
    return out


def summary(masks=False, nonfinite=0):
    """A summary as evaluate makes it: no pixel above 40 px (an empty band), one pair with non-finite predictions."""
    rec = records([{"valid": 100, "epe_sum": 150.0, "outliers": 3, "n_s0_10": 90, "sum_s0_10": 100.0, "n_s10_40": 10,
                    "sum_s10_40": 50.0, "nonfinite": nonfinite},
                   {"valid": 50, "epe_sum": 25.0, "n_s0_10": 50, "sum_s0_10": 25.0}], masks)
    s = E.summarize(rec, [120, 60], "val.txt", occlusions=masks)
    s.update({"batch": 1, "sizes": 1, "wall": 0.5, "busy": {"forward": 0.1}, "not_finite": ["val.txt:1"] if nonfinite else []})
    return s


@pytest.mark.parametrize("masks", [False, True])
def test_printed_lines_match_caffes_pattern(masks):
    s = summary(masks)
    lines = T.val_lines(2000, s)
    assert lines[0] == "Iteration 2000, Testing net (#0)"
    got = [CAFFE_TEST.search(l).groups() for l in lines[1:]]
    keys = ["epe", "epe_pair_mean", "fl_percent", "s0-10", "s10-40", "s40+"]
    if masks:
        keys += ["epe_matched", "epe_unmatched", "d0-10", "d10-60", "d60-140"]
    assert [k for _, k, _ in got] == keys and [int(i) for i, _, _ in got] == list(range(len(keys)))
    value = {k: v for _, k, v in got}
    assert float(value["epe"]) == pytest.approx(175.0 / 150, rel=1e-5) and value["s40+"] == "nan"
    assert float(value["fl_percent"]) == pytest.approx(2.0, rel=1e-5)
    assert all(math.isfinite(float(v)) or v == "nan" for v in value.values())


def test_not_finite_pairs_get_one_line_and_the_log():
    s = summary(nonfinite=4)
    lines = T.val_lines(7, s)
    extra = [l for l in lines if not CAFFE_TEST.search(l) and not l.startswith("Iteration")]
    assert extra == ["    1 validation pairs have a prediction that is not finite"]
    rec = json.loads(T.val_record(7, s, 0.25, 1.5))
    assert rec["iter"] == 7 and rec["not_finite"] == ["val.txt:1"] and rec["s40+"] is None
    assert rec["handover_s"] == 0.25 and rec["wall_s"] == 1.5
    assert list(rec)[1:-2] == list(s)                                  # the summary's keys, in order, between the two
    assert "NaN" not in T.val_record(7, s, 0.25, 1.5)


# ---- the hand-over check on Net.param_layers tables ----
CONV = lambda name, co, ci, lr=1.0: (name, "Convolution", "", [(co, ci, 3, 3), (co,)], [lr, lr])
AUG = lambda name, h, w: (name, "DataAugmentation", "c", [(1, 1, 1, 1), (1, 3, h, w), (1, 3, 1, 1)], [0.0, 0.0, 0.0])
SCALE = ("scale_conv1", "Convolution", "t", [(2, 2, 1, 1)], [0.0])


def test_handover_accepts_matching_nets():
    train = [AUG("img0s_aug", 320, 448), CONV("conv1", 16, 6), CONV("predict", 2, 16)]
    deploy = [AUG("img0s_aug", 436, 1024), CONV("conv1", 16, 6), CONV("predict", 2, 16, 0.0), SCALE]
    E.check_handover(train, deploy)                                    # crops differ: the augmentation adjusts its blobs
    E.check_handover([CONV("net1_conv1", 16, 6, 0.0)] + train, deploy)  # frozen layers the deploy net lacks are left out


def test_handover_refusals():
    train = [CONV("conv1", 16, 6), CONV("predict", 2, 16)]
    with pytest.raises(RunError, match="^the training net trains layer predict, which d.prototxt lacks$"):
        E.check_handover(train, [CONV("conv1", 16, 6), SCALE], "d.prototxt")
    with pytest.raises(RunError, match="layer net1_conv1 of d.prototxt gets no weights from the training net"):
        E.check_handover(train, train + [CONV("net1_conv1", 16, 6)], "d.prototxt")
    with pytest.raises(RunError, match="layer conv1 has blobs"):
        E.check_handover(train, [CONV("conv1", 32, 6), CONV("predict", 2, 16)])
    E.check_handover([("c", "Convolution", "", [(1, 1, 16, 6)], [1.0])], [("c", "Convolution", "", [(16, 6)], [1.0])])


# ---- refused flags ----
@pytest.fixture
def files(tmp_path):
    """A solver, a model, a training list and a validation list of 48 x 32 frames, and a deploy template."""
    r = np.random.default_rng(0)
    lines = []
    for i in range(3):
        a = write_pnm(tmp_path / ("a%d.ppm" % i), r.integers(0, 256, (32, 48, 3), dtype=np.uint8))
        b = write_pnm(tmp_path / ("b%d.ppm" % i), r.integers(0, 256, (32, 48, 3), dtype=np.uint8))
        f = str(tmp_path / ("f%d.flo" % i))
        write_flo(f, r.normal(0, 3, (32, 48, 2)).astype(np.float32))
        lines.append("%s %s %s\n" % (a, b, f))
    (tmp_path / "train.txt").write_text("".join(lines))
    (tmp_path / "val.txt").write_text("".join(lines[:2]))
    (tmp_path / "bad.txt").write_text(lines[0] + "x.ppm y.ppm z.flo\n")
    (tmp_path / "occ.txt").write_text("only_one.pgm\n")
    (tmp_path / "s.prototxt").write_text('type: "Adam"\nbase_lr: 1e-3\nlr_policy: "fixed"\nmax_iter: 4\n')
    (tmp_path / "m.prototxt").write_text("name: \"m\"\n")
    (tmp_path / "d.prototxt").write_text("name: \"d\"\n")
    return tmp_path


def refused(monkeypatch, capsys, files, extra):
    import flownet2_b200 as F

    def no_net(*a, **k):
        raise AssertionError("a net was built before the refusal")
    monkeypatch.setattr(F, "Net", no_net)
    capsys.readouterr()
    argv = ["--solver", str(files / "s.prototxt"), "--model", str(files / "m.prototxt"), "--data", str(files / "train.txt"),
            "--crop", "48x32", "--batch", "1"]
    assert T.main(argv + [x.format(d=files) for x in extra]) == 2
    err = capsys.readouterr().err
    assert err.startswith("error: ") and err.count("\n") == 1, err
    return err


VAL = ["--val", "{d}/val.txt", "--val-model", "{d}/d.prototxt", "--val-interval", "2"]


@pytest.mark.parametrize("extra,message", [
    (["--val-model", "{d}/d.prototxt"], "--val-model needs --val"),
    (["--val-interval", "5"], "--val-interval needs --val"),
    (["--val-batch", "2"], "--val-batch needs --val"),
    (["--no-val-initial"], "--no-val-initial needs --val"),
    (["--val-log", "{d}/log.jsonl"], "--val-log needs --val"),
    (["--val-occlusions", "{d}/occ.txt"], "--val-occlusions needs --val"),
    (["--val-objects", "{d}/occ.txt"], "--val-objects needs --val"),
    (["--val", "{d}/val.txt", "--val-interval", "2"], "--val needs --val-model"),
    (["--val", "{d}/val.txt", "--val-model", "{d}/d.prototxt"], "--val needs --val-interval"),
    (VAL[:-1] + ["0"], "--val-interval must be at least 1, got 0"),
    (VAL + ["--val-batch", "0"], "--val-batch must be at least 1, got 0"),
    (["--val", "{d}/nothing.txt"] + VAL[2:], "nothing.txt: no such validation list"),
    (VAL[:2] + ["--val-model", "{d}/nothing.prototxt"] + VAL[4:], "nothing.prototxt: no such deploy prototxt template"),
    (["--val", "{d}/bad.txt"] + VAL[2:], "bad.txt:2: x.ppm: no such file"),
    (VAL + ["--val-occlusions", "{d}/occ.txt"], "occ.txt"),
])
def test_refusals_exit_2_with_one_line_before_any_net(monkeypatch, capsys, files, extra, message):
    assert message in refused(monkeypatch, capsys, files, extra)
