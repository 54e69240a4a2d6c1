"""GPU: the evaluate command end to end.  Over a list of two frame sizes with .flo and both PFM byte orders as ground truth,
evaluate's per-pair records at --batch 1 equal the float32 metrics of the .flo files flownet2_b200.run writes for the same
list (the same predictions, bit for bit); --batch 3 agrees within the project's 1e-4 flow bound; the command prints its JSON
line and writes one --per-pair row per list line."""
import json
import os

import numpy as np
import pytest

from flownet2_b200 import FLOW_ERROR_FIELDS
from flownet2_b200 import evaluate as E
from flownet2_b200 import run as R
from flownet2_b200.files import read_flow, read_list, write_flo, write_pfm
from tests.flow_error_ref import assert_records_match, flow_error_ref
from tests.test_run_flownet_cpu import write_pnm
from tests.test_run_flownet_gpu import chairs_frames

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELD = {f: i for i, f in enumerate(FLOW_ERROR_FIELDS)}
A, B = (128, 96), (192, 64)
SPEC = [(A, "flo"), (B, "pfm"), (A, "pfm_be"), (B, "flo"), (A, "flo")]


def ground_truth(size, seed):
    """(H, W, 2) float32 flow over the three speed bands, with a NaN row, unknown (1e10) pixels and a NaN v component."""
    w, h = size
    r = np.random.default_rng(seed)
    f = (r.standard_normal((h, w, 2)) * r.choice([3.0, 20.0, 50.0], (h, w, 1))).astype(np.float32)
    f[h // 3] = np.nan
    f[5:9, 11, 0] = 1e10
    f[2, 3:40, 1] = np.nan
    return f


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    """Frames, ground truth and the two lists (evaluate's img0 img1 gt; run's img0 img1 out.flo) over SPEC."""
    d = tmp_path_factory.mktemp("eval")
    ev, rn = [], []
    for i, (size, kind) in enumerate(SPEC):
        f0, f1 = chairs_frames(size, 300 + i)
        a, b = write_pnm(d / ("p%d_0.ppm" % i), f0), write_pnm(d / ("p%d_1.ppm" % i), f1)
        gt = ground_truth(size, 400 + i)
        if kind == "flo":
            g = str(d / ("g%d.flo" % i))
            write_flo(g, gt)
        else:
            g = write_pfm(str(d / ("g%d.pfm" % i)), np.concatenate([gt, np.zeros_like(gt[:, :, :1])], axis=2),
                          big_endian=kind == "pfm_be")
        ev.append("%s %s %s\n" % (a, b, g))
        rn.append("%s %s %s\n" % (a, b, d / ("out%d.flo" % i)))
    (d / "val.txt").write_text("".join(ev))
    (d / "run.txt").write_text("".join(rn))
    return d


@pytest.fixture(scope="module", params=["FlowNet2-S", "FlowNet2"])
def model(request, scene, fn2):
    net = fn2.Net(fn2.fill_template(fn2.model_template(request.param), 128, 128), None, fn2.TEST, batch=1)
    net.fill_params(1701)
    path = scene / ("%s.caffemodel" % request.param)
    path.write_bytes(net.to_caffemodel())
    del net
    return str(path), os.path.join(ROOT, "models", "%s_deploy.prototxt.template" % request.param)


def test_evaluate_equals_metrics_of_run_outputs(fn2, scene, model, tmp_path, capsys):
    weights, template = model
    samples = read_list(str(scene / "val.txt"))
    assert R.main([weights, template, str(scene / "run.txt")]) == 0
    want, peak = [], 1.0
    for i, s in enumerate(samples):
        pred = fn2.read_flo(str(scene / ("out%d.flo" % i)))[None]
        peak = max(peak, float(np.abs(pred).max()))
        gt = read_flow(s.flow).transpose(2, 0, 1)[None]
        assert np.isnan(gt).any() and (gt == 1e10).any()
        want.append(flow_error_ref(pred, gt)[0])
    want = np.array(want)

    summary, rec1 = E.evaluate(weights, template, samples, batch=1)
    assert_records_match(rec1, want)
    assert summary["pairs"] == 5 and summary["not_finite"] == [] and summary["sizes"] == 2
    for k, v in E.summarize(want, [w * h for (w, h), _ in SPEC], "val.txt").items():
        assert summary[k] == pytest.approx(v, rel=1e-12), k
    assert summary["valid_px"] + summary["invalid_px"] == sum(w * h for (w, h), _ in SPEC)
    assert all(rec1[:, FIELD["n_s0_10"]] > 0) and all(rec1[:, FIELD["n_s40"]] > 0) and rec1[:, FIELD["outliers"]].sum() > 0

    # the command at --batch 3, with the per-pair file
    tsv = tmp_path / "pairs.tsv"
    capsys.readouterr()
    assert E.main([weights, template, str(scene / "val.txt"), "--batch", "3", "--per-pair", str(tsv)]) == 0
    line = capsys.readouterr().out.strip().splitlines()
    assert len(line) == 1
    out = json.loads(line[0])
    for k in ("pairs", "valid_px", "invalid_px", "nonfinite_px", "epe", "epe_pair_mean", "fl_percent", "s0-10", "s10-40", "s40+",
              "batch", "wall"):
        assert k in out, k
    assert out["batch"] == 3 and out["pairs"] == 5 and out["valid_px"] == summary["valid_px"]
    rows = tsv.read_text().splitlines()
    assert len(rows) == 1 + len(samples) and rows[3].startswith(samples[2].where + "\t")

    _, rec3 = E.evaluate(weights, template, read_list(str(scene / "val.txt")), batch=3)
    for f in ("valid", "nonfinite", "n_s0_10", "n_s10_40", "n_s40"):                 # decided by the ground truth alone
        assert np.array_equal(rec3[:, FIELD[f]], rec1[:, FIELD[f]]), f
    counted = rec1[:, FIELD["valid"]]
    bound = 2 * np.sqrt(2) * 1e-4 * peak                          # both flows within 1e-4 (of max(1, |flow|)) of float64
    assert np.all(np.abs(rec3[:, FIELD["epe_sum"]] - rec1[:, FIELD["epe_sum"]]) <= bound * counted)
    assert np.all(np.abs(rec3[:, FIELD["outliers"]] - rec1[:, FIELD["outliers"]]) <= 2)
    assert abs(out["epe"] - summary["epe"]) <= bound
