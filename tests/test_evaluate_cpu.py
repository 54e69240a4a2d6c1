"""Host side of the evaluate command (flownet2_b200.evaluate): arguments, the refusals that name their list line, the summary's
arithmetic, and the recombination of per-rank records.  No GPU needed."""
import json
import re

import numpy as np
import pytest

from flownet2_b200 import FLOW_ERROR_FIELDS
from flownet2_b200 import evaluate as E, files as FI
from flownet2_b200.files import RunError, write_flo, write_pfm
from flownet2_b200.run import shard
from tests.test_run_flownet_cpu import write_pnm

FIELD = {f: i for i, f in enumerate(FLOW_ERROR_FIELDS)}


def test_arguments():
    a = E.parse_args(["w.caffemodel", "t.template", "val.txt"])
    assert (a.caffemodel, a.deployproto, a.listfile, a.batch, a.per_pair, a.gpu) == ("w.caffemodel", "t.template", "val.txt", 1,
                                                                                     None, 0)
    a = E.parse_args(["w", "t", "l", "--batch", "8", "--per-pair", "o.tsv", "--gpu", "2"])
    assert (a.batch, a.per_pair, a.gpu) == (8, "o.tsv", 2)
    with pytest.raises(SystemExit):
        E.parse_args(["w", "t"])
    with pytest.raises(SystemExit):
        E.parse_args(["w", "t", "l", "extra"])


@pytest.fixture
def files(tmp_path):
    """A model and template that exist, two 9x7 frames and flows in every accepted form."""
    r = np.random.default_rng(0)
    f = r.integers(0, 256, (7, 9, 3), dtype=np.uint8)
    d = {"model": tmp_path / "m.caffemodel", "proto": tmp_path / "t.template"}
    d["model"].write_bytes(b"")
    d["proto"].write_text("")
    d["a"], d["b"] = write_pnm(tmp_path / "a.ppm", f), write_pnm(tmp_path / "b.ppm", f)
    flow = r.standard_normal((7, 9, 2)).astype(np.float32)
    d["flo"] = str(tmp_path / "g.flo")
    write_flo(d["flo"], flow)
    d["pfm"] = write_pfm(str(tmp_path / "g.pfm"), np.concatenate([flow, flow[:, :, :1]], axis=2))
    d["wide"] = str(tmp_path / "wide.flo")
    write_flo(d["wide"], np.zeros((7, 10, 2), np.float32))
    d["png"] = str(tmp_path / "g.png")
    open(d["png"], "wb").write(b"\x89PNG")
    d["dir"] = tmp_path
    return d


def refused(files, capsys, lines, match):
    lst = files["dir"] / "val.txt"
    lst.write_text("".join(l + "\n" for l in lines))
    assert E.main([str(files["model"]), str(files["proto"]), str(lst)]) == 2
    err = capsys.readouterr().err
    assert re.search(match, err), err


def test_refusals_name_the_list_line(files, capsys):
    a, b = files["a"], files["b"]
    good = "%s %s %s" % (a, b, files["flo"])
    refused(files, capsys, [good, "", "%s %s %s" % (a, b, files["dir"] / "none.flo")], r"val\.txt:3: .*none\.flo: no such file")
    refused(files, capsys, [good, "%s %s %s" % (a, b, files["wide"])], r"val\.txt:2: .*wide\.flo is 10x7 but its frames are 9x7")
    refused(files, capsys, ["%s %s %s" % (a, b, files["png"])], r"val\.txt:1: .*g\.png: flows must be \.flo or \.pfm files")
    refused(files, capsys, [good, good + " occ.png"], r"val\.txt:2: an occlusion field")
    refused(files, capsys, ["%s %s" % (a, b)], r"val\.txt:1: 2 fields")
    refused(files, capsys, [], r"val\.txt: the list holds no pairs")
    lst = files["dir"] / "ok.txt"
    lst.write_text(good + "\n" + "%s %s %s\n" % (a, b, files["pfm"]))
    samples = FI.read_list(str(lst))
    FI.probe(samples, ground_truth=True)                                            # a .flo and a PFM in one list are fine
    assert [s.size for s in samples] == [(9, 7)] * 2 and [s.flow_header.nbytes for s in samples] == [9 * 7 * 8, 9 * 7 * 12]
    assert E.main([str(files["dir"] / "none.caffemodel"), str(files["proto"]), str(lst)]) == 2
    assert "none.caffemodel: no such caffemodel" in capsys.readouterr().err


def synthetic_records(n, seed):
    """Plausible per-pair records: band counts summing to valid - nonfinite, sums of EPEs, outliers within the counted pixels."""
    r = np.random.default_rng(seed)
    rec = np.zeros((n, len(FLOW_ERROR_FIELDS)))
    for i in range(n):
        nb = r.integers(0, 500, 3)
        sb = nb * r.uniform(0.1, 20.0, 3)
        bad = 1 + r.integers(0, 3) if i % 5 == 4 else 0
        rec[i, FIELD["n_s0_10"]], rec[i, FIELD["n_s10_40"]], rec[i, FIELD["n_s40"]] = nb
        rec[i, FIELD["sum_s0_10"]], rec[i, FIELD["sum_s10_40"]], rec[i, FIELD["sum_s40"]] = sb
        rec[i, FIELD["nonfinite"]] = bad
        rec[i, FIELD["valid"]] = nb.sum() + bad
        rec[i, FIELD["epe_sum"]] = sb.sum()
        rec[i, FIELD["outliers"]] = r.integers(0, nb.sum() + 1)
    return rec


def test_summary_arithmetic():
    rec = synthetic_records(7, 1)
    rec[3] = 0                                                          # a pair without a valid pixel
    rec[3, FIELD["valid"]] = 0
    pixels = np.full(7, 2000)
    s = E.summarize(rec, pixels, "val.txt")
    valid, nonfinite = rec[:, FIELD["valid"]], rec[:, FIELD["nonfinite"]]
    counted = valid - nonfinite
    assert s["pairs"] == 7 and s["valid_px"] == valid.sum() and s["invalid_px"] == 14000 - valid.sum()
    assert s["nonfinite_px"] == nonfinite.sum() > 0
    assert s["epe"] == rec[:, FIELD["epe_sum"]].sum() / counted.sum()
    has = counted > 0
    assert s["epe_pair_mean"] == pytest.approx(np.mean(rec[has, FIELD["epe_sum"]] / counted[has]), rel=1e-15)
    assert not has[3] and has.sum() == 6
    assert s["fl_percent"] == pytest.approx(100 * rec[:, FIELD["outliers"]].sum() / counted.sum(), rel=1e-15)
    for key, n, total in (("s0-10", "n_s0_10", "sum_s0_10"), ("s10-40", "n_s10_40", "sum_s10_40"), ("s40+", "n_s40", "sum_s40")):
        assert s[key] == pytest.approx(rec[:, FIELD[total]].sum() / rec[:, FIELD[n]].sum(), rel=1e-15)
    json.dumps(s)                                                       # plain numbers only
    rec[:, FIELD["n_s40"]] = rec[:, FIELD["sum_s40"]] = 0
    assert E.summarize(rec, pixels, "val.txt")["s40+"] is None          # an empty band
    with pytest.raises(RunError, match=r"val\.txt: no ground-truth pixel is valid in any of its 7 pairs"):
        E.summarize(np.zeros((7, len(FLOW_ERROR_FIELDS))), pixels, "val.txt")


def test_per_pair_rows(tmp_path):
    rec = synthetic_records(4, 2)
    rec[1] = 0

    class S(object):
        def __init__(self, i):
            self.where, self.img0, self.img1, self.flow = "val.txt:%d" % (i + 1), "a%d.ppm" % i, "b%d.ppm" % i, "f%d.flo" % i

    samples = [S(i) for i in range(4)]
    p = tmp_path / "pairs.tsv"
    E.write_per_pair(str(p), samples, rec)
    rows = [l.split("\t") for l in p.read_text().splitlines()]
    assert rows[0] == ["where", "img0", "img1", "flow", "valid", "epe", "fl_percent"] and len(rows) == 5
    assert rows[2][:5] == ["val.txt:2", "a1.ppm", "b1.ppm", "f1.flo", "0"] and rows[2][5:] == ["nan", "nan"]
    counted = rec[0, FIELD["valid"]] - rec[0, FIELD["nonfinite"]]
    assert float(rows[1][5]) == pytest.approx(rec[0, FIELD["epe_sum"]] / counted, rel=1e-8)
    assert [s.where for s in E.not_finite(samples, rec)] == []
    rec[2, FIELD["nonfinite"]] = 1
    assert [s.where for s in E.not_finite(samples, rec)] == ["val.txt:3"]


@pytest.mark.parametrize("n", [1, 5, 12, 13])
def test_rank_recombination_is_bit_exact(n):
    rec = np.concatenate([synthetic_records(n, 3), np.full((n, 1), 436.0 * 1024)], axis=1)
    want = E.summarize(rec[:, :-1], rec[:, -1], "val.txt")
    for world in (1, 2, 3, 4, 8):
        shards = [np.array([rec[i] for i in shard(range(n), world, r)]).reshape(-1, rec.shape[1]) for r in range(world)]
        back = E.combine_shards(shards)
        assert np.array_equal(back.view(np.uint64), rec.view(np.uint64)), world
        assert E.summarize(back[:, :-1], back[:, -1], "val.txt") == want, world
