"""GPU: the train command's --val.  Each validation's records equal evaluate() on the snapshot of the same iteration, bit for
bit (plain, and KITTI flows with occlusion masks); snapshots, solverstates and display lines are the same with and without
--val; the kept deploy nets allocate nothing from the second validation on; a resumed run validates at its first iteration
and matches the uninterrupted run; two ranks validate one list between them; and the hand-over check refuses a deploy net
that does not fit the training net."""
import json
import os
import re

import numpy as np
import pytest

from flownet2_b200 import evaluate as E
from flownet2_b200 import kitti as K
from flownet2_b200 import train as T
from flownet2_b200.files import read_list, write_pnm
from tests.test_train_data_gpu import TINY_NET, scene

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY_DEPLOY = """name: "tiny"
input: "img0"
input_shape { dim: 1 dim: 3 dim: $TARGET_HEIGHT$ dim: $TARGET_WIDTH$ }
input: "img1"
input_shape { dim: 1 dim: 3 dim: $TARGET_HEIGHT$ dim: $TARGET_WIDTH$ }
layer { name: "scale0" type: "Eltwise" bottom: "img0" top: "img0s" eltwise_param { operation: SUM coeff: 0.00392156862745 } }
layer { name: "scale1" type: "Eltwise" bottom: "img1" top: "img1s" eltwise_param { operation: SUM coeff: 0.00392156862745 } }
layer { name: "concat" type: "Concat" bottom: "img0s" bottom: "img1s" top: "pair" }
layer { name: "conv1" type: "Convolution" bottom: "pair" top: "conv1"
  convolution_param { num_output: 16 kernel_size: 3 pad: 1 weight_filler { type: "msra" } bias_filler { type: "constant" } } }
layer { name: "relu1" type: "ReLU" bottom: "conv1" top: "conv1" relu_param { negative_slope: 0.1 } }
layer { name: "predict" type: "Convolution" bottom: "conv1" top: "predict_flow_final"
  convolution_param { num_output: 2 kernel_size: 3 pad: 1 weight_filler { type: "msra" } bias_filler { type: "constant" } } }
"""
SOLVER = ('type: "Adam"\nbase_lr: 1e-3\nlr_policy: "step"\ngamma: 0.5\nstepsize: 4\nmax_iter: %d\nsnapshot: %d\n'
          'snapshot_prefix: "%s"\ndisplay: 2\n')
TIMING = re.compile(r" \(.*?\)")


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def same_summary(a, b):
    drop = ("wall", "busy", "iter", "handover_s", "wall_s")
    return {k: v for k, v in a.items() if k not in drop} == {k: v for k, v in b.items() if k not in drop}


@pytest.fixture
def scored(monkeypatch, fn2):
    """Every Validator.score call of the test: (validator, summary, records, engine allocations made during the call)."""
    got = []
    score = E.Validator.score

    def wrap(self, weights):
        n0 = fn2.device_allocations()[0]
        summary, records = score(self, weights)
        got.append((self, summary, records, fn2.device_allocations()[0] - n0))
        return summary, records
    monkeypatch.setattr(E.Validator, "score", wrap)
    return got


def kitti_scene(d, n, w, h, seed):
    """n pairs of w x h frames with KITTI PNG flows (a third of the pixels invalid) and occlusion masks -> (list, masks)."""
    r = np.random.default_rng(seed)
    lines, masks = [], []
    for i in range(n):
        a = write_pnm(d / ("k%d_%d_0.ppm" % (seed, i)), r.integers(0, 256, (h, w, 3), dtype=np.uint8))
        b = write_pnm(d / ("k%d_%d_1.ppm" % (seed, i)), r.integers(0, 256, (h, w, 3), dtype=np.uint8))
        f = r.normal(0, 8, (h, w, 2)).astype(np.float32)
        f[r.random((h, w)) < 0.3] = np.nan
        g = str(d / ("k%d_%d.png" % (seed, i)))
        K.write_kitti_flow(g, f)
        masks.append(write_pnm(d / ("o%d_%d.pgm" % (seed, i)), np.where(r.random((h, w)) < 0.2, 255, 0).astype(np.uint8)))
        lines.append("%s %s %s\n" % (a, b, g))
    return lines, masks


def tiny_files(fn2, d, kitti):
    """The training list (48 x 32), a validation list of two frame sizes (occlusion masks with kitti), the TINY_NET model, its
    deploy template and initial weights."""
    if kitti:
        train, _ = kitti_scene(d, 7, 48, 32, 1)
        (d / "train.txt").write_text("".join(train))
        v0, m0 = kitti_scene(d, 3, 48, 32, 2)
        v1, m1 = kitti_scene(d, 2, 40, 24, 3)
        (d / "occ.txt").write_text("".join(m + "\n" for m in m0 + m1))
        lst = str(d / "train.txt")
    else:
        for sub in ("t", "v0", "v1"):
            (d / sub).mkdir()
        lst = scene(d / "t", 7, 48, 32)
        v0 = open(scene(d / "v0", 3, 48, 32, seed=5)).readlines()
        v1 = open(scene(d / "v1", 2, 40, 24, seed=6)).readlines()
    (d / "val.txt").write_text("".join(v0 + v1))
    (d / "tiny.prototxt.template").write_text(TINY_NET)
    (d / "tiny_deploy.prototxt.template").write_text(TINY_DEPLOY)
    net = fn2.Net(fn2.fill_train_template(TINY_NET, 48, 32, 48, 32, 2), None, fn2.TRAIN)
    net.fill_params(3)
    (d / "init.caffemodel").write_bytes(net.to_caffemodel())
    return lst


def run_train(capsys, d, sub, lst, max_iter, snap, extra, kitti=False):
    (d / sub).mkdir(exist_ok=True)
    os.chdir(d / sub)
    (d / sub / "s.prototxt").write_text(SOLVER % (max_iter, snap, "tiny"))
    capsys.readouterr()
    argv = ["--solver", "s.prototxt", "--model", str(d / "tiny.prototxt.template"), "--data", lst, "--crop", "48x32",
            "--batch", "2"] + (["--kitti"] if kitti else []) + extra
    assert T.main(argv) == 0
    return capsys.readouterr().out.splitlines()


def val_args(d, kitti, interval=2):
    return (["--val", str(d / "val.txt"), "--val-model", str(d / "tiny_deploy.prototxt.template"), "--val-interval",
             str(interval), "--val-log", "val.jsonl"] + (["--val-occlusions", str(d / "occ.txt")] if kitti else []))


def evaluate_file(d, weights, kitti):
    return E.evaluate(str(weights), str(d / "tiny_deploy.prototxt.template"), read_list(str(d / "val.txt")), batch=1,
                      kitti=kitti, occlusions=str(d / "occ.txt") if kitti else None)


@pytest.mark.parametrize("kitti", [False, True], ids=["flo", "kitti-occlusions"])
def test_validation_equals_evaluate_of_each_snapshot(fn2, tmp_path, monkeypatch, capsys, scored, kitti):
    monkeypatch.chdir(tmp_path)
    lst = tiny_files(fn2, tmp_path, kitti)
    init = ["--weights", str(tmp_path / "init.caffemodel")]
    out = run_train(capsys, tmp_path, "val", lst, 6, 2, init + val_args(tmp_path, kitti), kitti)
    plain = run_train(capsys, tmp_path, "plain", lst, 6, 2, init, kitti)
    # validations at 0, N, 2N and the end; each equals evaluate() on that iteration's weights
    log = [json.loads(l) for l in open(tmp_path / "val" / "val.jsonl")]
    assert [r["iter"] for r in log] == [0, 2, 4, 6] and len(scored) == 4
    for rec, (_, summary, records, _) in zip(log, scored):
        k = rec["iter"]
        weights = tmp_path / "init.caffemodel" if k == 0 else tmp_path / "val" / ("tiny_iter_%d.caffemodel" % k)
        want, want_records = evaluate_file(tmp_path, weights, kitti)
        assert np.array_equal(bits(records), bits(want_records)), k
        assert same_summary(rec, want) and same_summary(summary, want), k
        assert rec["handover_s"] > 0 and rec["wall_s"] >= rec["handover_s"]
        if kitti:
            assert want["invalid_px"] > 0 and want["epe_matched"] is not None and want["epe_unmatched"] is not None
    assert any(not np.array_equal(bits(scored[0][2]), bits(s[2])) for s in scored[1:])      # the weights moved
    # the printed validations, and the rest of the output as without --val
    tests = [l for l in out if "Testing net" in l]
    assert tests == ["Iteration %d, Testing net (#0)" % k for k in (0, 2, 4, 6)]
    outputs = [l for l in out if "Test net output #" in l]
    assert len(outputs) == 4 * len(T.score_keys(log[0]))
    rest = [TIMING.sub("", l) for l in out if "Test" not in l]
    assert rest == [TIMING.sub("", l) for l in plain] and "Optimization Done." in rest
    names = sorted(f for f in os.listdir(tmp_path / "plain") if f.startswith("tiny_iter_"))
    assert len(names) == 6
    for f in names:
        assert (tmp_path / "val" / f).read_bytes() == (tmp_path / "plain" / f).read_bytes(), f


def test_resumed_run_validates_at_its_first_iteration(fn2, tmp_path, monkeypatch, capsys, scored):
    monkeypatch.chdir(tmp_path)
    lst = tiny_files(fn2, tmp_path, False)
    init = ["--weights", str(tmp_path / "init.caffemodel")]
    run_train(capsys, tmp_path, "a", lst, 6, 2, init + val_args(tmp_path, False))
    run_train(capsys, tmp_path, "b", lst, 4, 4, init)
    out = run_train(capsys, tmp_path, "b", lst, 6, 2, ["--snapshot", "tiny_iter_4.solverstate"] + val_args(tmp_path, False))
    assert [l for l in out if "Testing net" in l] == ["Iteration 4, Testing net (#0)", "Iteration 6, Testing net (#0)"]
    a = {r["iter"]: r for r in map(json.loads, open(tmp_path / "a" / "val.jsonl"))}
    b = [json.loads(l) for l in open(tmp_path / "b" / "val.jsonl")]
    assert [r["iter"] for r in b] == [4, 6]
    for r in b:
        assert same_summary(r, a[r["iter"]]), r["iter"]
    assert np.array_equal(bits(scored[2][2]), bits(scored[4][2])) and np.array_equal(bits(scored[3][2]), bits(scored[5][2]))


def test_flownet2_c_validation_and_its_allocations(fn2, tmp_path, monkeypatch, capsys, scored):
    """FlowNet2-C trained at a 192 x 128 crop from fill_params, validated with the C deploy template every iteration."""
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("FN2_SEED", "5")
    lst = scene(tmp_path, 5, 224, 160)
    (tmp_path / "v").mkdir()
    (tmp_path / "val.txt").write_text(open(scene(tmp_path / "v", 2, 224, 160, seed=9)).read())
    deploy = os.path.join(ROOT, "models", "FlowNet2-C_deploy.prototxt.template")
    model = os.path.join(ROOT, "models", "FlowNet2-C_train.prototxt.template")
    (tmp_path / "s.prototxt").write_text(SOLVER % (4, 1, "c"))
    argv = ["--solver", "s.prototxt", "--model", model, "--data", lst, "--crop", "192x128", "--batch", "2", "--val",
            str(tmp_path / "val.txt"), "--val-model", deploy, "--val-interval", "1", "--val-log", "val.jsonl"]
    assert T.main(argv) == 0
    assert len(scored) == 5 and all(s[3] == 0 for s in scored[1:]), [s[3] for s in scored]   # kept nets: no new buffers
    val = scored[0][0]
    (net,) = val.nets.values()
    w, h = 224, 160
    sx, sy = w / (np.ceil(w / 64) * 64), h / (np.ceil(h / 64) * 64)
    assert np.array_equal(net.param("scale_conv1")[:, :, 0, 0], np.diag(np.float32([sx, sy])))   # defined by the template
    samples = read_list(str(tmp_path / "val.txt"))
    train = fn2.Net(T.model_text(model, (192, 128), (224, 160), 2), None, fn2.TRAIN)
    train.fill_params(5)
    (tmp_path / "c_iter_0.caffemodel").write_bytes(train.to_caffemodel())
    for k, (_, summary, records, _) in enumerate(scored):
        want, want_records = E.evaluate(str(tmp_path / ("c_iter_%d.caffemodel" % k)), deploy, samples)
        assert np.array_equal(bits(records), bits(want_records)), k
        assert same_summary(summary, want) and np.isfinite(want["epe"]), k


def _world2_worker(rank, port, tmp, lst, model, val, deploy, q):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=2)
    try:
        os.chdir(os.path.join(tmp, "r%d" % rank))
        a = T.parse_args(["--solver", "s.prototxt", "--model", model, "--data", lst, "--crop", "48x32", "--batch", "2",
                          "--val", val, "--val-model", deploy, "--val-interval", "2", "--val-log", "val.jsonl"])
        with open("out.txt", "w") as out:
            T.train(a, world=2, rank=rank, device=0, out=out)
        q.put((rank, sorted(os.listdir("."))))
    finally:
        dist.destroy_process_group()


def test_two_ranks_validate_the_list_between_them(fn2, tmp_path):
    import torch.multiprocessing as mp
    tiny_files(fn2, tmp_path, False)
    lst = str(tmp_path / "t" / "list.txt")
    for r in (0, 1):
        (tmp_path / ("r%d" % r)).mkdir()
        (tmp_path / ("r%d" % r) / "s.prototxt").write_text(SOLVER % (4, 2, "w2"))
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() % 2000) + 7
    args = (str(tmp_path), lst, str(tmp_path / "tiny.prototxt.template"), str(tmp_path / "val.txt"),
            str(tmp_path / "tiny_deploy.prototxt.template"), q)
    procs = [ctx.Process(target=_world2_worker, args=(r, port) + args) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in procs)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert "val.jsonl" in res[0] and "val.jsonl" not in res[1]
    assert "Testing net" not in (tmp_path / "r1" / "out.txt").read_text()
    printed = (tmp_path / "r0" / "out.txt").read_text()
    assert [l for l in printed.splitlines() if "Testing net" in l] == ["Iteration %d, Testing net (#0)" % k for k in (0, 2, 4)]
    log = [json.loads(l) for l in open(tmp_path / "r0" / "val.jsonl")]
    samples = read_list(str(tmp_path / "val.txt"))
    deploy = str(tmp_path / "tiny_deploy.prototxt.template")
    for r in log[1:]:
        want, _ = E.evaluate(str(tmp_path / "r0" / ("w2_iter_%d.caffemodel" % r["iter"])), deploy, samples)
        assert same_summary(r, want) and r["pairs"] == 5, r["iter"]


STAGES = ["FlowNet2-C", "FlowNet2-CS", "FlowNet2-CSS", "FlowNet2-SD", "FlowNet2"]


def test_handover_check(fn2, tmp_path, monkeypatch, capsys):
    (tmp_path / "v").mkdir()
    samples = read_list(scene(tmp_path / "v", 1, 64, 64))
    trains = {s: fn2.Net(fn2.fill_train_template(fn2.train_template(s), 192, 128, 192, 128, 1), None, fn2.TRAIN) for s in STAGES}
    deploy = lambda s: os.path.join(ROOT, "models", "%s_deploy.prototxt.template" % s)
    for s in STAGES:                                                    # each stage's deploy net takes its training net
        E.Validator(deploy(s), samples).check_handover(trains[s])
    with pytest.raises(E.RunError, match="trains layer conv1, which .*FlowNet2-CSS_deploy.prototxt.template lacks"):
        E.Validator(deploy("FlowNet2-CSS"), samples).check_handover(trains["FlowNet2-C"])
    with pytest.raises(E.RunError, match="trains layer net2_conv1, which .*FlowNet2-C_deploy.prototxt.template lacks"):
        E.Validator(deploy("FlowNet2-C"), samples).check_handover(trains["FlowNet2-CS"])
    # the command refuses before iteration 0
    monkeypatch.chdir(tmp_path)
    lst = scene(tmp_path, 3, 224, 160)
    (tmp_path / "s.prototxt").write_text(SOLVER % (2, 0, "x"))
    capsys.readouterr()
    assert T.main(["--solver", "s.prototxt", "--model", os.path.join(ROOT, "models", "FlowNet2-CS_train.prototxt.template"),
                   "--data", lst, "--crop", "192x128", "--batch", "1", "--val", str(tmp_path / "v" / "list.txt"),
                   "--val-model", deploy("FlowNet2-C"), "--val-interval", "1"]) == 2
    cap = capsys.readouterr()
    assert cap.err.count("\n") == 1 and "net2_conv1" in cap.err and "Iteration" not in cap.out
