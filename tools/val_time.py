"""Time the train command's validation (--val) on an H100, for the FlowNet2-C stage and the fusion stage (FlowNet2):

  * hand-over: the training net's weights into the kept deploy nets, as a validation does it -- Net.to_caffemodel() of the
    training net (448 x 320 crop, batch 8, fill_params weights), then Net.copy_from of those bytes into the deploy net; the
    median over --reps, each ending in a device synchronise;
  * validation: one Validator.score pass over --pairs Sintel-size (1024 x 436) pairs at --val-batch 1, after a first pass
    that builds the deploy net; the median wall time over --reps passes;
  * evaluate: the evaluate command on the same list and the same weights as a snapshot file, in a process of its own; its
    process wall time (interpreter, import and net build included) and the summary's own wall;
  * memory: the device memory in use (cudaMemGetInfo) with the FlowNet2-C training net alone, after one training step, and
    after the first validation pass, so the difference is what the kept deploy net and the scoring buffers add;
  * the card's name and power limit, read in the same run.

Prints one JSON line.

    python tools/val_time.py [--pairs 16] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.eval_time import card, make_list  # noqa: E402

CROP, DATA, BATCH = (448, 320), (512, 384), 8


def used():
    import torch
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    return total - free


def stage(name, listfile, d, reps, measure_memory):
    import torch
    import flownet2_b200 as F
    from flownet2_b200 import evaluate as E
    from flownet2_b200.files import read_list
    out = {}
    base = used()
    net = F.Net(F.fill_train_template(F.train_template(name), CROP[0], CROP[1], DATA[0], DATA[1], BATCH), None, F.TRAIN)
    net.fill_params(1701)
    if measure_memory:
        solver = F.Solver('type: "Adam"\nbase_lr: 1e-4\nlr_policy: "fixed"\nmax_iter: 10\n', net)
        r = np.random.default_rng(0)
        feed = {"img0": r.uniform(0, 255, net.blobs["img0"].shape).astype(np.float32),
                "img1": r.uniform(0, 255, net.blobs["img1"].shape).astype(np.float32),
                "flow_gt": r.normal(0, 5, net.blobs["flow_gt"].shape).astype(np.float32)}
        out["mem_train_net_bytes"] = used() - base
        solver.step(1, lambda: feed)
        out["mem_after_step_bytes"] = used() - base
    template = os.path.join(ROOT, "models", "%s_deploy.prototxt.template" % name)
    val = E.Validator(template, read_list(listfile))
    val.check_handover(net)
    weights = net.to_caffemodel()
    summary, _ = val.score(weights)                                     # builds the kept deploy net
    if measure_memory:
        out["mem_after_validation_bytes"] = used() - base
        out["mem_validation_adds_bytes"] = out["mem_after_validation_bytes"] - out["mem_after_step_bytes"]
    (deploy,) = val.nets.values()
    handover, to_cm, passes = [], [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        w = net.to_caffemodel()
        t1 = time.perf_counter()
        deploy.copy_from(w)
        deploy.sync()
        handover.append(time.perf_counter() - t0)
        to_cm.append(t1 - t0)
    for _ in range(reps):
        t0 = time.perf_counter()
        s, _ = val.score(weights)
        passes.append(time.perf_counter() - t0)
        assert s["epe"] == summary["epe"]
    path = os.path.join(d, "%s.caffemodel" % name)
    with open(path, "wb") as f:
        f.write(weights)
    t0 = time.perf_counter()
    p = subprocess.run([sys.executable, "-m", "flownet2_b200.evaluate", path, template, listfile], capture_output=True,
                       text=True, cwd=ROOT)
    cli = time.perf_counter() - t0
    if p.returncode != 0:
        raise SystemExit("evaluate failed: %s" % p.stderr.strip().splitlines()[-1])
    got = json.loads(p.stdout.strip().splitlines()[-1])
    assert got["epe"] == summary["epe"], (got["epe"], summary["epe"])
    out.update({"caffemodel_mb": len(weights) / 1e6, "handover_s": float(np.median(handover)),
                "to_caffemodel_s": float(np.median(to_cm)), "validation_pass_s": float(np.median(passes)),
                "validation_pairs_per_s": summary["pairs"] / float(np.median(passes)), "evaluate_process_s": cli,
                "evaluate_summary_wall_s": got["wall"], "epe": summary["epe"]})
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--pairs", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("val_time.py measures on the GPU; no CUDA device is visible")
    name, watts = card(0)
    with tempfile.TemporaryDirectory() as d:
        listfile = make_list(d, a.pairs, 7)[0]
        res = {"card": name, "power_limit_w": watts, "pairs": a.pairs, "size": "1024x436", "train_crop": "%dx%dx%d" % (
            CROP + (BATCH,)), "val_batch": 1}
        for i, stage_name in enumerate(("FlowNet2-C", "FlowNet2")):
            res[stage_name] = stage(stage_name, listfile, d, a.reps, i == 0)
            import gc
            gc.collect()
            torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
