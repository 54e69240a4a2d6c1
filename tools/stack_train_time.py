"""Time one training step of the stacked FlowNet2 stages (CS on a frozen C, CSS on a frozen CS, the fusion network on a frozen
CSS and SD) on one GPU, and count the gradient bytes a data-parallel step would all-reduce.

A step is clear_param_diffs + forward + backward; CUDA events on the net's stream bracket it and the step ends in a stream
synchronise.  The card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/stack_train_time.py [--stages FlowNet2-CS FlowNet2-CSS FlowNet2] [--warmup 3] [--steps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card(index):
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                       capture_output=True, text=True, check=True)
    name, watts = [x.strip() for x in q.stdout.strip().split(",")]
    return name, float(watts)


def time_stage(F, torch, stage, crop, data, batch, warmup, steps):
    proto = F.fill_train_template(F.train_template(stage), crop[0], crop[1], data[0], data[1], batch)
    net = F.Net(proto, None, F.TRAIN)
    net.fill_params(1701)
    r = np.random.default_rng(7)
    net.set_input("img0", r.uniform(0, 255, (batch, 3, data[1], data[0])).astype(np.float32))
    net.set_input("img1", r.uniform(0, 255, (batch, 3, data[1], data[0])).astype(np.float32))
    net.set_input("flow_gt", (3 * r.standard_normal((batch, 2, data[1], data[0]))).astype(np.float32))
    stream = torch.cuda.ExternalStream(net.stream)

    def step():
        net.clear_param_diffs()
        net.forward_async()
        net.backward_async()

    for _ in range(warmup):
        step()
    net.sync()
    ms = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        step()
        b.record(stream)
        net.sync()
        ms.append(a.elapsed_time(b))
    return {"step_ms_median": float(np.median(ms)), "step_ms_min": float(np.min(ms)), "steps": steps,
            "grad_arena_bytes": int(net.param_diff_arena()[1]), "trainable_span_bytes": int(net.trainable_diff_span()[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stages", nargs="+", default=["FlowNet2-CS", "FlowNet2-CSS", "FlowNet2"])
    ap.add_argument("--crop", nargs=2, type=int, default=[448, 320])
    ap.add_argument("--data", nargs=2, type=int, default=[512, 384])
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("stack_train_time.py needs a GPU")
    import flownet2_b200 as F
    name, watts = card(torch.cuda.current_device())
    res = {"card": name, "power_limit_w": watts, "crop": args.crop, "data": args.data, "batch": args.batch, "stages": {}}
    for s in args.stages:
        res["stages"][s] = time_stage(F, torch, s, args.crop, args.data, args.batch, args.warmup, args.steps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
