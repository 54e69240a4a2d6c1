"""Time LpqLoss against L1Loss (l2_per_location, the end-point error) on an H100.

  * kernels: forward + backward of each loss at the largest loss bottom of any models/*_train.prototxt.template at a 448x320
    crop, batch 8, laid out like the net's blobs (channel-fast, pixel stride padded to 4 floats).  --calls back-to-back
    forward + backward pairs are captured into one CUDA graph and CUDA events bracket each of --reps replays; the median per pair
    is reported with the bytes it must move (forward: both bottoms read; backward: both read again and both diffs written) and
    that rate's share of 3.35 TB/s (H100 SXM HBM3 data sheet).  LpqLoss runs at (p, q) = (2, 0.5), the end-point error L1Loss
    computes, and at (1, 0.4), the fine-tuning loss, whose powf calls the end-point error does not make;
  * solver step: one FlowNet2-C training iteration (Adam, 448x320, batch 8, inputs in place) with the template's five L1Loss
    layers swapped for LpqLoss (p 1, q 0.4), against the unchanged template: host clock around --steps solver.step(1) calls,
    the median reported;
  * the card's name and power limit, read in the same run.

Prints one JSON line.

    python tools/lpq_time.py [--calls 50] [--reps 7] [--warmup 3] [--steps 20]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12
CROP_W, CROP_H, DATA_W, DATA_H, BATCH = 448, 320, 512, 384, 8
SOLVER = ('type: "Adam"\nbase_lr: 1e-4\nlr_policy: "multistep"\ngamma: 0.5\nstepvalue: 400000\nstepvalue: 600000\n'
          'momentum: 0.9\nmomentum2: 0.999\nweight_decay: 0.0004\nmax_iter: 1200000\n')


def card(index):
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                       capture_output=True, text=True, check=True)
    name, watts = [x.strip() for x in q.stdout.strip().split(",")]
    return name, float(watts)


def largest_train_loss():
    """(N, C, H, W) of the largest loss bottom of any models/*_train.prototxt.template at the crop and batch above."""
    import glob
    from flownet2_b200 import fill_train_template, train_template
    from tests.util import net_losses
    best = None
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "models")
    for f in sorted(glob.glob(os.path.join(root, "*_train.prototxt.template"))):
        model = os.path.basename(f)[:-len("_train.prototxt.template")]
        for _, chw in net_losses(fill_train_template(train_template(model), CROP_W, CROP_H, DATA_W, DATA_H, BATCH)):
            if best is None or np.prod(chw) > np.prod(best):
                best = chw
    return (BATCH,) + tuple(best)


def to_lpq(proto, param):
    """The prototxt with every L1Loss layer an LpqLoss layer with `param` (loss weights kept)."""
    out, n = re.subn(r'type: "L1Loss"', 'type: "LpqLoss"', proto)
    out = re.sub(r"l1_loss_param\s*\{[^}]*\}", "lpq_loss_param { %s }" % param, out)
    return out, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lpq_time.py needs a GPU")
    import flownet2_b200 as F
    from flownet2_b200 import ops
    name, watts = card(torch.cuda.current_device())
    result = {"gpu": name, "power_limit_w": watts}

    # ---- kernels ----
    shape = largest_train_loss()
    n, c, h, w = shape
    g = torch.Generator(device="cuda").manual_seed(7)

    def blob():
        p = torch.zeros((n, 4 * ((c + 3) // 4), h, w), device="cuda").contiguous(memory_format=torch.channels_last)
        v = p[:, :c]
        v.copy_(3 * torch.randn((n, c, h, w), device="cuda", generator=g))
        return v

    pred, gt, d0, d1 = blob(), blob(), blob(), blob()
    gt[0, :, 10:40, 20:90] = float("nan")
    top = torch.ones(1, device="cuda")
    ws = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
    pairs = {
        "l1loss_epe": (lambda: ops.l1loss(pred, gt, l2_per_location=True, workspace=ws),
                       lambda st: ops.l1loss_backward(pred, gt, l2_per_location=True, state=st, top_diff=top, out0=d0, out1=d1)),
    }
    for p, q in ((2.0, 0.5), (1.0, 0.4)):
        state = ops.lpqloss(pred, gt, p=p, q=q, workspace=ws)[1]
        pairs["lpqloss_p%g_q%g" % (p, q)] = (
            lambda state=state: ops.lpqloss(pred, gt, p=None, q=None, state=state, workspace=ws),
            lambda st: ops.lpqloss_backward(pred, gt, state=st, top_diff=top, out0=d0, out1=d1))
    nbytes = 6 * 4 * n * c * h * w
    kern = {}
    for key, (fwd, bwd) in pairs.items():
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                bwd(fwd()[1])
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(args.calls):
                bwd(fwd()[1])
        graph.replay()
        torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            graph.replay()
            z.record()
            z.synchronize()
            times.append(a.elapsed_time(z) * 1e3 / args.calls)
        us = float(np.median(times))
        kern[key] = {"us": round(us, 2), "bytes": nbytes, "tb_per_s": round(nbytes / us * 1e-6, 3),
                     "hbm_fraction": round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)}
    result["loss_shape"] = list(shape)
    result["kernels_fwd_bwd"] = kern

    # ---- one FlowNet2-C solver step ----
    base = F.fill_train_template(F.train_template("FlowNet2-C"), CROP_W, CROP_H, DATA_W, DATA_H, BATCH)
    lpq, swapped = to_lpq(base, "p: 1 q: 0.4")
    assert swapped == 5, swapped
    r = np.random.default_rng(7)
    inputs = {"img0": r.uniform(0, 255, (BATCH, 3, DATA_H, DATA_W)).astype(np.float32),
              "img1": r.uniform(0, 255, (BATCH, 3, DATA_H, DATA_W)).astype(np.float32),
              "flow_gt": (3 * r.standard_normal((BATCH, 2, DATA_H, DATA_W))).astype(np.float32)}
    steps = {}
    for key, proto in (("l1loss_template", base), ("lpqloss_p1_q0.4", lpq)):
        net = F.Net(proto, None, F.TRAIN)
        net.fill_params(1701)
        for k, v in inputs.items():
            net.set_input(k, v)
        solver = F.get_solver(SOLVER, net)
        solver.step(args.warmup)
        times = []
        for _ in range(args.steps):
            t = time.perf_counter()
            solver.step(1)
            times.append((time.perf_counter() - t) * 1e3)
        steps[key] = {"ms": round(float(np.median(times)), 3), "loss": round(float(solver.smoothed_loss), 4)}
        del solver, net
    result["solver_step_flownet2_c"] = steps
    print(json.dumps(result))


if __name__ == "__main__":
    main()
