"""Time the evaluate command against run, and the fn2_flow_error kernel, on an H100.

  * pipelines: a synthetic list generated from --seed in a temporary directory, --pairs pairs of 1024x436 frames (Sintel's
    size, PPM) with .flo ground truth, through FlowNet2 with fill_params weights.  flownet2_b200.evaluate.evaluate and
    flownet2_b200.run.run each take the list at --batch 1 and 8, after one warm-up call per batch; pairs/s is the pair count
    over the call's wall time without its build time (reading the weights, constructing the net), and both are reported;
  * kernel: fn2_flow_error on 8 x 2 x 436 x 1024, the prediction as the NHWC buffer the net fills and the ground truth NCHW;
    --calls back-to-back calls are captured into one CUDA graph and CUDA events bracket each of --reps replays; the median per
    call is reported with the bytes it must read (N H W 16: pred and gt, float2 each) and that rate's share of 3.35 TB/s
    (H100 SXM HBM3 data sheet);
  * the card's name and power limit, read in the same run.

Prints one JSON line.

    python tools/eval_time.py [--pairs 32] [--seed 0] [--calls 100] [--reps 7]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12
W, H = 1024, 436


def card(index):
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                       capture_output=True, text=True, check=True)
    name, watts = [x.strip() for x in q.stdout.strip().split(",")]
    return name, float(watts)


def make_list(d, pairs, seed):
    """--pairs frame pairs with .flo ground truth -> (evaluate's list, run's list)."""
    from flownet2_b200.files import write_flo, write_pnm
    r = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    ev, rn = [], []
    for i in range(pairs):
        base = (127 + 60 * np.sin(xx / (17.0 + i)) * np.cos(yy / 23.0))[:, :, None] + r.integers(-20, 21, (H, W, 3))
        f0 = np.clip(base, 0, 255).astype(np.uint8)
        f1 = np.roll(f0, (1 + i % 3, 2), axis=(0, 1))
        a, b = write_pnm(os.path.join(d, "f%d_0.ppm" % i), f0), write_pnm(os.path.join(d, "f%d_1.ppm" % i), f1)
        g = os.path.join(d, "g%d.flo" % i)
        write_flo(g, (r.standard_normal((H, W, 2)) * 10).astype(np.float32))
        ev.append("%s %s %s\n" % (a, b, g))
        rn.append("%s %s %s\n" % (a, b, os.path.join(d, "o%d.flo" % i)))
    for name, lines in (("val.txt", ev), ("run.txt", rn)):
        with open(os.path.join(d, name), "w") as f:
            f.write("".join(lines))
    return os.path.join(d, "val.txt"), os.path.join(d, "run.txt")


def pipelines(d, template, pairs, seed):
    import flownet2_b200 as F
    from flownet2_b200 import evaluate, run
    from flownet2_b200.files import read_list
    net = F.Net(F.fill_template(F.model_template("FlowNet2"), 128, 128), None, F.TEST, batch=1)
    net.fill_params(1701)
    weights = os.path.join(d, "w.caffemodel")
    with open(weights, "wb") as f:
        f.write(net.to_caffemodel())
    del net
    val, rl = make_list(d, pairs, seed)
    out = {}
    for batch in (1, 8):
        evaluate.evaluate(weights, template, read_list(val)[:batch], batch=batch)       # warm-up
        run.run(weights, template, read_list(rl, ground_truth=False)[:batch], batch=batch)
        s, _ = evaluate.evaluate(weights, template, read_list(val), batch=batch)
        r = run.run(weights, template, read_list(rl, ground_truth=False), batch=batch)
        for name, wall, build in (("evaluate", s["wall"], s["busy"]["build"]), ("run", r["wall"], r["busy"]["build"])):
            out["%s_b%d" % (name, batch)] = {"pairs_per_s": pairs / (wall - build), "wall_s": wall, "build_s": build}
    return out


def kernel(calls, reps):
    import torch
    from flownet2_b200 import ops
    N = 8
    r = torch.Generator(device="cuda").manual_seed(1)
    pred = torch.randn((N, H, W, 2), device="cuda", generator=r).permute(0, 3, 1, 2)
    gt = torch.randn((N, 2, H, W), device="cuda", generator=r) * 10
    out = torch.empty((N, 10), dtype=torch.float64, device="cuda")
    ws = torch.empty(ops.flow_error_workspace_bytes(N, H, W), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):
            ops.flow_error(pred, gt, out=out, workspace=ws)
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(calls):
                ops.flow_error(pred, gt, out=out, workspace=ws)
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) * 1e-3 / calls)
    t = float(np.median(times))
    nbytes = N * H * W * 16
    return {"shape": [N, 2, H, W], "us": t * 1e6, "bytes": nbytes, "gb_per_s": nbytes / t / 1e9,
            "hbm_share": nbytes / t / HBM_BYTES_PER_S}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--pairs", type=int, default=32)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("eval_time.py needs a GPU")
    torch.cuda.set_device(0)
    name, watts = card(0)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    template = os.path.join(root, "models", "FlowNet2_deploy.prototxt.template")
    t0 = time.perf_counter()
    with tempfile.TemporaryDirectory() as d:
        res = {"card": name, "power_limit_w": watts, "frames": [W, H], "pairs": a.pairs}
        res["kernel"] = kernel(a.calls, a.reps)
        res.update(pipelines(d, template, a.pairs, a.seed))
    res["total_s"] = time.perf_counter() - t0
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
