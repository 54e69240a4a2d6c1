"""Training throughput fed from files against fed from device-resident tensors (flownet2_b200.data).

    python tools/train_data_time.py [--samples 48] [--steps 40] [--warmup 5]

Writes a seeded FlyingChairs-shaped dataset (512x384 frames) to a temporary directory twice: PPM + .flo, and PNG + big-endian
PFM.  Times FlowNet2-C training (448x320 crop, batch 8, Adam) fed (a) from device-resident tensors, the ceiling, and (b) from
the files through FlowDataset, in alternating rounds on one net.  Reports iterations/s, the dataset's per-stage busy times
per iteration, the mean time the net's stream waited for a slot, each iteration split into [ms, ms inside the feed call,
ms in the rest of Solver.step], and the card's name and power limit.  Needs a GPU.
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def write_dataset(d, n, kind, seed):
    """n samples of 512x384 frames and flows: kind 'ppm' (PPM + .flo) or 'png' (PNG + big-endian PFM) -> list path."""
    from PIL import Image
    from flownet2_b200.files import write_flo, write_pfm, write_pnm
    r = np.random.default_rng(seed)
    W, H = 512, 384
    base = r.integers(0, 256, (H + 8, W + 8, 3), dtype=np.uint8)
    lines = []
    for i in range(n):
        dy, dx = r.integers(0, 8, 2)
        f0 = base[dy:dy + H, dx:dx + W]
        f1 = np.roll(f0, (1, 2), axis=(0, 1))
        paths = []
        for j, f in enumerate((f0, f1)):
            p = os.path.join(d, "%s%04d_%d.%s" % (kind, i, j, kind))
            if kind == "ppm":
                write_pnm(p, f)
            else:
                Image.fromarray(f).save(p, compress_level=1)
            paths.append(p)
        v = r.normal(0, 10, (H, W, 3)).astype(np.float32)
        fl = os.path.join(d, "%s%04d.%s" % (kind, i, "flo" if kind == "ppm" else "pfm"))
        write_flo(fl, v[:, :, :2]) if kind == "ppm" else write_pfm(fl, v, big_endian=True)
        lines.append(" ".join(paths + [fl]))
    lst = os.path.join(d, "%s.txt" % kind)
    with open(lst, "w") as f:
        f.write("\n".join(lines) + "\n")
    return lst


def timed(torch, solver, steps, feed):
    """-> (iterations/s, ms per iteration, ms per iteration spent inside the feed call).  The rest of an iteration is the
    Solver's own: its enqueues, the device's step and the loss read that ends every iteration."""
    in_feed = [0.0]

    def feed_timed():
        t = time.perf_counter()
        out = feed()
        in_feed[0] += time.perf_counter() - t
        return out

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    solver.step(steps, feed_timed)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return steps / wall, wall / steps * 1e3, in_feed[0] / steps * 1e3


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--samples", type=int, default=48)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("train_data_time: no CUDA device; this tool measures the GPU and has no fallback")
    import flownet2_b200 as F
    from flownet2_b200 import data as D
    B, (CW, CH) = 8, (448, 320)
    solver_text = 'type: "Adam"\nbase_lr: 1e-4\nmomentum: 0.9\nmomentum2: 0.999\nlr_policy: "fixed"\nmax_iter: 1000000\n'
    res = {"card": card(), "crop": "%dx%d" % (CW, CH), "batch": B, "samples": a.samples, "cpus": os.cpu_count(),
           "reader_threads": min(16, os.cpu_count() or 4)}
    with tempfile.TemporaryDirectory() as d:
        for kind in ("ppm", "png"):
            t0 = time.perf_counter()
            lst = write_dataset(d, a.samples, kind, 1701)
            ds = D.FlowDataset(lst, B)
            W, H = ds.size
            net = F.Net(F.fill_train_template(F.train_template("FlowNet2-C"), CW, CH, W, H, B), None, F.TRAIN)
            net.fill_params(1701)
            solver = F.Solver(solver_text, net)
            # (a) the ceiling: batches already on the device
            dev = [dict(zip(("img0", "img1", "flow_gt"), (torch.from_numpy(x).cuda() for x in ds.host_batch(k))))
                   for k in range(4)]
            it = iter(range(10 ** 9))
            feed_a = lambda: dev[next(it) % len(dev)]
            ds.bind(net)
            timed(torch, solver, a.warmup, feed_a)
            timed(torch, solver, a.warmup, ds)
            ra, rb = [], []
            b0 = ds.busy()
            for _ in range(a.rounds):
                ra.append(timed(torch, solver, a.steps, feed_a))
                rb.append(timed(torch, solver, a.steps, ds))
            rates_a, rates_b = [x[0] for x in ra], [x[0] for x in rb]
            b1 = ds.busy()
            n = b1["calls"] - b0["calls"]
            per = {k: (b1[k] - b0[k]) / n * 1e3 for k in ("read", "host_wait", "h2d", "convert", "stream_wait")}
            ds.close()
            res[kind] = {"device_fed_it_s": [round(x, 2) for x in rates_a], "file_fed_it_s": [round(x, 2) for x in rates_b],
                         "file_vs_device": round(float(np.mean(rates_b) / np.mean(rates_a)), 4),
                         "per_iter_ms": {k: round(v, 3) for k, v in per.items()},
                         # an iteration split into the feed call and the Solver's rest, for each feed
                         "device_fed_ms": [[round(x[1], 2), round(x[2], 2), round(x[1] - x[2], 2)] for x in ra],
                         "file_fed_ms": [[round(x[1], 2), round(x[2], 2), round(x[1] - x[2], 2)] for x in rb],
                         "setup_s": round(time.perf_counter() - t0, 1)}
            print(json.dumps({kind: res[kind]}), flush=True)
            del solver, net, dev
            torch.cuda.empty_cache()
    res["card_after"] = card()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
