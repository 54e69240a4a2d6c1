"""Time the flow colour coding on an H100: the two device kernels, and run with and without --visualize.

  * kernels: fn2_flow_max_radius and fn2_flow_to_color_png_rows (and the dense fn2_flow_to_color) at 8 x 2 x 436 x 1024, the
    flow a padded NHWC view (16 B a pixel, as the nets' output); --calls back-to-back calls are captured into one CUDA graph
    and CUDA events bracket each of --reps replays (kitti_time.timed); the median per call is reported with the bytes the
    kernel must move (max radius: 8 B read per pixel, the sectors of a 16-B pixel stride count 16; colour: the same read plus
    3 B written, and a filter byte per row) and that rate's share of 3.35 TB/s (H100 SXM HBM3 data sheet);
  * run: FlowNet2 with fill_params weights over --pairs 1024x436 frame pairs (PPM) at --batch 8, writing .flo, without and
    with --visualize, alternated over --rounds after a warm-up call of each; pairs/s is the pair count over the call's wall
    time without its build time, and write_s the writer thread's busy time (.flo writes, and with --visualize the deflate);
  * the card's name and power limit, read in the same run.

Prints one JSON line.

    python tools/viz_time.py [--pairs 32] [--rounds 2] [--calls 100] [--reps 7]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.eval_time import HBM_BYTES_PER_S, card  # noqa: E402
from tools.kitti_time import timed  # noqa: E402

W, H = 1024, 436


def kernels(calls, reps):
    import torch
    from flownet2_b200 import ops
    N = 8
    g = torch.Generator(device="cuda").manual_seed(1)
    pad = torch.randn((N, H, W, 4), device="cuda", generator=g) * 20
    flow = pad.permute(0, 3, 1, 2)[:, :2]
    radius = torch.empty(N, device="cuda")
    rows = torch.empty(N * H * (1 + 3 * W), dtype=torch.uint8, device="cuda")
    dense = torch.empty(N * H * W * 3, dtype=torch.uint8, device="cuda")
    px = N * H * W
    out = {}
    for name, fn, nbytes in (
            ("flow_max_radius", lambda: ops.flow_max_radius(flow, radius), px * 16),
            ("flow_to_color_png_rows", lambda: ops.flow_to_color_png_rows(flow, rows, max_radius=radius),
             px * 16 + rows.numel()),
            ("flow_to_color", lambda: ops.flow_to_color(flow, out=dense, max_radius=radius), px * 16 + dense.numel()),
            ("max_radius_and_png_rows", lambda: ops.flow_to_color_png_rows(flow, rows, max_radius=ops.flow_max_radius(flow, radius)),
             px * 32 + rows.numel())):
        t = timed(fn, calls, reps)
        out[name] = {"us": t * 1e6, "bytes": nbytes, "tb_per_s": nbytes / t / 1e12,
                     "share_of_hbm": nbytes / t / HBM_BYTES_PER_S}
    return out


def make_list(d, pairs, seed):
    from flownet2_b200.files import write_pnm
    r = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    lines = []
    for i in range(pairs):
        base = (127 + 60 * np.sin(xx / (17.0 + i)) * np.cos(yy / 23.0))[:, :, None] + r.integers(-20, 21, (H, W, 3))
        f0 = np.clip(base, 0, 255).astype(np.uint8)
        f1 = np.roll(f0, (1 + i % 3, 2), axis=(0, 1))
        a, b = write_pnm(os.path.join(d, "f%d_0.ppm" % i), f0), write_pnm(os.path.join(d, "f%d_1.ppm" % i), f1)
        lines.append("%s %s %s\n" % (a, b, os.path.join(d, "o%d.flo" % i)))
    path = os.path.join(d, "run.txt")
    with open(path, "w") as f:
        f.write("".join(lines))
    return path


def runs(d, template, lst, pairs, rounds, batch):
    import flownet2_b200 as F
    from flownet2_b200 import run
    from flownet2_b200.files import read_list
    net = F.Net(F.fill_template(F.model_template("FlowNet2"), 128, 128), None, F.TEST, batch=1)
    net.fill_params(1701)
    weights = os.path.join(d, "w.caffemodel")
    with open(weights, "wb") as f:
        f.write(net.to_caffemodel())
    del net
    out = {"plain": [], "visualize": []}
    for vis in (False, True):
        run.run(weights, template, read_list(lst, ground_truth=False)[:batch], batch=batch, visualize=vis)         # warm-up
    for _ in range(rounds):
        for name, vis in (("plain", False), ("visualize", True)):
            s = run.run(weights, template, read_list(lst, ground_truth=False), batch=batch, visualize=vis)
            out[name].append({"pairs_per_s": pairs / (s["wall"] - s["busy"]["build"]), "wall_s": s["wall"],
                              "write_s": s["busy"]["write"], "forward_s": s["busy"]["forward"], "d2h_s": s["busy"]["d2h"]})
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--pairs", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("viz_time.py needs a GPU")
    torch.cuda.set_device(0)
    name, watts = card(0)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    template = os.path.join(root, "models", "FlowNet2_deploy.prototxt.template")
    t0 = time.perf_counter()
    with tempfile.TemporaryDirectory() as d:
        res = {"card": name, "power_limit_w": watts, "frames": [W, H], "pairs": a.pairs, "batch": a.batch,
               "cpus": os.cpu_count()}
        res["kernels"] = kernels(a.calls, a.reps)
        res["run"] = runs(d, template, make_list(d, a.pairs, a.seed), a.pairs, a.rounds, a.batch)
    res["total_s"] = time.perf_counter() - t0
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
