"""Time the forward-backward occlusion check on an H100: the device kernel, and run with and without --backward.

  * kernel: fn2_flow_fb_occlusion at 8 x 436 x 1024 on smooth synthetic flows (a slow rotation plus a sinusoid, displacements
    of a few pixels, the backward flow the forward one negated plus a little noise), both flows padded NHWC views (16 B a
    pixel, as the nets' output) and the mask dense; --calls back-to-back calls are captured into one CUDA graph and CUDA
    events bracket each of --reps replays (kitti_time.timed); the median per call is reported with the bytes the kernel must
    move (the forward flow's 16-B pixels, the backward flow's once, the mask's byte: 33 B a pixel) and that rate's share of
    3.35 TB/s (H100 SXM HBM3 data sheet);
  * run: FlowNet2 with fill_params weights over --pairs 1024x436 frame pairs (PPM) at --batch 8, writing .flo, without and
    with --backward, alternated over --rounds after a warm-up call of each; pairs/s is the pair count over the call's wall
    time without its build time;
  * the card's name and power limit, read in the same run.

Prints one JSON line.

    python tools/fb_time.py [--pairs 32] [--rounds 2] [--calls 100] [--reps 7]
"""
import argparse
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.eval_time import HBM_BYTES_PER_S, card  # noqa: E402
from tools.kitti_time import timed  # noqa: E402
from tools.viz_time import H, W, make_list  # noqa: E402


def kernel(calls, reps):
    import torch
    from flownet2_b200 import ops
    N = 8
    yy, xx = torch.meshgrid(torch.arange(H, device="cuda", dtype=torch.float32),
                            torch.arange(W, device="cuda", dtype=torch.float32), indexing="ij")
    fwd_pad = torch.zeros((N, H, W, 4), device="cuda")
    for n in range(N):
        a = 0.002 * (n + 1)
        fwd_pad[n, ..., 0] = -a * (yy - H / 2) + 3 * torch.sin(xx / 50.0 + n)
        fwd_pad[n, ..., 1] = a * (xx - W / 2) + 2 * torch.cos(yy / 40.0)
    g = torch.Generator(device="cuda").manual_seed(1)
    bwd_pad = -fwd_pad + 0.3 * torch.randn(fwd_pad.shape, device="cuda", generator=g)
    fwd, bwd = fwd_pad.permute(0, 3, 1, 2)[:, :2], bwd_pad.permute(0, 3, 1, 2)[:, :2]
    mask = torch.empty((N, H, W), dtype=torch.uint8, device="cuda")
    px = N * H * W
    nbytes = px * (16 + 16 + 1)
    t = timed(lambda: ops.flow_fb_occlusion(fwd, bwd, out=mask), calls, reps)
    return {"us": t * 1e6, "bytes": nbytes, "tb_per_s": nbytes / t / 1e12, "share_of_hbm": nbytes / t / HBM_BYTES_PER_S,
            "flagged_share": float((mask != 0).float().mean())}


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
    out = {"plain": [], "backward": []}
    for bwd in (False, True):
        run.run(weights, template, read_list(lst, ground_truth=False)[:batch], batch=batch, backward=bwd)       # warm-up
    for _ in range(rounds):
        for name, bwd in (("plain", False), ("backward", True)):
            s = run.run(weights, template, read_list(lst, ground_truth=False), batch=batch, backward=bwd)
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
        sys.exit("fb_time.py needs a GPU")
    torch.cuda.set_device(0)
    name, watts = card(0)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    template = os.path.join(root, "models", "FlowNet2_deploy.prototxt.template")
    t0 = time.perf_counter()
    with tempfile.TemporaryDirectory() as d:
        res = {"card": name, "power_limit_w": watts, "frames": [W, H], "pairs": a.pairs, "batch": a.batch,
               "cpus": os.cpu_count()}
        res["kernel"] = kernel(a.calls, a.reps)
        res["run"] = runs(d, template, make_list(d, a.pairs, a.seed), a.pairs, a.rounds, a.batch)
    res["total_s"] = time.perf_counter() - t0
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
