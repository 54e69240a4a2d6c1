"""Time fn2_occlusion_boundary_dist2 and fn2_flow_error_regions on an H100, next to fn2_flow_error.

At 8 x 436 x 1024 (a Sintel batch), with seeded blob masks and flows: each op's --calls back-to-back calls are captured into one
CUDA graph and CUDA events bracket each of --reps replays; the median per call is reported with the bytes the op moves and
that rate in GB/s:
  * distance: the mask (1 byte per pixel) and the int32 plane written by the column pass's downward sweep, read and written
    by its upward sweep, read and written by the row pass: 21 bytes per pixel;
  * regions (both masks): the two flows (16 bytes), both masks (2) and the distance (4): 22 bytes per pixel;
  * flow_error: the two flows, 16 bytes per pixel.
The card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/flow_regions_time.py [--calls 100] [--reps 7]
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.eval_time import card  # noqa: E402

N, H, W = 8, 436, 1024


def timed(fn, calls, reps):
    """Median seconds per call of fn() over reps replays of a graph of `calls` calls."""
    import torch
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(calls):
                fn()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) * 1e-3 / calls)
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("flow_regions_time.py needs a GPU")
    torch.cuda.set_device(0)
    from flownet2_b200 import ops
    from tests.test_flow_regions_gpu import blobs
    name, watts = card(0)
    occ = torch.from_numpy(blobs(N, H, W, 1)).cuda()
    obj = torch.from_numpy(blobs(N, H, W, 2, sigma=9.0)).cuda()
    r = torch.Generator(device="cuda").manual_seed(1)
    pred = torch.randn((N, H, W, 2), device="cuda", generator=r).permute(0, 3, 1, 2)
    gt = torch.randn((N, 2, H, W), device="cuda", generator=r) * 10
    dist2 = torch.empty((N, H, W), dtype=torch.int32, device="cuda")
    reg = torch.empty((N, 21), dtype=torch.float64, device="cuda")
    err = torch.empty((N, 10), dtype=torch.float64, device="cuda")
    ws = torch.empty(max(ops.flow_error_regions_workspace_bytes(N, H, W), ops.flow_error_workspace_bytes(N, H, W)),
                     dtype=torch.uint8, device="cuda")
    ops.occlusion_boundary_dist2(occ, out=dist2)
    px = N * H * W
    res = {"card": name, "power_limit_w": watts, "shape": [N, H, W]}
    for key, fn, per_px in (("distance", lambda: ops.occlusion_boundary_dist2(occ, out=dist2), 21),
                            ("regions", lambda: ops.flow_error_regions(pred, gt, occ=occ, obj=obj, dist2=dist2, out=reg,
                                                                      workspace=ws), 22),
                            ("flow_error", lambda: ops.flow_error(pred, gt, out=err, workspace=ws), 16)):
        t = timed(fn, a.calls, a.reps)
        res[key] = {"us": t * 1e6, "bytes": px * per_px, "gb_per_s": px * per_px / t / 1e9}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
