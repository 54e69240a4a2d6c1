"""Time the element-wise entry points (fn2_relu_backward, fn2_axpby, fn2_eltwise_sum, fn2_copy) at the shapes FlowNet2 gives them.

Each case is warmed up, then `--launches` back-to-back calls are captured into one CUDA graph (so that the host's call
overhead does not hide the kernel), and CUDA events bracket each replay; the median over `--reps` replays is reported per
launch, in microseconds.  Views are laid out like the net's blobs: channel-fast with the pixel stride padded
to 4 floats below 32 channels and to a multiple of 32 above.  The card's name and power limit are read in the same run.
FN2_LIB selects the library, so two builds can be compared by alternating runs.  Prints one JSON line.

    python tools/elementwise_time.py [--launches 200] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card(index):
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                       capture_output=True, text=True, check=True)
    name, watts = [x.strip() for x in q.stdout.strip().split(",")]
    return name, float(watts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    import flownet2_b200 as F
    from flownet2_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(7)

    def blob(n, c, h, w):
        """A channel-fast view with the net's padded pixel stride."""
        cs = 4 * ((c + 3) // 4) if c < 32 else 32 * ((c + 31) // 32)
        p = torch.zeros((n, cs, h, w), device="cuda").contiguous(memory_format=torch.channels_last)
        v = p[:, :c]
        v.copy_(torch.randn((n, c, h, w), device="cuda", generator=g))
        return v

    def nchw(n, c, h, w):
        return torch.randn((n, c, h, w), device="cuda", generator=g)

    cases = {}
    # ReLU backward of FlowNet2-C's conv / deconv tops at a 448x320 crop, batch 8, in place as the fused conv+ReLU runs it
    for c, h, w in ((64, 160, 224), (128, 80, 112), (256, 40, 56), (512, 20, 28), (1024, 5, 7)):
        y, dy = blob(8, c, h, w), blob(8, c, h, w)
        cases["relu_bwd_c%d_%dx%d" % (c, w, h)] = lambda y=y, dy=dy: ops.relu_backward(y, dy, 0.1, out=dy)
    # gradient accumulation into the concat blobs of FlowNet2-C (conv3_1's 473-channel input, the 1026-channel concat5)
    for c, h, w in ((473, 40, 56), (1026, 10, 14)):
        x, y = blob(8, c, h, w), blob(8, c, h, w)
        cases["axpby_c%d_%dx%d" % (c, w, h)] = lambda x=x, y=y: ops.axpby(x, 1.0, y, 1.0)
    # FlowNet2 deploy at 1024x436, 4 pairs: the warp block's error (3 channels) and flow rescaling (2), the input and output
    # layout conversions
    n, h, w = 4, 436, 1024
    for c in (2, 3):
        a, b, o = blob(n, c, h, w), blob(n, c, h, w), blob(n, c, h, w)
        cases["eltwise_c%d_%dx%d" % (c, w, h)] = lambda a=a, b=b, o=o: ops.eltwise_sum([a, b], [1.0, -1.0], out=o)
    src3, dst3 = nchw(n, 3, h, w), blob(n, 3, h, w)
    cases["copy_nchw_to_nhwc_c3_%dx%d" % (w, h)] = lambda: ops.copy(src3, dst3)
    src2, dst2 = blob(n, 2, h, w), nchw(n, 2, h, w)
    cases["copy_nhwc_to_nchw_c2_%dx%d" % (w, h)] = lambda: ops.copy(src2, dst2)

    name, watts = card(torch.cuda.current_device())
    res = {"card": name, "power_limit_w": watts, "lib": F.lib_path(), "launches": args.launches, "us": {}}
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for key, fn in cases.items():
        for _ in range(20):
            fn()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(args.launches):
                fn()
        graph.replay()
        times = []
        for _ in range(args.reps):
            start.record()
            graph.replay()
            stop.record()
            stop.synchronize()
            times.append(start.elapsed_time(stop) * 1e3 / args.launches)
        times.sort()
        res["us"][key] = round(times[len(times) // 2], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
