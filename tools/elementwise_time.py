"""Time the element-wise and streaming entry points (fn2_relu_backward, fn2_axpby, fn2_eltwise_sum, fn2_copy, FlowWarp, Resample,
ChannelNorm, the warp block, Downsample and L1Loss) at the shapes FlowNet2 and its training step give them.

Each case is warmed up, then `--launches` back-to-back calls are captured into one CUDA graph (so that the host's call
overhead does not hide the kernel), and CUDA events bracket each replay; the median over `--reps` replays is reported per
launch, in microseconds.  Views are laid out like the net's blobs: channel-fast with the pixel stride padded
to 4 floats below 32 channels and to a multiple of 32 above.  The card's name and power limit are read in the same run.
FN2_LIB selects the library, so two builds can be compared by alternating runs.  Prints one JSON line.

    python tools/elementwise_time.py [--launches 200] [--reps 5]
"""
import argparse
import ctypes as C
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
    # the warp block between stacked networks and the layers it fuses: flow up-sampled x4 from 109x256, 3-channel images
    img0, img1, flow = blob(n, 3, h, w), blob(n, 3, h, w), blob(n, 2, h, w)
    flow.mul_(8.0)
    small = blob(n, 2, 109, 256)
    small.mul_(8.0)
    warped, err, norm, full, scaled = blob(n, 3, h, w), blob(n, 3, h, w), blob(n, 1, h, w), blob(n, 2, h, w), blob(n, 2, h, w)
    cases["flow_warp_c3_%dx%d" % (w, h)] = lambda: ops.flow_warp(img1, flow, out=warped)
    cases["resample_flow_256x109_to_%dx%d" % (w, h)] = lambda: ops.resample(small, h, w, 2)
    cases["resample_image_%dx%d_to_%dx448" % (w, h, w)] = lambda: ops.resample(img0, 448, w, 2)
    cases["channel_norm_c3_%dx%d" % (w, h)] = lambda: ops.channel_norm(err, out=norm)
    cases["warp_block_%dx%d" % (w, h)] = lambda: ops.warp_block(small, img0, img1, 0.05, out=(full, warped, err, norm, scaled))
    # mean subtraction of the 3-channel input images (per pixel and per channel)
    top, mpp, mpc = nchw(n, 3, h, w), nchw(1, 3, h, w), torch.rand(3, device="cuda", generator=g)
    cases["mean_subtract_pp_c3_%dx%d" % (w, h)] = lambda: ops.mean_subtract(top, mpp, mpc, True)
    cases["mean_subtract_pc_c3_%dx%d" % (w, h)] = lambda: ops.mean_subtract(top, None, mpc, False)
    # FlowNet2-C training step at a 448x320 crop, batch 8: the ground truth's Downsample to each pyramid level, and the
    # end-point-error L1Loss forward + backward there
    gt = blob(8, 2, 320, 448)
    lib = F.lib()
    epe = F.fn2_l1loss_desc(1, 0, 0, 0.0, 0.0)

    def l1loss(pred, gtl, diff, ws, nbytes, state, one):
        dp, dg, dd = ops.desc(pred), ops.desc(gtl), ops.desc(diff)
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        F.check(lib.fn2_l1loss_forward(C.byref(dp), C.byref(dg), C.byref(epe), C.c_void_p(state.data_ptr()), None,
                                       C.c_void_p(ws.data_ptr()), C.c_size_t(nbytes), st))
        F.check(lib.fn2_l1loss_backward(C.byref(dp), C.byref(dg), C.byref(epe), C.c_void_p(state.data_ptr()), C.c_void_p(one.data_ptr()),
                                        C.byref(dd), None, 0, 0, st))

    for s in (4, 8, 16, 32, 64):
        th, tw = 320 // s, 448 // s
        lvl = blob(8, 2, th, tw)
        cases["downsample_448x320_to_%dx%d" % (tw, th)] = lambda lvl=lvl, th=th, tw=tw: ops.downsample(gt, th, tw, out=lvl)
        pred, diff = blob(8, 2, th, tw), blob(8, 2, th, tw)
        nb = C.c_size_t()
        F.check(lib.fn2_l1loss_workspace_bytes(8, th, tw, C.byref(nb)))
        ws, state, one = torch.zeros(nb.value, dtype=torch.uint8, device="cuda"), torch.zeros(4, device="cuda"), torch.ones(1, device="cuda")
        cases["l1loss_epe_fwd_bwd_%dx%d" % (tw, th)] = (lambda pred=pred, lvl=lvl, diff=diff, ws=ws, nb=nb.value, state=state, one=one:
                                                       l1loss(pred, lvl, diff, ws, nb, state, one))

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
