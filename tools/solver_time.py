"""Time the solver on FlowNet2-C 448x320, batch 8 (BASELINE config 5) with the FlowNet2 schedule's Adam (weight decay, multistep).

  * update kernel: device time of the fused Adam update pass per call (torch.profiler, CUDA activities, over --updates calls of
    fn2_solver_apply_update), the bytes it must move (4 floats read and 4 written per trainable parameter: data, diff, m, v),
    the achieved bandwidth and its share of 3.35 TB/s (H100 SXM HBM3 data sheet);
  * apply_update: CUDA events on the net's stream around whole fn2_solver_apply_update calls (update pass plus the re-packing
    of the updated convolution weights);
  * solver.step next to clear_param_diffs + forward + backward alone, host clock around calls that end in a stream synchronise.
  * the reference arm, when build/solver_ref/libref_solver.so exists (tests/golden/make_solver_ref_golden.py compile): the
    reference's own AdamUpdate kernel (adam_solver.cu:6-16) launched once per trainable blob, as AdamSolver::ComputeUpdateValue
    does, CUDA events over --updates rounds.  The reference also runs a cuBLAS axpy per blob for Regularize and one for
    Net::Update, which this arm leaves out;
  * the card's name and power limit, read in the same run.

End-to-end times are taken with the profiler off; the profiled window comes last.  Prints one JSON line.

    python tools/solver_time.py [--warmup 3] [--steps 10] [--updates 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12
SOLVER = ('type: "Adam"\nbase_lr: 1e-4\nlr_policy: "multistep"\ngamma: 0.5\nstepvalue: 400000\nstepvalue: 600000\n'
          'momentum: 0.9\nmomentum2: 0.999\nweight_decay: 0.0004\nmax_iter: 1200000\n')


def card(index):
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                       capture_output=True, text=True, check=True)
    name, watts = [x.strip() for x in q.stdout.strip().split(",")]
    return name, float(watts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--crop", nargs=2, type=int, default=[448, 320])
    ap.add_argument("--data", nargs=2, type=int, default=[512, 384])
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--updates", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("solver_time.py needs a GPU")
    import flownet2_b200 as F
    name, watts = card(torch.cuda.current_device())
    (cw, ch), (dw, dh), b = args.crop, args.data, args.batch
    proto = F.fill_train_template(F.train_template("FlowNet2-C"), cw, ch, dw, dh, b)
    net = F.Net(proto, None, F.TRAIN)
    net.fill_params(1701)
    r = np.random.default_rng(7)
    inputs = {"img0": r.uniform(0, 255, (b, 3, dh, dw)).astype(np.float32),
              "img1": r.uniform(0, 255, (b, 3, dh, dw)).astype(np.float32),
              "flow_gt": (3 * r.standard_normal((b, 2, dh, dw))).astype(np.float32)}
    for k, v in inputs.items():
        net.set_input(k, v)
    solver = F.get_solver(SOLVER, net)
    stream = torch.cuda.ExternalStream(net.stream)

    # trainable parameters (lr_mult != 0; DataAugmentation's blobs are state): what the update pass reads and writes
    from oracle.net import get, getall, parse_prototxt
    trainable, blobs = 0, []
    shape = (F.C.c_int * 4)()
    layers = dict(zip(net.layer_names, net.layer_types))
    parsed = {get(l, "name").strip('"'): l for l in getall(parse_prototxt(proto), "layer")}
    for lname in net.layer_names:
        i = 0
        specs = getall(parsed.get(lname, []), "param")
        while F.lib().fn2_net_param_shape(net._h, lname.encode(), i, shape) == 0:
            lr = float(get(specs[i], "lr_mult", 1)) if i < len(specs) else 1.0
            if layers[lname] != "DataAugmentation" and lr != 0:
                trainable += int(np.prod(list(shape)))
                blobs.append(int(np.prod(list(shape))))
            i += 1
    update_bytes = 8 * 4 * trainable

    # forward + backward alone, then whole solver steps (profiler off)
    def fwd_bwd():
        net.clear_param_diffs()
        net.forward_async()
        net.backward_async()
        net.sync()

    for _ in range(args.warmup):
        fwd_bwd()
    t = time.perf_counter()
    for _ in range(args.steps):
        fwd_bwd()
    fb_ms = (time.perf_counter() - t) * 1e3 / args.steps
    solver.step(args.warmup)                       # the inputs stay in place: no feed
    t = time.perf_counter()
    solver.step(args.steps)
    step_ms = (time.perf_counter() - t) * 1e3 / args.steps

    # whole apply_update calls, CUDA events on the net's stream
    a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(args.updates):
        F.check(F.lib().fn2_solver_apply_update(solver._h))
    z.record(stream)
    net.sync()
    apply_ms = a.elapsed_time(z) / args.updates

    # the update kernel alone (profiled window)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.updates):
            F.check(F.lib().fn2_solver_apply_update(solver._h))
        net.sync()
    kern_us = [e.device_time_total for e in prof.key_averages() if "solver_update_kernel" in e.key]
    calls = [e.count for e in prof.key_averages() if "solver_update_kernel" in e.key]
    kernel_ms = (sum(kern_us) / max(sum(calls), 1)) / 1e3 if calls else float("nan")
    reference = "not run: build/solver_ref/libref_solver.so is not built (tests/golden/make_solver_ref_golden.py compile)"
    from tests.golden import make_solver_ref_golden as G
    if os.path.exists(G.LIB):
        lib = G.load()
        g, m, v = (torch.zeros(trainable, device="cuda") for _ in range(3))
        offs = np.concatenate([[0], np.cumsum(blobs)[:-1]]) * 4

        def ref_round():
            for n, o in zip(blobs, offs):
                lib.ref_adam_update(n, g.data_ptr() + int(o), m.data_ptr() + int(o), v.data_ptr() + int(o), 0.9, 0.999, 1e-8, 1e-4)

        ref_round()
        torch.cuda.synchronize()
        a.record()
        for _ in range(args.updates):
            ref_round()
        z.record()
        torch.cuda.synchronize()
        reference = {"adam_update_per_blob_ms": a.elapsed_time(z) / args.updates, "blobs": len(blobs),
                     "excludes": "the per-blob cuBLAS axpys of Regularize and Net::Update"}
    res = {"card": name, "power_limit_w": watts, "crop": args.crop, "data": args.data, "batch": b,
           "trainable_params": trainable, "update_kernel_ms": kernel_ms, "update_bytes": update_bytes,
           "update_tb_per_s": update_bytes / (kernel_ms * 1e-3) / 1e12,
           "update_share_of_3_35_tb_per_s": update_bytes / (kernel_ms * 1e-3) / HBM_BYTES_PER_S,
           "apply_update_ms": apply_ms, "solver_step_ms": step_ms, "forward_backward_ms": fb_ms,
           "reference_arm": reference}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
