"""Time KITTI flow PNGs on an H100: the host decode, the two device kernels, and run / evaluate with KITTI files against .flo.

  * host: --pairs synthetic KITTI ground-truth PNGs of 1242x375 (a smooth flow with half its pixels invalid, written by
    kitti.write_kitti_flow); the median time of kitti.read_payload per file on one thread, and the pool's throughput (files/s)
    reading every file once with 1, 4, 8 and 16 threads;
  * kernels: fn2_flow_to_tensor (FLOW_KITTI) and fn2_flow_to_kitti_png_rows at 8 x 2 x 375 x 1242; --calls back-to-back calls are
    captured into one CUDA graph and CUDA events bracket each of --reps replays; the median per call is reported with the bytes
    the kernel must move (decode: 6 B read + 8 B written per pixel; encode: 8 B read + 6 B written per pixel, plus the filter
    bytes) and that rate's share of 3.35 TB/s (H100 SXM HBM3 data sheet);
  * pipelines: FlowNet2 with fill_params weights over the --pairs frame pairs (PPM): run at --batch 1 and 4 writing .flo
    against --kitti PNGs, and evaluate at --batch 1 with .flo ground truth against the same ground truth as KITTI PNGs; each
    after a warm-up call; pairs/s is the pair count over the call's wall time without its build time;
  * the card's name and power limit, read in the same run.

Prints one JSON line.

    python tools/kitti_time.py [--pairs 16] [--seed 0] [--calls 100] [--reps 7]
"""
import argparse
import json
import os
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.eval_time import HBM_BYTES_PER_S, card  # noqa: E402

W, H = 1242, 375


def make_lists(d, pairs, seed):
    """Frames and ground truth -> paths of {kitti, flo: evaluate's lists; run_flo, run_png: run's lists} and the PNGs."""
    from flownet2_b200 import kitti
    from flownet2_b200.files import write_flo, write_pnm
    r = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    lines = {k: [] for k in ("kitti", "flo", "run_flo", "run_png")}
    pngs = []
    for i in range(pairs):
        base = (127 + 60 * np.sin(xx / (17.0 + i)) * np.cos(yy / 23.0))[:, :, None] + r.integers(-20, 21, (H, W, 3))
        f0 = np.clip(base, 0, 255).astype(np.uint8)
        f1 = np.roll(f0, (1 + i % 3, 2), axis=(0, 1))
        a, b = write_pnm(os.path.join(d, "f%d_0.ppm" % i), f0), write_pnm(os.path.join(d, "f%d_1.ppm" % i), f1)
        gt = np.stack([20 * np.sin(xx / (50.0 + i)) + xx / 40, 5 * np.cos(yy / 30.0)], axis=2).astype(np.float32)
        gt[r.random((H, W)) < 0.5] = np.nan
        png = kitti.write_kitti_flow(os.path.join(d, "g%d.png" % i), gt)
        flo = os.path.join(d, "g%d.flo" % i)
        write_flo(flo, kitti.read_kitti_flow(png))
        pngs.append(png)
        for k, g in (("kitti", png), ("flo", flo), ("run_flo", os.path.join(d, "o%d.flo" % i)),
                     ("run_png", os.path.join(d, "o%d.png" % i))):
            lines[k].append("%s %s %s\n" % (a, b, g))
    out = {}
    for k, v in lines.items():
        out[k] = os.path.join(d, k + ".txt")
        with open(out[k], "w") as f:
            f.write("".join(v))
    return out, pngs


def host(pngs):
    from flownet2_b200 import kitti
    infos = [kitti.probe(p) for p in pngs]
    bufs = [np.empty(i.nbytes, np.uint8) for i in infos]
    one = []
    for _ in range(2):
        for p, i, b in zip(pngs, infos, bufs):
            t0 = time.perf_counter()
            kitti.read_payload(p, i, b)
            one.append(time.perf_counter() - t0)
    out = {"file_bytes_mean": float(np.mean([os.path.getsize(p) for p in pngs])),
           "decode_ms_per_file": float(np.median(one)) * 1e3}
    for n in (1, 4, 8, 16):
        with ThreadPoolExecutor(max_workers=n) as pool:
            list(pool.map(kitti.read_payload, pngs, infos, bufs))                       # warm the threads
            t0 = time.perf_counter()
            for _ in range(2):
                list(pool.map(kitti.read_payload, pngs, infos, bufs))
            out["pool_files_per_s_%d" % n] = 2 * len(pngs) / (time.perf_counter() - t0)
    return out


def timed(fn, calls, reps):
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


def kernels(calls, reps):
    import torch
    from flownet2_b200 import FLOW_KITTI, ops
    N = 8
    r = torch.Generator(device="cuda").manual_seed(1)
    payload = torch.randint(0, 256, (N * H * W * 6,), dtype=torch.uint8, device="cuda", generator=r)
    flow = torch.randn((N, 2, H, W), device="cuda", generator=r) * 30
    rows = torch.empty((N, H, 1 + 6 * W), dtype=torch.uint8, device="cuda")
    out = {}
    for name, fn, nbytes in (
            ("flow_to_tensor_kitti", lambda: ops.flow_to_tensor(payload, FLOW_KITTI, 0, flow), N * H * W * 14),
            ("flow_to_kitti_png_rows", lambda: ops.flow_to_kitti_png_rows(flow, rows), N * H * W * 8 + rows.numel())):
        t = timed(fn, calls, reps)
        out[name] = {"shape": [N, 2, H, W], "us": t * 1e6, "bytes": nbytes, "gb_per_s": nbytes / t / 1e9,
                     "hbm_share": nbytes / t / HBM_BYTES_PER_S}
    return out


def pipelines(d, template, lists, pairs):
    import flownet2_b200 as F
    from flownet2_b200 import evaluate, run
    from flownet2_b200.files import read_list
    net = F.Net(F.fill_template(F.model_template("FlowNet2"), 128, 128), None, F.TEST, batch=1)
    net.fill_params(1701)
    weights = os.path.join(d, "w.caffemodel")
    with open(weights, "wb") as f:
        f.write(net.to_caffemodel())
    del net
    rate = lambda s: {"pairs_per_s": pairs / (s["wall"] - s["busy"]["build"]), "wall_s": s["wall"],
                      "write_s": s["busy"].get("write"), "forward_s": s["busy"]["forward"]}
    out = {}
    for batch in (1, 4):
        for name, lst, kitti in (("run_flo", lists["run_flo"], False), ("run_kitti", lists["run_png"], True)):
            run.run(weights, template, read_list(lst, ground_truth=False)[:batch], batch=batch, kitti=kitti)           # warm-up
            out["%s_b%d" % (name, batch)] = rate(run.run(weights, template, read_list(lst, ground_truth=False), batch=batch,
                                                                kitti=kitti))
    for name, lst, kitti in (("evaluate_flo", lists["flo"], False), ("evaluate_kitti", lists["kitti"], True)):
        evaluate.evaluate(weights, template, read_list(lst)[:1], kitti=kitti)
        s, _ = evaluate.evaluate(weights, template, read_list(lst), kitti=kitti)
        out[name + "_b1"] = {"pairs_per_s": pairs / (s["wall"] - s["busy"]["build"]), "wall_s": s["wall"],
                             "epe": s["epe"], "decode_s": s["busy"]["decode"]}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--pairs", type=int, default=16)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("kitti_time.py needs a GPU")
    torch.cuda.set_device(0)
    name, watts = card(0)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    template = os.path.join(root, "models", "FlowNet2_deploy.prototxt.template")
    t0 = time.perf_counter()
    with tempfile.TemporaryDirectory() as d:
        res = {"card": name, "power_limit_w": watts, "frames": [W, H], "pairs": a.pairs, "cpus": os.cpu_count()}
        res["kernels"] = kernels(a.calls, a.reps)
        lists, pngs = make_lists(d, a.pairs, a.seed)
        res["host"] = host(pngs)
        res.update(pipelines(d, template, lists, a.pairs))
    res["total_s"] = time.perf_counter() - t0
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
