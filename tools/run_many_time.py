#!/usr/bin/env python
"""Files in to .flo out: the image-file driver (flownet2_b200.run) against the per-pair public path.

    python tools/run_many_time.py [--pairs 64] [--width 1024] [--height 436] [--model FlowNet2] [--out DIR]

Writes `--pairs` seeded synthetic frame pairs (half PPM, half PNG when Pillow imports) and a caffemodel from
Net.fill_params under DIR (a temporary directory by default, removed at the end), then times, with the host clock around
work that ends in a synchronise:
  (a) the per-pair public path: one Net, read_image + image_to_blob + net.forward + write_flo per pair;
  (b) the driver at --batch 1;
  (c) the driver at --batch 4.
Net construction (with checking the inputs and reading the weights) is timed apart from the pairs.  Prints one JSON line: pairs/s of each, the driver's per-stage busy
seconds (decode: host, summed over the pool's threads; h2d, forward, d2h: device events; write: host), the GPU's name
and power limit read in the same run, and whether (a) and (b) wrote bit-identical files.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:
        return {"gpu": None, "power_limit": None, "error": str(e)}


def write_pairs(d, n, w, h, seed=1701):
    from flownet2_b200 import files as FI
    try:
        from PIL import Image
    except ImportError:
        Image = None
    r = np.random.default_rng(seed)
    lines = []
    for i in range(n):
        a = r.integers(0, 256, (h, w, 3), dtype=np.uint8)
        b = np.clip(np.roll(a, (1, 2), axis=(0, 1)).astype(np.int16) + r.integers(-3, 4, a.shape), 0, 255).astype(np.uint8)
        paths = []
        for j, f in enumerate((a, b)):
            if i % 2 and Image is not None:
                p = os.path.join(d, "f%03d_%d.png" % (i, j))
                Image.fromarray(f).save(p)
            else:
                p = os.path.join(d, "f%03d_%d.ppm" % (i, j))
                with open(p, "wb") as fh:
                    fh.write(b"P6\n%d %d\n255\n" % (w, h) + f.tobytes())
            paths.append(p)
        lines.append(paths)
    assert all(FI.probe_image(p)[:2] == (w, h) for l in lines for p in l)
    return lines


def write_list(path, lines, outdir):
    os.makedirs(outdir, exist_ok=True)
    outs = [os.path.join(outdir, "out%03d.flo" % i) for i in range(len(lines))]
    with open(path, "w") as f:
        for (a, b), o in zip(lines, outs):
            f.write("%s %s %s\n" % (a, b, o))
    return outs


def public_path(F, FI, model, template, lines, outs, w, h):
    """(a): what a user of the Python API writes today, one pair per forward."""
    import torch
    t0 = time.perf_counter()
    net = F.Net(F.fill_template(open(template).read(), w, h), model, F.TEST, batch=1)
    build = time.perf_counter() - t0
    t1 = time.perf_counter()
    for (a, b), o in zip(lines, outs):
        flow = net.forward(img0=F.image_to_blob(FI.read_image(a)), img1=F.image_to_blob(FI.read_image(b)))["predict_flow_final"]
        F.write_flo(o, flow[0])
    torch.cuda.synchronize()
    wall = time.perf_counter() - t1
    del net
    return {"pairs_per_s": len(lines) / wall, "wall_s": wall, "build_s": build}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--height", type=int, default=436)
    ap.add_argument("--model", default="FlowNet2")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import gc
    import torch
    import flownet2_b200 as F
    from flownet2_b200 import files as FI, run as R
    assert torch.cuda.is_available(), "run_many_time.py measures on a GPU; there is no CPU fallback"
    torch.cuda.set_device(0)
    d = args.out or tempfile.mkdtemp(prefix="run_many_time_")
    os.makedirs(d, exist_ok=True)
    try:
        w, h = args.width, args.height
        template = os.path.join(ROOT, "models", "%s_deploy.prototxt.template" % args.model)
        net = F.Net(F.fill_template(open(template).read(), w, h), None, F.TEST, batch=1)
        net.fill_params(1701)
        model = os.path.join(d, "weights.caffemodel")
        with open(model, "wb") as f:
            f.write(net.to_caffemodel())
        del net
        gc.collect()
        lines = write_pairs(d, args.pairs, w, h)
        res = {"workload": "%s deploy, %d pairs of %dx%d frames (PPM and PNG), files in to .flo out" % (args.model, args.pairs, w, h)}
        res.update(gpu_info())
        outs_a = write_list(os.path.join(d, "a.txt"), lines, os.path.join(d, "a"))
        res["a_public_path"] = public_path(F, FI, model, template, lines, outs_a, w, h)
        gc.collect()
        for key, batch in (("b_driver_batch1", 1), ("c_driver_batch4", 4)):
            lst = os.path.join(d, "%s.txt" % key)
            outs = write_list(lst, lines, os.path.join(d, key))
            s = R.run(model, template, FI.read_list(lst, ground_truth=False), batch=batch)
            torch.cuda.synchronize()
            run_s = s["wall"] - s["busy"]["build"]
            res[key] = {"pairs_per_s": args.pairs / run_s, "wall_s": run_s, "build_s": s["busy"]["build"],
                        "busy_s": {k: v for k, v in s["busy"].items() if k != "build"}, "not_finite": len(s["not_finite"])}
            if batch == 1:
                res["a_b_bit_identical"] = all(open(x, "rb").read() == open(y, "rb").read() for x, y in zip(outs_a, outs))
        res["note"] = ("pairs_per_s excludes build_s: net construction, reading the weights and, for (b) and (c), reading the "
                       "frame headers; the first forward (eager pass and graph capture) is inside every timed window")
        print(json.dumps(res), flush=True)
    finally:
        if args.out is None:
            shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
