"""Time every NT = 128 plain-mode layer of FlowNet2 (the per-tap engine's FP16 route) at bench.py's shapes, for one or more
builds of libfn2.so, alternating them.

    python tools/conv128_time.py [--libs A.so B.so ...] [--rounds 3] [--iters 20] [--json OUT]

Each round runs every library once, in a process of its own (FN2_LIB), so the builds take turns on the card.  Per layer and
library: the median over rounds of the mean time per call (CUDA events around --iters calls after 3 warm-up calls), GFLOP
(algorithmic: 2 N Co Ho Wo Ci kh kw for a convolution, 2 N Ci H W Co kh kw for a deconvolution), TFLOP/s, and the bytes the
K steps of the plan read from L2: per 128 x 128 x 32 tile step 16 KB of activations plus the weight tiles (32 KB as TF32 hi/lo,
24 KB as three FP16 tiles; --wbytes picks which the table assumes per library, default 32 for the first, 24 for the others).
The card's name, power limit and maximum SM clock are read in the same call.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N, WIDTH, HEIGHT = 4, 1024, 436


def layers():
    """(name, ci, h, w, co, k, s, p, deconv) of the FlowNet2 deploy layers the per-tap engine runs at NT = 128 in plain mode"""
    import flownet2_b200 as F
    from flownet2_b200 import fn2_conv_desc
    from tests.util import deploy_convs
    out = []
    for name, ci, h, w, co, (k, _), s, (p, _), deconv, _ in deploy_convs("FlowNet2", WIDTH, HEIGHT):   # square kernels there
        d = fn2_conv_desc(ci, co, k, k, s, s, p, p, int(deconv), 1, 1, 0.1, 0, 1024)
        pl = (C.c_int32 * 8)()
        F.check(F.lib().fn2_conv_plan(C.byref(d), N, h, w, (ci + 31) // 32 * 32, pl))
        if pl[0] == 128 and pl[3] == 0:
            out.append((name, ci, h, w, co, k, s, p, bool(deconv), list(pl)))
    return out


def child(iters):
    import torch
    from flownet2_b200 import ops, lib, check, fn2_conv_desc
    l = lib()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    res = {}
    for name, ci, h, w, co, k, s, p, deconv, pl in layers():
        g = torch.Generator(device="cuda").manual_seed(1)
        cp = (ci + 31) // 32 * 32
        x = torch.randn(N, cp, h, w, generator=g, device="cuda").clamp_min(0).contiguous(memory_format=torch.channels_last)[:, :ci]
        wt = torch.randn((ci, co, k, k) if deconv else (co, ci, k, k), generator=g, device="cuda") * (2.0 / (ci * k * k)) ** 0.5
        b = torch.zeros(co, device="cuda")
        d = fn2_conv_desc(ci, co, k, k, s, s, p, p, int(deconv), 1, 1, 0.1, 2, 0)
        nf = C.c_size_t()
        check(l.fn2_conv_packed_floats(C.byref(d), cp, C.byref(nf)))
        packed = torch.empty(nf.value, device="cuda")
        check(l.fn2_conv_pack_weights(C.byref(d), cp, C.c_void_p(wt.data_ptr()), C.c_void_p(packed.data_ptr()), st))
        ho, wo = C.c_int(), C.c_int()
        check(l.fn2_conv_out_shape(C.byref(d), h, w, C.byref(ho), C.byref(wo)))
        out = torch.empty(N, co, ho.value, wo.value, device="cuda").contiguous(memory_format=torch.channels_last)
        wb = C.c_size_t()
        check(l.fn2_conv_workspace_bytes(C.byref(d), N, h, w, C.byref(wb)))
        ws = torch.empty(max(wb.value, 16) // 4 + 1, device="cuda")
        dx, do = ops.desc(x), ops.desc(out)

        def go():
            check(l.fn2_conv_forward(C.byref(d), C.byref(dx), C.c_void_p(packed.data_ptr()), C.c_void_p(b.data_ptr()), C.byref(do),
                                     C.c_void_p(ws.data_ptr()), wb.value, st))
        for _ in range(3):
            go()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            go()
        e1.record()
        torch.cuda.synchronize()
        res[name] = e0.elapsed_time(e1) / iters
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", nargs="+", default=[os.path.join(ROOT, "flownet2_b200", "libfn2.so")])
    ap.add_argument("--wbytes", nargs="+", type=int, default=None, help="weight KB per tile step assumed for each library")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    ap.add_argument("--child", action="store_true")
    a = ap.parse_args()
    if a.child:
        return child(a.iters)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    wkb = a.wbytes or [32] + [24] * (len(a.libs) - 1)
    runs = {lib: [] for lib in a.libs}
    for _ in range(a.rounds):
        for lib in a.libs:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--iters", str(a.iters)], capture_output=True,
                               text=True, env=dict(os.environ, FN2_LIB=os.path.abspath(lib)), cwd=ROOT)
            if r.returncode:
                sys.exit("child failed for %s:\n%s" % (lib, r.stderr[-3000:]))
            runs[lib].append(json.loads(r.stdout.strip().splitlines()[-1]))
    print("card: %s" % card)
    table = []
    for name, ci, h, w, co, k, s, p, deconv, pl in layers():
        ho = (h - 1) * s - 2 * p + k if deconv else (h + 2 * p - k) // s + 1
        wo = (w - 1) * s - 2 * p + k if deconv else (w + 2 * p - k) // s + 1
        gf = 2.0 * N * co * ci * k * k * (h * w if deconv else ho * wo) / 1e9
        row = {"layer": name, "shape": [ci, h, w, co, k, s, p, int(deconv)], "gflop": gf, "tile_steps": pl[1] * pl[2]}
        for lib, kb in zip(a.libs, wkb):
            ts = sorted(r[name] for r in runs[lib])
            ms = ts[len(ts) // 2]
            row[lib] = {"ms": ms, "spread_ms": ts[-1] - ts[0], "tflops": gf / ms, "l2_mb": pl[1] * pl[2] * (16 + kb) / 1024.0}
        table.append(row)
    hdr = "%-16s %7s" % ("layer", "GFLOP") + "".join(" | %8s %7s %7s" % ("ms", "TFLOP/s", "L2 MB") for _ in a.libs)
    print("libraries: " + ", ".join("%s (W %d KB/step)" % (lib, kb) for lib, kb in zip(a.libs, wkb)))
    print(hdr)
    tot = [0.0] * len(a.libs)
    for row in table:
        line = "%-16s %7.1f" % (row["layer"], row["gflop"])
        for i, lib in enumerate(a.libs):
            e = row[lib]
            tot[i] += e["ms"]
            line += " | %8.3f %7.1f %7.0f" % (e["ms"], e["tflops"], e["l2_mb"])
        print(line)
    gft = sum(r["gflop"] for r in table)
    print("%-16s %7.1f" % ("total", gft) + "".join(" | %8.3f %7.1f %7s" % (t, gft / t, "") for t in tot))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        json.dump({"card": card, "libs": a.libs, "rows": table, "total_ms": tot}, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
