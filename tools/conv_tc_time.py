"""Time every FlowNet2 layer the per-tap tensor-core engine runs (plain K blocks, tap groups, kernel rows; every NT) at bench.py's
shapes, for one or more builds of libfn2.so, alternating them.

    python tools/conv_tc_time.py [--libs A.so B.so ...] [--rounds 3] [--iters 20] [--json OUT]

Each layer runs on the bottom the net gives it: the nets' padded pixel stride and a 1 KB guard band of NaN (the `pad` layout of
tests/conv_ref.py), so that a small-Ci layer plans in the mode the net runs it in, and at the net's batch (a layer on both
images, net1_conv1, at twice the pairs).  Each round runs every library once, in a process of its own (FN2_LIB), so the builds
take turns on the card.  Per layer: its plan (NT, mode 0 plain / 1 tap groups / 2 kernel rows), GFLOP (algorithmic:
2 N Co Ho Wo Ci kh kw for a convolution, 2 N Ci H W Co kh kw for a deconvolution), and per library the median over rounds of
the mean time per call (CUDA events around --iters calls after 3 warm-up calls), TFLOP/s, the operand route its packed weights
show (FP16 or TF32) and the bytes the plan's K steps read from L2: 16 KB of activations per step plus the weight stage, 2 NT 128 B
as TF32 hi / lo or 2 NT 64 B as the FP16 tiles W_A and W_B (the packing's third tile, W_C, is not read).  The card's name, power
limit and maximum SM clock are read in the same call.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PAIRS, WIDTH, HEIGHT = 4, 1024, 436
MODES = {0: "plain", 1: "group", 2: "row"}


def _desc(ci, co, k, s, p, deconv):
    from flownet2_b200 import fn2_conv_desc
    from tests.conv_ref import guard_bytes
    return fn2_conv_desc(ci, co, k, k, s, s, p, p, int(deconv), 1, 1, 0.1, 2, guard_bytes("pad"))


def layers():
    """(name, N, ci, h, w, co, k, s, p, deconv, plan8) of the FlowNet2 deploy layers the per-tap engine runs"""
    import flownet2_b200 as F
    from flownet2_b200 import fill_template, model_template
    from tests.conv_ref import cstride
    from tests.util import net_walk
    convs, _, _, io = net_walk(fill_template(model_template("FlowNet2"), WIDTH, HEIGHT))
    out = []
    for name, ci, h, w, co, (k, _), s, (p, _), deconv, _ in convs:                 # square kernels there
        n = PAIRS * len(io[name][0])                                               # conv1 of FlowNetC: both images
        pl = (C.c_int32 * 8)()
        F.check(F.lib().fn2_conv_plan(C.byref(_desc(ci, co, k, s, p, deconv)), n, h, w, cstride(ci), pl))
        if pl[0] > 0 and pl[3] in MODES:
            out.append((name, n, ci, h, w, co, k, s, p, bool(deconv), list(pl)))
    return out


def child(iters):
    import torch
    from flownet2_b200 import ops, lib, check
    from tests.conv_ref import bottom
    l = lib()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    res = {}
    for name, n, ci, h, w, co, k, s, p, deconv, pl in layers():
        g = torch.Generator(device="cuda").manual_seed(1)
        x = bottom(torch.randn(n, ci, h, w, generator=g, device="cuda").clamp_min(0), "pad")
        cis = x.stride(3)
        wt = torch.randn((ci, co, k, k) if deconv else (co, ci, k, k), generator=g, device="cuda") * (2.0 / (ci * k * k)) ** 0.5
        b = torch.zeros(co, device="cuda")
        d = _desc(ci, co, k, s, p, deconv)
        nf = C.c_size_t()
        check(l.fn2_conv_packed_floats(C.byref(d), cis, C.byref(nf)))
        packed = torch.empty(nf.value, device="cuda")
        check(l.fn2_conv_pack_weights(C.byref(d), cis, C.c_void_p(wt.data_ptr()), C.c_void_p(packed.data_ptr()), st))
        ho, wo = C.c_int(), C.c_int()
        check(l.fn2_conv_out_shape(C.byref(d), h, w, C.byref(ho), C.byref(wo)))
        out = torch.empty(n, co, ho.value, wo.value, device="cuda").contiguous(memory_format=torch.channels_last)
        wb = C.c_size_t()
        check(l.fn2_conv_workspace_bytes(C.byref(d), n, h, w, C.byref(wb)))
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
        # the tensor-core part of the packed weights (behind the SIMT copy), from which the parent tells the route
        res[name] = [e0.elapsed_time(e1) / iters, nf.value - k * k * ci * co]
    print(json.dumps(res))


def f16_route(ci, co, k, pl, tc_floats):
    """whether packed tensor-core weights of tc_floats floats are the FP16 route's: 48 floats per output channel and K block
    (plain: taps x 32-channel blocks; kernel rows: the plan's K steps), then 4 (tc_f16_tile_floats)"""
    blocks = pl[2] if pl[3] == 2 else k * k * ((ci + 31) // 32)
    return pl[3] != 1 and tc_floats == 48 * blocks * co + 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", nargs="+", default=[os.path.join(ROOT, "flownet2_b200", "libfn2.so")])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    ap.add_argument("--child", action="store_true")
    a = ap.parse_args()
    if a.child:
        return child(a.iters)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    runs = {lib: [] for lib in a.libs}
    for _ in range(a.rounds):
        for lib in a.libs:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--iters", str(a.iters)], capture_output=True,
                               text=True, env=dict(os.environ, FN2_LIB=os.path.abspath(lib)), cwd=ROOT)
            if r.returncode:
                sys.exit("child failed for %s:\n%s" % (lib, r.stderr[-3000:]))
            runs[lib].append(json.loads(r.stdout.strip().splitlines()[-1]))
    print("card: %s" % card)
    print("libraries: " + ", ".join(a.libs))
    table = []
    for name, n, ci, h, w, co, k, s, p, deconv, pl in layers():
        ho = (h - 1) * s - 2 * p + k if deconv else (h + 2 * p - k) // s + 1
        wo = (w - 1) * s - 2 * p + k if deconv else (w + 2 * p - k) // s + 1
        gf = 2.0 * n * co * ci * k * k * (h * w if deconv else ho * wo) / 1e9
        row = {"layer": name, "n": n, "shape": [ci, h, w, co, k, s, p, int(deconv)], "plan": pl, "gflop": gf, "tile_steps": pl[1] * pl[2]}
        for lib in a.libs:
            ts = sorted(r[name][0] for r in runs[lib])
            ms = ts[len(ts) // 2]
            f16 = f16_route(ci, co, k, pl, runs[lib][0][name][1])
            wb = 2 * pl[0] * (64 if f16 else 128)
            row[lib] = {"ms": ms, "spread_ms": ts[-1] - ts[0], "tflops": gf / ms, "route": "FP16" if f16 else "TF32",
                        "l2_mb": pl[1] * pl[2] * (16384 + wb) / 2 ** 20}
        table.append(row)
    print("%-20s %4s %-5s %7s" % ("layer", "NT", "mode", "GFLOP") + "".join(" | %8s %7s %4s %7s" % ("ms", "TFLOP/s", "op", "L2 MB")
                                                                          for _ in a.libs))
    groups = {}
    for row in table:
        pl = row["plan"]
        line = "%-20s %4d %-5s %7.1f" % (row["layer"], pl[0], MODES[pl[3]], row["gflop"])
        g = groups.setdefault("NT %d %s" % (pl[0], MODES[pl[3]]), [0.0, [0.0] * len(a.libs)])
        g[0] += row["gflop"]
        for i, lib in enumerate(a.libs):
            e = row[lib]
            g[1][i] += e["ms"]
            line += " | %8.3f %7.1f %4s %7.0f" % (e["ms"], e["tflops"], e["route"], e["l2_mb"])
        print(line)
    for key, (gf, ms) in sorted(groups.items()):
        print("%-31s %7.1f" % (key, gf) + "".join(" | %8.3f %7.1f %4s %7s" % (t, gf / t, "", "") for t in ms))
    tot = [sum(row[lib]["ms"] for row in table) for lib in a.libs]
    gft = sum(r["gflop"] for r in table)
    print("%-31s %7.1f" % ("total", gft) + "".join(" | %8.3f %7.1f %4s %7s" % (t, gft / t, "", "") for t in tot))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        json.dump({"card": card, "libs": a.libs, "rows": table, "total_ms": tot}, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
