"""Records the tensor-core engines' host-side plan (fn2_conv_plan) and the conv workspace size (fn2_conv_workspace_bytes) over a
sweep of layer descriptors into tests/golden/conv_plan_golden.npz; test_host_cpu.py checks that the library still plans the same.

    FN2_LIB=<libfn2.so of the commit to record> python tests/golden/make_conv_plan_golden.py

The sweep: convolutions and deconvolutions with k 1-7, stride 1-2, Ci 3-1024 and Co multiples of 16 (plus Co = 2, which the
engines do not take) at three map sizes; the small-Ci packing cases with and without a guard band and with a wider pixel
stride; the conv / deconv layers of FlowNet2 at the BASELINE input (1024 x 448) with N = 1, 4 and 8; and the backward-data
descriptors (fn2_conv_backward_data_desc) of all those layers.  Deconvolutions with fewer taps than the stride (a parity
class that no tap reaches) are left out: the tensor-core engine does not take them.  The plan needs no GPU; without one the
SM count is 132, as on an H100 SXM.

Rows: desc (the int fields of fn2_conv_desc; negative_slope is 0.1), shape (N, H, W, ci_stride), plan8, workspace bytes, and
`uniform`: the recorded plan split every tile of the layer (first split tile 0), whose partial tiles the workspace holds as
[tile][split][128 pixels][NT]."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from flownet2_b200 import fn2_conv_desc, lib  # noqa: E402

INT_FIELDS = ["ci", "co", "kh", "kw", "stride_h", "stride_w", "pad_h", "pad_w", "deconv", "has_bias", "relu", "engine",
              "input_guard_bytes", "out_pad_h", "out_pad_w"]

# FlowNet2 conv / deconv layers at the BASELINE input 1024 x 448: (Ci, Co, k, stride, pad, deconv, H, W) of the layer's bottom
FLOWNET2 = [
    (3, 64, 7, 2, 3, 0, 448, 1024), (64, 128, 5, 2, 2, 0, 224, 512), (128, 256, 5, 2, 2, 0, 112, 256),      # FlowNetC
    (256, 32, 1, 1, 0, 0, 56, 128), (473, 256, 3, 1, 1, 0, 56, 128), (256, 512, 3, 2, 1, 0, 56, 128),
    (512, 512, 3, 1, 1, 0, 28, 64), (512, 512, 3, 2, 1, 0, 28, 64), (512, 512, 3, 1, 1, 0, 14, 32),
    (512, 1024, 3, 2, 1, 0, 14, 32), (1024, 1024, 3, 1, 1, 0, 7, 16), (1024, 2, 3, 1, 1, 0, 7, 16),
    (1024, 512, 4, 2, 1, 1, 7, 16), (2, 2, 4, 2, 1, 1, 7, 16), (1026, 2, 3, 1, 1, 0, 14, 32), (1026, 256, 4, 2, 1, 1, 14, 32),
    (770, 2, 3, 1, 1, 0, 28, 64), (770, 128, 4, 2, 1, 1, 28, 64), (386, 2, 3, 1, 1, 0, 56, 128), (386, 64, 4, 2, 1, 1, 56, 128),
    (194, 2, 3, 1, 1, 0, 112, 256),
    (12, 64, 7, 2, 3, 0, 448, 1024), (64, 128, 5, 2, 2, 0, 224, 512), (128, 256, 5, 2, 2, 0, 112, 256),   # FlowNetS
    (256, 256, 3, 1, 1, 0, 56, 128),
    (6, 64, 3, 1, 1, 0, 448, 1024), (64, 64, 3, 2, 1, 0, 448, 1024), (64, 128, 3, 1, 1, 0, 224, 512),      # FlowNet-SD
    (128, 128, 3, 2, 1, 0, 224, 512), (128, 128, 3, 1, 1, 0, 112, 256), (128, 256, 3, 2, 1, 0, 112, 256),
    (1026, 512, 3, 1, 1, 0, 14, 32), (770, 256, 3, 1, 1, 0, 28, 64), (386, 128, 3, 1, 1, 0, 56, 128),
    (194, 64, 3, 1, 1, 0, 112, 256), (512, 32, 3, 1, 1, 0, 14, 32), (256, 16, 3, 1, 1, 0, 28, 64),
    (11, 64, 3, 1, 1, 0, 448, 1024), (64, 64, 3, 2, 1, 0, 448, 1024), (64, 128, 3, 1, 1, 0, 224, 512),     # fusion
    (128, 128, 3, 2, 1, 0, 224, 512), (128, 128, 3, 1, 1, 0, 112, 256), (128, 32, 4, 2, 1, 1, 112, 256),
    (162, 32, 3, 1, 1, 0, 224, 512), (162, 16, 4, 2, 1, 1, 224, 512), (82, 16, 3, 1, 1, 0, 448, 1024),
    (16, 2, 3, 1, 1, 0, 448, 1024),
]


def stride_of(ci):
    """Blob::compute_cstride: padded channel count of an NHWC blob."""
    return (ci + 3) // 4 * 4 if ci < 32 else (ci + 31) // 32 * 32


def cases():
    out = []

    def add(ci, co, k, s, p, deconv, N, H, W, cis=None, guard=1024):
        if deconv and k < s:
            return
        d = fn2_conv_desc(ci, co, k, k, s, s, p, p, deconv, 1, 1, 0.1, 0, guard)
        out.append((d, N, H, W, cis if cis is not None else stride_of(ci)))

    for deconv in (0, 1):
        for k in range(1, 8):
            for s in (1, 2):
                for ci in (3, 8, 16, 32, 96, 473, 1024):
                    for co in (2, 16, 32, 64, 128, 1024):
                        for N, H, W in ((4, 7, 16), (4, 56, 128), (1, 224, 512)):
                            add(ci, co, k, s, (k - 1) // 2, deconv, N, H, W)
    for ci in (3, 4, 6, 12, 16):
        for k in (3, 5, 7):
            for s in (1, 2):
                for extra in (0, 8):
                    for guard in (0, 1024):
                        for N, H, W in ((4, 448, 1024), (1, 56, 128)):
                            add(ci, 64, k, s, (k - 1) // 2, 0, N, H, W, cis=stride_of(ci) + extra, guard=guard)
    for N in (1, 4, 8):
        for ci, co, k, s, p, deconv, H, W in FLOWNET2:
            add(ci, co, k, s, p, deconv, N, H, W)
    # the adjoint of every layer so far: a forward operator on the top diff (Ho x Wo), whose pixel stride is the padded Co
    bwd = []
    for d, N, H, W, _ in out:
        ho, wo, bd, flip = C.c_int(), C.c_int(), fn2_conv_desc(), C.c_int()
        assert lib().fn2_conv_out_shape(C.byref(d), H, W, C.byref(ho), C.byref(wo)) == 0
        assert lib().fn2_conv_backward_data_desc(C.byref(d), H, W, C.byref(bd), C.byref(flip)) == 0
        if bd.deconv and (bd.kh < bd.stride_h or bd.kw < bd.stride_w):
            continue
        bwd.append((bd, N, ho.value, wo.value, stride_of(bd.ci)))
    return out + bwd


def main():
    l = lib()
    rows = cases()
    desc = np.zeros((len(rows), len(INT_FIELDS)), np.int32)
    shape = np.zeros((len(rows), 4), np.int32)
    plan = np.zeros((len(rows), 8), np.int32)
    ws = np.zeros(len(rows), np.int64)
    uniform = np.zeros(len(rows), bool)
    for i, (d, N, H, W, cis) in enumerate(rows):
        o = (C.c_int32 * 8)()
        assert l.fn2_conv_plan(C.byref(d), N, H, W, cis, o) == 0
        b = C.c_size_t()
        assert l.fn2_conv_workspace_bytes(C.byref(d), N, H, W, C.byref(b)) == 0
        p = list(o)
        uniform[i] = p[0] > 0 and p[4] == 0 and p[5] > 1
        desc[i] = [getattr(d, f) for f in INT_FIELDS]
        shape[i] = (N, H, W, cis)
        plan[i] = p
        ws[i] = b.value
    np.savez_compressed(os.path.join(HERE, "conv_plan_golden.npz"), desc=desc, shape=shape, plan=plan, ws=ws, uniform=uniform)
    print("wrote %d plans (%d uniform splits, %d taps-on-N)" % (len(rows), uniform.sum(), (plan[:, 3] == 3).sum()))


if __name__ == "__main__":
    main()
