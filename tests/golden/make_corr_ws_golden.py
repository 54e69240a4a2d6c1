"""Records the Correlation / Correlation1D workspace queries (fn2_correlation_workspace_bytes,
fn2_correlation_backward_workspace_bytes, fn2_correlation1d_backward_workspace_bytes) over a sweep of layer shapes into
tests/golden/corr_ws_golden.npz; test_host_cpu.py checks the library's queries against it.

    FN2_LIB=<libfn2.so of the commit to record> python tests/golden/make_corr_ws_golden.py

The sweep: MULTIPLY and SUBTRACT, kernel_size 1 / 3, stride_1 1 / 2, pad = max_displacement and pad < max_displacement,
R = max_displacement / stride_2 of 2 / 3 / 4 / 10 with stride_2 1-3, C 8 / 40 / 64 / 256 and N 1 / 4 on a 48 x 64 map, for
the 2-D layer and the three directions of the 1-D layer; and FlowNet2-C's layer at the BASELINE input (conv3 features of
1024 x 448: 256 x 56 x 128, N 1 / 4 / 8).  No GPU is needed.

Rows: params (dims, N, C, H, W, pad, k, md, s1, s2, single_direction, corr_type), fwd (forward workspace bytes; -1 for the 1-D
layer, which takes none) and bwd (backward workspace bytes)."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from flownet2_b200 import lib  # noqa: E402

FIELDS = ["dims", "N", "C", "H", "W", "pad", "k", "md", "s1", "s2", "single_direction", "corr_type"]


def cases():
    out = []
    for typ in (0, 1):
        for k in (1, 3):
            for s1 in (1, 2):
                for R in (2, 3, 4, 10):
                    for s2 in (1, 2, 3):
                        md = R * s2
                        for pad in (md, md // 2):
                            for Cc in (8, 40, 64, 256):
                                for N in (1, 4):
                                    out.append((2, N, Cc, 48, 64, pad, k, md, s1, s2, 0, typ))
                                    for sd in (-1, 0, 1):
                                        out.append((1, N, Cc, 48, 64, pad, k, md, s1, s2, sd, typ))
    for N in (1, 4, 8):
        out.append((2, N, 256, 56, 128, 20, 1, 20, 1, 2, 0, 0))
    return out


def main():
    l = lib()
    rows = cases()
    fwd = np.full(len(rows), -1, np.int64)
    bwd = np.zeros(len(rows), np.int64)
    for i, (dims, N, Cc, H, W, pad, k, md, s1, s2, sd, typ) in enumerate(rows):
        b = C.c_size_t()
        if dims == 2:
            assert l.fn2_correlation_workspace_bytes(N, Cc, H, W, pad, k, md, s1, s2, typ, C.byref(b)) == 0
            fwd[i] = b.value
            assert l.fn2_correlation_backward_workspace_bytes(N, Cc, H, W, pad, k, md, s1, s2, typ, C.byref(b)) == 0
        else:
            assert l.fn2_correlation1d_backward_workspace_bytes(N, Cc, H, W, pad, k, md, s1, s2, sd, typ, C.byref(b)) == 0
        bwd[i] = b.value
    np.savez_compressed(os.path.join(HERE, "corr_ws_golden.npz"), params=np.array(rows, np.int32), fwd=fwd, bwd=bwd)
    print("wrote %d shapes (%d with a forward workspace)" % (len(rows), (fwd > 0).sum()))


if __name__ == "__main__":
    main()
