"""Records the packed weight size of a convolution (fn2_conv_packed_floats: the SIMT weights plus those of the tensor-core engine
that owns the layer) over the descriptor sweep of make_conv_plan_golden.py, each with its input pixel stride, into
tests/golden/conv_packed_golden.npz; test_conv_tc_host_cpu.py checks that the library still packs into the same sizes.

    FN2_LIB=<libfn2.so of the commit to record> python tests/golden/make_conv_packed_golden.py

The size does not depend on the batch or the map size, so each (descriptor, pixel stride) pair is recorded once.
Rows: desc (the int fields of fn2_conv_desc; negative_slope is 0.1), ci_stride, floats."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from flownet2_b200 import lib  # noqa: E402
from tests.golden.make_conv_plan_golden import INT_FIELDS, cases  # noqa: E402


def main():
    l = lib()
    rows = {}
    for d, _, _, _, cis in cases():
        key = tuple(getattr(d, f) for f in INT_FIELDS) + (cis,)
        if key in rows:
            continue
        n = C.c_size_t()
        assert l.fn2_conv_packed_floats(C.byref(d), cis, C.byref(n)) == 0
        rows[key] = n.value
    keys = sorted(rows)
    desc = np.array([k[:-1] for k in keys], np.int32)
    cis = np.array([k[-1] for k in keys], np.int32)
    floats = np.array([rows[k] for k in keys], np.int64)
    np.savez_compressed(os.path.join(HERE, "conv_packed_golden.npz"), desc=desc, ci_stride=cis, floats=floats)
    print("wrote %d packed sizes" % len(keys))


if __name__ == "__main__":
    main()
