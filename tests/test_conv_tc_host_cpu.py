"""CPU tests of the tensor-core engines' host side: the packed weight size of every layer in the descriptor sweep of
tests/golden/make_conv_plan_golden.py, as recorded by tests/golden/make_conv_packed_golden.py.  The size covers the SIMT weights,
then the packed weights of the engine that owns the layer: the taps-on-N layout, or the per-tap layout of the layer's route
(TF32 per tap, tap groups, kernel rows, or FP16 with the tail that holds the largest |w|)."""
import ctypes as C
import os

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_conv_packed_floats_golden(fn2):
    from flownet2_b200 import fn2_conv_desc
    from tests.golden.make_conv_plan_golden import INT_FIELDS
    lib = fn2.lib()
    g = np.load(os.path.join(GOLD, "conv_packed_golden.npz"))
    assert len(g["floats"]) > 2000
    bad = []
    for row, cis, want in zip(g["desc"], g["ci_stride"], g["floats"]):
        d = fn2_conv_desc(**dict(zip(INT_FIELDS, (int(v) for v in row))), negative_slope=0.1)
        n = C.c_size_t()
        assert lib.fn2_conv_packed_floats(C.byref(d), int(cis), C.byref(n)) == 0
        if n.value != int(want):
            bad.append((row.tolist(), int(cis), int(want), n.value))
    assert not bad, (len(bad), bad[:5])
