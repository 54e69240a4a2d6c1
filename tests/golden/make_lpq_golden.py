"""Generates tests/golden/lpq_golden.npz by running the REFERENCE's own LpqLossLayer on the cases of lpq_cases.py, in GPU mode:
forward, then backward with the top diff set to the case's loss weight.

The reference library that oracle/ref_shim/build_ref.py builds does not contain LpqLoss, so this script links its own copy:
the same recipe (the reference's sources compiled where they lie, with the same shim and flags) with lpq_loss_layer added, into
the git-ignored oracle/_ref/lpq/libref_caffe.so.  The objects are shared with the main recipe's.

    python tests/golden/make_lpq_golden.py --build       (where the reference checkout is: compile and link the library)
    python tests/golden/make_lpq_golden.py [outbase]      (on a GPU machine the built library travelled to)
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import lpq_cases as LC  # noqa: E402
from oracle import ref as R  # noqa: E402


LPQ_LIB = os.path.join(ROOT, "oracle", "_ref", "lpq", "libref_caffe.so")


def build_reference(force=False):
    """oracle/ref_shim/build_ref.py's build with lpq_loss_layer (lpq_loss_layer.cpp / .cu) added, linked into LPQ_LIB."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("build_ref", os.path.join(ROOT, "oracle", "ref_shim", "build_ref.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    m.LAYERS = m.LAYERS + ["lpq_loss_layer"]
    m.LIB = LPQ_LIB
    os.makedirs(os.path.dirname(LPQ_LIB), exist_ok=True)
    return m.build(force)


def run_case(name):
    c = LC.LPQ_CASES[name]
    bottoms = LC.lpq_inputs(name)
    bl = [R.Blob(shape=b.shape) for b in bottoms]
    for b, a in zip(bl, bottoms):
        b.set(a)
    tl = [R.Blob()]
    layer = R.Layer(c["text"], 1)
    layer.setup(bl, tl)
    layer.forward()
    out = {"top0": tl[0].get().reshape(tl[0].shape if tl[0].shape else (1,))}
    tl[0].set(np.full(tl[0].shape, c["top_diff"], np.float32), diff=True)
    for b in bl:
        b.set(np.zeros(b.shape, np.float32), diff=True)
    layer.backward([True] * len(bl))
    for i, b in enumerate(bl):
        out["bdiff%d" % i] = b.get(diff=True)
    return out


def main():
    if "--build" in sys.argv:
        print(build_reference(force="--force" in sys.argv))
        return
    outbase = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "lpq_golden")
    assert os.path.exists(LPQ_LIB), "%s is not built: run this script with --build where the reference checkout is" % LPQ_LIB
    R.LIB_PATH = LPQ_LIB
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    R.set_mode(True, 0)
    g, meta = {}, {"device": torch.cuda.get_device_name(0), "cases": {}}
    for name in LC.LPQ_CASES:
        out = run_case(name)
        for k, v in out.items():
            g["L/%s/%s" % (name, k)] = v
        meta["cases"][name] = {k: [list(v.shape), int(np.isnan(v).sum())] for k, v in out.items()}
        print(name, float(out["top0"][0]), meta["cases"][name], flush=True)
    np.savez_compressed(outbase + ".npz", **g)
    with open(outbase + ".json", "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)
    print("wrote", outbase + ".npz", os.path.getsize(outbase + ".npz"), "bytes")


if __name__ == "__main__":
    main()
