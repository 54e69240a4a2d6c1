"""Outputs of the REFERENCE's own solver update kernels (src/caffe/solvers/sgd_solver.cu SGDUpdate, adam_solver.cu AdamUpdate),
against which tests/test_solver_ref_gpu.py holds the engine's fused update.

Two steps, as the reference checkout and the GPU are on different machines:

  python tests/golden/make_solver_ref_golden.py compile     # where /root/reference is: the two .cu files, compiled where they
                                                           # lie with oracle/_ref's include paths and flags (nvcc's default
                                                           # -fmad=true, like the reference Makefile), plus the small C shim
                                                           # below, into build/solver_ref/libref_solver.so (git-ignored)
  python tests/golden/make_solver_ref_golden.py run OUT    # on the GPU: run them on the seeded cases of CASES, write OUT (.npz)

The inputs are regenerated from the seeds by inputs(); only the reference's outputs are stored (ref_solver_update.npz).
tools/solver_time.py uses the same library, when present, as the reference arm of its timing.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "build", "solver_ref")
LIB = os.path.join(OUT, "libref_solver.so")

SHIM = r'''
namespace caffe {
template <typename Dtype> void sgd_update_gpu(int N, Dtype* g, Dtype* h, Dtype momentum, Dtype local_rate);
template <typename Dtype> void adam_update_gpu(int N, Dtype* g, Dtype* m, Dtype* v, Dtype beta1, Dtype beta2, Dtype eps_hat,
                                               Dtype corrected_local_rate);
}
extern "C" int ref_sgd_update(int n, float* g, float* h, float momentum, float local_rate) {
  try { caffe::sgd_update_gpu<float>(n, g, h, momentum, local_rate); return 0; } catch (...) { return -1; }
}
extern "C" int ref_adam_update(int n, float* g, float* m, float* v, float b1, float b2, float eps, float rate) {
  try { caffe::adam_update_gpu<float>(n, g, m, v, b1, b2, eps, rate); return 0; } catch (...) { return -1; }
}
'''

# (name, solver text, iteration the solver is restored at); every parameter has lr_mult 1 and no weight decay, so the gradient
# reaches SGDUpdate / AdamUpdate as it is
CASES = [
    ("sgd_m0", 'type: "SGD"\nbase_lr: 0.05\nlr_policy: "fixed"\nmomentum: 0\n', 7),
    ("sgd_m09", 'type: "SGD"\nbase_lr: 0.05\nlr_policy: "fixed"\nmomentum: 0.9\n', 7),
    ("adam", 'type: "Adam"\nbase_lr: 0.05\nlr_policy: "fixed"\nmomentum: 0.9\nmomentum2: 0.999\ndelta: 1e-8\n', 7),
]
COUNT = 5813               # the learnable floats of tests/test_solver_ref_gpu.NET: 16x3x3x3 + 16 + 37x16x3x3 + 37


def inputs(seed, n=COUNT):
    """Data, gradient, history (m) and v of one case.  Within an element the gradient and the history share a sign and the data
    has the other one, so no sum in the update cancels and a distance in units in the last place measures the arithmetic,
    not the conditioning of the case."""
    r = np.random.default_rng(seed)
    s = r.choice(np.array([-1.0, 1.0], np.float32), n)
    g = (s * (0.05 + np.abs(r.standard_normal(n)))).astype(np.float32)
    h = (s * 0.1 * (0.05 + np.abs(r.standard_normal(n)))).astype(np.float32)
    v = (1e-2 * (0.05 + np.abs(r.standard_normal(n)))).astype(np.float32)
    w = (-s * (1 + np.abs(r.standard_normal(n)))).astype(np.float32)
    return w, g, h, v


def scalars(text, it):
    """(momentum, momentum2, delta, local_rate or corrected local rate) as the reference passes them (sgd_solver.cpp:213-217,
    adam_solver.cpp:26-44), float32."""
    from tests import solver_oracle as SO
    import flownet2_b200 as F
    p = F.solver_params(text)
    rate, _ = SO.learning_rate(p, it, 0)
    local_rate = np.float32(rate) * np.float32(1)
    if p["type"] == "Adam":
        local_rate = local_rate * SO.adam_correction(p, it)
    return np.float32(p["momentum"]), np.float32(p["momentum2"]), np.float32(p["delta"]), np.float32(local_rate)


def compile_lib():
    from oracle.ref_shim import build_ref as B
    B.build()                                       # libref_caffe.so, which provides what the glog stand-in refers to
    os.makedirs(OUT, exist_ok=True)
    shim = os.path.join(OUT, "solver_shim.cu")
    with open(shim, "w") as f:
        f.write(SHIM)
    srcs = [os.path.join(B.REF, "src/caffe/solvers", s) for s in ("sgd_solver.cu", "adam_solver.cu")] + [shim]
    inc = sum((["-I", i] for i in B.INCLUDES), [])
    cmd = [B.NVCC] + B.ARCH + ["-O2", "-std=c++14", "-ccbin", "/usr/bin/g++", "-Xcompiler", "-fPIC,-w", "-w", "-shared"] + \
        B.DEFS + inc + srcs + ["-o", LIB, "-L", os.path.dirname(B.LIB), "-lref_caffe",
                               "-Xlinker", "-rpath,$ORIGIN/../../oracle/_ref"]
    subprocess.run(cmd, check=True)
    return LIB


def load():
    lib = C.CDLL(LIB)
    lib.ref_sgd_update.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_float]
    lib.ref_adam_update.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_float] * 4
    return lib


def run(out):
    import torch
    lib = load()
    res = {}
    for k, (name, text, it) in enumerate(CASES):
        w, g, h, v = inputs(100 + k)
        b1, b2, eps, rate = scalars(text, it)
        tg, th, tv = (torch.from_numpy(a.copy()).cuda() for a in (g, h, v))
        torch.cuda.synchronize()
        if name.startswith("adam"):
            rc = lib.ref_adam_update(g.size, tg.data_ptr(), th.data_ptr(), tv.data_ptr(), b1, b2, eps, rate)
        else:
            rc = lib.ref_sgd_update(g.size, tg.data_ptr(), th.data_ptr(), b1, rate)
        assert rc == 0
        torch.cuda.synchronize()
        res[name + "_diff"], res[name + "_hist"] = tg.cpu().numpy(), th.cpu().numpy()
        if name.startswith("adam"):
            res[name + "_v"] = tv.cpu().numpy()
    np.savez_compressed(out, **res)


if __name__ == "__main__":
    if sys.argv[1] == "compile":
        print(compile_lib())
    else:
        run(sys.argv[2])
