"""In-tree build of libfn2.so (nvcc, sm_90a only).

    python -m flownet2_b200.build            # incremental
    python -m flownet2_b200.build --force

Objects go to flownet2_b200/csrc/build/, the library to flownet2_b200/libfn2.so (both git-ignored).
nvcc cross-compiles without a GPU.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(CSRC, "build")
LIB = os.path.join(HERE, "libfn2.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden,-Wall,-Wno-unused-function",
          "-ccbin", "/usr/bin/g++", "-Xptxas", "-v"]

# (source, extra flags)
SOURCES = [
    ("fn2_runtime.cu", []),
    ("fn2_ops.cu", ["-fmad=false"]),        # bit-exact streaming layers, see file header
    ("fn2_corr.cu", []),
    ("fn2_corr_fast.cu", []),
    ("fn2_corr_bwd.cu", []),
    ("fn2_conv.cu", []),
    ("fn2_conv_nhwc.cu", []),
    ("fn2_conv_tc.cu", []),
    ("fn2_conv_tn.cu", []),
    ("fn2_train.cu", []),
    ("fn2_loss.cu", []),
    ("fn2_solver.cu", ["-fmad=false"]),     # bit-exact update, see file header
    ("fn2_eval.cu", ["-fmad=false"]),       # per-pixel EPE restated exactly in float32, see file header
    ("caffe/proto.cpp", []),
    ("caffe/blob.cpp", []),
    ("caffe/layers.cpp", []),
    ("caffe/net.cpp", []),
    ("caffe/hdf5_min.cpp", []),
    ("caffe/png_unfilter.cpp", []),
    ("caffe/solver.cpp", []),
    ("caffe/capi.cpp", []),
]


def _deps_hash(src, flags):
    h = hashlib.sha1()
    h.update(" ".join(flags).encode())
    for root in (CSRC, os.path.join(CSRC, "caffe"), os.path.join(HERE, "..", "include")):
        for fn in sorted(os.listdir(root)):
            if fn.endswith((".cuh", ".hpp", ".h")):
                with open(os.path.join(root, fn), "rb") as f:
                    h.update(f.read())
    with open(os.path.join(CSRC, src), "rb") as f:
        h.update(f.read())
    return h.hexdigest()


def _compile(item):
    src, extra = item
    obj = os.path.join(BUILD, src.replace("/", "_") + ".o")
    stamp = obj + ".sha1"
    flags = ARCH + COMMON + extra
    want = _deps_hash(src, flags)
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == want and "--force" not in sys.argv:
        return obj, ""
    cmd = [NVCC] + flags + ["-x", "cu", "-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    with open(stamp, "w") as f:
        f.write(want)
    return obj, r.stderr


def build(verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        results = list(ex.map(_compile, SOURCES))
    objs = [o for o, _ in results]
    log = "".join("==== %s\n%s" % (s[0], l) for s, (_, l) in zip(SOURCES, results) if l)
    if log:
        with open(os.path.join(BUILD, "ptxas.log"), "a") as f:
            f.write(log)
        if verbose:
            print(log)
    newest = max(os.path.getmtime(o) for o in objs)
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < newest or "--force" in sys.argv:
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-Xlinker", "--no-undefined",
                                                                "-ccbin", "/usr/bin/g++"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv))
