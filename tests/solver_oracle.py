"""Restatement of Caffe's solver arithmetic, for the solver tests.

* learning_rate: SGDSolver::GetLearningRate (src/caffe/solvers/sgd_solver.cpp:27-63) in the reference's types: pow(float, int)
  in double (the int overload promotes), pow(float, float) and exp(float) as the C library's powf / expf (the float
  overloads <math.h> makes visible), float32 arithmetic around them.
* update: one SGDSolver::ApplyUpdate (sgd_solver.cpp:102-116) of one parameter blob, float32 numpy, every product and sum
  rounded on its own except the multiply-adds the reference's nvcc build fuses in SGDUpdate and AdamUpdate (fma below), in the
  order the reference writes them:
    ClipGradients :81-99 (scale_diff), Normalize :119-142 (caffe_gpu_scal), Regularize :145-204 (axpy of data / sign(data)),
    SGDUpdate sgd_solver.cu:6-12, AdamUpdate adam_solver.cu:6-16 with adam_solver.cpp:26-44, Blob::Update (data -= diff).
* clip_scale: ClipGradients' factor from a float64 sum of squares.
* SolverState (caffe.proto:247-252) wire format, written and read without protobuf.
"""
import ctypes
import ctypes.util
import math

import numpy as np

f32 = np.float32
_LIBM = ctypes.CDLL(ctypes.util.find_library("m"))
_LIBM.powf.restype = _LIBM.expf.restype = ctypes.c_float
_LIBM.powf.argtypes = [ctypes.c_float, ctypes.c_float]
_LIBM.expf.argtypes = [ctypes.c_float]


def powf(x, y):
    return f32(_LIBM.powf(float(x), float(y)))


def expf(x):
    return f32(_LIBM.expf(float(x)))


def learning_rate(p, it, current_step):
    """-> (rate as float32, current_step)."""
    pol, base, gamma, power = p["lr_policy"], f32(p["base_lr"]), f32(p["gamma"]), f32(p["power"])
    if pol == "fixed":
        return base, current_step
    if pol == "step":
        current_step = it // int(p["stepsize"])
        return f32(float(base) * math.pow(float(gamma), current_step)), current_step
    if pol == "exp":
        return f32(float(base) * math.pow(float(gamma), it)), current_step
    if pol == "inv":
        x = f32(1) + gamma * f32(it)
        return base * powf(x, -power), current_step
    if pol == "multistep":
        sv = p["stepvalue"]
        if current_step < len(sv) and it >= sv[current_step]:
            current_step += 1
        return f32(float(base) * math.pow(float(gamma), current_step)), current_step
    if pol == "poly":
        x = f32(1) - f32(it) / f32(p["max_iter"])
        return base * powf(x, power), current_step
    if pol == "sigmoid":
        arg = -gamma * (f32(it) - f32(p["stepsize"]))
        return base * (f32(1) / (f32(1) + expf(arg))), current_step
    raise ValueError(pol)


def adam_correction(p, it):
    t = it + 1
    return f32(math.sqrt(1.0 - math.pow(float(f32(p["momentum2"])), t)) / (1.0 - math.pow(float(f32(p["momentum"])), t)))


def fma(a, b, c):
    """float32 fused multiply-add: the product of two float32 is exact in the 64-bit significand of long double, so the only
    roundings are of the sum (to 64 bits, then to 24; a second rounding changes the result only with probability ~2^-40)."""
    ld = np.longdouble
    return (np.asarray(a, ld) * np.asarray(b, ld) + np.asarray(c, ld)).astype(np.float32)


def clip_scale(diffs, clip):
    """diffs: the trainable gradients.  -> float32 scale (1 when the norm is within clip)."""
    sumsq = sum(float(np.dot(d.astype(np.float64), d.astype(np.float64))) for d in diffs)
    l2 = f32(math.sqrt(sumsq))
    return f32(clip) / l2 if l2 > f32(clip) else f32(1)


def update(p, rate, it, w, g, h0, h1, lr_mult, decay_mult, scale=None):
    """One parameter blob.  -> (w, g, h0, h1) after the update; h1 is Adam's v (None for SGD)."""
    w, g, h0 = (np.asarray(a, np.float32).copy() for a in (w, g, h0))
    if scale is not None:
        g = g * f32(scale)
    if int(p["iter_size"]) != 1:
        g = g * (f32(1) / f32(p["iter_size"]))
    local_decay = f32(p["weight_decay"]) * f32(decay_mult)
    if local_decay != 0:
        r = np.sign(w).astype(np.float32) if p["regularization_type"] == "L1" else w
        g = local_decay * r + g
    local_rate = f32(rate) * f32(lr_mult)
    if p["type"] == "Adam":
        b1, b2 = f32(p["momentum"]), f32(p["momentum2"])
        h1 = np.asarray(h1, np.float32).copy()
        h0 = fma(f32(1) - b1, g, h0 * b1)                                   # adam_solver.cu:11-12 as nvcc fuses them
        h1 = fma(f32(1) - b2, g * g, h1 * b2)
        g = (local_rate * adam_correction(p, it)) * h0 / (np.sqrt(h1) + f32(p["delta"]))
    else:
        h0 = fma(f32(p["momentum"]), h0, local_rate * g)                    # sgd_solver.cu:10 as nvcc fuses it
        g = h0.copy()
    return w - g, g, h0, h1


# ---- SolverState wire format ----
def _varint(b, i):
    v, s = 0, 0
    while True:
        c = b[i]
        i += 1
        v |= (c & 0x7F) << s
        if not c & 0x80:
            return v, i
        s += 7


def _put_varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _field(fn, wt):
    return _put_varint((fn << 3) | wt)


def _ld(fn, payload):
    return _field(fn, 2) + _put_varint(len(payload)) + payload


def parse_blob(b):
    shape, data, i = [], [], 0
    while i < len(b):
        key, i = _varint(b, i)
        fn, wt = key >> 3, key & 7
        assert wt == 2, (fn, wt)
        n, i = _varint(b, i)
        sub = b[i:i + n]
        i += n
        if fn == 5:
            data.append(np.frombuffer(sub, "<f4"))
        elif fn == 7:
            j = 0
            while j < len(sub):
                k2, j = _varint(sub, j)
                m, j = _varint(sub, j)
                dims, q = sub[j:j + m], 0
                j += m
                while q < len(dims):
                    d, q = _varint(dims, q)
                    shape.append(d)
    return shape, (np.concatenate(data) if data else np.zeros(0, np.float32))


def parse_state(b):
    """-> {iter, current_step, learned_net, history: [(shape, float32 array)]}."""
    out, i = {"iter": 0, "current_step": 0, "learned_net": "", "history": []}, 0
    while i < len(b):
        key, i = _varint(b, i)
        fn, wt = key >> 3, key & 7
        if wt == 0:
            v, i = _varint(b, i)
            out[{1: "iter", 4: "current_step"}[fn]] = v
            continue
        n, i = _varint(b, i)
        sub = b[i:i + n]
        i += n
        if fn == 2:
            out["learned_net"] = sub.decode()
        elif fn == 3:
            out["history"].append(parse_blob(sub))
    return out


def write_state(it, current_step, learned_net, history):
    """history: [(shape, float32 array)] -> SolverState bytes."""
    o = _field(1, 0) + _put_varint(it) + _ld(2, learned_net.encode())
    for shape, data in history:
        dims = b"".join(_put_varint(d) for d in shape)
        o += _ld(3, _ld(5, np.asarray(data, "<f4").tobytes()) + _ld(7, _ld(1, dims)))
    return o + _field(4, 0) + _put_varint(current_step)
