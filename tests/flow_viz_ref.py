"""numpy restatement of the flow colour code of include/fn2_flow.h (the Middlebury colour wheel), the reference of
tests/test_flow_viz_cpu.py and tests/test_flow_viz_gpu.py.  rad, the rad <= 1 branch, the scale and every product are float32
as the kernel computes them; only atan2 is float64, rounded to float32 and then divided by the float32 pi as the kernel does."""
import numpy as np

SEGMENTS = (("RY", 15), ("YG", 6), ("GC", 4), ("CB", 11), ("BM", 13), ("MR", 6))
F32 = np.float32


def wheel():
    """(55, 3) int wheel: entry i of each segment in integer arithmetic."""
    rows = []
    for name, n in SEGMENTS:
        for i in range(n):
            up, down = 255 * i // n, 255 - 255 * i // n
            rows.append({"RY": (255, up, 0), "YG": (down, 255, 0), "GC": (0, 255, up), "CB": (0, down, 255),
                         "BM": (up, 0, 255), "MR": (255, 0, down)}[name])
    return np.array(rows, np.int64)


def known(flow):
    """(..., 2) flow -> bool (...): both components finite and |u|, |v| <= 1e9."""
    f = np.asarray(flow, np.float32)
    with np.errstate(invalid="ignore"):
        return (np.abs(f) <= F32(1e9)).all(axis=-1)


def max_radius(flow_hw2):
    """Largest float32 sqrt(u^2 + v^2) over the known pixels of one (H, W, 2) flow; -1 when none is known."""
    f = np.asarray(flow_hw2, np.float32)
    k = known(f)
    if not k.any():
        return F32(-1)
    u, v = f[..., 0][k], f[..., 1][k]
    return np.sqrt(u * u + v * v).max().astype(np.float32)


def scale_of(flow_hw2, max_flow=None):
    """The colour scale of one image: max_flow, else its max radius, 1 when that is not positive."""
    if max_flow is not None:
        return F32(max_flow)
    m = max_radius(flow_hw2)
    return m if m > 0 else F32(1)


def colour(flow_hw2, scale):
    """(H, W, 2) flow and a float32 scale -> (H, W, 3) uint8 RGB."""
    f = np.asarray(flow_hw2, np.float32)
    ok = known(f)
    with np.errstate(invalid="ignore", over="ignore"):
        fx, fy = np.where(ok, f[..., 0], 0) / F32(scale), np.where(ok, f[..., 1], 0) / F32(scale)
        fx, fy = fx.astype(np.float32), fy.astype(np.float32)
        rad = np.sqrt(fx * fx + fy * fy)
        a = np.arctan2(-fy.astype(np.float64), -fx.astype(np.float64)).astype(np.float32) / F32(np.pi)
        fk = (a + F32(1)) / F32(2) * F32(54)
        k0 = fk.astype(np.int64)
        k1 = (k0 + 1) % 55
        fr = fk - k0.astype(np.float32)
        w = wheel().astype(np.float32)
        out = np.zeros(f.shape[:-1] + (3,), np.uint8)
        for c in range(3):
            col = (F32(1) - fr) * w[k0, c] / F32(255) + fr * w[k1, c] / F32(255)
            col = np.where(rad <= F32(1), F32(1) - rad * (F32(1) - col), col * F32(0.75)).astype(np.float32)
            out[..., c] = np.where(ok, (F32(255) * col).astype(np.int64), 0)
    return out


def flow_to_color(flow_hw2, max_flow=None):
    return colour(flow_hw2, scale_of(flow_hw2, max_flow))


def paeth_rows(rgb):
    """(H, W, 3) uint8 -> (H, 1 + 3 W) uint8 PNG scanlines, each Paeth-filtered (type 4) with 3 bytes per pixel."""
    raw = np.ascontiguousarray(rgb, np.uint8).reshape(rgb.shape[0], -1).astype(np.int16)
    a = np.zeros_like(raw)
    a[:, 3:] = raw[:, :-3]
    b = np.zeros_like(raw)
    b[1:] = raw[:-1]
    c = np.zeros_like(raw)
    c[1:] = a[:-1]
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    pred = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
    rows = ((raw - pred) & 0xff).astype(np.uint8)
    return np.concatenate([np.full((rows.shape[0], 1), 4, np.uint8), rows], axis=1)
