"""Float64 reference of FlowNet2's correlation class, forward and backward, in torch on any device.

The class is MULTIPLY, kernel_size 1, stride_1 1, pad = max_displacement (md), md % stride_2 == 0: the top has the bottoms'
H x W, and top channel t = i * D + j (D = 2 R + 1, R = md / stride_2) compares bottom 0 at pixel q with bottom 1 at q + disp(t),
disp(t) = ((i - R) * stride_2, (j - R) * stride_2), zero outside the image (correlation_layer.cu, CorrelateData and its two
backward kernels).  Each operation is a shift-and-sum over the displacement grid:

    forward      out[:, t]  = sum_c a * shift(b, disp t) / C
    d bottom 0   d0         = sum_t td[:, t] * shift(b, disp t) / C
    d bottom 1   d1         = sum_t shift^-1(td[:, t] * a, disp t) / C

Every function also returns the same operation applied to the absolute values of its inputs (`absref`): the sum of the
magnitudes of the products, which the error bounds of the kernels are stated against.  A NaN input propagates exactly where
it meets a product (zero fill outside the image is 0, not NaN).  tests/test_corr_ref_cpu.py pins this module to the oracle.
"""
import torch


def radius(md, s2):
    assert md % s2 == 0, "the FlowNet2 class needs md % stride_2 == 0"
    return md // s2


def displacements(md, s2):
    """[(dy, dx)] in top-channel order."""
    R = radius(md, s2)
    D = 2 * R + 1
    return [((t // D - R) * s2, (t % D - R) * s2) for t in range(D * D)]


def _pad(x, md):
    return torch.nn.functional.pad(x, (md, md, md, md))


def _fwd(a, b, md, s2):
    N, C, H, W = a.shape
    bp = _pad(b, md)
    disp = displacements(md, s2)
    out = torch.empty((N, len(disp), H, W), dtype=torch.float64, device=a.device)
    for t, (dy, dx) in enumerate(disp):
        out[:, t] = (a * bp[:, :, md + dy:md + dy + H, md + dx:md + dx + W]).sum(1)
    return out / C


def _bwd0(b, td, md, s2):
    N, C, H, W = b.shape
    bp = _pad(b, md)
    d0 = torch.zeros((N, C, H, W), dtype=torch.float64, device=b.device)
    for t, (dy, dx) in enumerate(displacements(md, s2)):
        d0 += td[:, t:t + 1] * bp[:, :, md + dy:md + dy + H, md + dx:md + dx + W]
    return d0 / C


def _bwd1(a, td, md, s2):
    N, C, H, W = a.shape
    acc = torch.zeros((N, C, H + 2 * md, W + 2 * md), dtype=torch.float64, device=a.device)
    for t, (dy, dx) in enumerate(displacements(md, s2)):
        acc[:, :, md + dy:md + dy + H, md + dx:md + dx + W] += td[:, t:t + 1] * a
    return acc[:, :, md:md + H, md:md + W] / C


def _f64(x):
    return torch.as_tensor(x).to(torch.float64)


def forward(a, b, md, s2):
    """a, b: (N, C, H, W) -> (out, absref), both float64 (N, D*D, H, W) on a's device."""
    a, b = _f64(a), _f64(b).to(_f64(a).device)
    return _fwd(a, b, md, s2), _fwd(a.abs(), b.abs(), md, s2)


def backward(a, b, td, md, s2):
    """a, b: (N, C, H, W), td: (N, D*D, H, W) -> (d0, d1, absref0, absref1), float64 on a's device."""
    a = _f64(a)
    b, td = _f64(b).to(a.device), _f64(td).to(a.device)
    return (_bwd0(b, td, md, s2), _bwd1(a, td, md, s2), _bwd0(b.abs(), td.abs(), md, s2), _bwd1(a.abs(), td.abs(), md, s2))


def gradients(a, b, td, md, s2):
    """The bottom gradients of `backward` without their absrefs: -> (d0, d1), float64 on a's device."""
    a = _f64(a)
    b, td = _f64(b).to(a.device), _f64(td).to(a.device)
    return _bwd0(b, td, md, s2), _bwd1(a, td, md, s2)
