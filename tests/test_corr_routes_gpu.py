"""Every route of the Correlation and Correlation1D layers (fn2_corr.cu, fn2_corr_fast.cu, fn2_corr_bwd.cu, and the
tensor-core correlation of fn2_conv_tc.cu) against the float64-accumulated oracle.

Each case is built to reach one route, and `test_corr_route_kernel` checks, with the CUDA profiler, that it runs that route's
kernel.  Tolerances: 1e-5 of the output scale for the forward and the fast backward, 2e-5 for the tiled backward.
"""
import ctypes as C
import zlib

import numpy as np
import pytest

from oracle import oracle as O
from tests.util import maxabs, rng

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def ops(fn2):
    from flownet2_b200 import ops as _ops
    return _ops


def dev(a, channels_last=False):
    t = torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    return t.contiguous(memory_format=torch.channels_last) if channels_last else t


def host(t):
    return t.contiguous().cpu().numpy()


# the kernels each route launches, as the profiler names them
FWD_KERNEL = {"tc": "conv_tc_kernel<128, 3>", "fast10": "corr_fast_kernel<10>", "fast4": "corr_fast_kernel<4>",
              "generic": "corr_generic_kernel(", "generic1d": "corr_generic_kernel("}
BWD_KERNELS = {"fast": ["corr_bwd_fast_kernel<1>", "corr_bwd_fast_kernel<-1>", "corr_shift_kernel("],
               "tiled": ["corr_apply_kernel<0>", "corr_apply_kernel<1>"]}

FWD_CASES = [
    # route, (N, C, H, W, pad, k, md, s1, s2, single_direction or None for the 2-D layer, type), channels_last, workspace
    ("tc", (2, 64, 24, 40, 20, 1, 20, 1, 2, None, 0), True, True),
    ("tc", (1, 32, 19, 27, 10, 1, 10, 1, 1, None, 0), True, True),
    ("fast10", (2, 64, 24, 40, 20, 1, 20, 1, 2, None, 0), False, True),      # NCHW
    ("fast10", (1, 40, 21, 37, 20, 1, 20, 1, 2, None, 0), True, True),       # C % 32 != 0
    ("fast4", (2, 32, 12, 14, 4, 1, 4, 1, 1, None, 0), False, True),
    ("fast4", (2, 32, 13, 17, 8, 1, 8, 1, 2, None, 0), True, True),
    ("generic", (2, 16, 11, 13, 3, 1, 3, 1, 1, None, 0), False, True),      # R = 3, pad = md
    ("generic", (1, 8, 13, 15, 4, 3, 3, 1, 1, None, 0), False, True),       # k = 3
    ("generic", (1, 8, 16, 18, 4, 3, 2, 2, 2, None, 0), True, True),        # stride_1 = 2
    ("generic", (1, 8, 12, 12, 2, 1, 4, 1, 2, None, 0), False, True),       # pad < md
    ("generic", (2, 16, 9, 10, 3, 1, 3, 1, 1, None, 1), True, True),        # SUBTRACT
    ("generic", (1, 256, 10, 12, 20, 1, 20, 1, 2, None, 0), True, False),   # FlowNet2-C's layer without workspace
    ("generic1d", (2, 16, 7, 19, 8, 1, 8, 1, 2, 0, 0), False, False),       # both directions
    ("generic1d", (2, 16, 7, 19, 8, 1, 8, 1, 2, -1, 0), True, False),       # left
    ("generic1d", (2, 16, 7, 19, 8, 1, 8, 1, 2, 1, 0), False, False),       # right
    ("generic1d", (1, 8, 11, 21, 4, 3, 4, 2, 1, 0, 0), False, False),       # k = 3, stride_1 = 2
    ("generic1d", (2, 8, 6, 15, 3, 1, 3, 1, 1, 0, 1), False, False),        # SUBTRACT
]
FWD_PARAMS = [pytest.param(route, case, cl, ws, id="%s-%s-%s%s" % (route, "nhwc" if cl else "nchw", "-".join(map(str, case)),
                                                                   "" if ws else "-nows"))
              for route, case, cl, ws in FWD_CASES]

BWD_CASES = [
    # route, (N, C, H, W, pad, k, md, s1, s2, single_direction or None, type), channels_last, extra kernels
    ("fast", (1, 32, 19, 45, 10, 1, 10, 1, 1, None, 0), True, []),
    ("fast", (2, 64, 24, 40, 20, 1, 20, 1, 2, None, 0), True, []),
    ("tiled", (1, 32, 19, 45, 10, 1, 10, 1, 1, None, 0), False, []),                           # identity G, NCHW
    ("tiled", (1, 4, 11, 12, 4, 3, 2, 2, 2, None, 0), False, ["corr_patchsum_kernel("]),       # patch sum
    ("tiled", (2, 16, 9, 10, 3, 1, 3, 1, 1, None, 1), False, ["corr_sign_kernel("]),           # SUBTRACT, identity G
    ("tiled", (1, 8, 12, 13, 2, 3, 2, 1, 2, None, 1), True,
     ["corr_sign_kernel(", "corr_patchsum_kernel("]),                                          # SUBTRACT, patch sum
    ("tiled", (2, 16, 7, 19, 8, 1, 8, 1, 2, 0, 0), False, []),                                 # 1-D, identity G
    ("tiled", (1, 8, 11, 21, 4, 3, 4, 2, 1, -1, 1), False, ["corr_sign_kernel(", "corr_patchsum_kernel("]),  # 1-D
]
BWD_PARAMS = [pytest.param(route, case, cl, extra, id="%s-%s-%s" % (route, "nhwc" if cl else "nchw", "-".join(map(str, case))))
              for route, case, cl, extra in BWD_CASES]


def bottoms(case):
    N, Cc, H, W = case[:4]
    r = rng(zlib.crc32(repr(case).encode()))
    return r.standard_normal((N, Cc, H, W)).astype(np.float32), r.standard_normal((N, Cc, H, W)).astype(np.float32), r


def forward(ops, case, a, b, cl, ws):
    N, Cc, H, W, pad, k, md, s1, s2, sd, typ = case
    if sd is None:
        return ops.correlation(dev(a, cl), dev(b, cl), pad, k, md, s1, s2, typ, use_workspace=ws)
    return ops.correlation1d(dev(a, cl), dev(b, cl), pad, k, md, s1, s2, sd, typ)


def kernels(fn):
    """Names of the kernels fn launches.  Now and then the profiler records no device activity at all for a short run; such
    an empty capture is taken again."""
    for _ in range(3):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if names:
            return names
    return names


@pytest.mark.parametrize("route,case,cl,ws", FWD_PARAMS)
def test_corr_route(ops, route, case, cl, ws):
    N, Cc, H, W, pad, k, md, s1, s2, sd, typ = case
    a, b, _ = bottoms(case)
    if sd is None:
        want = O.correlation_fwd(a, b, pad, k, md, s1, s2, typ, exact_order=False)
    else:
        want = O.correlation1d_fwd(a, b, pad, k, md, s1, s2, sd, typ)
    got = host(forward(ops, case, a, b, cl, ws))
    assert maxabs(got, want) <= 1e-5 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("route,case,cl,ws", FWD_PARAMS)
def test_corr_route_kernel(ops, route, case, cl, ws):
    """The case runs the kernel of its route and no other forward route's."""
    a, b, _ = bottoms(case)
    names = kernels(lambda: forward(ops, case, a, b, cl, ws))
    for r, kname in FWD_KERNEL.items():
        assert any(kname in n for n in names) == (kname == FWD_KERNEL[route]), (route, sorted(names))


@pytest.mark.parametrize("route,case,cl,extra", BWD_PARAMS)
def test_corr_backward_route(ops, route, case, cl, extra):
    N, Cc, H, W, pad, k, md, s1, s2, sd, typ = case
    a, b, r = bottoms(case)
    if sd is None:
        tc, th, tw = ops.correlation_shape(H, W, pad, k, md, s1, s2)
    else:
        tc, th, tw = ops.correlation1d_shape(H, W, pad, k, md, s1, s2, sd)
    td = r.standard_normal((N, tc, th, tw)).astype(np.float32)
    if sd is None and typ == 0:
        w0, w1 = O.correlation_bwd(a, b, td, pad, k, md, s1, s2)
    else:
        w0, w1 = O.correlation_bwd_ex(a, b, td, pad, k, md, s1, s2, typ, sd is not None, sd or 0)
    da, db, dtd = dev(a, cl), dev(b, cl), dev(td, cl)
    if sd is None:
        run = lambda: ops.correlation_backward(da, db, dtd, pad, k, md, s1, s2, typ)          # noqa: E731
    else:
        run = lambda: ops.correlation1d_backward(da, db, dtd, pad, k, md, s1, s2, sd, typ)    # noqa: E731
    g0, g1 = run()
    tol = 1e-5 if route == "fast" else 2e-5
    assert maxabs(host(g0), w0) <= tol * max(1.0, np.abs(w0).max())
    assert maxabs(host(g1), w1) <= tol * max(1.0, np.abs(w1).max())
    names = kernels(run)
    for r_, knames in BWD_KERNELS.items():
        for kname in knames:
            assert any(kname in n for n in names) == (r_ == route), (route, sorted(names))
    for kname in ("corr_patchsum_kernel(", "corr_sign_kernel("):
        assert any(kname in n for n in names) == (kname in extra), (route, sorted(names))


def test_corr_forward_workspace_too_small(ops, fn2):
    """A non-null workspace smaller than the query's need is an error, not a silent fall-back to another route."""
    N, Cc, H, W = 1, 64, 16, 20
    a = dev(np.ones((N, Cc, H, W), np.float32), True)
    out = torch.empty((N, 441, H, W), device="cuda").contiguous(memory_format=torch.channels_last)
    need = C.c_size_t()
    assert fn2.lib().fn2_correlation_workspace_bytes(N, Cc, H, W, 20, 1, 20, 1, 2, 0, C.byref(need)) == 0
    assert need.value > 0
    ws = torch.zeros(need.value // 4, dtype=torch.uint8, device="cuda")
    d, dt = ops.desc(a), ops.desc(out)
    rc = fn2.lib().fn2_correlation_forward(C.byref(d), C.byref(d), C.byref(dt), 20, 1, 20, 1, 2, 0, C.c_void_p(ws.data_ptr()),
                                           C.c_size_t(ws.numel()), None)
    assert rc == -5                                                         # FN2_ERR_WORKSPACE
