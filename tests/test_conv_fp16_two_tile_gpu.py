"""The FP16 route's two-tile K step (NT = 128, plain K blocks) on the device.

* The forward reads W_A and W_B only: with every W_C tile of the packed weights overwritten by NaN, the route cases of
  tests/test_conv_fp16_split_gpu.py give the same output, bit for bit, as with the intact packing.
* Low halves below FP16's normal range: pixels whose channels spread over 2^-30 .. 1, so that many lo'' = fp16(a 2^-e - hi) are
  subnormal, against the float64 reference within 1e-6 of the sum of |a w| per output.
"""
import numpy as np
import pytest

from tests.conv_ref import case, reference
from tests.test_conv_fp16_split_gpu import ROUTE_CASES, TOL, _scaled_draw
from tests.test_conv_tc_routes_gpu import out_hw, plan_of, prepare, sample, weight_shape

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

F16_NAN = 0x7E00


@pytest.mark.parametrize("c", ROUTE_CASES, ids=lambda c: c.name)
def test_forward_does_not_read_wc(c):
    x, w, b = _scaled_draw(c, 31)
    r = prepare(c, x, w, b)
    r.go()
    intact = r.wide.clone()
    packed = r.go.keep[1]
    # behind the SIMT copy: [tap][channel block][W_A | W_B | W_C][Co][32 halves], then the 4 floats of the largest |w|
    kh, kw = c.k
    blocks = kh * kw * ((c.Ci + 31) // 32)
    simt = kh * kw * c.Ci * c.Co
    tiles = packed[simt:simt + blocks * 3 * c.Co * 16].view(torch.int16).view(blocks, 3, c.Co * 32)
    assert packed.numel() == simt + blocks * 48 * c.Co + 4
    tiles[:, 2] = F16_NAN
    r.go()
    torch.cuda.synchronize()
    assert bool(torch.isfinite(intact[:, 16:16 + c.Co]).all())
    assert torch.equal(intact.view(torch.int32), r.wide.view(torch.int32))


SUBNORMAL_CASES = [
    case("f16_lo_subnormal_conv", 2, 96, 20, 30, 128, 3, 1, 1),
    case("f16_lo_subnormal_conv_s2", 1, 256, 24, 40, 128, 3, 2, 1, bias=False),
    case("f16_lo_subnormal_d_k4", 1, 256, 13, 19, 128, 4, 2, 1, True),
]


@pytest.mark.parametrize("c", SUBNORMAL_CASES, ids=lambda c: c.name)
def test_low_halves_below_normal_range(c):
    pl = plan_of(c)
    assert pl[0] == 128 and pl[3] == 0
    g = torch.Generator(device="cuda").manual_seed(37)
    x = torch.randn((c.N, c.Ci, c.H, c.W), generator=g, device="cuda")
    x = x * 2.0 ** (-30 * torch.rand(x.shape, generator=g, device="cuda"))          # each pixel's channels: 2^-30 .. 1
    ws = weight_shape(c)
    w = torch.randn(ws, generator=g, device="cuda") * np.sqrt(2.0 / (ws[1] * ws[2] * ws[3]))
    b = torch.randn(c.Co, generator=g, device="cuda") if c.bias else None
    r = prepare(c, x, w, b)
    r.go()
    ho, wo = out_hw(c)
    n, oy, ox = sample(c, pl, ho, wo, 5)
    want = reference(c, x.double(), w.double(), None, n, oy, ox)
    mag = reference(c, x.double().abs(), w.double().abs(), None, n, oy, ox)
    got = r.out[n, :, oy, ox].double()
    if b is not None:                                 # bias and leaky ReLU (slope 0.1) after the sum, as prepare() asks
        z = want + b.double()
        want, mag = torch.where(z > 0, z, 0.1 * z), mag + b.double().abs()
    assert bool(torch.isfinite(got).all())
    err = ((got - want).abs() / mag.clamp_min(1e-300))
    assert float(err.max()) <= TOL, float(err.max())
