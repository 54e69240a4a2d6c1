"""The FP16 operand route of the per-tap tensor-core engine (NT = 128, plain K blocks) on the device.

* The packed weights of small layers, read back, against the numpy restatement of tests/test_conv_fp16_split_cpu.py bit for
  bit: the three FP16 tiles of every K block in K-slot order, and the bits of the layer's largest |w| behind them.
* Every NT = 128 route -- convolution, every deconvolution parity class, both K-split regimes, channel tails -- against the
  float64 reference on inputs where the scale matters: 8 x 8 pixel blocks whose channels lie 1e-20 .. 1e20 apart in magnitude,
  weights up to 1e4.  Per output, within 1e-6 of the sum of |a w| over its reduction (an unscaled FP16 split would overflow or
  flush whole blocks).
* The mean signed error of same-sign sums at two FlowNet2 shapes stays within 4e-8: TRUNC_LOSS_PER_MMA_F16's compensation
  is in place.
"""
import ctypes as C
import math

import numpy as np
import pytest

from tests.conv_ref import _check, _lib, case, reference
from tests.test_conv_fp16_split_cpu import channel, pack_f16, wexp
from tests.test_conv_tc_routes_gpu import out_hw, plan_of, prepare, sample, shrink, weight_shape

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ROUTE_CASES = [
    case("f16_conv", 2, 96, 20, 30, 128, 3, 1, 1),                        # 3 K blocks, tw 32
    case("f16_conv_s2_ci473", 1, 473, 30, 40, 256, 3, 2, 1, bias=False),    # Ci tail 473, two Co tiles, stride 2
    case("f16_split_all", 1, 512, 7, 16, 128, 3, 1, 1),                     # every tile split, 8 ranges
    case("f16_split_tail", 1, 473, 150, 128, 128, 3, 1, 1, bias=False),     # the last wave's tiles split
    case("f16_ci40", 1, 40, 33, 150, 128, 3, 1, 1),                         # Ci tail of 8, two tile columns
    case("f16_d_k3_odd", 1, 1024, 4, 6, 128, 3, 2, 1, True),                # classes of 4 / 2 / 2 / 1 taps, split
    case("f16_d_k4", 1, 256, 13, 19, 256, 4, 2, 1, True),                   # four classes of 4 taps
    case("f16_d_k2", 2, 64, 15, 17, 128, 2, 2, 0, True),                    # one tap per class
    case("f16_d_k5", 1, 96, 11, 14, 128, 5, 2, 2, True),                    # 9 / 6 / 6 / 4 taps
    case("f16_d_s1", 1, 64, 20, 30, 128, 3, 1, 1, True),                    # stride-1 deconvolution: one class
]
TOL = 1e-6


def test_route_cases_are_f16_plans():
    """Every case runs the per-tap engine at NT = 128 in plain mode; both K-split regimes and several parity classes appear."""
    pls = [plan_of(c) for c in ROUTE_CASES]
    assert all(pl[0] == 128 and pl[3] == 0 for pl in pls)
    assert any(pl[5] > 1 and pl[4] == 0 for pl in pls) and any(pl[5] > 1 and pl[4] > 0 for pl in pls)


def _packed(c, w):
    from flownet2_b200 import fn2_conv_desc
    (kh, kw), (sh, sw), (ph, pw) = c.k, c.s, c.p
    d = fn2_conv_desc(c.Ci, c.Co, kh, kw, sh, sw, ph, pw, int(c.deconv), 1, 1, 0.1, 2, 0)
    cis = (c.Ci + 31) // 32 * 32
    nf = C.c_size_t()
    _check(_lib().fn2_conv_packed_floats(C.byref(d), cis, C.byref(nf)))
    packed = torch.full((nf.value,), float("nan"), device="cuda")
    _check(_lib().fn2_conv_pack_weights(C.byref(d), cis, w.data_ptr(), packed.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    simt = kh * kw * c.Ci * c.Co
    return packed[simt:].cpu().numpy()


@pytest.mark.parametrize("c", [case("pk_conv", 1, 40, 8, 8, 128, 3, 1, 1), case("pk_deconv", 1, 64, 8, 8, 256, 4, 2, 1, True)],
                         ids=lambda c: c.name)
@pytest.mark.parametrize("scale", [1e-3, 1e4])
def test_packing_bit_for_bit(c, scale):
    r = np.random.default_rng(5)
    w = (r.standard_normal(weight_shape(c)) * scale * 10.0 ** r.uniform(-8, 0, weight_shape(c))).astype(np.float32)
    got = _packed(c, torch.from_numpy(w).cuda())
    kh, kw = c.k
    cb = (c.Ci + 31) // 32
    tiles = 48 * kh * kw * c.Co * cb
    assert got.size == tiles + 4
    assert got[tiles:tiles + 1].view(np.uint32)[0] == np.abs(w).max().view(np.uint32)
    f = wexp(np.abs(w).max())
    # [tap][channel block][W_A | W_B | W_C][Co][32 slots]; Caffe layout (Co, Ci, kh, kw), a deconvolution's (Ci, Co, kh, kw)
    wt = w.transpose(2, 3, 1, 0) if c.deconv else w.transpose(2, 3, 0, 1)           # (kh, kw, Co, Ci)
    wt = np.concatenate([wt, np.zeros(wt.shape[:3] + (cb * 32 - c.Ci,), np.float32)], 3).reshape(kh * kw, c.Co, cb, 32)
    wt = wt[..., [channel(s) for s in range(32)]].transpose(0, 2, 1, 3)                # (tap, block, Co, slot)
    want = np.stack(pack_f16(wt, f), 2)                                                # (tap, block, 3, Co, slot)
    assert np.array_equal(got[:tiles].view(np.uint16), want.reshape(-1).view(np.uint16))


def _scaled_draw(c, seed):
    """bottom with one magnitude 10^u, u in [-20, 20], per 8 x 8 pixel block (N(0,1) channels), weights N(0,1) 10^[-4, 4]"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((c.N, c.Ci, c.H, c.W), generator=g, device="cuda")
    u = torch.rand((c.N, 1, (c.H + 7) // 8, (c.W + 7) // 8), generator=g, device="cuda") * 40 - 20
    x = x * (10.0 ** u).repeat_interleave(8, 2).repeat_interleave(8, 3)[:, :, :c.H, :c.W]
    ws = weight_shape(c)
    w = torch.randn(ws, generator=g, device="cuda") * 10.0 ** (torch.rand(ws, generator=g, device="cuda") * 8 - 4)
    b = torch.randn(c.Co, generator=g, device="cuda") if c.bias else None
    return x, w, b


@pytest.mark.parametrize("c", ROUTE_CASES, ids=lambda c: c.name)
def test_f16_route_scaled(c):
    x, w, b = _scaled_draw(c, 17)
    r = prepare(c, x, w, b)
    r.go()
    ho, wo = out_hw(c)
    n, oy, ox = sample(c, plan_of(c), ho, wo, 3)
    want = reference(c, x.double(), w.double(), None, n, oy, ox)
    mag = reference(c, x.double().abs(), w.double().abs(), None, n, oy, ox)
    got = r.out[n, :, oy, ox].double()
    if b is not None:                                 # bias and leaky ReLU (slope 0.1) after the sum, as prepare() asks
        z = want + b.double()
        want, mag = torch.where(z > 0, z, 0.1 * z), mag + b.double().abs()
    assert bool(torch.isfinite(got).all())
    err = ((got - want).abs() / mag.clamp_min(1e-300))
    assert float(err.max()) <= TOL, float(err.max())


@pytest.mark.parametrize("c", [case("deploy-net1_conv3_1", 4, 473, 56, 128, 256, 3, 1, 1, bias=False, layout="pad"),
                               case("deploy-net1_deconv4", 4, 1026, 14, 32, 256, 4, 2, 1, True, bias=False, layout="pad")],
                         ids=lambda c: c.name)
def test_f16_shrink(c):
    """Same-sign sums (post-ReLU bottom, positive weights): mean signed error within 4e-8 of the mean |output|, the
    SHRINK_BOUND of these layers in tests/test_conv_tc_routes_gpu.py.  Without the compensation (TRUNC_LOSS_PER_MMA_F16 = 0)
    these cases shrink by 6.6e-8 on an H100 80GB HBM3 (700 W)."""
    g = torch.Generator(device="cuda").manual_seed(23)
    x = torch.randn((c.N, c.Ci, c.H, c.W), generator=g, device="cuda").clamp_min(0)
    ws = weight_shape(c)
    w = (torch.randn(ws, generator=g, device="cuda") * math.sqrt(2.0 / (ws[1] * ws[2] * ws[3]))).abs()
    r = prepare(c, x, w, None)
    r.go()
    ho, wo = out_hw(c)
    n, oy, ox = sample(c, plan_of(c), ho, wo, 3)
    want = reference(c, x, w, None, n, oy, ox)
    sh = shrink(r.out[n, :, oy, ox].double(), want)
    print("%s shrink %.3g" % (c.name, sh))
    assert abs(sh) <= 4e-8, sh
