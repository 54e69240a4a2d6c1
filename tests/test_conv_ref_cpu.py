"""tests/conv_ref.py on the CPU: the float64 reference against the oracle, the enumeration of the layers the default engine runs
on SIMT, and the concat offsets the nets' zero-copy children get."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import conv_ref as R
from tests.util import net_walk

torch = pytest.importorskip("torch")

# (N, Ci, H, W, Co, k, stride, pad, deconv): stride 1 and 2, kernels 1 x 1, 3 x 3 and 4 x 4, odd maps
CASES = [
    (2, 5, 9, 11, 3, 3, 1, 1, False), (1, 4, 10, 13, 2, 3, 2, 1, False), (2, 6, 7, 9, 4, 1, 1, 0, False),
    (1, 3, 11, 10, 2, 1, 2, 0, False), (1, 2, 12, 15, 2, 4, 2, 1, False), (2, 3, 5, 7, 2, 4, 2, 1, True),
    (1, 4, 6, 5, 3, 3, 1, 1, True), (1, 2, 4, 6, 2, 3, 2, 1, True), (1, 3, 5, 4, 2, 1, 2, 0, True),
    (1, 2, 6, 7, 3, 4, 1, 2, True),
]
IDS = ["%s_k%d_s%d_p%d" % ("deconv" if c[8] else "conv", c[5], c[6], c[7]) for c in CASES]


def _every_pixel(shape):
    return torch.ones(shape, dtype=torch.bool).nonzero().unbind(1)


def _oracle(x, w, b, c):
    N, Ci, H, W, Co, k, s, p, deconv = c
    return (O.deconv_fwd if deconv else O.conv_fwd)(x, w, b, s, p, f64acc=True)


def _rows(a):
    return a.transpose(0, 2, 3, 1).reshape(-1, a.shape[1])


@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_ref_at_equals_oracle_exactly_on_integers(c):
    """Small integers make every sum exact in float32: ref_at and the oracle agree bit for bit."""
    N, Ci, H, W, Co, k, s, p, deconv = c
    r = np.random.default_rng(11)
    x = r.integers(-8, 9, (N, Ci, H, W)).astype(np.float32)
    w = r.integers(-8, 9, (Ci, Co, k, k) if deconv else (Co, Ci, k, k)).astype(np.float32)
    want = _oracle(x, w, None, c)
    n, oy, ox = _every_pixel(want.shape[:1] + want.shape[2:])
    got = R.ref_at(torch.from_numpy(x), torch.from_numpy(w), deconv, (s, s), (p, p), n, oy, ox).numpy()
    assert np.array_equal(got, _rows(want).astype(np.float64))


@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_reference_matches_oracle(c):
    """`reference` (bias and leaky ReLU) on N(0, 1) data agrees with the oracle to within its float32 steps: the rounding of the
    float64 sum, and on the negative side the float32 slope 0.1f (1.5e-8 from 0.1) and the rounding of the product."""
    N, Ci, H, W, Co, k, s, p, deconv = c
    r = np.random.default_rng(12)
    x = r.standard_normal((N, Ci, H, W)).astype(np.float32)
    w = r.standard_normal((Ci, Co, k, k) if deconv else (Co, Ci, k, k)).astype(np.float32)
    b = r.standard_normal(Co).astype(np.float32)
    want = O.relu(_oracle(x, w, b, c), 0.1)
    cc = R.case("c", N, Ci, H, W, Co, k, s, p, deconv)
    n, oy, ox = _every_pixel(want.shape[:1] + want.shape[2:])
    want = _rows(want)
    got = R.reference(cc, torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), n, oy, ox).numpy()
    assert (np.abs(got - want) <= 3 * 2.0 ** -24 * np.abs(got)).all()


@pytest.mark.parametrize("c", [CASES[0], CASES[1], CASES[4], CASES[5], (1, 3, 9, 8, 2, 3, 2, 1, False)],
                         ids=["conv_s1", "conv_s2", "conv_k4_s2", "upsampler", "conv_s2_outpad"])
def test_adjoint_reference_is_the_data_gradient(fn2, c):
    """The reference of a data-gradient operator (adjoint) equals the oracle's bottom gradient of its layer, and the operator's
    output has the bottom's shape (out_pad where the layer's last window does not reach the bottom's edge)."""
    N, Ci, H, W, Co, k, s, p, deconv = c
    r = np.random.default_rng(13)
    x = r.integers(-4, 5, (N, Ci, H, W)).astype(np.float32)
    w = r.integers(-4, 5, (Ci, Co, k, k) if deconv else (Co, Ci, k, k)).astype(np.float32)
    top = _oracle(x, w, None, c)
    dy = r.integers(-4, 5, top.shape).astype(np.float32)
    a = R.adjoint("a", N, Ci, H, W, Co, k, s, p, deconv)
    assert (a.N, a.Ci, a.H, a.W) == dy.shape and a.fwd[9] == Ci
    n, oy, ox = _every_pixel((N, H, W))
    got = R.reference(a, torch.from_numpy(dy), torch.from_numpy(w), None, n, oy, ox).numpy()
    want = O.conv_bwd(x, w, dy, s, p, deconv)[0]
    assert np.array_equal(got, _rows(want).astype(np.float64))


@pytest.mark.parametrize("c", [CASES[1], CASES[4], CASES[5], CASES[7], CASES[9]], ids=lambda c: "x".join(map(str, c[5:8])))
def test_taps_at_counts_the_taps_inside(c):
    N, Ci, H, W, Co, k, s, p, deconv = c
    cc = R.case("c", N, Ci, H, W, Co, k, s, p, deconv)
    ho, wo = (s * (H - 1) + k - 2 * p, s * (W - 1) + k - 2 * p) if deconv else ((H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1)
    n, oy, ox = _every_pixel((N, ho, wo))
    got = R.taps_at(cc, n, oy, ox).numpy()
    want = []
    for y, x_ in zip(oy.tolist(), ox.tolist()):
        t = 0
        for ky in range(k):
            for kx in range(k):
                if deconv:
                    ty, tx = y + p - ky, x_ + p - kx
                    t += ty % s == 0 and tx % s == 0 and 0 <= ty // s < H and 0 <= tx // s < W
                else:
                    t += 0 <= y * s - p + ky < H and 0 <= x_ * s - p + kx < W
        want.append(t)
    assert np.array_equal(got, np.array(want, np.float64))


def _text(kind, model):
    from flownet2_b200 import fill_template, fill_train_template, model_template, train_template
    if kind == "deploy":
        return fill_template(model_template(model), 1024, 436)
    return fill_train_template(train_template(model), 448, 320, 512, 384, 1)


TEMPLATES = [("deploy", m) for m in R.DEPLOY_MODELS] + [("train", m) for m in R.TRAIN_MODELS]


@pytest.mark.parametrize("kind,model", TEMPLATES, ids=["%s-%s" % t for t in TEMPLATES])
def test_enumeration_finds_every_predictor_and_upsampler(fn2, kind, model):
    """The layers of a template the default engine runs on SIMT are exactly its predict_flow and upsample_flow layers (and
    FlowNet2's scale_conv1); in a training graph every upsampler's data-gradient operator runs there too, reading its top diff
    as the concat child the upsampler writes."""
    text = _text(kind, model)
    convs = [c[0] for c in net_walk(text)[0]]
    flow = {n for n in convs if "predict_flow" in n or "upsample_flow" in n}
    assert flow
    layers = R.net_simt_layers(text, 4, "", kind == "train")
    fwd = {L.case.name for L in layers if not L.case.fwd}
    assert fwd == flow | ({"scale_conv1"} if "scale_conv1" in convs else set()), sorted(fwd ^ flow)
    for L in layers:
        assert not L.case.name.startswith("dgrad-") or (L.case.fwd and L.case.fwd[5] and isinstance(L.bottom, tuple))
        if "upsample_flow" in L.case.name and not L.case.fwd:
            assert L.top is not None, L.case.name
    dgrad = {L.case.name[len("dgrad-"):] for L in layers if L.case.fwd}
    assert dgrad == ({n for n in flow if "upsample_flow" in n} if kind == "train" else set())


def test_concat_offsets():
    """upsampled_flow6_to_5 is channels [1024, 1026) of concat5 in FlowNet2-C's training graph (after conv5_1 and deconv5),
    at concat5's pixel stride of 1056; an upsampler's top in the fusion network is a child too."""
    text = _text("train", "FlowNet2-C")
    _, _, concats, io = net_walk(text)
    assert io["upsample_flow6to5"][1] == ["upsampled_flow6_to_5"]
    assert concats["upsampled_flow6_to_5"] == ("concat5", 1024, 1026)
    alias = R.aliased(text)
    assert alias["upsampled_flow6_to_5"] == (1024, 1026) and R.cstride(1026) == 1056
    assert alias["upsampled_flow3_to_2"] == (192, 194) and R.cstride(194) == 224
    off, stride, fill, guard = R.concat_child(*alias["upsampled_flow6_to_5"])
    assert (off, stride(2), fill, guard) == (1024, 1056, "junk", True)
    deploy = _text("deploy", "FlowNet2")
    tops = {net_walk(deploy)[3]["fuse_upsample_flow1to0"][1][0]}
    assert {R.aliased(deploy).get(t) for t in tops} == {(80, 82)}
