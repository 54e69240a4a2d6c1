"""The float64 Net::Backward of tests/net_grad64.py against the CPU oracle (OracleNet / PrunedOracleNet with float64
accumulation): FlowNet2-C's deploy graph under seeds on its five flow predictions, the pruned FlowNet2-CS and FlowNet2-SD
training graphs under their losses, and each restated operator on small random cases.

The oracle rounds every layer's result to float32, so every gradient must agree to within that rounding, compounded over the
layers it passed through: TOL of each tensor's largest entry.  The reference runs here in torch on the CPU; on the GPU
(tests/test_net_grad_train_shapes_gpu.py) the same code runs on the device.
"""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from oracle.net import OracleNet, get, getall
from tests.net_grad64 import NetGrad64, conv_backward64, correlation_backward64, l1loss_bwd64, l1loss_fwd64
from tests.stack_oracle import PrunedOracleNet
from tests.util import rng, smooth_images

TOL = 4e-7
SEEDS = ["predict_flow6", "predict_flow5", "predict_flow4", "predict_flow3", "predict_flow2"]


def rel(got, want):
    got, want = np.asarray(torch.as_tensor(got).double()), np.asarray(want, np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    return float(np.abs(got - want).max()) / max(float(np.abs(want).max()), 1e-30)


def t64(a):
    return torch.from_numpy(np.ascontiguousarray(a)).double()


def compare(D, P, oD, oP, blobs=()):
    """Every parameter gradient of the oracle, and the diffs of `blobs`, within TOL; -> number of tensors compared."""
    assert sorted(P) == sorted(oP)
    worst = {}
    for name, grads in oP.items():
        assert len(P[name]) == len(grads), name
        for i, g in enumerate(grads):
            worst["%s[%d]" % (name, i)] = rel(P[name][i].reshape(g.shape), g)
    for b in blobs:
        worst[b] = rel(D[b], oD[b])
    bad = {k: v for k, v in worst.items() if v > TOL}
    assert not bad, bad
    return len(worst)


# ---- whole graphs ------------------------------------------------------------------------------------------------------------
def test_flownet_c_deploy_graph_matches_oracle(fn2):
    """test_flownet_c_backward_matches_oracle's case: FlowNet2-C at 192 x 100, batch 1, seeds on the five predictions."""
    w, h = 192, 100
    proto = fn2.fill_template(fn2.model_template("FlowNet2-C"), w, h)
    onet = OracleNet(proto, None, batch=1, f64acc=True, synth_seed=7)
    img0, img1 = smooth_images(rng(7), 1, h, w)
    B = onet.forward(img0=img0, img1=img1)
    r = rng(8)
    seeds = {s: r.standard_normal(B[s].shape).astype(np.float32) for s in SEEDS}
    oD, oP = onet.backward(**seeds)
    net = NetGrad64(proto, {k: [t64(a) for a in v] for k, v in onet.weights.items()})
    D, P = net.backward({k: t64(v) for k, v in B.items()}, {k: t64(v) for k, v in seeds.items()})
    blobs = ["conv1a", "conv1b", "conv2a", "conv2b", "conv3a", "conv3b", "corr", "conv_redir", "conv3_1", "deconv5", "conv6_1",
             "blob20", "concat2"]
    blobs = [b for b in blobs if b in oD]
    assert compare(D, P, oD, oP, blobs) >= 40 + 10
    # the layer-local forward of every convolution against the oracle's
    for l in onet.layers:
        if get(l, "type") in ("Convolution", "Deconvolution") and get(l, "name") in P:
            for t, y in net.conv_forward(get(l, "name"), {k: t64(v) for k, v in B.items()}).items():
                assert rel(y, B[t]) <= TOL, (get(l, "name"), t)


def _center_crop(x, ch, cw):
    H, W = x.shape[2:]
    y0, x0 = (H - ch) // 2, (W - cw) // 2
    return np.ascontiguousarray(x[:, :, y0:y0 + ch, x0:x0 + cw])


def oracle_train_forward(onet, inputs, cw, ch):
    """OracleNet's forward over a training graph.  The augmentation layers run forward only and are out of this test's reach:
    a centred crop without the random transform, and zero augmentation parameters, stand in for them."""
    B = dict(inputs)
    for l in onet.layers:
        typ, bots, tops = get(l, "type"), [B[b] for b in getall(l, "bottom")], getall(l, "top")
        if typ == "Input":
            continue
        if typ in ("DataAugmentation", "FlowAugmentation"):
            B[tops[0]] = _center_crop(bots[0], ch, cw)
            for t in tops[1:]:
                B[t] = np.zeros((bots[0].shape[0], 42, 1, 1), np.float32)
        elif typ == "GenerateAugmentationParameters":
            B[tops[0]] = np.zeros_like(bots[0])
        else:
            for t, v in zip(tops, onet.run_layer(l, bots)):
                B[t] = v
    onet.blobs = B
    return B


@pytest.mark.parametrize("stage", ["FlowNet2-CS", "FlowNet2-SD"])
def test_pruned_training_graph_matches_oracle(fn2, stage):
    """The stacked training graphs at the crop of tests/test_stack_train_gpu.py, batch 2: the losses, the trained parameter
    gradients, and every blob diff the two share."""
    cw, ch, dw, dh, batch = 192, 128, 224, 160, 2
    proto = fn2.fill_train_template(fn2.train_template(stage), cw, ch, dw, dh, batch)
    onet = PrunedOracleNet(proto, None, f64acc=True, synth_seed=11)
    img0, img1 = smooth_images(rng(12), batch, dh, dw)
    gt = (3 * rng(13).standard_normal((batch, 2, dh, dw))).astype(np.float32)
    gt[0, :, 60:75, 80:110] = np.nan                              # invalid ground truth
    B = oracle_train_forward(onet, {"img0": img0, "img1": img1, "flow_gt": gt}, cw, ch)
    oD, oP = onet.backward()
    net = NetGrad64(proto, {k: [t64(a) for a in v] for k, v in onet.weights.items()})
    blobs = {k: t64(v) for k, v in B.items()}
    D, P = net.backward(blobs)
    assert sorted(P) == sorted(net.trained()) and len(P) >= 20
    shared = [b for b in D if b in oD and not b.startswith("flow_loss") and not b.endswith("loss")]
    assert len(shared) >= 20
    compare(D, P, oD, oP, shared)
    for name in net.losses():
        l = net.by_name[name]
        want = float(B[getall(l, "top")[0]].reshape(-1)[0])
        assert abs(float(net.loss(name, blobs)) - want) <= TOL * abs(want), name


# ---- single operators on small random cases ----------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 32, 9, 13), (2, 64, 12, 7)])
@pytest.mark.parametrize("s2", [1, 2])
def test_correlation_backward(shape, s2):
    r = rng(sum(shape) + s2)
    a, b = (r.standard_normal(shape).astype(np.float32) for _ in range(2))
    md = 4 if s2 == 2 else 3
    l = [("name", "c"), ("correlation_param", [("pad", str(md)), ("kernel_size", "1"), ("max_displacement", str(md)),
                                               ("stride_1", "1"), ("stride_2", str(s2))])]
    tc, th, tw, _, _ = O.correlation_shape(shape[2], shape[3], md, 1, md, 1, s2)
    td = r.standard_normal((shape[0], tc, th, tw)).astype(np.float32)
    w0, w1 = O.correlation_bwd_ex(a, b, td, md, 1, md, 1, s2, 0)
    g0, g1 = correlation_backward64(l, t64(a), t64(b), t64(td))
    assert rel(g0, w0) <= TOL and rel(g1, w1) <= TOL


def test_correlation_outside_the_class_is_refused():
    l = [("name", "c"), ("correlation_param", [("pad", "3"), ("kernel_size", "3"), ("max_displacement", "3")])]
    x = torch.zeros((1, 4, 5, 5), dtype=torch.float64)
    with pytest.raises(NotImplementedError):
        correlation_backward64(l, x, x, x)


L1_FLAGS = [dict(l2_per_location=l2, normalize_by_num_entries=nb, l2_prescale_by_channels=pc, plateau=pl, epsilon=eps)
            for l2 in (False, True) for nb in (False, True) for pc in ((False, True) if l2 else (False,))
            for pl, eps in ((0.0, 1e-2), (0.3, 1e-3))]


@pytest.mark.parametrize("two", [True, False])
@pytest.mark.parametrize("flags", L1_FLAGS, ids=lambda f: "-".join("%s=%s" % (k[:6], v) for k, v in sorted(f.items())))
def test_l1loss(flags, two):
    r = rng(5)
    b0 = r.standard_normal((2, 3, 7, 9)).astype(np.float32)
    b1 = r.standard_normal(b0.shape).astype(np.float32) if two else None
    b0[0, 1, 2, 3] = np.nan                                        # invalid entries are masked
    b0[1, :, 4, 5] = np.nan
    b0[1, 0, 0, :4] = (b1[1, 0, 0, :4] if two else 0) + np.float32(0.01)     # inside the plateau
    want, _ = O.l1loss_fwd(b0, b1, **flags)
    got = float(l1loss_fwd64(t64(b0), t64(b1) if two else None, **flags))
    assert abs(got - want) <= TOL * abs(want)
    w0, w1 = O.l1loss_bwd(b0, b1, 0.7, **flags)
    g0, g1 = l1loss_bwd64(t64(b0), t64(b1) if two else None, 0.7, **flags)
    assert rel(g0, w0) <= TOL and rel(g1, w1) <= TOL


# (N, Ci, H, W, Co, k, stride, pad, deconv)
CONV_CASES = [(2, 5, 9, 11, 7, 3, 1, 1, False), (1, 6, 10, 13, 4, 5, 2, 2, False), (2, 4, 11, 8, 6, 3, 2, 1, False),
              (2, 4, 5, 7, 3, 4, 2, 1, True), (1, 3, 6, 5, 5, 5, 2, 2, True), (2, 6, 7, 9, 2, 3, 1, 1, True)]


@pytest.mark.parametrize("c", CONV_CASES, ids=lambda c: "%s_k%d_s%d_%dx%d" % ("d" if c[8] else "c", c[5], c[6], c[2], c[3]))
def test_conv_backward_and_forward(c):
    N, Ci, H, W, Co, k, s, p, deconv = c
    r = rng(sum(c[:8]))
    x = r.standard_normal((N, Ci, H, W)).astype(np.float32)
    w = r.standard_normal((Ci, Co, k, k) if deconv else (Co, Ci, k, k)).astype(np.float32)
    b = r.standard_normal(Co).astype(np.float32)
    y = (O.deconv_fwd if deconv else O.conv_fwd)(x, w, b, s, p, f64acc=True)
    dy = r.standard_normal(y.shape).astype(np.float32)
    want = O.conv_bwd(x, w, dy, s, p, deconv)
    got = conv_backward64(t64(x), t64(w), t64(dy), deconv, (s, s), (p, p))
    for g, wt in zip(got, want):
        assert rel(g, wt) <= TOL
    # the layer-local forward, followed by an in-place leaky ReLU
    typ = "Deconvolution" if deconv else "Convolution"
    proto = ('layer { name: "in" type: "Input" top: "x" input_param { shape { dim: %d dim: %d dim: %d dim: %d } } }\n'
             'layer { name: "l" type: "%s" bottom: "x" top: "y" convolution_param { num_output: %d kernel_size: %d stride: %d '
             'pad: %d } }\nlayer { name: "r" type: "ReLU" bottom: "y" top: "y" relu_param { negative_slope: 0.1 } }\n'
             % (N, Ci, H, W, typ, Co, k, s, p))
    net = NetGrad64(proto, {"l": [t64(w), t64(b)]})
    got = net.conv_forward("l", {"x": t64(x)})["y"]
    assert rel(got, O.relu(y, 0.1)) <= TOL
    # backward through the ReLU from its top data, both parameters
    D, P = net.backward({"x": t64(x), "y": t64(O.relu(y, 0.1))}, {"y": t64(dy)})
    gx, gw, gb = O.conv_bwd(x, w, O.relu_bwd(O.relu(y, 0.1), dy, 0.1), s, p, deconv)
    assert rel(P["l"][0], gw) <= TOL and rel(P["l"][1], gb) <= TOL and "x" not in D


def test_shared_weights_and_fan_out_sum():
    """A convolution with two bottoms sums its weight gradient over both; a blob read by two layers sums their gradients; an
    Eltwise scales by its coefficients and a Concat slices its top diff."""
    proto = ('force_backward: true\n'
             'layer { name: "in" type: "Input" top: "a" top: "b" input_param { shape { dim: 2 dim: 3 dim: 6 dim: 8 } '
             'shape { dim: 2 dim: 3 dim: 6 dim: 8 } } }\n'
             'layer { name: "c" type: "Convolution" bottom: "a" bottom: "b" top: "ca" top: "cb" '
             'convolution_param { num_output: 3 kernel_size: 3 pad: 1 } }\n'
             'layer { name: "e" type: "Eltwise" bottom: "ca" bottom: "a" top: "e" eltwise_param { operation: SUM coeff: 2 '
             'coeff: -0.5 } }\n'
             'layer { name: "k" type: "Concat" bottom: "e" bottom: "cb" top: "k" }\n')
    r = rng(3)
    a, b = (r.standard_normal((2, 3, 6, 8)).astype(np.float32) for _ in range(2))
    w = r.standard_normal((3, 3, 3, 3)).astype(np.float32)
    ca, cb = (O.conv_fwd(x, w, None, 1, 1, f64acc=True) for x in (a, b))
    dk = r.standard_normal((2, 6, 6, 8)).astype(np.float32)
    net = NetGrad64(proto, {"c": [t64(w), torch.zeros(3, dtype=torch.float64)]})
    blobs = {"a": t64(a), "b": t64(b), "ca": t64(ca), "cb": t64(cb), "e": t64(2 * ca - 0.5 * a)}
    D, P = net.backward(blobs, {"k": t64(dk)})
    ga, gwa, gba = O.conv_bwd(a, w, 2 * dk[:, :3], 1, 1)
    gb, gwb, gbb = O.conv_bwd(b, w, dk[:, 3:], 1, 1)
    assert rel(D["a"], ga.astype(np.float64) - 0.5 * dk[:, :3]) <= TOL and rel(D["b"], gb) <= TOL
    assert rel(P["c"][0], gwa.astype(np.float64) + gwb) <= TOL and rel(P["c"][1], gba.astype(np.float64) + gbb) <= TOL
