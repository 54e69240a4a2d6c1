"""GPU parity of the gradient path (SURVEY.md 8 row N1, BASELINE config 5): ConvolutionLayer / DeconvolutionLayer::Backward_gpu
through the C-ABI against the float64 oracle (oracle.conv_bwd, itself pinned to the reference's ConvolutionLayer::Backward in
tests/golden/train_golden.npz), and Net::Backward over the FlowNet2-C graph against OracleNet.backward.

Tolerances are relative to the largest gradient entry of each tensor: the data gradient runs through the 3xTF32 tensor-core
engine (same error budget as the forward pass, 1e-5), the weight gradient is an fp32 FMA reduction over up to N*H*W terms.
"""
import numpy as np
import pytest

from oracle import oracle as O
from oracle.net import OracleNet
from tests.util import maxabs, rng, smooth_images

from flownet2_b200 import ops as OPS

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def rel(got, want):
    return maxabs(got, want) / max(float(np.abs(want).max()), 1e-30)


def dev(a, channels_last=False):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t.contiguous(memory_format=torch.channels_last) if channels_last else t


# (name, N, Ci, H, W, Co, k, stride, pad, deconv, channels_last)
CONV_BWD_CASES = [
    ("c3x3_s1", 2, 16, 12, 20, 24, 3, 1, 1, False, True),
    ("c3x3_s1_wide", 1, 64, 24, 40, 64, 3, 1, 1, False, True),            # adjoint runs on the tensor-core engine
    ("c5x5_s2", 2, 8, 21, 27, 16, 5, 2, 2, False, True),                  # adjoint output smaller than the bottom
    ("c7x7_s2_img", 2, 3, 32, 48, 16, 7, 2, 3, False, False),             # first layer: plain NCHW bottom
    ("c1x1", 2, 32, 9, 11, 8, 1, 1, 0, False, True),
    ("c3x3_s2_wide", 1, 128, 16, 24, 256, 3, 2, 1, False, True),
    ("c3x3_s2_odd", 2, 32, 17, 23, 64, 3, 2, 1, False, True),             # odd bottom: no extra rows; adjoint has Co = 32
    ("c3x3_s2_even", 2, 32, 18, 24, 64, 3, 2, 1, False, True),            # even bottom: one extra row / column (out_pad)
    ("predict", 2, 96, 6, 10, 2, 3, 1, 1, False, True),                   # predict_flow: Co = 2
    ("d4x4_s2", 2, 32, 6, 8, 16, 4, 2, 1, True, True),
    ("d4x4_s2_flow", 2, 2, 6, 8, 2, 4, 2, 1, True, True),                 # upsample_flow: 2 -> 2
    ("d4x4_s2_wide", 1, 256, 8, 12, 128, 4, 2, 1, True, True),
    ("c3x3_473", 2, 473, 10, 14, 256, 3, 1, 1, False, True),              # conv3_1: channel tail of the 128-row tiles
    ("c3x3_s2_tiny", 2, 160, 5, 7, 192, 3, 2, 1, False, True),            # 3 x 4 output map: one K segment per row, mostly zero fill
    ("c5x5_s2_w57", 1, 64, 41, 57, 128, 5, 2, 2, False, True),            # odd width: the parity planes differ in length
    ("d4x4_s2_1026", 1, 130, 5, 7, 64, 4, 2, 1, True, True),              # deconv: the shifted map is the top diff
]


@pytest.mark.parametrize("case", CONV_BWD_CASES, ids=[c[0] for c in CONV_BWD_CASES])
def test_conv_backward_matches_oracle(fn2, case):
    name, N, Ci, H, W, Co, k, s, p, deconv, cl = case
    r = rng(sum(ord(c) for c in name))
    x = r.standard_normal((N, Ci, H, W)).astype(np.float32)
    w = (r.standard_normal((Ci, Co, k, k) if deconv else (Co, Ci, k, k)) / np.sqrt(Ci * k * k)).astype(np.float32)
    if deconv:
        Ho, Wo = s * (H - 1) + k - 2 * p, s * (W - 1) + k - 2 * p
    else:
        Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    dy = r.standard_normal((N, Co, Ho, Wo)).astype(np.float32)
    gx, gw, gb = OPS.conv2d_backward(dev(x, cl), dev(w), dev(dy, cl), s, p, deconv)
    torch.cuda.synchronize()
    wx, ww, wb = O.conv_bwd(x, w, dy, s, p, deconv)
    assert rel(gx.cpu().numpy(), wx) <= 1e-5, ("bottom diff", rel(gx.cpu().numpy(), wx))
    assert rel(gw.cpu().numpy(), ww) <= 1e-5, ("weight diff", rel(gw.cpu().numpy(), ww))
    assert rel(gb.cpu().numpy(), wb) <= 1e-5, ("bias diff", rel(gb.cpu().numpy(), wb))


@pytest.mark.parametrize("case", [CONV_BWD_CASES[0], CONV_BWD_CASES[2], CONV_BWD_CASES[7], CONV_BWD_CASES[9]], ids=lambda c: c[0] + "_simt")
def test_conv_backward_simt_engine(fn2, case):
    """`engine: CAFFE` (fn2_conv_desc.engine = 1): gradients on the exact-FP32 SIMT kernels instead of the tensor cores."""
    name, N, Ci, H, W, Co, k, s, p, deconv, cl = case
    r = rng(sum(ord(c) for c in name) + 1)
    x = r.standard_normal((N, Ci, H, W)).astype(np.float32)
    w = (r.standard_normal((Ci, Co, k, k) if deconv else (Co, Ci, k, k)) / np.sqrt(Ci * k * k)).astype(np.float32)
    Ho, Wo = (s * (H - 1) + k - 2 * p, s * (W - 1) + k - 2 * p) if deconv else ((H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1)
    dy = r.standard_normal((N, Co, Ho, Wo)).astype(np.float32)
    gx, gw, gb = OPS.conv2d_backward(dev(x, cl), dev(w), dev(dy, cl), s, p, deconv, engine=1)
    wx, ww, wb = O.conv_bwd(x, w, dy, s, p, deconv)
    assert rel(gx.cpu().numpy(), wx) <= 1e-5 and rel(gw.cpu().numpy(), ww) <= 1e-5 and rel(gb.cpu().numpy(), wb) <= 1e-5


def test_conv_backward_params_accumulates(fn2):
    r = rng(5)
    x = r.standard_normal((2, 8, 10, 12)).astype(np.float32)
    w = r.standard_normal((16, 8, 3, 3)).astype(np.float32)
    dy = r.standard_normal((2, 16, 10, 12)).astype(np.float32)
    _, gw, gb = OPS.conv2d_backward(dev(x, True), dev(w), dev(dy, True), 1, 1, False, need_input_grad=False)
    gw2, gb2 = gw.clone(), gb.clone()
    OPS.conv2d_backward(dev(x, True), dev(w), dev(dy, True), 1, 1, False, need_input_grad=False, accumulate=True, out=(gw2, gb2))
    torch.cuda.synchronize()
    assert rel(gw2.cpu().numpy(), 2 * gw.cpu().numpy()) <= 1e-6
    assert rel(gb2.cpu().numpy(), 2 * gb.cpu().numpy()) <= 1e-6


@pytest.mark.parametrize("slope", [0.0, 0.1])
def test_relu_backward_and_axpby(fn2, slope):
    r = rng(9)
    y = r.standard_normal((2, 5, 7, 9)).astype(np.float32)
    y[0, 0, 0, :3] = 0.0
    d = r.standard_normal(y.shape).astype(np.float32)
    got = OPS.relu_backward(dev(y, True), dev(d, True), slope).cpu().numpy()
    assert np.array_equal(got, O.relu_bwd(y, d, slope))
    a, b = dev(y, True), dev(d)
    want = (np.float32(0.5) * y + np.float32(2.0) * d).astype(np.float32)
    OPS.axpby(a, 0.5, b, 2.0)
    assert maxabs(b.cpu().numpy(), want) <= 1e-6


# ---- whole-net gradients ------------------------------------------------------------------------------------------------
SEEDS = ["predict_flow6", "predict_flow5", "predict_flow4", "predict_flow3", "predict_flow2"]


def test_flownet_c_backward_matches_oracle(fn2):
    w, h, batch = 192, 100, 1
    proto = fn2.fill_template(fn2.model_template("FlowNet2-C"), w, h)
    net = fn2.Net(proto, None, fn2.TEST, batch=batch)
    net.fill_params(7)
    weights = net.to_caffemodel()
    img0, img1 = smooth_images(rng(7), batch, h, w)
    net.forward(img0=img0, img1=img1)
    r = rng(8)
    seeds = {s: r.standard_normal(net.blobs[s].shape).astype(np.float32) for s in SEEDS}
    net.clear_param_diffs()
    net.backward(**seeds)
    need = dict(zip(net.layer_names, net.layer_need_backward()))
    assert need["conv1"] and need["corr"] and need["Concat2"] and not need["Resample_final"] and not need["img0s_aug"]
    onet = OracleNet(proto, weights, batch=batch, f64acc=True)
    B = onet.forward(img0=img0, img1=img1)
    # differentiate at the ENGINE's activations: a pre-activation within rounding of zero (conv3b has some: 1e-8 against 8e-8)
    # must not pick different sides of the ReLU kink in the two implementations
    for k in list(B):
        if k not in ("img0", "img1"):
            assert maxabs(net.blobs[k].data, B[k]) <= 1e-4 * max(1.0, float(np.abs(B[k]).max())), k
            B[k] = net.blobs[k].data
    D, P = onet.backward(**seeds)
    worst = {}
    for lname, grads in P.items():
        for i, g in enumerate(grads):
            got = net.param(lname, i, diff=True).reshape(g.shape)
            worst["%s[%d]" % (lname, i)] = rel(got, g)
    bad = {k: v for k, v in worst.items() if v > 2e-5}
    assert not bad, bad
    assert len(worst) >= 40
    # (concat tops are not compared: the fused ReLUs of their zero-copy children differentiate in place inside them)
    for blob in ("conv1a", "conv1b", "conv2a", "conv2b", "conv3a", "conv3b", "corr", "conv_redir", "conv3_1", "deconv5", "conv6_1"):
        assert rel(net.get_diff(blob), D[blob]) <= 2e-5, (blob, rel(net.get_diff(blob), D[blob]))
    # parameter gradients accumulate across calls until cleared (net.cpp:935-955)
    first = net.param("conv3_1", 0, diff=True)
    net.forward(img0=img0, img1=img1)
    net.backward(**seeds)
    assert rel(net.param("conv3_1", 0, diff=True), 2 * first) <= 1e-6
    net.clear_param_diffs()
    net.sync()
    assert not net.param("conv3_1", 0, diff=True).any()


def test_backward_without_fusion_or_aliasing_is_the_same(fn2, monkeypatch):
    """The fused conv+ReLU derivative and the zero-copy concat gradient slices against the plain layer-by-layer execution."""
    w, h, batch = 128, 64, 2
    proto = fn2.fill_template(fn2.model_template("FlowNet2-C"), w, h)
    img0, img1 = smooth_images(rng(3), batch, h, w)
    r = rng(4)
    res = []
    for plain in (False, True):
        if plain:
            monkeypatch.setenv("FN2_NO_FUSE", "1")
            monkeypatch.setenv("FN2_NO_ALIAS", "1")
        net = fn2.Net(proto, None, fn2.TEST, batch=batch)
        net.fill_params(5)
        net.forward(img0=img0, img1=img1)
        if not res:
            seeds = {s: r.standard_normal(net.blobs[s].shape).astype(np.float32) for s in SEEDS}
        net.clear_param_diffs()
        net.backward(**seeds)
        res.append({n: net.param(n, 0, diff=True) for n, t in zip(net.layer_names, net.layer_types) if t in ("Convolution", "Deconvolution")
                    and net.layer_need_backward()[net.layer_names.index(n)]})
    assert len(res[0]) >= 20
    for k in res[0]:
        assert rel(res[0][k], res[1][k]) <= 1e-5, (k, rel(res[0][k], res[1][k]))


# ---- training-side layers against the reference's recorded outputs (tests/golden/train_golden.npz) and the oracle -----------
import os      # noqa: E402
import sys     # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import train_cases as TC                                       # noqa: E402
from tests.refcheck import TRAIN_TOL, train_oracle_eval        # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_golden.npz")


def single_layer_net(fn2, case, bottoms):
    names = [n for n in __import__("re").findall(r'bottom:\s*"([^"]+)"', case["text"])]
    shapes = "".join(" shape { %s }" % " ".join("dim: %d" % d for d in b.shape) for b in bottoms)
    proto = ('force_backward: true\nlayer { name: "in" type: "Input" %s input_param {%s } }\nlayer { %s }\n'
             % (" ".join('top: "%s"' % n for n in names), shapes, case["text"]))
    net = fn2.Net(proto, None, fn2.TEST)
    return net, names


@pytest.mark.parametrize("name", list(TC.TRAIN_CASES))
def test_training_layers_match_reference_and_oracle(fn2, name):
    c = TC.TRAIN_CASES[name]
    bottoms, params, r = TC.train_inputs(name)
    net, names = single_layer_net(fn2, c, bottoms)
    lname = net.layer_names[-1]
    if params is not None:
        from oracle.net import write_caffemodel
        net.copy_from(write_caffemodel([(lname, net.layer_types[-1], params)]))
    top = net.outputs[0]
    out = {"top0": net.forward(**dict(zip(names, bottoms)))[top]}
    k = c["kind"]
    if k == "conv_bwd":
        net.clear_param_diffs()
        net.backward(**{top: r.standard_normal(out["top0"].shape).astype(np.float32)})
        out["bdiff0"] = net.get_diff(names[0])
        out["pdiff0"] = net.param(lname, 0, diff=True)
        out["pdiff1"] = net.param(lname, 1, diff=True)
    elif k == "l1loss":
        net.backward(**{top: np.full(net.blobs[top].shape, c["top_diff"], np.float32)})
        for i, n in enumerate(names):
            out["bdiff%d" % i] = net.get_diff(n)
    want_o = train_oracle_eval(name)
    gold = np.load(GOLD) if os.path.exists(GOLD) else None
    assert gold is not None, "tests/golden/train_golden.npz is missing"
    tol = 5 * TRAIN_TOL[k]
    for key, got in out.items():
        for label, want in (("oracle", want_o[key]), ("reference", gold["T/%s/%s" % (name, key)])):
            want = np.asarray(want)
            g = np.asarray(got).reshape(want.shape)
            scale = max(float(np.nanmax(np.abs(want))), 1e-6)
            assert maxabs(g, want) <= tol * scale, (name, key, label, maxabs(g, want), scale)


def test_l1loss_accumulates_into_a_shared_bottom(fn2):
    """predict_flow blobs feed both the loss and the next decoder stage: the loss gradient must ADD to what the other consumer wrote."""
    proto = ('force_backward: true\n'
             'layer { name: "in" type: "Input" top: "a" top: "gt" input_param { shape { dim: 2 dim: 2 dim: 6 dim: 8 } shape { dim: 2 dim: 2 dim: 6 dim: 8 } } }\n'
             'layer { name: "scale" type: "Eltwise" bottom: "a" top: "a2" eltwise_param { operation: SUM coeff: 3 } }\n'
             'layer { name: "l1" type: "L1Loss" bottom: "a" bottom: "gt" top: "loss1" loss_weight: 0.5 l1_loss_param { l2_per_location: true } }\n'
             'layer { name: "l2" type: "L1Loss" bottom: "a2" bottom: "gt" top: "loss2" loss_weight: 2 }\n')
    net = fn2.Net(proto, None, fn2.TEST)
    r = rng(21)
    a = r.standard_normal((2, 2, 6, 8)).astype(np.float32)
    gt = r.standard_normal((2, 2, 6, 8)).astype(np.float32)
    out = net.forward(a=a, gt=gt)
    l1, _ = O.l1loss_fwd(a, gt, l2_per_location=True)
    l2, _ = O.l1loss_fwd(3 * a, gt)
    assert abs(float(out["loss1"].reshape(-1)[0]) - l1) <= 1e-5 * l1 and abs(float(out["loss2"].reshape(-1)[0]) - l2) <= 1e-5 * l2
    net.backward()
    g1, _ = O.l1loss_bwd(a, gt, 0.5, l2_per_location=True)
    g2, h2 = O.l1loss_bwd(3 * a, gt, 2.0)
    assert maxabs(net.get_diff("a"), g1 + 3 * g2) <= 1e-6
    assert maxabs(net.get_diff("gt"), -g1 + h2) <= 1e-6


def test_flownet_c_training_net_step(fn2):
    """The authored FlowNet2-C training graph (models/FlowNet2-C_train.prototxt.template): random augmentation of both frames and
    of the ground truth, multi-scale end-point-error losses, backward.  Every training-side layer is checked in place against the
    oracle given the blobs the net itself produced; the conv stack's gradients are covered by the deploy-graph test above."""
    cw, ch, dw, dh, batch = 192, 128, 224, 160, 2     # predict_flow6 is 2 x 3 (a 1-row level divides by zero in Downsample)
    proto = fn2.fill_train_template(fn2.train_template("FlowNet2-C"), cw, ch, dw, dh, batch)
    net = fn2.Net(proto, None, fn2.TRAIN)
    net.fill_params(11)
    img0, img1 = smooth_images(rng(12), batch, dh, dw)
    r = rng(13)
    gt = (3 * r.standard_normal((batch, 2, dh, dw))).astype(np.float32)
    gt[0, :, 60:75, 80:110] = np.nan                              # invalid ground truth
    net.clear_param_diffs()
    out = net.forward(img0=img0, img1=img1, flow_gt=gt)
    B = lambda n: net.blobs[n].data
    p0, p1 = B("img0_aug_params"), B("img1_aug_params")
    assert p0.shape == (batch, 42, 1, 1) and np.abs(p0).max() > 0 and maxabs(p0, p1) > 0
    assert B("img0_aug").shape == (batch, 3, ch, cw)
    want = O.flow_augmentation(gt, p0, p1, cw, ch)
    got = B("flow_gt_aug")
    both = ~np.isnan(want) & ~np.isnan(got)
    # nearest-neighbour lookup into a white-noise field: a source position within rounding of x.5 may pick the neighbouring sample
    off = np.abs(got[both] - want[both]) > 2e-5 * max(1.0, np.abs(want[both]).max())
    assert both.mean() > 0.9 and off.mean() < 2e-3, (both.mean(), off.mean())
    total = 0.0
    for lvl, wgt in ((6, 0.32), (5, 0.08), (4, 0.02), (3, 0.01), (2, 0.005)):
        pf, g = B("predict_flow%d" % lvl), B("blob_gt%d" % lvl)
        assert maxabs(g, O.downsample_fwd(B("scaled_flow_gt_aug"), pf.shape[2], pf.shape[3])) <= 1e-5
        loss, _ = O.l1loss_fwd(pf, g, l2_per_location=True)
        mine = float(out["flow_loss%d" % lvl].reshape(-1)[0])
        assert abs(mine - loss) <= 1e-5 * abs(loss), (lvl, mine, loss)
        total += wgt * mine
    assert np.isfinite(total)
    net.backward()
    pf, g = B("predict_flow2"), B("blob_gt2")
    g0, _ = O.l1loss_bwd(pf, g, 0.005, l2_per_location=True)
    assert rel(net.get_diff("predict_flow2"), g0) <= 1e-5
    for lname in ("conv1", "conv3", "conv_redir", "conv6_1", "deconv2", "predict_flow2", "upsample_flow6to5"):
        gw = net.param(lname, 0, diff=True)
        assert np.isfinite(gw).all() and np.abs(gw).max() > 0, lname
    need = dict(zip(net.layer_names, net.layer_need_backward()))
    assert need["corr"] and need["flow_loss6"] and not need["Downsample6"] and not need["flow_aug"] and not need["img0s_aug"]


def _random_conv_cases(count, seed):
    r = np.random.default_rng(seed)
    cases = []
    while len(cases) < count:
        deconv = bool(r.integers(0, 4) == 0)
        k = int(r.choice([1, 2, 3, 4, 5, 7]))
        s = int(r.choice([1, 1, 2, 2, 3]))
        p = int(r.integers(0, (k + 1) // 2 + 1))
        N = int(r.integers(1, 4))
        Ci = int(r.choice([1, 2, 3, 5, 8, 17, 32, 48, 70, 130]))
        Co = int(r.choice([1, 2, 4, 16, 24, 33, 64, 96, 144]))
        H, W = int(r.integers(k + 1, 30)), int(r.integers(k + 1, 45))
        if deconv:
            if s * (H - 1) + k - 2 * p < 1 or s * (W - 1) + k - 2 * p < 1 or p > k - 1:
                continue
            H, W = min(H, 12), min(W, 14)
        elif H + 2 * p < k or W + 2 * p < k or p > k - 1:
            continue
        cases.append(("rand%d_%s_c%d_o%d_k%d_s%d_p%d_%dx%dx%d" % (len(cases), "d" if deconv else "c", Ci, Co, k, s, p, N, H, W),
                      N, Ci, H, W, Co, k, s, p, deconv, True))
    return cases


RANDOM_CONV_CASES = _random_conv_cases(16, 2024)


@pytest.mark.parametrize("case", RANDOM_CONV_CASES, ids=[c[0] for c in RANDOM_CONV_CASES])
def test_conv_backward_random_shapes(fn2, case):
    """Seeded random layer shapes (odd channel counts, even kernels, stride 3, one-pixel-wide tails): every gradient path the engine
    may pick (tensor-core weight gradient with / without tap grouping, padded adjoints, SIMT fall-backs) against the float64 oracle."""
    test_conv_backward_matches_oracle(fn2, case)


def test_loss_net_gradients_match_reference_net(fn2):
    """The engine's Net::Forward / Backward on the FlowNet2-C graph with five EPE losses against the reference's own Net semantics
    recorded in train_golden.npz (oracle.ref.RefNet with Split layers): losses and every parameter gradient."""
    from oracle.net import synth_weights
    gold = np.load(GOLD)
    assert "N/lossnet/loss2" in gold.files, "train_golden.npz has no whole-net gradients"
    proto, ins = TC.loss_net_proto(), TC.loss_net_inputs()
    small = fn2.fill_template(fn2.model_template("FlowNet2-C"), 64, 64)
    _, cm = synth_weights(small, TC.LOSS_NET["seed"], fn2.fill_template(fn2.model_template("FlowNet2-C"), TC.LOSS_NET["w"], TC.LOSS_NET["h"]))
    net = fn2.Net(proto, cm, fn2.TEST, batch=TC.LOSS_NET["batch"])
    out = net.forward(**ins)
    for lvl in TC.LOSS_NET["weights"]:
        want = float(gold["N/lossnet/loss%d" % lvl][0])
        assert abs(float(out["flow_loss%d" % lvl].reshape(-1)[0]) - want) <= 5e-5 * abs(want), lvl
    net.clear_param_diffs()
    net.backward()
    for k in [k for k in gold.files if k.startswith("N/lossnet/grad/")]:
        _, _, _, name, i = k.split("/")
        want = gold[k]
        got = TC.grad_signature(name, int(i), net.param(name, int(i), diff=True))
        scale = float(np.abs(want).max())
        assert np.abs(got - want).max() <= 5e-5 * scale, (k, float(np.abs(got - want).max()), scale)      # measured: 2.2e-6


def test_explicit_split_layers_load_and_sum_gradients(fn2):
    """A prototxt that already went through the reference's InsertSplits (explicit Split layers, split_layer.cpp): forward copies,
    backward sums the top diffs -- the same gradients as the implicit fan-out."""
    shape = "dim: 2 dim: 4 dim: 6 dim: 8"
    head = 'force_backward: true\nlayer { name: "in" type: "Input" top: "a" input_param { shape { %s } } }\n' % shape
    tail = ('layer { name: "s1" type: "Eltwise" bottom: "%s" top: "b1" eltwise_param { operation: SUM coeff: 2 } }\n'
            'layer { name: "s2" type: "Eltwise" bottom: "%s" top: "b2" eltwise_param { operation: SUM coeff: -3 } }\n'
            'layer { name: "l1" type: "L1Loss" bottom: "b1" top: "loss1" loss_weight: 1 }\n'
            'layer { name: "l2" type: "L1Loss" bottom: "b2" top: "loss2" loss_weight: 0.5 l1_loss_param { l2_per_location: true } }\n')
    split = 'layer { name: "a_in_0_split" type: "Split" bottom: "a" top: "a_in_0_split_0" top: "a_in_0_split_1" }\n'
    a = rng(31).standard_normal((2, 4, 6, 8)).astype(np.float32)
    grads = []
    for proto in (head + tail % ("a", "a"), head + split + tail % ("a_in_0_split_0", "a_in_0_split_1")):
        net = fn2.Net(proto, None, fn2.TEST)
        out = net.forward(a=a)
        net.backward()
        grads.append((net.get_diff("a"), float(out["loss1"].reshape(-1)[0]), float(out["loss2"].reshape(-1)[0])))
    assert "Split" in fn2.Net(head + split + tail % ("a_in_0_split_0", "a_in_0_split_1"), None, fn2.TEST).layer_types
    assert grads[0][1:] == grads[1][1:]
    assert np.abs(grads[0][0]).max() > 0 and maxabs(grads[0][0], grads[1][0]) <= 1e-6
