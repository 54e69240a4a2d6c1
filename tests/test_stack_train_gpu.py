"""The stacked FlowNet2 training schedule on the GPU (models/FlowNet2-CS_train, -CSS_train, -SD_train, FlowNet2_train): backward
runs on the trained sub-network and its losses only, frozen parameters get no gradient, the losses and the trained gradients
match the float64 oracle with Caffe's need-backward pruning (tests/stack_oracle.py), the warp blocks run fused in TRAIN phase
bit-identically to the layer chain, the trainable span of the gradient arena, and the weight hand-over between stages.

Crops are multiples of 64 with predict_flow6 at 3 x 2 (a 1-row level divides by zero in Downsample)."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle.net import get, getall, parse_prototxt
from tests.stack_oracle import PrunedOracleNet
from tests.util import maxabs, rng, smooth_images

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

STAGES = {"FlowNet2-CS": "net2_", "FlowNet2-CSS": "net3_", "FlowNet2-SD": "", "FlowNet2": "fuse_"}
CW, CH, DW, DH, BATCH = 192, 128, 224, 160, 2
CONV = ("Convolution", "Deconvolution")


def rel(got, want):
    return maxabs(got, want) / max(float(np.abs(want).max()), 1e-30)


def trained(name, pre):
    """Layer of the stage's trained sub-network (SD trains the unprefixed layers)."""
    return name.startswith(pre) and (pre != "" or not name.startswith(("net", "fuse_")))


def train_step(fn2, stage, seed=11):
    proto = fn2.fill_train_template(fn2.train_template(stage), CW, CH, DW, DH, BATCH)
    net = fn2.Net(proto, None, fn2.TRAIN)
    net.fill_params(seed)
    img0, img1 = smooth_images(rng(12), BATCH, DH, DW)
    gt = (3 * rng(13).standard_normal((BATCH, 2, DH, DW))).astype(np.float32)
    net.clear_param_diffs()
    out = net.forward(img0=img0, img1=img1, flow_gt=gt)
    net.backward()
    net.sync()
    return proto, net, out


def conv_layers(net):
    return [n for n, t in zip(net.layer_names, net.layer_types) if t in CONV]


@pytest.mark.parametrize("stage", list(STAGES))
def test_backward_runs_only_on_the_trained_subnetwork(fn2, stage):
    pre = STAGES[stage]
    proto, net, out = train_step(fn2, stage)
    need = dict(zip(net.layer_names, net.layer_need_backward()))
    for n, t in zip(net.layer_names, net.layer_types):
        want = t == "L1Loss" or (trained(n, pre) and t in CONV + ("ReLU", "Concat") and not n.endswith("Concat_input"))
        assert need[n] == want, (n, t, need[n])
    n_trained = 0
    for n in conv_layers(net):
        for i in (0, 1):
            d = net.param(n, i, diff=True)
            if trained(n, pre):
                assert np.isfinite(d).all() and np.abs(d).max() > 0, (n, i)
                n_trained += 1
            else:
                assert not d.any(), (n, i)
    assert n_trained >= 22
    # every loss against the oracle's L1 loss on the net's own blobs
    losses = [l for l in getall(parse_prototxt(proto), "layer") if get(l, "type") == "L1Loss"]
    assert len(losses) == (3 if stage == "FlowNet2" else 5)
    for l in losses:
        pred, gt = getall(l, "bottom")
        want, _ = O.l1loss_fwd(net.blobs[pred].data, net.blobs[gt].data, l2_per_location=True)
        got = float(out[getall(l, "top")[0]].reshape(-1)[0])
        assert np.isfinite(got) and abs(got - want) <= 1e-5 * abs(want), (get(l, "name"), got, want)


@pytest.mark.parametrize("stage", ["FlowNet2-CS", "FlowNet2"])
def test_trained_gradients_match_pruned_oracle(fn2, stage):
    pre = STAGES[stage]
    proto, net, _ = train_step(fn2, stage)
    onet = PrunedOracleNet(proto, net.to_caffemodel(), f64acc=True)
    # differentiate at the ENGINE's activations (a pre-activation within rounding of zero must not pick different sides of a ReLU)
    onet.blobs = {b: net.blobs[b].data for b in net.blob_names}
    _, P = onet.backward()
    assert sorted(P) == sorted(n for n in conv_layers(net) if trained(n, pre))
    worst = {}
    for lname, grads in P.items():
        for i, g in enumerate(grads):
            worst["%s[%d]" % (lname, i)] = rel(net.param(lname, i, diff=True).reshape(g.shape), g)
    bad = {k: v for k, v in worst.items() if v > 2e-5}
    assert not bad, bad


@pytest.mark.parametrize("stage", ["FlowNet2-CS", "FlowNet2"])
def test_fused_warp_block_in_train_phase_is_bit_identical(fn2, monkeypatch, stage):
    runs = []
    for fused in (True, False):
        if not fused:
            monkeypatch.setenv("FN2_NO_WARPFUSE", "1")
        _, net, _ = train_step(fn2, stage)
        blobs = {b: net.blobs[b].data for b in net.blob_names}
        diffs = {(n, i): net.param(n, i, diff=True) for n in conv_layers(net) for i in (0, 1)}
        runs.append((net.launches_per_forward, blobs, diffs))
    assert runs[0][0] < runs[1][0], (runs[0][0], runs[1][0])              # the fusion actually happened
    for b in runs[0][1]:
        assert np.array_equal(runs[0][1][b], runs[1][1][b], equal_nan=True), b
    for k in runs[0][2]:
        assert np.array_equal(runs[0][2][k], runs[1][2][k]), k
    assert np.abs(runs[0][1]["net2_in_err_norm"]).max() > 0


def test_trainable_span_covers_exactly_the_trained_parameters(fn2):
    from flownet2_b200 import parallel as PAR
    pre = STAGES["FlowNet2"]
    _, net, _ = train_step(fn2, "FlowNet2")
    full, span = PAR.grad_arena_tensor(net), PAR.grad_arena_tensor(net, trainable_only=True)
    padded = lambda a: (a.size + 63) // 64 * 64
    want = sum(padded(net.param(n, i)) for n in conv_layers(net) if trained(n, pre) for i in (0, 1))
    assert span.numel() == want and 0 < span.numel() < full.numel() // 10
    assert span.data_ptr() + 4 * span.numel() == full.data_ptr() + 4 * full.numel()      # the fusion net sits at the end
    span.fill_(1.0)
    torch.cuda.synchronize()
    for n in conv_layers(net):
        for i in (0, 1):
            d = net.param(n, i, diff=True)
            assert (d == 1).all() if trained(n, pre) else not d.any(), (n, i)
    # the C training graph trains everything after the augmentation
    proto = fn2.fill_train_template(fn2.train_template("FlowNet2-C"), CW, CH, DW, DH, BATCH)
    c = fn2.Net(proto, None, fn2.TRAIN)
    assert c.trainable_diff_span()[1] == 4 * sum(padded(c.param(n, i)) for n in conv_layers(c) for i in (0, 1))


def test_c_weights_with_prefix_drive_net1_of_css(fn2):
    w, h = 192, 128
    img0, img1 = smooth_images(rng(21), 1, h, w)
    c = fn2.Net(fn2.fill_template(fn2.model_template("FlowNet2-C"), w, h), None, fn2.TEST, batch=1)
    c.fill_params(31)
    cm = c.to_caffemodel()
    css = fn2.Net(fn2.fill_template(fn2.model_template("FlowNet2-CSS"), w, h), None, fn2.TEST, batch=1)
    css.fill_params(32)
    css.copy_from(cm)                       # the preprocessing state, by name (the C layers have no match and are ignored)
    css.copy_from(cm, prefix="net1_")
    c.forward(img0=img0, img1=img1)
    css.forward(img0=img0, img1=img1)
    want = c.blobs["predict_flow2"].data
    got = css.blobs["net1_predict_flow2"].data
    assert np.abs(want).max() > 0 and rel(got, want) <= 1e-6, rel(got, want)
    assert np.array_equal(css.param("net1_conv3_1", 0), c.param("conv3_1", 0))


def test_cs_caffemodel_loads_into_css_train_and_leaves_net3_alone(fn2):
    def make(stage, seed):
        net = fn2.Net(fn2.fill_train_template(fn2.train_template(stage), CW, CH, DW, DH, BATCH), None, fn2.TRAIN)
        net.fill_params(seed)
        return net
    cs, css = make("FlowNet2-CS", 41), make("FlowNet2-CSS", 42)
    before = {(n, i): css.param(n, i) for n in conv_layers(css) for i in (0, 1)}
    css.copy_from(cs.to_caffemodel())
    moved = 0
    for (n, i), b in before.items():
        got = css.param(n, i)
        if n.startswith("net3_"):
            assert np.array_equal(got, b), (n, i)
        else:
            assert np.array_equal(got, cs.param(n, i)) and (i == 1 or not np.array_equal(got, b)), (n, i)    # biases start at 0
            moved += 1
    assert moved == 2 * len([n for n in conv_layers(cs)])
