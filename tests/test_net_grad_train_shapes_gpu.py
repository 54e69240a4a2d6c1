"""Whole-net gradients at the training shape (train.py --crop 448x320 --batch 8): Net::Backward of FlowNet2-C, -CS, -CSS, -SD and
the fusion stage against the float64 Net::Backward of tests/net_grad64.py, evaluated on the device at the engine's own
activations (pinned to the CPU oracle by tests/test_net_grad64_cpu.py).

At this shape the graphs run plans the toy shapes of test_train_gpu.py and test_stack_train_gpu.py never reach together --
data-gradient operators at NT = 128 in plain mode (the FP16 operand route), K-split tiles, the fast correlation backward --
with batch 8 in the host layers: concat gradient slices at the real channel strides, the Co-padded scratch diff of
BackwardData, accumulation into bottoms with several consumers, the fused ReLU derivative in place.  The second-iteration case
checks that a solver step repacks the forward weights, the FP16 weight scale and the adjoint operator's weights.

Tolerances are those of the toy-shape tests: 2e-5 of each tensor's largest entry for gradients
(test_flownet_c_backward_matches_oracle), 1e-6 of max(1, largest |entry|) for a convolution's top (test_conv_tc_routes_gpu.py)
and 1e-6 relative for a loss.  Each case prints the worst error of every tensor it compared.
"""
import ctypes as C
import gc
import re
import time

import numpy as np
import pytest

from oracle.net import get, getall
from tests.conv_ref import adjoint, case
from tests.net_grad64 import CONV, NetGrad64
from tests.util import kernels_per_case, rng, smooth_images, train_convs

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

CW, CH, DW, DH, BATCH = 448, 320, 512, 384, 8
GRAD_TOL, FWD_TOL, LOSS_TOL = 2e-5, 1e-6, 1e-6
STAGES = {"FlowNet2-CS": "net2_", "FlowNet2-CSS": "net3_", "FlowNet2-SD": "", "FlowNet2": "fuse_"}
# the blob diffs test_flownet_c_backward_matches_oracle compares (not the concat tops: the fused ReLUs of their zero-copy
# children differentiate in place inside them)
C_BLOBS = ("conv1a", "conv1b", "conv2a", "conv2b", "conv3a", "conv3b", "corr", "conv_redir", "conv3_1", "deconv5", "conv6_1")


class EngineBlobs(object):
    """The engine's blobs as float64 device tensors, read on first use."""

    def __init__(self, net):
        self.net, self.cache = net, {}

    def __getitem__(self, name):
        if name not in self.cache:
            self.cache[name] = torch.from_numpy(self.net.blobs[name].data).cuda().double()
        return self.cache[name]

    def shape_of(self, name):
        return self.net.blobs[name].shape


def engine_params(net, ref):
    """{layer: [weight, bias]} on the device for the convolutions the reference differentiates."""
    return {n: [torch.from_numpy(net.param(n, i)).cuda() for i in (0, 1)]
            for n, need in ref.layer_need.items() if need and get(ref.by_name[n], "type") in CONV}


def rel(got, want):
    got = torch.as_tensor(got).to(want.device).double().reshape(want.shape)
    return float((got - want).abs().max()) / max(float(want.abs().max()), 1e-30)


def inputs(seed=12):
    img0, img1 = smooth_images(rng(seed), BATCH, DH, DW)
    gt = (3 * rng(seed + 1).standard_normal((BATCH, 2, DH, DW))).astype(np.float32)
    gt[0, :, 100:130, 200:260] = np.nan                            # invalid ground truth
    return {"img0": img0, "img1": img1, "flow_gt": gt}


def make_net(fn2, stage, seed=11):
    proto = fn2.fill_train_template(fn2.train_template(stage), CW, CH, DW, DH, BATCH)
    net = fn2.Net(proto, None, fn2.TRAIN)
    net.fill_params(seed)
    return proto, net


def step(net, feed=None):
    net.clear_param_diffs()
    out = net.forward(**(feed or {}))
    net.backward()
    net.sync()
    return out


def check_gradients(net, P, worst):
    """Every parameter gradient of the reference within GRAD_TOL; every other convolution parameter's diff exactly 0."""
    for name, grads in P.items():
        for i, g in enumerate(grads):
            worst["%s[%d]" % (name, i)] = rel(torch.from_numpy(net.param(name, i, diff=True)), g)
    frozen = 0
    for n, t in zip(net.layer_names, net.layer_types):
        if t in CONV and n not in P:
            for i in (0, 1):
                assert not net.param(n, i, diff=True).any(), (n, i)
                frozen += 1
    return frozen


def check_losses(ref, blobs, out, worst):
    for name in ref.losses():
        top = getall(ref.by_name[name], "top")[0]
        want = float(ref.loss(name, blobs))
        got = float(out[top].reshape(-1)[0])
        worst[name] = abs(got - want) / abs(want)


def check_forwards(ref, names, blobs, worst):
    for n in names:
        for t, want in ref.conv_forward(n, blobs).items():
            worst["fwd " + t] = float((blobs[t] - want).abs().max()) / max(1.0, float(want.abs().max()))
            del want


def report(stage, worst, limits):
    print("\n%s: %d tensors" % (stage, len(worst)))
    for k, v in sorted(worst.items(), key=lambda kv: -kv[1]):
        print("  %-32s %.3g" % (k, v))
    bad = {k: v for k, v in worst.items() if v > limits(k)}
    assert not bad, bad


def limit(key):
    if key.startswith("fwd "):
        return FWD_TOL
    if "loss" in key:
        return LOSS_TOL
    return GRAD_TOL


def plans(model, trained):
    """Forward and data-gradient plans (fn2_conv_plan, the helpers of test_conv_tc_routes_gpu.py) of the trained convolutions
    at this shape: -> {name: (forward plan, data-gradient plan or None)}."""
    from tests.test_conv_tc_routes_gpu import plan_of
    out = {}
    for name, ci, h, w, co, k, s, p, deconv, _ in train_convs(model, CW, CH):
        if name not in trained:
            continue
        fwd = plan_of(case("fwd-" + name, BATCH, ci, h, w, co, k, s, p, deconv, layout="pad"))
        bwd = None
        if ci > 16:                                    # the layers on the input images get no data gradient
            bwd = plan_of(adjoint("dgrad-" + name, BATCH, ci, h, w, co, k, s, p, deconv))
        out[name] = (fwd, bwd)
    return out


@pytest.fixture(autouse=True)
def release():
    """The machines are shared: each case's net and float64 tensors go before the next case starts."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def module_budget():
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    print("\nmodule wall time %.1f s, peak device memory (torch) %.2f GB" % (time.time() - t0,
                                                                              torch.cuda.max_memory_allocated() / 2 ** 30))


# ---- FlowNet2-C ------------------------------------------------------------------------------------------------------------
def test_flownet_c_at_training_shape(fn2):
    proto, net = make_net(fn2, "FlowNet2-C")
    out = step(net, inputs())
    ref = NetGrad64(proto, None)
    ref.params = engine_params(net, ref)
    blobs = EngineBlobs(net)
    worst = {}
    check_losses(ref, blobs, out, worst)
    D, P = ref.backward(blobs, keep=C_BLOBS)
    assert sorted(P) == sorted(ref.trained()) and len(P) >= 20
    check_gradients(net, P, worst)
    assert sum(1 for k in worst if k.endswith("]")) >= 40
    for b in C_BLOBS:
        worst["diff " + b] = rel(torch.from_numpy(net.get_diff(b)), D[b])
    del D, P
    check_forwards(ref, ref.trained(), blobs, worst)
    # the plans the toy shapes do not reach
    pl = plans("FlowNet2-C", set(ref.trained()))
    f16 = [n for n, (_, b) in pl.items() if b and b[0] == 128 and b[3] == 0]
    split = [n for n, (f, b) in pl.items() if f[5] > 1 or (b and b[5] > 1)]
    print("plans: data gradient at NT 128, plain mode: %s; K split: %s" % (f16, split))
    assert f16 and split
    need = C.c_size_t()
    cin = net.blobs["conv3a"].shape
    fn2.check(fn2.lib().fn2_correlation_backward_workspace_bytes(cin[0], cin[1], cin[2], cin[3], 20, 1, 20, 1, 2, 0,
                                                                  C.byref(need)))
    assert need.value == 4 * cin[0] * cin[2] * cin[3] * 441                 # the fast route's shape: the staged top diff
    got, = kernels_per_case([lambda: (net.backward_async(), net.sync())])
    print("correlation backward kernels: %s" % sorted(k for k in got if "corr" in k))
    assert any("corr_bwd_fast_kernel" in k for k in got), sorted(got)
    report("FlowNet2-C", worst, limit)


# ---- the stacked stages ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stage", list(STAGES))
def test_stacked_stage_at_training_shape(fn2, stage):
    proto, net = make_net(fn2, stage)
    out = step(net, inputs())
    ref = NetGrad64(proto, None)
    ref.params = engine_params(net, ref)
    pre = STAGES[stage]
    assert ref.trained() and all(n.startswith(pre) and (pre or not n.startswith(("net", "fuse_"))) for n in ref.trained())
    blobs = EngineBlobs(net)
    worst = {}
    check_losses(ref, blobs, out, worst)
    _, P = ref.backward(blobs, keep=())
    frozen = check_gradients(net, P, worst)
    assert frozen >= (0 if stage == "FlowNet2-SD" else 2 * 20), frozen
    del P
    pl = plans(stage, set(ref.trained()))
    print("plans: data gradient at NT 128, plain mode: %s; K split: %s"
          % ([n for n, (_, b) in pl.items() if b and b[0] == 128 and b[3] == 0],
             [n for n, (f, b) in pl.items() if f[5] > 1 or (b and b[5] > 1)]))
    report(stage, worst, limit)


# ---- a second iteration after a solver step ----------------------------------------------------------------------------------
def with_lr_mults(proto, mults):
    """The prototxt with the lr_mult of the weight and of the bias of each layer in mults set to mults[layer]."""
    chunks = proto.split("layer {")
    done = 0
    for i, c in enumerate(chunks):
        m = re.search(r'name:\s*"([^"]+)"', c)
        if m and m.group(1) in mults:
            vals = iter(mults[m.group(1)])
            chunks[i] = re.sub(r"lr_mult:\s*[0-9.eE+-]+", lambda _: "lr_mult: %r" % next(vals), c)
            done += 1
    assert done == len(mults)
    return "layer {".join(chunks)


def test_second_iteration_uses_the_updated_weights(fn2):
    """Solver.step(1) with SGD, then forward and backward again: the gradients and the convolutions' tops match the reference
    at the updated weights, and the reference at the old weights misses them by at least 10 x the tolerance, so a stale
    forward packing, FP16 weight scale or adjoint packing cannot pass.  Gradient-to-weight ratios span four orders of magnitude
    across the layers, so one learning rate that moves every weight tensor would blow up the others: each layer's lr_mult,
    from the gradients of a first pass, moves its weights by about 3 % and its bias by at most as much as its weights."""
    proto, net = make_net(fn2, "FlowNet2-C")
    feed = inputs()
    step(net, feed)
    ref = NetGrad64(proto, None)
    names = ref.trained()
    mults = {}
    for n in names:
        w, gw, gb = (torch.from_numpy(net.param(n, i, diff=d)).double().norm() for i, d in ((0, False), (0, True), (1, True)))
        mults[n] = (float(0.03 * w / gw), float(0.03 * w / max(gw, gb)))
    del net
    gc.collect()
    proto = with_lr_mults(proto, mults)
    net = fn2.Net(proto, None, fn2.TRAIN)
    net.fill_params(11)
    ref = NetGrad64(proto, None)
    assert ref.trained() == names
    old = engine_params(net, ref)
    solver = fn2.get_solver('type: "SGD"\nbase_lr: 1\nlr_policy: "fixed"\n', net)
    solver.step(1, feed=lambda: feed)
    new = engine_params(net, ref)
    moved = {n: float((new[n][0] - old[n][0]).norm() / old[n][0].norm()) for n in names}
    print("\nrelative weight change min %.3g max %.3g" % (min(moved.values()), max(moved.values())))
    assert min(moved.values()) >= 0.01, moved
    out = step(net)
    blobs = EngineBlobs(net)
    worst, stale = {}, {}
    for params, w in ((new, worst), (old, stale)):
        ref.params = params
        _, P = ref.backward(blobs, keep=())
        for name, grads in P.items():
            for i, g in enumerate(grads):
                w["%s[%d]" % (name, i)] = rel(torch.from_numpy(net.param(name, i, diff=True)), g)
        del P
        check_forwards(ref, names, blobs, w)
    ref.params = new
    check_losses(ref, blobs, out, worst)
    grad_miss = max(v for k, v in stale.items() if not k.startswith("fwd "))
    fwd_miss = max(v for k, v in stale.items() if k.startswith("fwd "))
    print("reference at the old weights: worst gradient miss %.3g, worst forward miss %.3g" % (grad_miss, fwd_miss))
    report("FlowNet2-C, second iteration", worst, limit)
    assert grad_miss >= 10 * GRAD_TOL and fwd_miss >= 10 * FWD_TOL
