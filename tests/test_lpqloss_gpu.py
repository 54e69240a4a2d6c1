"""GPU: LpqLoss (fn2_lpqloss_forward / backward, include/fn2_lpq.h, and the LpqLoss layer) against the REFERENCE's own layer
(tests/golden/lpq_golden.npz) and the oracle; views, accumulation, the setup checks, and the p/q schedule following the Solver's
iteration through CUDA-graph replays, restores and iter_size."""
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import lpq_cases as LC  # noqa: E402
import train_cases as TC  # noqa: E402
from oracle import oracle as O  # noqa: E402
from tests import lpq_oracle as LO  # noqa: E402
from tests.refcheck import TRAIN_TOL  # noqa: E402
from tests.util import device_view, maxabs, rng  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(HERE, "golden", "lpq_golden.npz")
TOL = 5 * TRAIN_TOL["l1loss"]                     # what the L1Loss layer test allows against the reference and the oracle


def rel(got, want):
    return maxabs(got, want) / max(float(np.nanmax(np.abs(np.asarray(want, np.float64)))), 1e-30)


@pytest.fixture(scope="module")
def gold():
    assert os.path.exists(GOLD), "tests/golden/lpq_golden.npz is missing"
    return np.load(GOLD)


def kinks(bots):
    d = bots[0] - bots[1] if len(bots) > 1 else bots[0]
    return d == 0


def oracle_out(name, zero_at_kink=True):
    c = LC.LPQ_CASES[name]
    bots = LC.lpq_inputs(name)
    b1 = bots[1] if len(bots) > 1 else None
    loss, _ = LO.lpqloss_fwd(bots[0], b1, **c["args"])
    g = LO.lpqloss_bwd(bots[0], b1, c["top_diff"], zero_at_kink=zero_at_kink, **c["args"])
    out = {"top0": np.array([loss], np.float32), "bdiff0": g[0]}
    if b1 is not None:
        out["bdiff1"] = g[1]
    return out


def single_layer_net(fn2, text, bottoms):
    names = re.findall(r'bottom:\s*"([^"]+)"', text)
    shapes = "".join(" shape { %s }" % " ".join("dim: %d" % d for d in b.shape) for b in bottoms)
    proto = ('force_backward: true\nlayer { name: "in" type: "Input" %s input_param {%s } }\nlayer { %s }\n'
             % (" ".join('top: "%s"' % n for n in names), shapes, text))
    return fn2.Net(proto, None, fn2.TEST), names


@pytest.mark.parametrize("name", list(LC.LPQ_CASES))
def test_layer_matches_reference_and_oracle(fn2, gold, name):
    c = LC.LPQ_CASES[name]
    bots = LC.lpq_inputs(name)
    net, names = single_layer_net(fn2, c["text"], bots)
    top = net.outputs[0]
    out = {"top0": net.forward(**dict(zip(names, bots)))[top].reshape(1)}
    net.backward(**{top: np.full(net.blobs[top].shape, c["top_diff"], np.float32)})
    for i, n in enumerate(names):
        out["bdiff%d" % i] = net.get_diff(n)
    k = kinks(bots)
    want_o = oracle_out(name)
    for key, got in out.items():
        ref = np.asarray(gold["L/%s/%s" % (name, key)])
        if c["deviation"] and key != "top0":
            # the reference's 0 / 0: NaN exactly at the exact-zero differences, where the engine writes 0
            assert np.array_equal(np.isnan(ref), k) and k.sum() >= 5
            assert np.all(got[k] == 0)
            ref = np.where(k, np.float32(0), ref)
        for label, want in (("oracle", want_o[key]), ("reference", ref)):
            assert rel(np.asarray(got).reshape(want.shape), want) <= TOL, (name, key, label, rel(got, want))


@pytest.mark.parametrize("layout", ["nchw", "nhwc", "pad", "slice"])
@pytest.mark.parametrize("name", ["lpq_1_04_norm", "lpq_c3"])
def test_kernels_on_views(fn2, layout, name):
    """Strided, channel-padded and concat-child views of both bottoms and both diffs; accumulate and overwrite."""
    import torch
    from flownet2_b200 import ops
    c = LC.LPQ_CASES[name]
    a = c["args"]
    kw = {k: a[k] for k in ("p_epsilon", "q_epsilon", "l2_prescale_by_channels", "normalize_by_num_entries")}
    b0, b1 = LC.lpq_inputs(name)
    want = oracle_out(name)
    v0, v1 = device_view(b0, layout), device_view(b1, layout)
    loss, state = ops.lpqloss(v0, v1, p=a["p"], q=a["q"], **kw)
    assert rel(loss.cpu().numpy(), want["top0"]) <= TOL
    st = state.cpu().numpy()
    assert st[4] == np.float32(a["p"]) and st[5] == np.float32(a["q"]) and st[3] == float((~np.isnan(b0 - b1)).sum())
    top = torch.tensor([c["top_diff"]], device="cuda")
    base = np.random.default_rng(3).standard_normal(b0.shape).astype(np.float32)
    o0, o1 = device_view(base, layout), device_view(base, layout)
    ops.lpqloss_backward(v0, v1, state=state, top_diff=top, out0=o0, out1=o1, accumulate0=True, accumulate1=False, **kw)
    torch.cuda.synchronize()
    assert rel(o0.cpu().numpy() - base, want["bdiff0"]) <= TOL
    assert rel(o1.cpu().numpy(), want["bdiff1"]) <= TOL
    if layout == "slice":                             # the channels outside the view keep their NaN
        assert torch.isnan(o0._base if o0._base is not None else o0).any()


def test_accumulates_into_a_bottom_shared_with_l1loss(fn2):
    proto = ('force_backward: true\n'
             'layer { name: "in" type: "Input" top: "a" top: "gt" input_param { shape { dim: 2 dim: 2 dim: 6 dim: 8 } shape { dim: 2 dim: 2 dim: 6 dim: 8 } } }\n'
             'layer { name: "l1" type: "L1Loss" bottom: "a" bottom: "gt" top: "loss1" loss_weight: 0.5 l1_loss_param { l2_per_location: true } }\n'
             'layer { name: "lpq" type: "LpqLoss" bottom: "a" bottom: "gt" top: "loss2" loss_weight: 2 lpq_loss_param { p: 2 q: 0.4 } }\n')
    net = fn2.Net(proto, None, fn2.TEST)
    r = rng(21)
    a = r.standard_normal((2, 2, 6, 8)).astype(np.float32)
    gt = r.standard_normal((2, 2, 6, 8)).astype(np.float32)
    gt[1, :, 2, 3] = np.nan
    out = net.forward(a=a, gt=gt)
    l2, _ = LO.lpqloss_fwd(a, gt, p=2, q=0.4)
    assert abs(float(out["loss2"].reshape(-1)[0]) - l2) <= 1e-5 * l2
    net.backward()
    g1, h1 = O.l1loss_bwd(a, gt, 0.5, l2_per_location=True)
    g2, h2 = LO.lpqloss_bwd(a, gt, 2.0, p=2, q=0.4)
    assert maxabs(net.get_diff("a"), g1 + g2) <= 1e-6 and maxabs(net.get_diff("gt"), h1 + h2) <= 1e-6


@pytest.mark.parametrize("param,msg", [
    ("p: 1 p: 2 q: 1 q: 1 pq_episode_starts_at_iter: 0", r"Incompatible sizes: \(pq_episode_starts_at_iter -> 1, p -> 2, q -> 2\)"),
    ("p_epsilon: 0.1", "Lpq schedule parameters must not be empty"),
    ("p: 1 p: 2 q: 1 q: 1 pq_episode_starts_at_iter: 0 pq_episode_starts_at_iter: 0",
     "pq_episode_starts_at_frame is not ordered or contains duplicates: 0 0"),
    ("p: 1 p: 2 q: 1 q: 1 pq_episode_starts_at_iter: 2 pq_episode_starts_at_iter: 5",
     "First entry in pq_episode_starts_at_frame is not 0, this is probably a mistake."),
])
def test_setup_checks(fn2, param, msg):
    proto = ('layer { name: "in" type: "Input" top: "a" input_param { shape { dim: 1 dim: 2 dim: 4 dim: 4 } } }\n'
             'layer { name: "lpq" type: "LpqLoss" bottom: "a" top: "loss" lpq_loss_param { %s } }\n' % param)
    with pytest.raises(fn2.Fn2Error, match=msg):
        fn2.Net(proto, None, fn2.TRAIN)


# ---- the schedule over the Solver's iteration -------------------------------------------------------------------------------
SCHEDULE = "p: 1 p: 2 q: 0.4 q: 1 pq_episode_starts_at_iter: 0 pq_episode_starts_at_iter: 3"
SMALL_NET = (
    'layer { name: "data" type: "Input" top: "img" top: "gt" input_param { shape { dim: 2 dim: 3 dim: 16 dim: 16 } '
    'shape { dim: 2 dim: 2 dim: 16 dim: 16 } } }\n'
    'layer { name: "conv1" type: "Convolution" bottom: "img" top: "h" convolution_param { num_output: 8 kernel_size: 3 pad: 1 '
    'weight_filler { type: "gaussian" std: 0.2 } bias_filler { type: "constant" value: 0.1 } } }\n'
    'layer { name: "relu1" type: "ReLU" bottom: "h" top: "h" }\n'
    'layer { name: "conv2" type: "Convolution" bottom: "h" top: "pred" convolution_param { num_output: 2 kernel_size: 3 pad: 1 '
    'weight_filler { type: "gaussian" std: 0.2 } } }\n'
    'layer { name: "loss" type: "LpqLoss" bottom: "pred" bottom: "gt" top: "loss" lpq_loss_param { %s q_epsilon: 0.01 } }\n')


def small_feed():
    r = rng(5)
    img = r.standard_normal((2, 3, 16, 16)).astype(np.float32)
    gt = (img[:, :2] * 0.5 - img[:, 2:] * 0.25).astype(np.float32)
    gt[0, :, 2:5, 3:7] = np.nan
    return lambda: {"img": img, "gt": gt}


def small(fn2, solver_text, lpq=SCHEDULE, seed=3):
    net = fn2.Net(SMALL_NET % lpq, None, fn2.TRAIN)
    net.fill_params(seed)
    return net, fn2.get_solver(solver_text, net)


def step_losses(solver, n, feed):
    out = []
    for _ in range(n):
        solver.step(1, feed)
        out.append(solver.smoothed_loss)
    return out


@pytest.mark.parametrize("iter_size", [1, 2])
def test_schedule_follows_the_solver_in_graph_mode(fn2, iter_size):
    """With the weights held (base_lr 0) every iteration's loss is the constant-(p, q) net's loss of its schedule step; the
    forward is a CUDA-graph replay from the second pass on, so a (p, q) captured into the graph would fail from iteration 3."""
    assert not os.environ.get("FN2_NO_GRAPH")
    text = 'type: "SGD"\nbase_lr: 0\nlr_policy: "fixed"\nmax_iter: 10\niter_size: %d\n' % iter_size
    net, solver = small(fn2, text)
    feed = small_feed()
    assert net.iter == 0
    losses = step_losses(solver, 6, feed)
    assert net.graph_active and net.iter == 5
    want = []
    for pq in ("p: 1 q: 0.4", "p: 2 q: 1"):
        ref, _ = small(fn2, text, lpq=pq)
        want.append(float(ref.forward(**feed())["loss"].reshape(-1)[0]))
    assert want[0] != want[1]
    assert losses == [want[0]] * 3 + [want[1]] * 3, (losses, want)
    pred, gt = net.blobs["pred"].data, feed()["gt"]
    assert abs(want[1] - LO.lpqloss_fwd(pred, gt, p=2, q=1)[0]) <= 1e-5 * want[1]


def test_restore_across_the_boundary_is_bit_identical(fn2, tmp_path):
    text = 'type: "SGD"\nbase_lr: 0.01\nmomentum: 0.9\nlr_policy: "fixed"\nmax_iter: 10\n'
    prefix = str(tmp_path / "snap")
    _, sol_a = small(fn2, text)
    run = step_losses(sol_a, 5, small_feed())
    _, sol_b = small(fn2, text + 'snapshot: 2\nsnapshot_prefix: "%s"\n' % prefix)
    assert step_losses(sol_b, 2, small_feed()) == run[:2]
    net_c, sol_c = small(fn2, text, seed=99)
    sol_c.restore(prefix + "_iter_2.solverstate")
    assert sol_c.iter == 2
    assert step_losses(sol_c, 3, small_feed()) == run[2:]
    # the same net stepped back to an earlier iteration picks the earlier step again
    sol_b.restore(prefix + "_iter_2.solverstate")
    assert step_losses(sol_b, 1, small_feed()) == run[2:3]


def test_warm_steps_allocate_nothing(fn2):
    import ctypes as C
    net, solver = small(fn2, 'type: "SGD"\nbase_lr: 0.01\nlr_policy: "fixed"\nmax_iter: 10\niter_size: 2\n')
    feed = small_feed()
    solver.step(2, feed)
    count = lambda: fn2.lib().fn2_device_allocations(C.byref(C.c_uint64()))
    before = count()
    solver.step(3, feed)                             # crosses the boundary at iteration 3
    assert count() == before and solver.iter == 5


def test_flownet_c_with_lpq_losses_matches_oracle(fn2):
    """The FlowNet2-C graph with its five end-point-error L1Loss layers replaced by LpqLoss (p 1, q 0.4, the fine-tuning loss, and
    p 2, q 0.5), against LpqOracleNet.backward (OracleNet with LpqLoss): losses and every parameter gradient, differentiated at
    the engine's activations."""
    from oracle.net import get, synth_weights
    proto = TC.loss_net_proto()
    n = proto.count('type: "L1Loss"')
    assert n == 5
    proto = proto.replace('type: "L1Loss"', 'type: "LpqLoss"')
    proto = proto.replace("l1_loss_param {\n    l2_per_location: true\n  }", "lpq_loss_param {\n    p: 1\n    q: 0.4\n  }", 3)
    proto = proto.replace("l1_loss_param {\n    l2_per_location: true\n  }", "lpq_loss_param {\n    p: 2\n    q: 0.5\n    l2_prescale_by_channels: true\n  }")
    assert proto.count('type: "LpqLoss"') == 5 and "l1_loss_param" not in proto
    ins = TC.loss_net_inputs()
    small_t = fn2.fill_template(fn2.model_template("FlowNet2-C"), 64, 64)
    _, cm = synth_weights(small_t, TC.LOSS_NET["seed"], fn2.fill_template(fn2.model_template("FlowNet2-C"), TC.LOSS_NET["w"], TC.LOSS_NET["h"]))
    net = fn2.Net(proto, cm, fn2.TEST, batch=TC.LOSS_NET["batch"])
    out = net.forward(**ins)
    onet = LO.LpqOracleNet(proto, cm, batch=TC.LOSS_NET["batch"], f64acc=True)
    B = onet.forward(**ins)
    for k in list(B):
        if k not in ins and not k.startswith("flow_loss"):
            assert maxabs(net.blobs[k].data, B[k]) <= 1e-4 * max(1.0, float(np.abs(B[k]).max())), k
            B[k] = net.blobs[k].data
    for lvl in TC.LOSS_NET["weights"]:
        want = float(LO.lpqloss_fwd(B["predict_flow%d" % lvl], ins["gt%d" % lvl], **LO.lpq_args(
            next(l for l in onet.layers if get(l, "name") == "flow_loss%d" % lvl)))[0])
        got = float(out["flow_loss%d" % lvl].reshape(-1)[0])
        assert abs(got - want) <= 5e-5 * abs(want), (lvl, got, want)
    net.clear_param_diffs()
    net.backward()
    _, P = onet.backward()
    worst = {}
    for lname, grads in P.items():
        for i, g in enumerate(grads):
            worst["%s[%d]" % (lname, i)] = rel(net.param(lname, i, diff=True).reshape(g.shape), g)
    assert len(worst) >= 40
    bad = {k: v for k, v in worst.items() if v > 5e-5}
    assert not bad, bad
