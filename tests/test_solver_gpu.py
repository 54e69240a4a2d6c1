"""The solver on the GPU: the fused update against the float32 restatement of Caffe's update (tests/solver_oracle.py) bit for
bit, on synthetic arenas and on the FlowNet2-C training graph; snapshot and resume; the frozen stages of a stacked network;
callback order; allocations; and that training lowers the loss."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle.net import get, getall, parse_prototxt
from tests import solver_oracle as SO
from tests.util import rng, smooth_images

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


# ---- helpers ----
def learnable(fn2, net):
    """Net::learnable_params order: [(layer, index, count, arena offset)], the arena padding every blob to 64 floats."""
    out, off = [], 0
    shape = (C.c_int * 4)()
    for name in net.layer_names:
        i = 0
        while fn2.lib().fn2_net_param_shape(net._h, name.encode(), i, shape) == 0:
            n = int(np.prod(list(shape)))
            out.append((name, i, n, off))
            off += (n + 63) // 64 * 64
            i += 1
    return out


def multipliers(net, text):
    """{(layer, index): (lr_mult, decay_mult)} from the prototxt's ParamSpecs (default 1); DataAugmentation's blobs are state,
    lr_mult 0 (data_augmentation_layer.cpp:48-65)."""
    layers = {get(l, "name").strip('"'): l for l in getall(parse_prototxt(text), "layer")}
    out = {}
    for name, typ in zip(net.layer_names, net.layer_types):
        specs = getall(layers[name], "param") if name in layers else []
        for i in range(8):
            if typ == "DataAugmentation":
                out[(name, i)] = (0.0, 0.0)
            elif i < len(specs):
                out[(name, i)] = (float(get(specs[i], "lr_mult", 1)), float(get(specs[i], "decay_mult", 1)))
            else:
                out[(name, i)] = (1.0, 1.0)
    return out


def arenas(fn2, net):
    from flownet2_b200 import parallel
    net.sync()
    return parallel.arena_tensor(net).cpu().numpy().copy(), parallel.grad_arena_tensor(net).cpu().numpy().copy()


def history(solver, params, adam):
    st = SO.parse_state(solver.state())
    h = [d for _, d in st["history"]]
    assert len(h) == len(params) * (2 if adam else 1)
    return h[:len(params)], (h[len(params):] if adam else [None] * len(params)), st


def check_update(p, it, cs, params, mults, before, grads, h_before, after, h_after, clip=None):
    """Every trainable blob: the restatement of the update of (data, diff, history) before equals the engine's after, bit for
    bit.  Frozen blobs: data unchanged, history zero."""
    (w0, _), (w1, g1) = before, after
    rate, _ = SO.learning_rate(p, it, cs)
    trainable = [k for k, (name, i, n, off) in enumerate(params) if mults[(name, i)][0] != 0]
    scale = None
    if clip is not None:                 # the engine's own scale: test_device_clip_scale_is_within_1e6_of_float64
        scale = SO.clip_scale([grads[params[k][3]:params[k][3] + params[k][2]] for k in trainable], clip)
    for k, (name, i, n, off) in enumerate(params):
        sl = slice(off, off + n)
        lr, dm = mults[(name, i)]
        if lr == 0:
            assert np.array_equal(w1[sl], w0[sl], equal_nan=True), name
            assert not np.any(h_after[0][k]) and (h_after[1][k] is None or not np.any(h_after[1][k])), name
            continue
        w, g, m, v = SO.update(p, rate, it, w0[sl], grads[sl], h_before[0][k], h_before[1][k], lr, dm, scale)
        assert w.tobytes() == w1[sl].tobytes(), (name, i, "data")
        assert g.tobytes() == g1[sl].tobytes(), (name, i, "diff")
        assert m.tobytes() == h_after[0][k].tobytes(), (name, i, "history")
        if v is not None:
            assert v.tobytes() == h_after[1][k].tobytes(), (name, i, "v")


# ---- 1. the update operator on synthetic arenas ----
ARENA_NET = (
    'layer { name: "in" type: "Input" top: "x" input_param { shape { dim: 1 dim: 3 dim: 8 dim: 8 } } }\n'
    'layer { name: "c1" type: "Convolution" bottom: "x" top: "y" param { lr_mult: 1 decay_mult: 1 } '
    'param { lr_mult: 2 decay_mult: 0 } convolution_param { num_output: 37 kernel_size: 3 } }\n'
    'layer { name: "c2" type: "Convolution" bottom: "y" top: "z2" param { lr_mult: 0 } param { lr_mult: 0 } '
    'convolution_param { num_output: 5 kernel_size: 3 } }\n'
    'layer { name: "c3" type: "Convolution" bottom: "y" top: "z3" param { lr_mult: 0.5 decay_mult: 3 } '
    'param { lr_mult: 1 decay_mult: 1 } convolution_param { num_output: 130 kernel_size: 5 } }\n'
    'layer { name: "d1" type: "Deconvolution" bottom: "y" top: "z4" '
    'convolution_param { num_output: 6 kernel_size: 4 stride: 2 } }\n')

CASES = {
    "sgd_m0_l2": dict(type="SGD", momentum=0.0, reg="L2", iter_size=1, clip=None),
    "sgd_m09_l1_iter3_clip": dict(type="SGD", momentum=0.9, reg="L1", iter_size=3, clip=0.5),
    "sgd_m09_l2_clip_inactive": dict(type="SGD", momentum=0.9, reg="L2", iter_size=1, clip=1e6),
    "adam_l2": dict(type="Adam", momentum=0.9, reg="L2", iter_size=1, clip=None),
    "adam_l1_iter3_clip": dict(type="Adam", momentum=0.9, reg="L1", iter_size=3, clip=0.5),
    "adam_l2_iter3": dict(type="Adam", momentum=0.8, reg="L2", iter_size=3, clip=None),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_update_is_the_restatement_bit_for_bit(fn2, case):
    from flownet2_b200 import parallel
    c = CASES[case]
    text = ('type: "%s"\nbase_lr: 0.05\nlr_policy: "step"\ngamma: 0.5\nstepsize: 3\nmomentum: %r\nmomentum2: 0.999\n'
            'delta: 1e-8\nweight_decay: 0.01\nregularization_type: "%s"\niter_size: %d\n'
            % (c["type"], c["momentum"], c["reg"], c["iter_size"]))
    if c["clip"] is not None:
        text += "clip_gradients: %r\n" % c["clip"]
    net = fn2.Net(ARENA_NET, None, fn2.TRAIN)
    net.fill_params(5)
    params, mults = learnable(fn2, net), multipliers(net, ARENA_NET)
    r = rng(77)
    data, grads = parallel.arena_tensor(net), parallel.grad_arena_tensor(net)
    data.copy_(torch.from_numpy(r.standard_normal(data.numel()).astype(np.float32)))
    grads.copy_(torch.from_numpy((0.1 * r.standard_normal(grads.numel())).astype(np.float32)))
    data.view(-1)[params[0][3]] = 0.0                                       # sign(0) = 0 under L1
    torch.cuda.synchronize()
    net.params_changed()
    solver = fn2.get_solver(text, net)
    adam = c["type"] == "Adam"
    hist = [r.standard_normal(n).astype(np.float32) * 0.01 for _, _, n, _ in params]
    hist += [np.abs(r.standard_normal(n)).astype(np.float32) * 1e-4 for _, _, n, _ in params] if adam else []
    shapes = [[n] for _, _, n, _ in params] * (2 if adam else 1)
    solver.restore(SO.write_state(7, 0, "", list(zip(shapes, hist))))
    assert solver.iter == 7
    h0, h1, _ = history(solver, params, adam)
    for k, (name, i, n, off) in enumerate(params):                          # frozen blobs keep a zero history
        if mults[(name, i)][0] == 0:
            assert not np.any(h0[k])
    before = arenas(fn2, net)
    fn2.check(fn2.lib().fn2_solver_apply_update(solver._h))
    after = arenas(fn2, net)
    ha0, ha1, st = history(solver, params, adam)
    assert st["iter"] == 8 and st["current_step"] == 7 // 3
    p = fn2.solver_params(text)
    check_update(p, 7, 0, params, mults, before, before[1], (h0, h1), after, (ha0, ha1), clip=c["clip"])
    # the padding between blobs keeps its values (a blob's last float4 stores back the pad floats it loaded)
    pad = np.ones(before[0].size, bool)
    for _, _, n, off in params:
        pad[off:off + n] = False
    assert np.array_equal(after[0][pad], before[0][pad]) and np.array_equal(after[1][pad], before[1][pad])


# ---- 2. the FlowNet2-C training graph ----
CW, CH, DW, DH, BATCH = 192, 128, 224, 160, 2


def feeder(seed=12):
    img0, img1 = smooth_images(rng(seed), BATCH, DH, DW)
    gt = (3 * rng(seed + 1).standard_normal((BATCH, 2, DH, DW))).astype(np.float32)
    return lambda: {"img0": img0, "img1": img1, "flow_gt": gt}


def test_flownet2c_adam_iterations_are_the_restatement(fn2):
    from flownet2_b200 import parallel
    proto = fn2.fill_train_template(fn2.train_template("FlowNet2-C"), CW, CH, DW, DH, BATCH)
    net = fn2.Net(proto, None, fn2.TRAIN)
    net.fill_params(11)
    text = ('type: "Adam"\nbase_lr: 1e-3\nlr_policy: "multistep"\ngamma: 0.5\nstepvalue: 2\nmomentum: 0.9\nmomentum2: 0.999\n'
            'weight_decay: 0.0004\niter_size: 2\nmax_iter: 3\n')
    solver = fn2.get_solver(text, net)
    params, mults = learnable(fn2, net), multipliers(net, proto)
    assert any(m[0] == 0 for m in mults.values()) and sum(1 for k in params if mults[k[:2]][0] != 0) > 20
    p = fn2.solver_params(text)
    seen = {}

    def ready():
        net.sync()
        seen["grads"] = parallel.grad_arena_tensor(net).cpu().numpy().copy()
        seen["data"] = parallel.arena_tensor(net).cpu().numpy().copy()
        seen["hist"] = history(solver, params, True)

    solver.add_callback(lambda: None, ready)
    cs = 0
    for it in range(3):
        solver.step(1, feeder())
        after = arenas(fn2, net)
        ha0, ha1, st = history(solver, params, True)
        h0, h1, _ = seen["hist"]
        check_update(p, it, cs, params, mults, (seen["data"], None), seen["grads"], (h0, h1), after, (ha0, ha1))
        _, cs = SO.learning_rate(p, it, cs)
        assert st["iter"] == it + 1 and st["current_step"] == cs
    assert cs == 1 and np.isfinite(solver.smoothed_loss)


# ---- 3. snapshot and resume ----
SMALL_NET = (
    'layer { name: "data" type: "Input" top: "img" top: "gt" input_param { shape { dim: 2 dim: 3 dim: 16 dim: 16 } '
    'shape { dim: 2 dim: 2 dim: 16 dim: 16 } } }\n'
    'layer { name: "conv1" type: "Convolution" bottom: "img" top: "h" convolution_param { num_output: 8 kernel_size: 3 pad: 1 '
    'weight_filler { type: "gaussian" std: 0.2 } bias_filler { type: "constant" value: 0.1 } } }\n'
    'layer { name: "relu1" type: "ReLU" bottom: "h" top: "h" }\n'
    'layer { name: "conv2" type: "Convolution" bottom: "h" top: "pred" param { lr_mult: 1 decay_mult: 1 } '
    'param { lr_mult: 2 decay_mult: 0 } convolution_param { num_output: 2 kernel_size: 3 pad: 1 '
    'weight_filler { type: "gaussian" std: 0.2 } } }\n'
    'layer { name: "loss" type: "L1Loss" bottom: "pred" bottom: "gt" top: "loss" }\n')
ADAM = ('type: "Adam"\nbase_lr: 0.01\nlr_policy: "multistep"\ngamma: 0.5\nstepvalue: 3\nstepvalue: 7\nmomentum: 0.9\n'
        'momentum2: 0.999\nweight_decay: 0.001\nmax_iter: 10\n')


def small_feed():
    r = rng(5)
    img = r.standard_normal((2, 3, 16, 16)).astype(np.float32)
    gt = (img[:, :2] * 0.5 - img[:, 2:] * 0.25).astype(np.float32)
    return lambda: {"img": img, "gt": gt}


def small(fn2, solver_text, seed=3):
    net = fn2.Net(SMALL_NET, None, fn2.TRAIN)
    net.fill_params(seed)
    return net, fn2.get_solver(solver_text, net)


def test_resume_is_bit_identical(fn2, tmp_path):
    prefix = str(tmp_path / "snap")
    net_a, sol_a = small(fn2, ADAM)
    sol_a.step(10, small_feed())
    net_b, sol_b = small(fn2, ADAM + 'snapshot: 5\nsnapshot_prefix: "%s"\n' % prefix)
    sol_b.step(5, small_feed())
    model, state = prefix + "_iter_5.caffemodel", prefix + "_iter_5.solverstate"
    assert os.path.exists(model) and os.path.exists(state)
    st = SO.parse_state(open(state, "rb").read())
    params = learnable(fn2, net_b)
    assert st["iter"] == 5 and st["current_step"] == 1 and st["learned_net"] == model
    assert [int(np.prod(s)) for s, _ in st["history"]] == [n for _, _, n, _ in params] * 2        # m of each, then v of each
    assert [s for s, _ in st["history"][:4]] == [[8, 3, 3, 3], [8], [2, 8, 3, 3], [2]]
    net_c, sol_c = small(fn2, ADAM, seed=99)                               # fresh weights, overwritten by the snapshot
    sol_c.restore(state)
    assert sol_c.iter == 5
    sol_c.step(5, small_feed())
    assert arenas(fn2, net_c)[0].tobytes() == arenas(fn2, net_a)[0].tobytes()
    assert sol_c.state() == sol_a.state() and net_c.to_caffemodel() == net_a.to_caffemodel()


def test_caffe_pb2_solverstate_restores(fn2):
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    raw = open(os.path.join(gold, "ref_pb2_solverstate.bin"), "rb").read()
    proto = ('layer { name: "in" type: "Input" top: "x" input_param { shape { dim: 1 dim: 3 dim: 6 dim: 6 } } }\n'
             'layer { name: "a" type: "Convolution" bottom: "x" top: "y" convolution_param { num_output: 4 kernel_size: 3 } }\n'
             'layer { name: "b" type: "Convolution" bottom: "y" top: "z" convolution_param { num_output: 2 kernel_size: 1 } }\n')
    net = fn2.Net(proto, None, fn2.TRAIN)
    net.fill_params(1)
    solver = fn2.get_solver('type: "Adam"\nbase_lr: 0.1\nlr_policy: "fixed"\n', net)
    buf = (C.c_char * len(raw)).from_buffer_copy(raw)
    fn2.check(fn2.lib().fn2_solver_restore(solver._h, buf, len(raw)))
    assert solver.iter == 1234
    assert solver.state("snap/flow_iter_1234.caffemodel") == raw               # iter, current_step and every history value
    sgd = fn2.get_solver('type: "SGD"\nbase_lr: 0.1\nlr_policy: "fixed"\n', net)
    with pytest.raises(fn2.Fn2Error, match="Incorrect length of history blobs"):
        fn2.check(fn2.lib().fn2_solver_restore(sgd._h, buf, len(raw)))


# ---- 4. frozen predecessors ----
def test_frozen_stage_is_untouched_under_adam_with_decay(fn2):
    proto = fn2.fill_train_template(fn2.train_template("FlowNet2-CS"), CW, CH, DW, DH, BATCH)
    net = fn2.Net(proto, None, fn2.TRAIN)
    net.fill_params(21)
    params, mults = learnable(fn2, net), multipliers(net, proto)
    frozen = [k for k, (name, i, n, off) in enumerate(params) if name.startswith("net1_")]
    assert frozen and all(mults[params[k][:2]][0] == 0 for k in frozen)
    w0 = arenas(fn2, net)[0]
    solver = fn2.get_solver('type: "Adam"\nbase_lr: 1e-3\nlr_policy: "fixed"\nweight_decay: 0.0004\nmomentum: 0.9\n', net)
    solver.step(2, feeder())
    w1 = arenas(fn2, net)[0]
    h0, h1, _ = history(solver, params, True)
    for k in frozen:
        name, i, n, off = params[k]
        assert w1[off:off + n].tobytes() == w0[off:off + n].tobytes(), name
        assert not np.any(h0[k]) and not np.any(h1[k]), name
    trained = [k for k, (name, i, n, off) in enumerate(params) if name.startswith("net2_")]
    assert any(w1[params[k][3]:params[k][3] + params[k][2]].tobytes() != w0[params[k][3]:params[k][3] + params[k][2]].tobytes()
               for k in trained)


# ---- 5. callback order ----
def test_gradients_zeroed_in_the_callback_leave_the_parameters(fn2):
    from flownet2_b200 import parallel
    net, solver = small(fn2, 'type: "SGD"\nbase_lr: 0.1\nlr_policy: "fixed"\nmomentum: 0.9\n')
    w0 = arenas(fn2, net)[0]
    calls = []
    solver.add_callback(lambda: calls.append("start"),
                        lambda: (calls.append("ready"), parallel.grad_arena_tensor(net).zero_(), torch.cuda.synchronize()))
    solver.step(2, small_feed())
    assert calls == ["start", "ready"] * 2
    assert arenas(fn2, net)[0].tobytes() == w0.tobytes()


# ---- 6. allocations ----
def test_warm_steps_allocate_nothing_and_destroy_frees(fn2):
    net = fn2.Net(SMALL_NET, None, fn2.TRAIN)
    net.fill_params(3)
    feed = small_feed()
    net.clear_param_diffs()
    net.forward(**feed())
    net.backward()                                        # the net's own lazy buffers
    live0 = fn2.device_allocations()[1]
    solver = fn2.get_solver(ADAM + "clip_gradients: 1\n", net)
    assert fn2.device_allocations()[1] > live0
    solver.step(1, feed)
    n1 = fn2.device_allocations()[0]
    solver.step(3, feed)
    assert fn2.device_allocations()[0] == n1
    del solver
    assert fn2.device_allocations()[1] == live0


# ---- 7. learning ----
def test_adam_overfits_one_batch(fn2):
    net, solver = small(fn2, 'type: "Adam"\nbase_lr: 0.01\nlr_policy: "fixed"\nmomentum: 0.9\nmomentum2: 0.999\n')
    feed = small_feed()
    solver.step(1, feed)
    start = solver.smoothed_loss
    solver.step(49, feed)
    assert solver.iter == 50 and solver.smoothed_loss < 0.5 * start, (start, solver.smoothed_loss)


def test_device_clip_scale_is_within_1e6_of_float64(fn2):
    """The engine's own scale, read off the update: SGD with lr 1, no momentum or decay makes the applied diff g * scale."""
    from flownet2_b200 import parallel
    net = fn2.Net(ARENA_NET, None, fn2.TRAIN)
    net.fill_params(5)
    params, mults = learnable(fn2, net), multipliers(net, ARENA_NET)
    grads = parallel.grad_arena_tensor(net)
    grads.copy_(torch.from_numpy((0.1 * rng(78).standard_normal(grads.numel())).astype(np.float32)))
    torch.cuda.synchronize()
    solver = fn2.get_solver('type: "SGD"\nbase_lr: 1\nlr_policy: "fixed"\nclip_gradients: 0.5\n', net)
    g0 = arenas(fn2, net)[1]
    fn2.check(fn2.lib().fn2_solver_apply_update(solver._h))
    g1 = arenas(fn2, net)[1]
    trainable = [np.arange(off, off + n) for name, i, n, off in params if mults[(name, i)][0] == 1]
    idx = np.concatenate(trainable)
    k = idx[np.argmax(np.abs(g0[idx]))]
    engine_scale = float(g1[k]) / float(g0[k])                  # g * scale rounded once: within 2^-24 of the scale
    exact = 0.5 / np.sqrt(sum(float(np.dot(g0[off:off + n].astype(np.float64), g0[off:off + n].astype(np.float64)))
                              for name, i, n, off in params if mults[(name, i)][0] != 0))
    assert exact < 1 and abs(engine_scale - exact) <= 1e-6 * exact, (engine_scale, exact)
