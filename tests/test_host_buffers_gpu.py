"""Host side of the Caffe-surface net: every gradient-accumulation route, and device memory.

Net::PlanBackward tells each layer, per bottom, whether to overwrite the bottom diff or add to it. Each accumulate case below
builds a net where input blob `a` (and `b`) feeds the layer under test and a second consumer, an Eltwise that runs first in
the backward pass, so the layer under test adds. The expected diff is the sum of the two contributions, each taken from a net
with only that consumer. Where the add is fn2_axpby(1, s, 1, d) the match is bit-exact; Eltwise fuses its coefficient into the
add (fmaf(coeff, dy, dx)), which may differ from the separately rounded sum by one float32 rounding.

The memory tests read fn2_device_allocations: a warm training step or deploy forward allocates nothing, and destroying the nets
returns every byte.
"""
import gc

import numpy as np
import pytest

from tests.util import rng, smooth_images

pytestmark = pytest.mark.gpu

N, H, W = 2, 12, 16


def _input(names_channels):
    shapes = "".join(" shape { dim: %d dim: %d dim: %d dim: %d }" % (N, c, H, W) for _, c in names_channels)
    tops = "".join(' top: "%s"' % n for n, _ in names_channels)
    return 'force_backward: true\nlayer { name: "in" type: "Input"%s input_param {%s } }\n' % (tops, shapes)


# the second consumer: runs after the layer under test in the forward pass, so first in the backward pass
SHARED = 'layer { name: "shared" type: "Eltwise" %s top: "e" eltwise_param { operation: SUM %s } }\n'

CORR = ('layer { name: "corr" type: "Correlation" bottom: "a" bottom: "b" top: "t" correlation_param { pad: %d kernel_size: %d '
        'max_displacement: %d stride_1: 1 stride_2: %d } }\n')
CONV = ('layer { name: "conv" type: "%s" bottom: "a" top: "t" convolution_param { num_output: %d kernel_size: %d stride: %d '
        'pad: %d weight_filler { type: "gaussian" std: 0.1 } bias_filler { type: "constant" value: 0.1 } } }\n')

# name -> (inputs, layer(s) under test, seeded tops, bottoms the second consumer shares, fused-scale tolerance)
CASES = {
    "relu": ([("a", 8)], 'layer { name: "relu" type: "ReLU" bottom: "a" top: "t" relu_param { negative_slope: 0.1 } }\n',
             ["t"], ["a"], False),
    "eltwise": ([("a", 8)], 'layer { name: "scale" type: "Eltwise" bottom: "a" top: "t" eltwise_param { operation: SUM coeff: -0.7 } }\n',
                ["t"], ["a"], True),
    "slice": ([("a", 8)], 'layer { name: "slice" type: "Slice" bottom: "a" top: "t" top: "t2" slice_param { axis: 1 slice_point: 3 } }\n',
              ["t", "t2"], ["a"], False),
    "concat_copy": ([("a", 6), ("b", 5)], 'layer { name: "cat" type: "Concat" bottom: "a" bottom: "b" top: "t" }\n',
                    ["t"], ["a"], False),
    # FlowNet2-C's geometry (k 1, pad = md = 20, stride_2 2, C % 32 == 0, channel-fast): the fast backward route
    "corr_fast": ([("a", 32), ("b", 32)], CORR % (20, 1, 20, 2), ["t"], ["a", "b"], False),
    "corr_tiled": ([("a", 12), ("b", 12)], CORR % (4, 3, 3, 1), ["t"], ["a", "b"], False),
    "conv": ([("a", 32)], CONV % ("Convolution", 24, 3, 1, 1), ["t"], ["a"], False),
    # 20 bottom channels: the adjoint convolution pads Co to 32 and runs through the scratch blob in any case
    "conv_pad_co": ([("a", 20)], CONV % ("Convolution", 24, 3, 2, 1), ["t"], ["a"], False),
    "conv_relu": ([("a", 32)], CONV % ("Convolution", 32, 3, 1, 1) +
                  'layer { name: "relu" type: "ReLU" bottom: "t" top: "t" relu_param { negative_slope: 0.1 } }\n',
                  ["t"], ["a"], False),
    "deconv": ([("a", 16)], CONV % ("Deconvolution", 8, 4, 2, 1), ["t"], ["a"], False),
    "deconv_20": ([("a", 20)], CONV % ("Deconvolution", 8, 4, 2, 1), ["t"], ["a"], False),
}


def _shared(bottoms):
    return SHARED % (" ".join('bottom: "%s"' % b for b in bottoms), " ".join("coeff: %g" % c for c in (3, -2)[:len(bottoms)]))


def _grads(fn2, proto, inputs, seeds, weights=None):
    """Input diffs of a net seeded with the tops of `seeds` it has."""
    net = fn2.Net(proto, None, fn2.TEST)
    if weights is not None:
        net.copy_from(weights)
    net.forward(**inputs)
    net.backward(**{k: v for k, v in seeds.items() if k in net.blob_names})
    return {k: net.get_diff(k) for k in inputs}


@pytest.mark.parametrize("case", sorted(CASES))
def test_layer_accumulates_into_a_shared_bottom(fn2, monkeypatch, case):
    monkeypatch.setenv("FN2_NO_ALIAS", "1")        # Concat runs its copy path
    ins, layer, tops, shared, fused_scale = CASES[case]
    r = rng(41)
    inputs = {n: r.standard_normal((N, c, H, W)).astype(np.float32) for n, c in ins}
    both = _input(ins) + layer + _shared(shared)
    net = fn2.Net(both, None, fn2.TEST)
    net.fill_params(7)
    weights = net.to_caffemodel()
    net.forward(**inputs)
    seeds = {t: r.standard_normal(net.blobs[t].shape).astype(np.float32) for t in tops + ["e"]}
    net.backward(**seeds)
    got = {n: net.get_diff(n) for n in inputs}

    g_layer = _grads(fn2, _input(ins) + layer, inputs, seeds, weights)
    g_shared = _grads(fn2, _input(ins) + _shared(shared), inputs, seeds)
    for n in shared:
        want = g_shared[n] + g_layer[n]
        assert np.abs(g_layer[n]).max() > 0 and np.abs(g_shared[n]).max() > 0
        if fused_scale:
            # fmaf(coeff, dy, dx) against fl(fl(coeff * dy) + dx): at most the rounding of the product plus one of the sum
            tol = np.spacing(np.abs(g_layer[n])) + np.spacing(np.abs(want))
            assert (np.abs(got[n] - want) <= tol).all(), case
        else:
            assert np.array_equal(got[n], want), (case, n, float(np.abs(got[n] - want).max()))
    for n in set(inputs) - set(shared):          # bottoms only the layer under test reads: overwritten, not added
        assert np.array_equal(got[n], g_layer[n]), (case, n)


def test_flow_warp_refuses_a_shared_bottom(fn2):
    proto = (_input([("a", 3), ("f", 2)]) +
             'layer { name: "warp" type: "FlowWarp" bottom: "a" bottom: "f" top: "t" }\n' + _shared(["a"]))
    net = fn2.Net(proto, None, fn2.TEST)
    r = rng(42)
    net.forward(a=r.standard_normal((N, 3, H, W)).astype(np.float32), f=r.standard_normal((N, 2, H, W)).astype(np.float32))
    with pytest.raises(fn2.Fn2Error, match="FlowWarp backward into a shared bottom is not supported"):
        net.backward(t=np.ones((N, 3, H, W), np.float32), e=np.ones((N, 3, H, W), np.float32))


def _allocations_during(fn2, run):
    before, _ = fn2.device_allocations()
    run()
    return fn2.device_allocations()[0] - before


def test_warm_steps_allocate_nothing_and_nets_free_everything(fn2):
    gc.collect()
    _, live_before = fn2.device_allocations()

    # the FlowNet2-C training step of test_train_gpu.test_flownet_c_training_net_step
    cw, ch, dw, dh, batch = 192, 128, 224, 160, 2
    train = fn2.Net(fn2.fill_train_template(fn2.train_template("FlowNet2-C"), cw, ch, dw, dh, batch), None, fn2.TRAIN)
    train.fill_params(11)
    img0, img1 = smooth_images(rng(12), batch, dh, dw)
    gt = (3 * rng(13).standard_normal((batch, 2, dh, dw))).astype(np.float32)
    for name, value in (("img0", img0), ("img1", img1), ("flow_gt", gt)):
        train.set_input(name, value)

    def step():
        train.forward_async()
        train.backward_async()
        train.sync()
    train.clear_param_diffs()
    step()                                                   # warm-up: workspaces, scratch blobs, gradient storage
    assert _allocations_during(fn2, step) == 0
    assert np.isfinite(train.get_diff("predict_flow2")).all()    # host transfers allocate their own temporaries

    deploy = fn2.Net(fn2.fill_template(fn2.model_template("FlowNet2-C"), 128, 96), None, fn2.TEST, batch=1)
    deploy.fill_params(1701)
    r = rng(14)
    deploy.set_input("img0", np.round(r.uniform(0, 255, (1, 3, 96, 128))).astype(np.float32))
    deploy.set_input("img1", np.round(r.uniform(0, 255, (1, 3, 96, 128))).astype(np.float32))

    def forward():
        deploy.forward_async()
        deploy.sync()
    forward()
    assert _allocations_during(fn2, forward) == 0
    assert _allocations_during(fn2, forward) == 0            # the graph replay, if the net captured one
    assert np.isfinite(deploy.blobs["predict_flow_final"].data).all()

    _, live = fn2.device_allocations()
    assert live > live_before
    del train, deploy
    gc.collect()
    assert fn2.device_allocations()[1] == live_before
