"""The stacked FlowNet2 training schedule without a GPU: the generator reproduces every committed template, the four stage
templates as the reference's own caffe_pb2 reads them (tests/golden/make_stack_train_proto_golden.py) against the engine's
parser, the oracle's need-backward pruning (tests/stack_oracle.py), and the all-reduce of the trainable span of the gradient
arena under gloo."""
import importlib.util
import json
import os

import numpy as np
import pytest

from oracle import net as onet
from oracle.net import OracleNet, get, getall
from tests.stack_oracle import PrunedOracleNet
from tests.test_host_cpu import canonical
from tests.util import rng

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
STAGES = {"FlowNet2-CS": "net2_", "FlowNet2-CSS": "net3_", "FlowNet2-SD": "", "FlowNet2": "fuse_"}


def _generator():
    spec = importlib.util.spec_from_file_location("gen_prototxt", os.path.join(ROOT, "models", "gen_prototxt.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_generator_reproduces_every_committed_template():
    g = _generator()
    for kind, table in (("deploy", g.MODELS), ("train", g.TRAIN_MODELS)):
        for name, fn in table.items():
            with open(os.path.join(ROOT, "models", "%s_%s.prototxt.template" % (name, kind))) as f:
                assert f.read() == fn(), (name, kind)
    assert set(g.TRAIN_MODELS) == {"FlowNet2-C"} | set(STAGES)


@pytest.mark.parametrize("stage", list(STAGES))
def test_stage_template_parser_matches_reference_protobuf(fn2, stage):
    ref = json.load(open(os.path.join(GOLD, "ref_pb2_stack_train_prototxt.json")))[stage]
    text = fn2.fill_train_template(fn2.train_template(stage), 448, 320, 512, 384, 8)
    msg = onet.parse_prototxt(canonical(fn2, text))
    layers = getall(msg, "layer")
    assert len(layers) == len(ref["layers"])
    for got, want in zip(layers, ref["layers"]):
        assert get(got, "name") == want["name"] and get(got, "type") == want["type"]
        assert getall(got, "bottom") == want["bottom"] and getall(got, "top") == want["top"]
        assert np.allclose([float(x) for x in getall(got, "loss_weight")], want["loss_weight"], rtol=1e-6)
        assert [x == "true" for x in getall(got, "propagate_down")] == want["propagate_down"]
        assert [[float(get(p, "lr_mult", 1)), float(get(p, "decay_mult", 1))] for p in getall(got, "param")] == want["param"]
        if "conv" in want:
            cp = get(got, "convolution_param")
            assert [int(get(cp, "num_output")), [int(x) for x in getall(cp, "kernel_size")], [int(x) for x in getall(cp, "stride")],
                    [int(x) for x in getall(cp, "pad")]] == want["conv"]
        if "coeff" in want:
            assert np.allclose([float(x) for x in getall(get(got, "eltwise_param"), "coeff")], want["coeff"], rtol=1e-6)
        if "aug" in want:
            ap = get(got, "augmentation_param")
            assert [int(get(ap, "crop_width", 0)), int(get(ap, "crop_height", 0))] == want["aug"]["crop"]
            assert get(ap, "mode", "add") == want["aug"]["mode"]
        if "shapes" in want:
            assert [[int(d) for d in getall(s, "dim")] for s in getall(get(got, "input_param"), "shape")] == want["shapes"]


@pytest.mark.parametrize("stage", list(STAGES))
def test_stage_freezes_every_predecessor_and_trains_the_newest(fn2, stage):
    """Every parameter of a frozen sub-network has lr_mult 0 and decay_mult 0; the trained one keeps the deploy templates'
    ParamSpecs; the losses sit on the trained sub-network; the names match the deploy graph, so a trained caffemodel loads there."""
    pre = STAGES[stage]
    layers = getall(onet.parse_prototxt(fn2.train_template(stage)), "layer")
    deploy_name = "FlowNet2-CSS" if stage == "FlowNet2-CS" else stage            # there is no CS deploy net; CS lives inside CSS
    deploy = {get(l, "name") for l in getall(onet.parse_prototxt(fn2.model_template(deploy_name)), "layer")}
    trained = frozen = 0
    for l in layers:
        if get(l, "type") not in ("Convolution", "Deconvolution"):
            continue
        name = get(l, "name")
        assert name in deploy, name
        lr = [(float(get(p, "lr_mult")), float(get(p, "decay_mult"))) for p in getall(l, "param")]
        if name.startswith(pre) and (pre or not name.startswith(("net", "fuse_"))):
            assert lr == [(1.0, 1.0), (1.0, 0.0)], name
            trained += 1
        else:
            assert lr == [(0.0, 0.0), (0.0, 0.0)], name
            frozen += 1
    assert trained >= 11 and (frozen > 0) == (stage != "FlowNet2-SD")
    losses = [l for l in layers if get(l, "type") == "L1Loss"]
    assert [getall(l, "bottom")[0] for l in losses] == ["%spredict_flow%d" % (pre, k) for k in ((2, 1, 0) if pre == "fuse_" else (6, 5, 4, 3, 2))]
    gts = {getall(l, "bottom")[0] for l in layers if get(l, "type") == "Downsample"}
    assert gts == {"flow_gt_aug" if stage == "FlowNet2" else "scaled_flow_gt_aug"}
    # the warp blocks read the augmented frames
    for l in layers:
        if get(l, "type") == "FlowWarp":
            assert getall(l, "bottom")[0] == "img1_aug"


# ---- the oracle's need-backward pruning ----------------------------------------------------------------------------------------
AUG_TYPES = ("DataAugmentation", "GenerateAugmentationParameters", "FlowAugmentation")


def _forward_train_graph(net, given):
    """OracleNet forward over a training graph from the augmentation's outputs (the oracle has no augmentation sampler): the
    layers in front of the augmentation, and the augmentation itself, are skipped."""
    B = net.blobs = dict(given)
    for l in net.layers:
        if get(l, "type") in ("Input",) + AUG_TYPES or any(b not in B for b in getall(l, "bottom")):
            continue
        for t, v in zip(getall(l, "top"), net.run_layer(l, [B[b] for b in getall(l, "bottom")])):
            B[t] = v
    return B


def test_pruned_oracle_stops_at_the_frozen_predecessor(fn2):
    cw, ch = 192, 128
    text = fn2.fill_train_template(fn2.train_template("FlowNet2-CS"), cw, ch, cw, ch, 1)
    r = rng(41)
    given = {"img0_aug": r.uniform(-0.5, 0.5, (1, 3, ch, cw)).astype(np.float32),
             "img1_aug": r.uniform(-0.5, 0.5, (1, 3, ch, cw)).astype(np.float32),
             "flow_gt_aug": (3 * r.standard_normal((1, 2, ch, cw))).astype(np.float32)}
    plain = OracleNet(text, None, synth_seed=5)
    _forward_train_graph(plain, given)
    with pytest.raises(NotImplementedError, match="ChannelNorm"):
        plain.backward()
    pruned = PrunedOracleNet(text, None, synth_seed=5)
    B = _forward_train_graph(pruned, given)
    D, P = pruned.backward()
    need = pruned.layer_need
    assert not any(need[get(l, "name")] for l in pruned.layers if get(l, "type") in ("ChannelNorm", "FlowWarp", "Resample"))
    assert not any(n.startswith("net1_") or n.startswith("net2_in_") for n in D) and "net2_input" not in D
    convs = [get(l, "name") for l in pruned.layers if get(l, "type") in ("Convolution", "Deconvolution")]
    assert sorted(P) == sorted(n for n in convs if n.startswith("net2_"))
    assert all(np.isfinite(g).all() and np.abs(g).max() > 0 for gs in P.values() for g in gs)
    assert np.isfinite(B["flow_loss2"]).all()


def test_pruned_oracle_keeps_the_c_graph_gradients(fn2):
    w, h = 128, 64
    proto = fn2.fill_template(fn2.model_template("FlowNet2-C"), w, h)
    r = rng(42)
    img0 = r.uniform(0, 255, (1, 3, h, w)).astype(np.float32)
    img1 = r.uniform(0, 255, (1, 3, h, w)).astype(np.float32)
    res = []
    for cls in (OracleNet, PrunedOracleNet):
        net = cls(proto, None, synth_seed=9)
        B = net.forward(img0=img0, img1=img1)
        seeds = {"predict_flow%d" % k: rng(43 + k).standard_normal(B["predict_flow%d" % k].shape).astype(np.float32) for k in range(2, 7)}
        res.append(net.backward(**seeds) + (net,))
    (D0, P0, _), (D1, P1, pruned) = res
    assert sorted(P0) == sorted(P1) and len(P1) >= 20
    for k in P0:
        assert all(np.array_equal(a, b) for a, b in zip(P0[k], P1[k])), k
    for k in D1:
        assert np.array_equal(D0[k], D1[k]), k
    # what the pruning drops is exactly the gradient of blobs nothing trainable lies under
    assert sorted(set(D0) - set(D1)) == sorted(k for k in D0 if not pruned.blob_need.get(k, False))


# ---- all-reduce of the trainable span (world size 2, gloo) ----------------------------------------------------------------------
def _span_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    from flownet2_b200 import parallel as PAR
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        # a frozen head of 960 floats, a trainable span of 320 at the end of the arena (the fusion stage's layout)
        arena = torch.full((1280,), -7.0 - rank)
        arena[960:] = float(rank + 1) * torch.arange(320, dtype=torch.float32)
        span = arena[960:]
        PAR.allreduce_gradients(span)
        ok = bool(torch.equal(arena[:960], torch.full((960,), -7.0 - rank)))
        ok = ok and bool(torch.allclose(arena[960:], 1.5 * torch.arange(320, dtype=torch.float32)))
        q.put((rank, ok))
    finally:
        dist.destroy_process_group()


def test_span_allreduce_world2_touches_only_the_span():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_span_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert sorted(res) == [(0, True), (1, True)]
