"""GPU parity: whole-net forward through the Caffe-surface engine (fn2_net_* C-ABI) vs the CPU
oracle executing the same prototxt with the same weights (exported as .caffemodel bytes and
re-read by the oracle's own wire-format parser).

Tolerance on predict_flow_final: 1e-4 max-abs (north_star).  Intermediate blobs are compared
relative to their magnitude (1e-4) to localise a failure.
"""
import numpy as np
import pytest

from oracle import oracle as O
from oracle.net import OracleNet
from tests.util import maxabs, rng, smooth_images

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def run_pair(fn2, model, width, height, batch, seed=1701, check_blobs=()):
    proto = fn2.fill_template(fn2.model_template(model), width, height)
    net = fn2.Net(proto, None, fn2.TEST, batch=batch)
    net.fill_params(seed)
    weights = net.to_caffemodel()
    img0, img1 = smooth_images(rng(seed), batch, height, width)
    out = net.forward(img0=img0, img1=img1)
    got = out["predict_flow_final"]
    assert got.shape == (batch, 2, height, width)
    onet = OracleNet(proto, weights, batch=batch, f64acc=True)
    ref = onet.forward(img0=img0, img1=img1)
    want = ref["predict_flow_final"]
    report = []
    for name in check_blobs:
        g, w = net.blobs[name].data, ref[name]
        report.append((name, maxabs(g, w), float(np.abs(w).max())))
    return net, got, want, report


@pytest.mark.parametrize("model,w,h,batch", [
    ("FlowNet2-S", 128, 96, 2),          # 96 rows -> adapted 128: exercises both Resample directions
    ("FlowNet2-C", 128, 128, 1),
    ("FlowNet2-C", 192, 100, 2),
])
def test_single_net_parity(fn2, model, w, h, batch):
    blobs = ["img0_nomean_resize", "conv3_1", "conv6_1", "predict_flow6", "predict_flow2"]
    net, got, want, report = run_pair(fn2, model, w, h, batch, check_blobs=blobs)
    for name, err, mag in report:
        assert err <= 1e-4 * max(1.0, mag), (name, err, mag)
    assert np.isfinite(got).all()
    assert np.abs(want).max() > 1e-3, "degenerate test: flow is ~0"
    assert maxabs(got, want) <= 1e-4, maxabs(got, want)


def test_css_parity(fn2):
    blobs = ["net1_predict_flow2", "net2_in_img1_warped", "net2_in_err_norm", "net2_predict_flow2", "net3_predict_flow2"]
    net, got, want, report = run_pair(fn2, "FlowNet2-CSS", 128, 128, 1, check_blobs=blobs)
    for name, err, mag in report:
        assert err <= 2e-4 * max(1.0, mag), (name, err, mag)
    assert maxabs(got, want) <= 1e-4, (maxabs(got, want), np.abs(want).max())      # strict north_star tolerance, |flow| ~ 25


def test_full_flownet2_parity(fn2):
    net, got, want, report = run_pair(fn2, "FlowNet2", 128, 64, 1, check_blobs=["fuse_input", "fuse_predict_flow0"])
    for name, err, mag in report:
        assert err <= 2e-4 * max(1.0, mag), (name, err, mag)
    assert maxabs(got, want) <= 1e-4, (maxabs(got, want), np.abs(want).max())      # strict north_star tolerance


def test_graph_replay_matches_eager(fn2):
    proto = fn2.fill_template(fn2.model_template("FlowNet2-C"), 128, 64)
    net = fn2.Net(proto, None, fn2.TEST, batch=2)
    net.fill_params(3)
    img0, img1 = smooth_images(rng(3), 2, 64, 128)
    first = net.forward(img0=img0, img1=img1)["predict_flow_final"]        # eager (allocations)
    second = net.forward(img0=img0, img1=img1)["predict_flow_final"]       # captured + replayed
    third = net.forward(img0=img0, img1=img1)["predict_flow_final"]        # replayed
    assert maxabs(first, second) == 0.0 and maxabs(first, third) == 0.0
    assert net.launches_per_forward > 0
    other0, other1 = smooth_images(rng(4), 2, 64, 128)
    changed = net.forward(img0=other0, img1=other1)["predict_flow_final"]
    assert maxabs(first, changed) > 0.0


def test_arena_written_on_device_refreshes_host_state(fn2):
    """What a non-root rank does after the NCCL broadcast (bench.py): its arena is overwritten ON THE DEVICE, then
    fn2_net_params_changed.  The replica must behave exactly like the source: same flow, and -- because the DataAugmentation
    iteration counter is read on the host -- it must reach CUDA-graph replay instead of re-estimating the mean forever."""
    proto = fn2.fill_template(fn2.model_template("FlowNet2-C"), 128, 64)
    src = fn2.Net(proto, None, fn2.TEST, batch=1)
    src.fill_params(9)
    dst = fn2.Net(proto, None, fn2.TEST, batch=1)
    from flownet2_b200 import parallel as P
    a, b = P.arena_tensor(src), P.arena_tensor(dst)
    assert a.numel() == b.numel() and float(b.abs().sum()) == 0.0
    b.copy_(a)
    torch.cuda.synchronize()
    dst.params_changed()
    img0, img1 = smooth_images(rng(9), 1, 64, 128)
    for _ in range(3):
        fa = src.forward(img0=img0, img1=img1)["predict_flow_final"]
        fb = dst.forward(img0=img0, img1=img1)["predict_flow_final"]
        assert maxabs(fa, fb) == 0.0
    assert src.graph_active and dst.graph_active
    from oracle.net import parse_caffemodel
    wa, wb = parse_caffemodel(src.to_caffemodel()), parse_caffemodel(dst.to_caffemodel())
    assert all(np.array_equal(x, y) for k in wa for x, y in zip(wa[k], wb[k]))          # host copies were re-read from the device


def test_concat_of_small_eltwise_outputs_keeps_both_halves(fn2):
    """Zero-copy Concat of two 2-channel Eltwise outputs: the float4 store of the first child must not zero the lanes that
    hold the second child's channels (ADVICE r1: px_view inferred padding ownership from strides)."""
    proto = '''name: "t" input: "a" input_shape { dim: 1 dim: 2 dim: 8 dim: 12 } input: "b" input_shape { dim: 1 dim: 2 dim: 8 dim: 12 }
    layer { name: "e1" type: "Eltwise" bottom: "a" top: "fa" eltwise_param { operation: SUM coeff: 20 } }
    layer { name: "e2" type: "Eltwise" bottom: "b" top: "fb" eltwise_param { operation: SUM coeff: 20 } }
    layer { name: "c" type: "Concat" bottom: "fa" bottom: "fb" top: "cat" }
    layer { name: "e3" type: "Eltwise" bottom: "cat" top: "out" eltwise_param { operation: SUM coeff: 0.5 } }'''
    net = fn2.Net(proto, None, fn2.TEST)
    r = rng(4)
    a = r.standard_normal((1, 2, 8, 12)).astype(np.float32)
    b = r.standard_normal((1, 2, 8, 12)).astype(np.float32)
    for _ in range(3):
        out = net.forward(a=a, b=b)["out"]
        assert np.array_equal(out, np.concatenate([a * 20, b * 20], 1) * np.float32(0.5))


def test_caffemodel_roundtrip_and_name_matching(fn2):
    proto = fn2.fill_template(fn2.model_template("FlowNet2-S"), 64, 64)
    a = fn2.Net(proto, None, fn2.TEST)
    a.fill_params(5)
    blob = a.to_caffemodel()
    b = fn2.Net(proto, blob, fn2.TEST)
    # conv weights survive the round trip bit for bit; DataAugmentation only takes the iteration count and
    # the per-channel mean when mean_per_pixel is false (adjust_blobs, data_augmentation_layer.cpp:172-183)
    from oracle.net import parse_caffemodel
    wa, wb = parse_caffemodel(blob), parse_caffemodel(b.to_caffemodel())
    assert wa.keys() == wb.keys()
    for k in wa:
        idx = [0, 2] if k.endswith("_aug") else range(len(wa[k]))
        for i in idx:
            assert np.array_equal(wa[k][i], wb[k][i]), (k, i)
    img0, img1 = smooth_images(rng(5), 1, 64, 64)
    fa = a.forward(img0=img0, img1=img1)["predict_flow_final"]
    fb = b.forward(img0=img0, img1=img1)["predict_flow_final"]
    assert maxabs(fa, fb) == 0.0


def test_flo_roundtrip_and_reference_files(fn2, tmp_path):
    flow = rng(6).standard_normal((2, 13, 17)).astype(np.float32)
    p = str(tmp_path / "x.flo")
    fn2.write_flo(p, flow)
    raw = open(p, "rb").read()
    assert raw[:4] == b"PIEH" and np.frombuffer(raw[4:12], np.int32).tolist() == [17, 13]
    # python twin of the reference writer: (H,W,2) interleaved (scripts/run-flownet.py:117-124)
    assert np.array_equal(np.frombuffer(raw[12:], np.float32).reshape(13, 17, 2), flow.transpose(1, 2, 0))
    assert np.array_equal(fn2.read_flo(p), flow)


AUG_PROTO = """
name: "aug_train"
input: "img"
input_shape { dim: 4 dim: 3 dim: 48 dim: 64 }
input: "img_b"
input_shape { dim: 4 dim: 3 dim: 48 dim: 64 }
layer {
  name: "aug" type: "DataAugmentation" bottom: "img" top: "aug" top: "params"
  augmentation_param {
    augment_during_test: true crop_width: 48 crop_height: 32 max_multiplier: 1
    mirror { rand_type: "bernoulli" prob: 0.5 }
    translate { rand_type: "uniform_bernoulli" mean: 0 spread: 0.1 prob: 1.0 }
    rotate { rand_type: "uniform_bernoulli" mean: 0 spread: 0.2 prob: 1.0 }
    zoom { rand_type: "uniform_bernoulli" exp: true mean: 0.1 spread: 0.1 prob: 1.0 }
    squeeze { rand_type: "uniform_bernoulli" exp: true mean: 0 spread: 0.1 prob: 1.0 }
    gamma { rand_type: "gaussian_bernoulli" exp: true mean: 0 spread: 0.2 prob: 1.0 }
    brightness { rand_type: "gaussian_bernoulli" mean: 0 spread: 0.05 prob: 1.0 }
    contrast { rand_type: "gaussian_bernoulli" exp: true mean: 0 spread: 0.2 prob: 1.0 }
    color { rand_type: "gaussian_bernoulli" exp: true mean: 0 spread: 0.1 prob: 1.0 }
    lmult_pow { rand_type: "uniform_bernoulli" exp: true mean: 0 spread: 0.2 prob: 1.0 }
    lmult_mult { rand_type: "uniform_bernoulli" exp: true mean: 0 spread: 0.2 prob: 1.0 }
    lmult_add { rand_type: "uniform_bernoulli" mean: 0 spread: 0.03 prob: 1.0 }
    sat_pow { rand_type: "uniform_bernoulli" exp: true mean: 0 spread: 0.2 prob: 1.0 }
    col_rotate { rand_type: "uniform_bernoulli" mean: 0 spread: 0.5 prob: 1.0 }
    shadow_angle { rand_type: "uniform" mean: 0 spread: 3.1 }
    shadow_distance { rand_type: "uniform" mean: 0 spread: 5 }
    shadow_strength { rand_type: "uniform" mean: 0.2 spread: 0.1 }
    chromatic_eigvec: 0.51 chromatic_eigvec: 0.56 chromatic_eigvec: 0.65 chromatic_eigvec: 0.79 chromatic_eigvec: 0.01
    chromatic_eigvec: -0.62 chromatic_eigvec: 0.35 chromatic_eigvec: -0.83 chromatic_eigvec: 0.44
  }
}
layer {
  name: "aug_b" type: "DataAugmentation" bottom: "img_b" bottom: "params" top: "aug_b"
  augmentation_param {
    augment_during_test: true crop_width: 48 crop_height: 32 max_multiplier: 1
    chromatic_eigvec: 0.51 chromatic_eigvec: 0.56 chromatic_eigvec: 0.65 chromatic_eigvec: 0.79 chromatic_eigvec: 0.01
    chromatic_eigvec: -0.62 chromatic_eigvec: 0.35 chromatic_eigvec: -0.83 chromatic_eigvec: 0.44
  }
}
"""

COEFF_DEFAULT = np.array([0, 0, 0, 0, 1, 1, 1, 0, 1, 1, 1, 1] + [1, 1, 1, 0, 0, 0, 1, 1, 1, 1, 1, 1, 0, 0, 0, 1, 1, 1, 1, 0, 1, 0] + [0] * 8,
                         np.float32)


def oracle_augment(x, params, crop_w, crop_h, eigvec, max_mult):
    """DataAugmentationLayer::Forward_gpu given the (N,42) coefficient blob, restated with the oracle's pieces."""
    N = x.shape[0]
    vals = np.where(np.abs(COEFF_DEFAULT) < 1e-3, params, np.exp(params)).astype(np.float32)      # array_to_coeff
    vals = np.where(np.abs(COEFF_DEFAULT - vals) < 1e-3, COEFF_DEFAULT, vals)                      # clear_defaults
    mats = np.stack([O.transmat_from_coeff(crop_w, crop_h, x.shape[3], x.shape[2], mirror=float(vals[n, 0]), angle=float(vals[n, 3]),
                                           dx=float(vals[n, 1]), dy=float(vals[n, 2]), zoom_x=float(vals[n, 4]), zoom_y=float(vals[n, 5]))
                     for n in range(N)])
    out = O.spatial_augmentation(x, mats, crop_h, crop_w)
    eig = vals[:, 12:34]
    if np.any(eig != COEFF_DEFAULT[12:34]):
        out = O.chromatic_eigen_augmentation(out, eig, O.chromatic_eigenspace(x, eigvec), max_mult)
    chroma = vals[:, 6:12]
    if np.any(chroma != COEFF_DEFAULT[6:12]):
        out = O.color_contrast_augmentation(out, chroma, max_mult)
    eff = np.zeros((N, 9), np.float32)
    eff[:, 0:4] = vals[:, 34:38]
    eff[:, 4], eff[:, 5] = np.cos(vals[:, 38]), np.sin(vals[:, 38])
    eff[:, 6:9] = vals[:, 39:42]
    if np.any((eff[:, 0] != 0) & (eff[:, 1] != 0)) or np.any(eff[:, 3] > 0) or np.any(eff[:, 7] > 0):
        out = O.apply_effects(out, eff, max_mult)
    return out, vals


def test_data_augmentation_training_path(fn2):
    """Sampled coefficients (params output blob) -> spatial + chromatic-eigen + chromatic + effect kernels; a second layer
    consumes the same coefficient blob.  The random STREAM is unpinned (boost in the reference), so the check is: whatever
    was sampled, the images are what the reference arithmetic gives for those coefficients, and the samples lie in the
    configured ranges."""
    net = fn2.Net(AUG_PROTO, None, fn2.TEST)
    r = rng(3)
    img = r.uniform(0, 1, (4, 3, 48, 64)).astype(np.float32)
    img_b = r.uniform(0, 1, (4, 3, 48, 64)).astype(np.float32)
    seen = []
    for it in range(3):
        net.forward(img=img, img_b=img_b)
        params = net.blobs["params"].data.reshape(4, 42).copy()
        seen.append(params)
        want, vals = oracle_augment(img, params, 48, 32, EIGVEC_T, 1.0)
        assert maxabs(net.blobs["aug"].data, want) <= 2e-5
        want_b, _ = oracle_augment(img_b, params, 48, 32, EIGVEC_T, 1.0)
        assert maxabs(net.blobs["aug_b"].data, want_b) <= 2e-5
        assert set(np.unique(vals[:, 0])) <= {0.0, 1.0}                                  # mirror
        assert np.all(np.abs(vals[:, 1:3]) <= 0.1 + 1e-6) and np.all(np.abs(vals[:, 3]) <= 0.2 + 1e-6)
        assert np.all(vals[:, 40] >= 0.1 - 1e-6) and np.all(vals[:, 40] <= 0.3 + 1e-6)  # shadow strength
    assert not np.array_equal(seen[0], seen[1])                                          # fresh samples every forward


EIGVEC_T = [0.51, 0.56, 0.65, 0.79, 0.01, -0.62, 0.35, -0.83, 0.44]


def test_full_size_properties(fn2, monkeypatch):
    """BASELINE.json's configuration (FlowNet2, 1024x436, 4 pairs) is too large for the CPU oracle; checked through
    size-independent properties instead: (1) replay determinism (eager pass == CUDA-graph replays, bit for bit),
    (2) batch independence: sample k of a batch-4 forward equals a batch-1 forward of that pair (different tile schedules and
    K splits, so within the flow tolerance, not bitwise), (3) the two convolution engines agree: wgmma 3xTF32 vs exact-FP32
    SIMT within 1e-4 of the flow scale, (4) correlation layer: tensor-core route vs the FP32 fast route on the net's own conv3
    features (NCHW copies, which the tensor-core route does not take)."""
    W, H, B = 1024, 436, 4
    proto = fn2.fill_template(fn2.model_template("FlowNet2"), W, H)
    img0, img1 = smooth_images(rng(99), B, H, W)
    net = fn2.Net(proto, None, fn2.TEST, batch=B)
    net.fill_params(1701)
    weights = net.to_caffemodel()
    f1 = net.forward(img0=img0, img1=img1)["predict_flow_final"].copy()
    f2 = net.forward(img0=img0, img1=img1)["predict_flow_final"].copy()      # captured into a graph here
    f3 = net.forward(img0=img0, img1=img1)["predict_flow_final"].copy()      # graph replay
    assert np.isfinite(f1).all() and f1.shape == (B, 2, H, W)
    assert maxabs(f1, f2) == 0.0 and maxabs(f1, f3) == 0.0
    scale = max(1.0, float(np.abs(f1).max()))
    if "net1_corr" in net.blobs:
        from flownet2_b200 import ops
        corr_tc = net.blobs["net1_corr"].data
        a, b = (torch.from_numpy(net.blobs[n].data).cuda() for n in ("net1_conv3a", "net1_conv3b"))
        corr_fp32 = ops.correlation(a, b, 20, 1, 20, 1, 2).cpu().numpy()
        corr_fp32 = np.where(corr_fp32 > 0, corr_fp32, corr_fp32 * np.float32(0.1))     # net1_ReLU_corr runs in place
        assert maxabs(corr_fp32, corr_tc) <= 1e-5 * max(1.0, float(np.abs(corr_fp32).max()))
    del net
    one = fn2.Net(proto, weights, fn2.TEST, batch=1)
    g = one.forward(img0=img0[2:3], img1=img1[2:3])["predict_flow_final"]
    assert maxabs(g, f1[2:3]) <= 1e-4 * scale, (maxabs(g, f1[2:3]), scale)
    del one
    monkeypatch.setenv("FN2_CONV_ENGINE", "simt")
    simt = fn2.Net(proto, weights, fn2.TEST, batch=B)
    h = simt.forward(img0=img0, img1=img1)["predict_flow_final"]
    assert maxabs(h, f1) <= 1e-4 * scale, (maxabs(h, f1), scale)


def test_fused_warp_block_is_bit_identical_to_the_layer_chain(fn2, monkeypatch):
    """Net::FuseWarpBlocks runs Resample -> FlowWarp -> Eltwise(1,-1) -> ChannelNorm (+ the Eltwise that rescales the flow) of every
    hand-over between stacked networks as one kernel; its five tops must equal the separate layers' bit for bit."""
    proto = fn2.fill_template(fn2.model_template("FlowNet2-CSS"), 192, 128)
    img0, img1 = smooth_images(rng(5), 2, 128, 192)
    blobs = ["net2_in_flow_full", "net2_in_img1_warped", "net2_in_err", "net2_in_err_norm", "net2_in_flow_scaled",
             "net3_in_flow_full", "net3_in_img1_warped", "net3_in_err_norm", "net3_in_flow_scaled", "predict_flow_final"]
    got = []
    for fused in (True, False):
        if not fused:
            monkeypatch.setenv("FN2_NO_WARPFUSE", "1")
        net = fn2.Net(proto, None, fn2.TEST, batch=2)
        net.fill_params(9)
        net.forward(img0=img0, img1=img1)
        got.append(({b: net.blobs[b].data for b in blobs}, net.launches_per_forward))
    assert got[0][1] < got[1][1], (got[0][1], got[1][1])                    # the fusion actually happened (8 launches fewer)
    for b in blobs:
        assert np.array_equal(got[0][0][b], got[1][0][b], equal_nan=True), b
    assert np.abs(got[0][0]["net2_in_err_norm"]).max() > 0


def test_weights_from_hdf5_equal_weights_from_caffemodel(fn2):
    """Net::CopyTrainedLayersFromHDF5 (net.cpp:823-870): the same weights as /data/<layer>/<index> datasets of an HDF5 file
    (recognised by its signature) must give the same flow, bit for bit, as the binary .caffemodel."""
    from oracle.net import parse_caffemodel
    from tests.util_h5 import write_caffemodel_h5
    proto = fn2.fill_template(fn2.model_template("FlowNet2-S"), 128, 64)
    a = fn2.Net(proto, None, fn2.TEST, batch=1)
    a.fill_params(13)
    binary = a.to_caffemodel()
    h5 = write_caffemodel_h5(parse_caffemodel(binary))
    img0, img1 = smooth_images(rng(13), 1, 64, 128)
    want = a.forward(img0=img0, img1=img1)["predict_flow_final"]
    b = fn2.Net(proto, h5, fn2.TEST, batch=1)
    got = b.forward(img0=img0, img1=img1)["predict_flow_final"]
    assert np.abs(want).max() > 1e-3 and np.array_equal(got, want)
    with pytest.raises(fn2.Fn2Error):
        fn2.Net(proto, h5[:4000], fn2.TEST, batch=1)                      # truncated file: loud failure, no partial load
