"""GPU: KITTI flow PNGs on the device.  fn2_flow_to_tensor (FLOW_KITTI) bit-exact against kitti.decode (and the uint16
quantisation), fn2_flow_to_kitti_png_rows byte-exact against kitti.paeth_rows(kitti.encode(...)), their refusals, and the three commands:
evaluate on a KITTI list equal to evaluate on the .flo twin list, the dataset's blobs equal to the .flo twin's, and run --kitti
writing the PNGs of the flows run writes as .flo."""
import os

import numpy as np
import pytest

from flownet2_b200 import data as D, evaluate as E, files as FI, kitti as K, run as R, train as T
from tests.test_run_flownet_cpu import write_pnm
from tests.test_run_flownet_gpu import chairs_frames
from tests.test_train_data_gpu import TINY_NET, train_net

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def raw_samples(r, n, h, w):
    """(n, h, w, 3) uint16 samples with the edge values 0, 32767, 32768, 65535 and invalid pixels (B = 0)."""
    s = r.integers(0, 65536, (n, h, w, 3)).astype(np.uint16)
    s[..., 2] = r.integers(0, 3, (n, h, w))
    flat = s.reshape(-1, 3)
    flat[:8] = [[0, 0, 1], [32767, 32768, 1], [32768, 32767, 7], [65535, 0, 65535], [0, 65535, 1], [5, 6, 0], [32768, 32768, 1],
                [65535, 65535, 0]]
    return s


@pytest.mark.parametrize("quant", [0, 1])
@pytest.mark.parametrize("layout", ["nchw", "pad", "slice"])
def test_flow_to_tensor_kitti_bit_exact(fn2, quant, layout):
    import torch
    from flownet2_b200 import ops
    n, h, w = 3, 5, 37                                        # H*W odd: the second payload starts 2 bytes past a 4-byte boundary
    s = raw_samples(np.random.default_rng(quant), n, h, w)
    want = K.decode(s).transpose(0, 3, 1, 2)
    if quant:
        want = D.uint16flow(want)
    payload = np.ascontiguousarray(s, ">u2").view(np.uint8).reshape(-1)
    fill = -7.0
    if layout == "nchw":
        parent, lo = torch.full((n, 2, h, w), fill, device="cuda"), 0
    else:
        parent, lo = torch.full((n, 4 if layout == "pad" else 8, h, w), fill, device="cuda").contiguous(
            memory_format=torch.channels_last), 0 if layout == "pad" else 2
    flags = fn2.FLOW_UINT16FLOW if quant else 0
    src = torch.from_numpy(payload.copy()).cuda()
    ops.flow_to_tensor(src, fn2.FLOW_KITTI, flags, parent[:, lo:lo + 2])
    torch.cuda.synchronize()
    got = parent.cpu().numpy()
    assert np.array_equal(bits(got[:, lo:lo + 2]), bits(want))
    assert (np.delete(got, range(lo, lo + 2), axis=1) == fill).all()          # channels outside the view are untouched
    assert np.isnan(want).any() and (np.isnan(want[:, 0]) == np.isnan(want[:, 1])).all()
    # pairs 1 and 2 alone, from a source that is only 2-byte aligned
    one = torch.full((2, 2, h, w), fill, device="cuda")
    ops.flow_to_tensor(src[h * w * 6:], fn2.FLOW_KITTI, flags, one)
    assert (src[h * w * 6:].data_ptr() & 3) == 2
    assert np.array_equal(bits(one.cpu().numpy()), bits(want[1:]))


def flow_with_edges(r, n, h, w):
    """(n, 2, h, w) float32 flow over +-600 px with NaN, +-Inf, huge and tiny values."""
    f = (r.standard_normal((n, 2, h, w)) * 200).astype(np.float32)
    edges = np.array([np.nan, np.inf, -np.inf, 1e30, -1e30, 512.0, -512.0, 511.984375, 511.99, -512.01, 0.0, -0.0, 1e-30,
                      0.015625, -0.015624], np.float32)
    flat = f.reshape(-1)
    flat[r.choice(flat.size, 3 * edges.size, replace=False)] = np.tile(edges, 3)
    return f


@pytest.mark.parametrize("layout", ["nchw", "nhwc", "slice", "strided"])
def test_flow_to_kitti_png_rows_byte_exact(fn2, layout):
    import torch
    from flownet2_b200 import ops
    n, h, w = 3, 7, 45
    f = flow_with_edges(np.random.default_rng(5), n, h, w)
    t = torch.from_numpy(f).cuda()
    if layout == "nhwc":
        src = t.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    elif layout == "slice":
        parent = torch.full((n, 6, h, w), float("nan"), device="cuda").contiguous(memory_format=torch.channels_last)
        parent[:, 3:5] = t
        src = parent[:, 3:5]
    elif layout == "strided":
        parent = torch.full((n, 2, h + 3, 2 * w), float("nan"), device="cuda")
        parent[:, :, 1:h + 1, ::2] = t
        src = parent[:, :, 1:h + 1, ::2]
    else:
        src = t
    out = torch.full((n * h * (1 + 6 * w) + 16,), 0xab, dtype=torch.uint8, device="cuda")
    ops.flow_to_kitti_png_rows(src, out)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    want = np.stack([K.paeth_rows(K.encode(f[i].transpose(1, 2, 0))) for i in range(n)])
    assert np.array_equal(got[:-16].reshape(n, h, -1), want)
    assert (got[-16:] == 0xab).all()
    dec = np.stack([K.decode(K.encode(f[i].transpose(1, 2, 0))) for i in range(n)])
    assert np.isnan(dec).any() and (dec[~np.isnan(dec)] >= -512).all() and (dec[~np.isnan(dec)] < 512).all()


def test_refusals(fn2):
    import torch
    from flownet2_b200 import ops
    src = torch.zeros(2 * 3 * 4 * 6 + 2, dtype=torch.uint8, device="cuda")
    dst = torch.zeros((2, 2, 3, 4), device="cuda")
    with pytest.raises(fn2.Fn2Error, match="flow_to_tensor: unknown flags 0x2"):
        ops.flow_to_tensor(src, fn2.FLOW_KITTI, 2, dst)
    with pytest.raises(fn2.Fn2Error, match="flow_to_tensor: dst must have 2 channels"):
        ops.flow_to_tensor(src, fn2.FLOW_KITTI, 0, torch.zeros((2, 3, 3, 4), device="cuda"))
    with pytest.raises(fn2.Fn2Error, match="flow_to_tensor: src must be 2-byte aligned"):
        ops.flow_to_tensor(src[1:], fn2.FLOW_KITTI, 0, dst)
    rows = torch.zeros(2 * 3 * (1 + 6 * 4), dtype=torch.uint8, device="cuda")
    with pytest.raises(fn2.Fn2Error, match="flow_to_kitti_png_rows: src must have 2 channels"):
        ops.flow_to_kitti_png_rows(torch.zeros((2, 3, 3, 4), device="cuda"), rows)
    d = ops.desc(dst)
    d.data += 2
    assert fn2.lib().fn2_flow_to_kitti_png_rows(d, rows.data_ptr(), None) == -1
    assert fn2.lib().fn2_last_error().decode() == "flow_to_kitti_png_rows: src must be 4-byte aligned"
    net = fn2.Net(fn2.fill_train_template(fn2.train_template("FlowNet2-C"), 64, 64, 64, 64, 1), None, fn2.TRAIN)
    with pytest.raises(fn2.Fn2Error, match=r"blob img0 must have shape \(N, 2, H, W\)"):
        net.set_input_flow_device("img0", src.data_ptr(), fn2.FLOW_KITTI)


# ---- the commands ----
def sparse_flow(r, w, h):
    """KITTI-like sparse ground truth: about half the pixels invalid, the rest within +-60 px."""
    f = (r.standard_normal((h, w, 2)) * r.choice([3.0, 20.0, 60.0], (h, w, 1))).astype(np.float32)
    f[r.random((h, w)) < 0.5] = np.nan
    f[: h // 4] = np.nan
    return f


def kitti_scene(d, spec, seed):
    """Frames and sparse KITTI ground truth over spec [(w, h)]: the KITTI list, its .flo twin (the decoded ground truth, NaN at
    invalid pixels), and run's lists with .flo and .png outputs."""
    r = np.random.default_rng(seed)
    lines = {"kitti": [], "flo": [], "run_flo": [], "run_png": []}
    for i, size in enumerate(spec):
        f0, f1 = chairs_frames(size, seed + i)
        a, b = write_pnm(d / ("p%d_0.ppm" % i), f0), write_pnm(d / ("p%d_1.ppm" % i), f1)
        png = K.write_kitti_flow(str(d / ("g%d.png" % i)), sparse_flow(r, *size))
        flo = str(d / ("g%d.flo" % i))
        FI.write_flo(flo, K.read_kitti_flow(png))
        for k, g in (("kitti", png), ("flo", flo), ("run_flo", d / ("o%d.flo" % i)), ("run_png", d / ("o%d.png" % i))):
            lines[k].append("%s %s %s\n" % (a, b, g))
    for k, v in lines.items():
        (d / ("%s.txt" % k)).write_text("".join(v))
    return {k: str(d / ("%s.txt" % k)) for k in lines}


@pytest.fixture(scope="module")
def flownet2s(tmp_path_factory, fn2):
    d = tmp_path_factory.mktemp("kitti")
    net = fn2.Net(fn2.fill_template(fn2.model_template("FlowNet2-S"), 128, 128), None, fn2.TEST, batch=1)
    net.fill_params(1701)
    path = d / "s.caffemodel"
    path.write_bytes(net.to_caffemodel())
    del net
    return d, str(path), os.path.join(ROOT, "models", "FlowNet2-S_deploy.prototxt.template")


def test_evaluate_kitti_equals_flo_twin(fn2, flownet2s, capsys):
    d, weights, template = flownet2s
    lists = kitti_scene(d, [(128, 96), (192, 64), (128, 96)], 500)
    for batch in (1, 2):
        s_png, rec_png = E.evaluate(weights, template, FI.read_list(lists["kitti"]), batch=batch, kitti=True)
        s_flo, rec_flo = E.evaluate(weights, template, FI.read_list(lists["flo"]), batch=batch)
        assert np.array_equal(rec_png, rec_flo), batch
        assert s_png["invalid_px"] > 0 and s_png["valid_px"] > 0
        for k in ("pairs", "valid_px", "invalid_px", "nonfinite_px", "epe", "epe_pair_mean", "fl_percent", "s0-10", "s10-40", "s40+"):
            assert s_png[k] == s_flo[k], k
    capsys.readouterr()
    assert E.main([weights, template, lists["kitti"], "--kitti"]) == 0
    assert E.main([weights, template, lists["flo"]]) == 0
    a, b = [__import__("json").loads(l) for l in capsys.readouterr().out.strip().splitlines()]
    assert {k: v for k, v in a.items() if k != "wall"} == {k: v for k, v in b.items() if k != "wall"}


def test_run_kitti_writes_the_png_of_run_flo(fn2, flownet2s):
    d, weights, template = flownet2s
    lists = kitti_scene(d, [(128, 96), (192, 64), (128, 96)], 600)
    for batch in (1, 2):
        assert R.main([weights, template, lists["run_flo"], "--batch", str(batch)]) == 0
        assert R.main([weights, template, lists["run_png"], "--batch", str(batch), "--kitti"]) == 0
        for i in range(3):
            flow = fn2.read_flo(str(d / ("o%d.flo" % i))).transpose(1, 2, 0)
            assert np.isfinite(flow).all()
            png = open(str(d / ("o%d.png" % i)), "rb").read()
            assert png == K.png_bytes(K.paeth_rows(K.encode(flow)), flow.shape[1], flow.shape[0]), (batch, i)
            got = K.read_kitti_flow(str(d / ("o%d.png" % i)))
            assert np.array_equal(got, K.decode(K.encode(flow)))


def test_kitti_sink_names_non_finite_pairs(fn2, capsys):
    import torch
    sink = R.KittiFiles()
    B, H, W = 3, 4, 5
    flow_dev = [torch.zeros((B, H, W, 2), device="cuda") for _ in range(2)]
    sink.bind(torch, B, H, W, flow_dev)
    flow_dev[1][1, 2, 3, 0] = float("inf")
    flow_dev[1][2, 0, 0, 1] = float("nan")
    sink.score(1)
    sink.host[1].copy_(sink.dev[1])
    pairs = [FI.Pair("l:%d" % i, "a", "b", os.devnull) for i in range(B)]
    sink.take(pairs, 1, 2)                                        # the third pair is padding
    assert [p.where for p in sink.bad] == ["l:1"]
    assert "l:1: the flow of a b is not finite" in capsys.readouterr().err


@pytest.mark.parametrize("encoding", ["uint16", "float"])
def test_dataset_kitti_blobs_equal_flo_twin(fn2, tmp_path, encoding):
    lists = kitti_scene(tmp_path, [(192, 128)] * 5, 700)
    ds = D.FlowDataset(lists["kitti"], 2, flow_encoding=encoding, kitti=True)
    twin = D.FlowDataset(lists["flo"], 2, flow_encoding=encoding)
    nets = [train_net(fn2, ds), train_net(fn2, twin)]
    ds.bind(nets[0])
    twin.bind(nets[1])
    for k in range(4):
        assert ds() == {} and twin() == {}
        for name in ("img0", "img1", "flow_gt"):
            assert np.array_equal(bits(nets[0].blobs[name].data), bits(nets[1].blobs[name].data)), (k, name)
        assert np.array_equal(bits(nets[0].blobs["flow_gt"].data), bits(ds.host_batch(k)[2]))
    assert np.isnan(nets[0].blobs["flow_gt"].data).any()
    ds.close()
    twin.close()


def test_train_command_kitti(fn2, tmp_path, monkeypatch, capsys):
    lists = kitti_scene(tmp_path, [(48, 32)] * 4, 800)
    model = tmp_path / "tiny.prototxt.template"
    model.write_text(TINY_NET)
    (tmp_path / "s.prototxt").write_text('type: "Adam"\nbase_lr: 1e-3\nlr_policy: "fixed"\nmax_iter: 3\ndisplay: 1\n'
                                         'snapshot_after_train: false\n')
    monkeypatch.setenv("FN2_SEED", "5")
    monkeypatch.chdir(tmp_path)
    args = ["--solver", "s.prototxt", "--model", str(model), "--crop", "48x32", "--batch", "2"]
    assert T.main(args + ["--data", lists["kitti"], "--kitti"]) == 0
    out_png = capsys.readouterr().out
    assert T.main(args + ["--data", lists["flo"]]) == 0
    out_flo = capsys.readouterr().out
    losses = lambda out: [l.split("loss = ")[1] for l in out.splitlines() if "loss = " in l]
    assert len(losses(out_png)) == 3 and losses(out_png) == losses(out_flo)
    assert all(np.isfinite(float(x)) for x in losses(out_png))
