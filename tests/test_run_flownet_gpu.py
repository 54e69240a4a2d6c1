"""8-bit frames converted on the device (fn2_frames_to_tensor, Net.set_input_image), blobs read back as NHWC, and the image-file
driver (flownet2_b200.run) against Net.forward and the float64 oracle."""
import gc
import os

import numpy as np
import pytest

from flownet2_b200 import run as R
from flownet2_b200.files import read_image
from tests.test_run_flownet_cpu import write_pnm

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TEMPLATE = os.path.join(ROOT, "models", "FlowNet2-C_deploy.prototxt.template")


def blob_of(frames):
    """(N, H, W[, K]) uint8 -> (N, 3, H, W) float32 as image_to_blob makes each frame, a gray frame broadcast (pycaffe)."""
    import flownet2_b200 as F
    out = [F.image_to_blob(f[:, :, 0] if f.ndim == 3 and f.shape[2] == 1 else f) for f in frames]
    return np.concatenate([np.broadcast_to(b, (1, 3) + b.shape[2:]) for b in out]).astype(np.float32)


def random_frames(r, n, h, w, k):
    return r.integers(0, 256, (n, h, w, k), dtype=np.uint8)


@pytest.mark.parametrize("k", [1, 3, 4])
@pytest.mark.parametrize("layout", ["nchw", "pad", "slice"])
def test_frames_to_tensor_bit_exact(fn2, k, layout):
    import torch
    from flownet2_b200 import ops
    n, h, w = 3, 5, 37                                        # odd W: W*K is odd for K = 1, 3
    fr = random_frames(np.random.default_rng(10 + k), n, h, w, k)
    want = blob_of(fr)
    dev = torch.from_numpy(fr).cuda()
    if layout == "nchw":
        parent, lo = torch.full((n, 3, h, w), float("nan"), device="cuda"), 0
    else:                                                     # channels_last parent: a 4-wide padded pixel, or channels 2..4 of 8
        parent, lo = torch.full((n, 4 if layout == "pad" else 8, h, w), float("nan"), device="cuda").contiguous(
            memory_format=torch.channels_last), 0 if layout == "pad" else 2
    dst = parent[:, lo:lo + 3]
    ops.frames_to_tensor(dev, dst)
    torch.cuda.synchronize()
    got = parent.cpu().numpy()
    assert np.array_equal(got[:, lo:lo + 3], want)
    rest = np.delete(got, range(lo, lo + 3), axis=1)
    assert np.isnan(rest).all()                               # channels outside the view are untouched


def flownet2c(fn2, w, h, batch, seed=1701):
    net = fn2.Net(fn2.fill_template(fn2.model_template("FlowNet2-C"), w, h), None, fn2.TEST, batch=batch)
    net.fill_params(seed)
    return net


def test_set_input_image_matches_set_input(fn2):
    W, H, B = 128, 96, 2
    net = flownet2c(fn2, W, H, B)
    r = np.random.default_rng(3)
    for k0, k1 in ((3, 4), (1, 3)):
        f0, f1 = random_frames(r, B, H, W, k0), random_frames(r, B, H, W, k1)
        b0, b1 = blob_of(f0), blob_of(f1)
        net.forward(img0=b0, img1=b1)                          # eager, then graph capture and replay below
        net.set_input("img0", b0)
        net.set_input("img1", b1)
        net.forward_async()
        want = net.blobs["predict_flow_final"].data
        net.set_input_image("img0", f0)
        net.set_input_image("img1", f1)
        assert np.array_equal(net.blobs["img0"].data, b0) and np.array_equal(net.blobs["img1"].data, b1)
        net.forward_async()
        got = net.blobs["predict_flow_final"].data
        assert np.array_equal(got, want) and np.isfinite(got).all()
    one = flownet2c(fn2, W, H, 1)
    g = random_frames(r, 1, H, W, 1)[0, :, :, 0]
    one.set_input_image("img0", g)                             # (H, W) for N = 1
    assert np.array_equal(one.blobs["img0"].data, blob_of(g[None]))
    with pytest.raises(fn2.Fn2Error, match="frames must be uint8"):
        one.set_input_image("img0", g.astype(np.float32))
    with pytest.raises(fn2.Fn2Error, match="channels must be 1, 3 or 4"):
        one.set_input_image("img0", np.zeros((H, W, 2), np.uint8))
    with pytest.raises(fn2.Fn2Error, match=r"blob predict_flow_final must have shape \(N, 3, H, W\)"):
        one.set_input_image("predict_flow_final", np.zeros((H, W, 3), np.uint8))


def test_get_blob_nhwc_is_the_transpose(fn2):
    net = flownet2c(fn2, 128, 96, 2)
    r = np.random.default_rng(4)
    net.set_input_image("img0", random_frames(r, 2, 96, 128, 3))
    net.set_input_image("img1", random_frames(r, 2, 96, 128, 3))
    net.forward_async()
    wide = [b for b in net.blob_names if net.blobs[b].shape[1] >= 32][:2]
    for name in ["predict_flow_final", "img0"] + wide:
        got = net.get_blob_nhwc(name)
        assert np.array_equal(got, net.blobs[name].data.transpose(0, 2, 3, 1)), name


def test_warm_frames_in_and_nhwc_out_allocate_nothing(fn2):
    import torch
    W, H, B = 128, 96, 2
    net = flownet2c(fn2, W, H, B)
    r = np.random.default_rng(5)
    f = torch.from_numpy(random_frames(r, 2 * B, H, W, 3)).cuda()
    flow = torch.empty((B, H, W, 2), device="cuda")
    host = [random_frames(r, B, H, W, 3) for _ in range(2)]

    def step():
        net.set_input_image_device("img0", f.data_ptr(), 3)
        net.set_input_image_device("img1", f[B:].data_ptr(), 3)
        net.forward_async()
        net.get_blob_nhwc_device("predict_flow_final", flow.data_ptr())
        net.set_input_image("img0", host[0])
        net.set_input_image("img1", host[1])
        net.forward_async()
        return net.get_blob_nhwc("predict_flow_final")

    for _ in range(3):
        step()
    n0 = fn2.device_allocations()[0]
    for _ in range(3):
        step()
    assert fn2.device_allocations()[0] == n0


# ---- the driver ----
def chairs_frames(size, seed):
    """A frame pair of `size` (w, h) cut from the FlyingChairs crop, the second shifted, both with seeded noise."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "chairs_crop.npz"))
    big = np.concatenate([g["img1"], np.concatenate([g["img0"], g["img0"][::-1]], axis=0)], axis=1)      # 128 x 192
    w, h = size
    r = np.random.default_rng(seed)
    a = big[:h, :w].astype(np.int16)
    b = np.roll(a, (1, 2), axis=(0, 1))
    noise = lambda x: np.clip(x + r.integers(-3, 4, x.shape), 0, 255).astype(np.uint8)
    return noise(a), noise(b)


@pytest.fixture(scope="module")
def scene(tmp_path_factory, fn2):
    """Five pairs in two sizes (128x96 and 192x64): PPM, PNG when Pillow imports, and one gray frame; the weights as a
    caffemodel written by fill_params."""
    d = tmp_path_factory.mktemp("run")
    try:
        from PIL import Image
    except ImportError:
        Image = None
    A, Bs = (128, 96), (192, 64)
    spec = [(A, "ppm"), (Bs, "png"), (A, "gray"), (Bs, "ppm"), (A, "png")]
    pairs = []
    for i, (size, kind) in enumerate(spec):
        f0, f1 = chairs_frames(size, 100 + i)
        paths = []
        for j, f in enumerate((f0, f1)):
            if kind == "gray" and j == 0:
                p = write_pnm(d / ("p%d_%d.pgm" % (i, j)), f.mean(axis=2).round().astype(np.uint8))
            elif kind == "png" and Image is not None:
                p = str(d / ("p%d_%d.png" % (i, j)))
                Image.fromarray(f).save(p)
            else:
                p = write_pnm(d / ("p%d_%d.ppm" % (i, j)), f)
            paths.append(p)
        pairs.append((size, paths[0], paths[1]))
    net = flownet2c(fn2, 64, 64, 1)
    model = d / "w.caffemodel"
    model.write_bytes(net.to_caffemodel())
    del net
    return d, str(model), pairs


def write_list(path, pairs, outdir):
    outs = [os.path.join(str(outdir), "out%d.flo" % i) for i in range(len(pairs))]
    os.makedirs(str(outdir), exist_ok=True)
    with open(str(path), "w") as f:
        f.write("\n")
        for (_, a, b), o in zip(pairs, outs):
            f.write("%s %s %s\n\n" % (a, b, o))
    return outs


def test_single_pair_equals_net_forward(fn2, scene, tmp_path):
    d, model, pairs = scene
    for i in (0, 2):                                          # RGB, and gray + RGB
        (w, h), a, b = pairs[i]
        out = str(tmp_path / ("single%d.flo" % i))
        assert R.main([model, TEMPLATE, a, b, out]) == 0
        net = fn2.Net(fn2.fill_template(open(TEMPLATE).read(), w, h), model, fn2.TEST, batch=1)
        want = net.forward(img0=blob_of([read_image(a)]), img1=blob_of([read_image(b)]))["predict_flow_final"][0]
        got = fn2.read_flo(out)
        assert got.shape == (2, h, w) and np.array_equal(got, want)


def test_many_pairs_against_oracle_and_single_pair(fn2, scene, tmp_path):
    from oracle.net import OracleNet
    d, model, pairs = scene
    lst = tmp_path / "pairs.txt"
    gc.collect()                                              # nets of earlier tests that are only garbage by now
    live0 = fn2.device_allocations()[1]
    outs = write_list(lst, pairs, tmp_path / "b2")
    assert R.main([model, TEMPLATE, str(lst), "--batch", "2"]) == 0
    assert fn2.device_allocations()[1] == live0                 # every net and staging buffer was freed
    weights = open(model, "rb").read()
    for size in ((128, 96), (192, 64)):
        idx = [i for i, p in enumerate(pairs) if p[0] == size]
        proto = fn2.fill_template(open(TEMPLATE).read(), *size)
        img0 = blob_of([read_image(pairs[i][1]) for i in idx])
        img1 = blob_of([read_image(pairs[i][2]) for i in idx])
        want = OracleNet(proto, weights, batch=len(idx), f64acc=True).forward(img0=img0, img1=img1)["predict_flow_final"]
        for j, i in enumerate(idx):
            got = fn2.read_flo(outs[i])
            err = float(np.abs(got.astype(np.float64) - want[j]).max())
            assert np.isfinite(got).all() and err <= 1e-4, (i, err)
    # batch 1: every file equals the single-pair run's
    outs1 = write_list(lst, pairs, tmp_path / "b1")
    assert R.main([model, TEMPLATE, str(lst)]) == 0
    assert fn2.device_allocations()[1] == live0
    for i, (_, a, b) in enumerate(pairs):
        single = str(tmp_path / ("s%d.flo" % i))
        assert R.main([model, TEMPLATE, a, b, single]) == 0
        assert open(single, "rb").read() == open(outs1[i], "rb").read(), i


def test_ranks_write_disjoint_shards(fn2, scene, tmp_path, monkeypatch, capsys):
    d, model, pairs = scene
    lst = tmp_path / "pairs.txt"
    outs = write_list(lst, pairs, tmp_path / "o")
    written = []
    for rank in (0, 1):
        monkeypatch.setenv("WORLD_SIZE", "2")
        monkeypatch.setenv("RANK", str(rank))
        monkeypatch.setenv("LOCAL_RANK", "0")
        before = set(os.listdir(str(tmp_path / "o")))
        assert R.main([model, TEMPLATE, str(lst), "--batch", "2"]) == 0
        written.append(set(os.listdir(str(tmp_path / "o"))) - before)
        assert "rank %d/2: %d pairs" % (rank, len(written[-1])) in capsys.readouterr().out
    assert not written[0] & written[1]
    assert written[0] | written[1] == set(os.path.basename(o) for o in outs)
    assert written[0] == set("out%d.flo" % i for i in (0, 2, 4))
