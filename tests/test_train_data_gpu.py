"""Training from files on the device: fn2_flow_to_tensor bit-exact against its numpy restatement, the dataset's blobs equal to
set_input of the host restatement, a Solver fed by the dataset equal to one fed by arrays, warm steps allocating nothing, and
the train command's interrupted run equal to an uninterrupted one."""
import os

import numpy as np
import pytest

from flownet2_b200 import data as D, train as T
from flownet2_b200.files import write_flo, write_pfm, write_pnm

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def special_flow(r, h, w, k):
    """(h, w, k) float32 flow with NaN, +-0, values truncating to 32767, below -32768, |v| >= 1024 and ordinary values."""
    v = r.normal(0, 40, (h, w, k)).astype(np.float32)
    s = np.array([np.nan, 0.0, -0.0, -0.01, 0.01, 1023.96875, 1023.97, 1024.0, -1024.0, -1024.03, -1024.04, 5000.0, -5000.0,
                  np.inf, -np.inf, 1e-30, -1e-30, 31.999, -31.999], np.float32)
    flat = v.reshape(-1)
    flat[r.choice(flat.size, 3 * s.size, replace=False)] = np.tile(s, 3)
    return v


def payload(v, kind):
    """The bytes of N flow files' payloads, back to back: v is (N, H, W, 3) top-down."""
    if kind == "flo":
        return np.ascontiguousarray(v[..., :2], "<f4").tobytes()
    return np.ascontiguousarray(v[:, ::-1], ">f4" if kind == "pfm-be" else "<f4").tobytes()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("kind", ["flo", "pfm", "pfm-be"])
@pytest.mark.parametrize("quant", [0, 1])
@pytest.mark.parametrize("layout", ["nchw", "pad", "slice"])
def test_flow_to_tensor_bit_exact(fn2, kind, quant, layout):
    import torch
    from flownet2_b200 import ops
    n, h, w = 3, 5, 37
    v = special_flow(np.random.default_rng(20 + quant), n * h, w, 3).reshape(n, h, w, 3)
    want = v[..., :2].transpose(0, 3, 1, 2)
    if quant:
        want = D.uint16flow(want)
    src = torch.from_numpy(np.frombuffer(payload(v, kind), np.uint8).copy()).cuda()
    fmt = {"flo": fn2.FLOW_FLO, "pfm": fn2.FLOW_PFM, "pfm-be": fn2.FLOW_PFM_BE}[kind]
    fill = -7.0
    if layout == "nchw":
        parent, lo = torch.full((n, 2, h, w), fill, device="cuda"), 0
    else:
        parent, lo = torch.full((n, 4 if layout == "pad" else 8, h, w), fill, device="cuda").contiguous(
            memory_format=torch.channels_last), 0 if layout == "pad" else 2
    ops.flow_to_tensor(src, fmt, fn2.FLOW_UINT16FLOW if quant else 0, parent[:, lo:lo + 2])
    torch.cuda.synchronize()
    got = parent.cpu().numpy()
    assert np.array_equal(bits(got[:, lo:lo + 2]), bits(want))
    assert (np.delete(got, range(lo, lo + 2), axis=1) == fill).all()          # channels outside the view are untouched


def test_flow_to_tensor_refusals(fn2):
    import torch
    from flownet2_b200 import ops
    src = torch.zeros(4 * 2 * 3 * 4 * 4, dtype=torch.uint8, device="cuda")
    dst = torch.zeros((1, 2, 3, 4), device="cuda")
    with pytest.raises(fn2.Fn2Error, match="format must be FN2_FLOW_FLO, FN2_FLOW_PFM, FN2_FLOW_PFM_BE or FN2_FLOW_KITTI, got 4"):
        ops.flow_to_tensor(src, 4, 0, dst)
    with pytest.raises(fn2.Fn2Error, match="unknown flags 0x2"):
        ops.flow_to_tensor(src, fn2.FLOW_FLO, 2, dst)
    with pytest.raises(fn2.Fn2Error, match="dst must have 2 channels"):
        ops.flow_to_tensor(src, fn2.FLOW_FLO, 0, torch.zeros((1, 3, 3, 4), device="cuda"))
    with pytest.raises(fn2.Fn2Error, match="src must be 4-byte aligned"):
        ops.flow_to_tensor(src[1:], fn2.FLOW_FLO, 0, dst)
    net = fn2.Net(fn2.fill_train_template(fn2.train_template("FlowNet2-C"), 64, 64, 64, 64, 1), None, fn2.TRAIN)
    with pytest.raises(fn2.Fn2Error, match=r"blob img0 must have shape \(N, 2, H, W\)"):
        net.set_input_flow_device("img0", src.data_ptr(), fn2.FLOW_FLO)


# ---- the dataset ----
def scene(d, n, w, h, kind="flo", seed=0):
    """n samples of w x h frames (PPM, one PNG when Pillow imports, one gray PGM) and flows with special values -> list path."""
    try:
        from PIL import Image
    except ImportError:
        Image = None
    r = np.random.default_rng(seed)
    lines = []
    for i in range(n):
        paths = []
        for j in range(2):
            f = r.integers(0, 256, (h, w, 3), dtype=np.uint8)
            if i == 1 and j == 0:
                paths.append(write_pnm(d / ("g%d.pgm" % i), f[:, :, 0]))
            elif i == 2 and Image is not None:
                paths.append(str(d / ("p%d_%d.png" % (i, j))))
                Image.fromarray(f).save(paths[-1])
            else:
                paths.append(write_pnm(d / ("p%d_%d.ppm" % (i, j)), f))
        v = special_flow(r, h, w, 3)
        if kind == "flo":
            fl = str(d / ("f%d.flo" % i))
            write_flo(fl, v[:, :, :2])
        else:
            fl = write_pfm(d / ("f%d.pfm" % i), v, big_endian=kind == "pfm-be")
        lines.append("%s %s %s" % (paths[0], paths[1], fl))
    p = d / "list.txt"
    p.write_text("\n".join(lines) + "\n")
    return str(p)


def train_net(fn2, ds, seed=1701):
    W, H = ds.size
    net = fn2.Net(fn2.fill_train_template(fn2.train_template("FlowNet2-C"), 192, 128, W, H, ds.batch), None, fn2.TRAIN)
    net.fill_params(seed)
    return net


@pytest.mark.parametrize("kind,encoding", [("flo", "uint16"), ("pfm-be", "uint16"), ("flo", "float")])
def test_dataset_blobs_equal_host_restatement(fn2, tmp_path, kind, encoding):
    ds = D.FlowDataset(scene(tmp_path, 5, 224, 160, kind), 2, flow_encoding=encoding)
    net = train_net(fn2, ds)
    ds.bind(net)
    for k in range(6):                                                   # 12 items over 5 samples: more than one wrap
        assert ds() == {}
        want = ds.host_batch(k)
        for name, a in zip(("img0", "img1", "flow_gt"), want):
            assert np.array_equal(bits(net.blobs[name].data), bits(a)), (k, name)
    b = ds.busy()
    assert b["calls"] == 6 and b["read"] > 0 and b["h2d"] > 0 and b["convert"] > 0
    ds.close()


def test_solver_fed_by_dataset_equals_solver_fed_by_arrays(fn2, tmp_path, monkeypatch):
    from tests.test_solver_gpu import arenas
    monkeypatch.setenv("FN2_SEED", "77")
    lst = scene(tmp_path, 5, 224, 160)
    solver_text = 'type: "Adam"\nbase_lr: 1e-4\nmomentum: 0.9\nmomentum2: 0.999\nlr_policy: "fixed"\nmax_iter: 3\n'
    ds = D.FlowDataset(lst, 2)
    host = D.FlowDataset(lst, 2)
    nets = [train_net(fn2, ds), train_net(fn2, ds)]
    solvers = [fn2.Solver(solver_text, n) for n in nets]
    ds.bind(nets[0])
    k = iter(range(100))

    def arrays():
        i0, i1, fl = host.host_batch(next(k))
        return {"img0": i0, "img1": i1, "flow_gt": fl}

    losses = [[], []]
    for _ in range(3):
        solvers[0].step(1, ds)
        solvers[1].step(1, arrays)
        for j in range(2):
            losses[j].append(solvers[j].smoothed_loss)
    assert losses[0] == losses[1] and all(np.isfinite(losses[0]))
    a, b = arenas(fn2, nets[0]), arenas(fn2, nets[1])
    assert np.array_equal(bits(a[0]), bits(b[0])) and np.array_equal(bits(a[1]), bits(b[1]))
    ds.close()


def test_warm_steps_with_the_dataset_allocate_nothing(fn2, tmp_path):
    ds = D.FlowDataset(scene(tmp_path, 5, 224, 160), 2)
    net = train_net(fn2, ds)
    solver = fn2.Solver('type: "Adam"\nbase_lr: 1e-4\nlr_policy: "fixed"\nmax_iter: 100\n', net)
    ds.bind(net)
    solver.step(3, ds)
    n0 = fn2.device_allocations()[0]
    solver.step(4, ds)
    assert fn2.device_allocations()[0] == n0
    ds.close()


# ---- the train command ----
TINY_NET = """name: "tiny"
layer { name: "data" type: "Input" top: "img0" top: "img1" top: "flow_gt"
  input_param { shape { dim: $BATCH$ dim: 3 dim: $DATA_HEIGHT$ dim: $DATA_WIDTH$ }
                shape { dim: $BATCH$ dim: 3 dim: $DATA_HEIGHT$ dim: $DATA_WIDTH$ }
                shape { dim: $BATCH$ dim: 2 dim: $DATA_HEIGHT$ dim: $DATA_WIDTH$ } } }
layer { name: "scale0" type: "Eltwise" bottom: "img0" top: "img0s" eltwise_param { operation: SUM coeff: 0.00392156862745 } }
layer { name: "scale1" type: "Eltwise" bottom: "img1" top: "img1s" eltwise_param { operation: SUM coeff: 0.00392156862745 } }
layer { name: "concat" type: "Concat" bottom: "img0s" bottom: "img1s" top: "pair" }
layer { name: "conv1" type: "Convolution" bottom: "pair" top: "conv1"
  convolution_param { num_output: 16 kernel_size: 3 pad: 1 weight_filler { type: "msra" } bias_filler { type: "constant" } } }
layer { name: "relu1" type: "ReLU" bottom: "conv1" top: "conv1" relu_param { negative_slope: 0.1 } }
layer { name: "predict" type: "Convolution" bottom: "conv1" top: "predict"
  convolution_param { num_output: 2 kernel_size: 3 pad: 1 weight_filler { type: "msra" } bias_filler { type: "constant" } } }
layer { name: "loss" type: "L1Loss" bottom: "predict" bottom: "flow_gt" top: "loss" loss_weight: 1
  l1_loss_param { l2_per_location: true } }
"""


def test_train_command_resume_equals_uninterrupted(fn2, tmp_path, monkeypatch, capsys):
    # 7 samples, batch 2, snapshot at 5: the resumed run starts at sequence position 10, which is not a multiple of 7, so its
    # batches differ from the ones a run restarted at position 0 would see
    lst = scene(tmp_path, 7, 48, 32)
    perm = D.FlowDataset(lst, 2).perm
    assert all(D.batch_keys(perm, 2, 5 + j) != D.batch_keys(perm, 2, j) for j in range(5))
    model = tmp_path / "tiny.prototxt.template"
    model.write_text(TINY_NET)
    net = fn2.Net(fn2.fill_train_template(TINY_NET, 48, 32, 48, 32, 2), None, fn2.TRAIN)
    net.fill_params(3)
    weights = tmp_path / "init.caffemodel"
    weights.write_bytes(net.to_caffemodel())
    del net
    solver = 'type: "Adam"\nbase_lr: 1e-3\nlr_policy: "step"\ngamma: 0.5\nstepsize: 4\nmax_iter: %d\nsnapshot: 5\n' \
             'snapshot_prefix: "tiny"\ndisplay: 2\n'
    for d, iters in (("a", 10), ("b", 5), ("c", 5)):
        (tmp_path / d).mkdir()
        (tmp_path / d / "s.prototxt").write_text(solver % iters)
        (tmp_path / d / "s10.prototxt").write_text(solver % 10)
    args = ["--model", str(model), "--data", lst, "--crop", "48x32", "--batch", "2"]
    monkeypatch.chdir(tmp_path / "a")
    assert T.main(["--solver", "s.prototxt", "--weights", str(weights)] + args) == 0
    out = capsys.readouterr().out
    assert "Iteration 10 (" in out and "Iteration 10, lr = 0.00025" in out and "Optimization Done." in out
    monkeypatch.chdir(tmp_path / "b")
    assert T.main(["--solver", "s.prototxt", "--weights", str(weights)] + args) == 0
    assert T.main(["--solver", "s10.prototxt", "--snapshot", "tiny_iter_5.solverstate"] + args) == 0
    for ext in ("caffemodel", "solverstate"):
        a = (tmp_path / "a" / ("tiny_iter_10." + ext)).read_bytes()
        assert a == (tmp_path / "b" / ("tiny_iter_10." + ext)).read_bytes(), ext
    assert (tmp_path / "a" / "tiny_iter_5.caffemodel").read_bytes() == (tmp_path / "b" / "tiny_iter_5.caffemodel").read_bytes()
    # the same resume with the data restarted at position 0, as the reference restarts it, ends elsewhere
    monkeypatch.chdir(tmp_path / "c")
    assert T.main(["--solver", "s.prototxt", "--weights", str(weights)] + args) == 0
    seek = D.FlowDataset.seek
    monkeypatch.setattr(D.FlowDataset, "seek", lambda self, k: seek(self, 0 if self.net is None else k))  # train's seek ignored
    assert T.main(["--solver", "s10.prototxt", "--snapshot", "tiny_iter_5.solverstate"] + args) == 0
    monkeypatch.undo()
    monkeypatch.chdir(tmp_path)
    assert (tmp_path / "c" / "tiny_iter_10.caffemodel").read_bytes() != (tmp_path / "a" / "tiny_iter_10.caffemodel").read_bytes()
    capsys.readouterr()
    assert T.main(["--solver", str(tmp_path / "b" / "s10.prototxt"), "--snapshot", str(tmp_path / "b" / "tiny_iter_5.solverstate"),
                   "--weights", str(weights)] + args) == 2
    assert "not both" in capsys.readouterr().err
    bad = tmp_path / "bad.txt"
    bad.write_text(open(lst).read() + "x.ppm y.ppm z.flo\n")
    assert T.main(["--solver", str(tmp_path / "a" / "s.prototxt")] + args[:2] + ["--data", str(bad)] + args[4:]) == 2
    assert capsys.readouterr().err.startswith("error: %s:8: x.ppm: no such file" % bad)


def test_seek_after_bind_delivers_that_batch(fn2, tmp_path):
    ds = D.FlowDataset(scene(tmp_path, 7, 224, 160), 2)
    net = train_net(fn2, ds)
    ds.bind(net)
    for k in (0, 1, 9, 3, 4, 20):                                        # forwards, backwards, jumps past a wrap
        if k != ds.next_batch:
            ds.seek(k)
        assert ds() == {} and ds.next_batch == k + 1
        for name, a in zip(("img0", "img1", "flow_gt"), ds.host_batch(k)):
            assert np.array_equal(bits(net.blobs[name].data), bits(a)), (k, name)
    ds.close()


def _world2_worker(rank, port, tmp, lst, model, q):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), FN2_SEED=str(11 + rank))   # different fills per rank
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=2)                # two ranks on one GPU: gloo over CUDA tensors
    try:
        import flownet2_b200 as F
        from flownet2_b200 import parallel as P
        os.chdir(os.path.join(tmp, "r%d" % rank))
        a = T.parse_args(["--solver", "s.prototxt", "--model", model, "--data", lst, "--crop", "48x32", "--batch", "2"])
        solver = T.train(a, world=2, rank=rank, device=0)
        arena = P.arena_tensor(solver.net).cpu().numpy().view(np.uint32).copy()
        q.put((rank, arena, sorted(os.listdir("."))))
    finally:
        dist.destroy_process_group()


def test_train_world2_broadcasts_allreduces_and_only_rank0_snapshots(fn2, tmp_path):
    import torch.multiprocessing as mp
    lst = scene(tmp_path, 7, 48, 32)
    model = tmp_path / "tiny.prototxt.template"
    model.write_text(TINY_NET)
    for r in (0, 1):
        (tmp_path / ("r%d" % r)).mkdir()
        (tmp_path / ("r%d" % r) / "s.prototxt").write_text(
            'type: "Adam"\nbase_lr: 1e-3\nlr_policy: "fixed"\nmax_iter: 4\nsnapshot: 2\nsnapshot_prefix: "w2"\n')
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_world2_worker, args=(r, port, str(tmp_path), lst, str(model), q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=300) for _ in procs), key=lambda x: x[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    (_, a0, files0), (_, a1, files1) = res
    assert np.array_equal(a0, a1)                          # one broadcast, then the same all-reduced update on both ranks
    assert files0 == ["s.prototxt", "w2_iter_2.caffemodel", "w2_iter_2.solverstate", "w2_iter_4.caffemodel",
                      "w2_iter_4.solverstate"]
    assert files1 == ["s.prototxt"]                        # only rank 0 writes snapshots
