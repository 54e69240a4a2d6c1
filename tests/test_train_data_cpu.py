"""Host side of training from files (flownet2_b200.data, flownet2_b200.train): CustomData's key order against libstdc++'s own
std::random_shuffle, the batch sequence, rank shards and resume, the refusals, the flow readers and the ground-truth
quantisation.  No GPU needed."""
import os

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import flownet2_b200 as F
from flownet2_b200 import data as D, files as FI, train as T
from flownet2_b200.files import RunError, write_flo, write_pfm, write_pnm
from tests.golden.make_train_data_golden import CASES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "train_data_golden.npz")


def make_list(d, n, w=9, h=7, flow="flo", seed=0):
    """n samples of w x h PPM frames and .flo / .pfm / .pfm-be flows in directory d -> list path."""
    r = np.random.default_rng(seed)
    lines = []
    for i in range(n):
        f0 = write_pnm(d / ("a%d.ppm" % i), r.integers(0, 256, (h, w, 3), dtype=np.uint8))
        f1 = write_pnm(d / ("b%d.ppm" % i), r.integers(0, 256, (h, w, 3), dtype=np.uint8))
        v = r.normal(0, 20, (h, w, 3)).astype(np.float32)
        if flow == "flo":
            fl = str(d / ("f%d.flo" % i))
            write_flo(fl, v[:, :, :2])
        else:
            fl = write_pfm(d / ("f%d.pfm" % i), v, big_endian=flow == "pfm-be")
        lines.append("%s %s %s" % (f0, f1, fl))
    p = d / "list.txt"
    p.write_text("\n" + "\n\n".join(lines) + "\n")
    return str(p)


# ---- the order ----
@pytest.mark.parametrize("name", sorted(CASES))
def test_permutation_equals_libstdcxx(name):
    n, seed, block, rs, re_, order = CASES[name]
    want = np.load(GOLDEN)[name]
    assert D.permutation(n, True, seed, block, rs, re_, order) == want.tolist()


def test_glibc_rand_and_unpermuted_ranges():
    r = D.GlibcRand(1)
    assert [r() for _ in range(3)] == [1804289383, 846930886, 1681692777]          # glibc's documented first rand() values
    assert D.permutation(10) == list(range(10))
    assert D.permutation(10, range_start=3, range_end=5) == [3, 4, 5]
    assert D.permutation(10, range_start=-4, range_end=99) == list(range(10))       # clamped as CustomData clamps them
    assert D.permutation(10, True, 77, block_size=1)[:10] == list(range(10))        # blocks of 1 shuffle nothing (n2 - 1)
    assert D.permutation(30, True, -5) == D.permutation(30, True, 1)                 # seed <= 0: glibc's initial state
    with pytest.raises(RunError, match="range end 2 is before range start 5"):
        D.permutation(10, range_start=5, range_end=2)


def test_sequence_wraps_shards_and_resumes():
    perm = D.permutation(5, True, 77)
    seq = [perm[i % 5] for i in range(100)]
    assert D.batch_keys(perm, 2, 2) == [perm[4], perm[0]]                          # straddles the end of the list
    assert [k for b in range(50) for k in D.batch_keys(perm, 2, b)] == seq
    r0 = [D.batch_keys(perm, 2, b, 2, 0) for b in range(25)]
    r1 = [D.batch_keys(perm, 2, b, 2, 1) for b in range(25)]
    assert [k for b in range(25) for k in r0[b] + r1[b]] == seq                     # two ranks interleave world 1's batches
    # resume after `it` iterations of iter_size 3, world 2: rank 1 continues at position (it * 3 * 2 + 1) * B
    it, iter_size = 4, 3
    assert D.batch_keys(perm, 2, it * iter_size, 2, 1) == seq[(it * iter_size * 2 + 1) * 2:][:2]


def test_dataset_host_state(tmp_path):
    lst = make_list(tmp_path, 5)
    ds = D.FlowDataset(lst, 2)
    assert ds.size == (9, 7) and ds.flow_format == F.FLOW_FLO and len(ds) == 5
    assert ds.perm == D.permutation(5, True, 77) and ds.keys(2) == [ds.perm[4], ds.perm[0]]
    assert D.FlowDataset(lst, 2, rand_permute=False).keys(0) == [0, 1]
    with pytest.raises(RunError, match="not bound"):
        ds()


# ---- refusals: each names the list line and the file ----
def refusal_cases(d):
    lst = make_list(d, 3)
    lines = open(lst).read().split("\n")                                         # ['', s0, '', s1, '', s2, '']
    a0, b0, f0 = lines[1].split()
    out = []

    def case(name, edit, msg, line=2):
        p = d / (name + ".txt")
        new = list(lines)
        new[1] = edit(a0, b0, f0)
        p.write_text("\n".join(new))
        out.append((name, str(p), r"%s:%d: .*%s" % (p, line, msg)))

    (d / "trunc.ppm").write_bytes(open(a0, "rb").read()[:-5])
    (d / "trunc.flo").write_bytes(open(f0, "rb").read()[:-1])
    (d / "tag.flo").write_bytes(b"PIEX" + open(f0, "rb").read()[4:])
    (d / "gray.pfm").write_bytes(b"Pf\n9 7\n-1.0\n" + bytes(9 * 7 * 4))
    write_flo(str(d / "big.flo"), np.zeros((7, 10, 2), np.float32))
    write_pnm(d / "big.ppm", np.zeros((8, 9, 3), np.uint8))
    write_pfm(d / "other.pfm", np.zeros((7, 9, 3), np.float32))
    (d / "flow.txt").write_bytes(b"")
    case("missing", lambda a, b, f: "%s %s %s" % (a, str(d / "nope.ppm"), f), r"nope\.ppm: no such file")
    case("truncated_frame", lambda a, b, f: "%s %s %s" % (d / "trunc.ppm", b, f), r"trunc\.ppm: truncated raster")
    case("truncated_flow", lambda a, b, f: "%s %s %s" % (a, b, d / "trunc.flo"), r"trunc\.flo: truncated payload")
    case("tag", lambda a, b, f: "%s %s %s" % (a, b, d / "tag.flo"), r"tag\.flo: \.flo tag is b'PIEX', expected 'PIEH'")
    case("pf_gray", lambda a, b, f: "%s %s %s" % (a, b, d / "gray.pfm"), r"gray\.pfm: a one-channel 'Pf' PFM")
    case("flow_size", lambda a, b, f: "%s %s %s" % (a, b, d / "big.flo"), r"big\.flo is 10x7 but its frames are 9x7")
    case("frame_size", lambda a, b, f: "%s %s %s" % (a, d / "big.ppm", f), r"is 9x7 but .*big\.ppm is 9x8")
    case("mixed_format", lambda a, b, f: "%s %s %s" % (a, b, d / "other.pfm"), r"other\.pfm is a little-endian \.pfm flow")
    case("other_ext", lambda a, b, f: "%s %s %s" % (a, b, d / "flow.txt"), r"flow\.txt: flows must be \.flo or \.pfm")
    case("occlusion", lambda a, b, f: "%s %s %s occ.png" % (a, b, f), r"an occlusion field \(occ\.png\)")
    case("fields", lambda a, b, f: "%s %s" % (a, b), r"2 fields, expected 'img0 img1 flow'")
    return out


def test_every_refusal_names_its_file_and_line(tmp_path):
    cases = refusal_cases(tmp_path)
    for name, lst, msg in cases:
        # mixed_format: the first sample is fine and sets the format; the refused file sits on the list's later line
        if name in ("flow_size", "frame_size", "mixed_format"):
            lines = open(lst).read().split("\n")
            lines[1], lines[3] = lines[3], lines[1]
            open(lst, "w").write("\n".join(lines))
            msg = msg.replace(":2:", ":4:")
        with pytest.raises(RunError, match=msg):
            D.FlowDataset(lst, 2)
    with pytest.raises(RunError, match="no such list file"):
        D.FlowDataset(str(tmp_path / "none.txt"), 2)


def test_train_command_refuses_with_status_2(tmp_path, capsys):
    cases = refusal_cases(tmp_path)
    solver = tmp_path / "solver.prototxt"
    solver.write_text('base_lr: 0.001\nlr_policy: "fixed"\nmax_iter: 1\n')
    model = os.path.join(ROOT, "models", "FlowNet2-C_train.prototxt.template")
    base = ["--solver", str(solver), "--model", model, "--crop", "8x8", "--batch", "2"]
    assert T.main(base + ["--data", cases[0][1]]) == 2
    err = capsys.readouterr().err
    assert err.startswith("error: %s:2: " % cases[0][1]) and err.count("\n") == 1
    assert T.main(base[:-4] + ["--crop", "448", "--batch", "2", "--data", cases[0][1]]) == 2
    assert "--crop must be WIDTHxHEIGHT, got 448" in capsys.readouterr().err
    assert T.main(base + ["--data", cases[0][1], "--weights", str(tmp_path / "w.caffemodel:net1_")]) == 2
    assert "w.caffemodel: no such weights file" in capsys.readouterr().err
    (tmp_path / "w.caffemodel").write_bytes(b"")
    (tmp_path / "x.solverstate").write_bytes(b"")
    assert T.main(base + ["--data", cases[0][1], "--weights", str(tmp_path / "w.caffemodel"),
                          "--snapshot", str(tmp_path / "x.solverstate")]) == 2           # caffe train refuses the pair too
    assert "give --snapshot to resume training or --weights to finetune, not both" in capsys.readouterr().err


def test_weights_and_template_helpers(tmp_path):
    w = tmp_path / "c.caffemodel"
    w.write_bytes(b"")
    assert T.parse_weights(["%s:net1_,%s" % (w, w)]) == [(str(w), "net1_"), (str(w), "")]
    text = T.model_text(os.path.join(ROOT, "models", "FlowNet2-C_train.prototxt.template"), (448, 320), (512, 384), 8)
    assert "dim: 8 dim: 3 dim: 384 dim: 512" in text and "crop_width: 448" in text and "$" not in text
    assert T.solver_display('display: 20\nbase_lr: 1\n') == 20 and T.solver_display("base_lr: 1") == 0
    assert T.rank_params({"snapshot": 5, "snapshot_after_train": True}, 1) == {"snapshot": 0, "snapshot_after_train": False}
    assert T.rank_params({"snapshot": 5, "snapshot_after_train": True}, 0) == {"snapshot": 5, "snapshot_after_train": True}


# ---- flow files ----
@pytest.mark.parametrize("kind", ["flo", "pfm", "pfm-be"])
def test_flow_payload_reader_equals_numpy(tmp_path, kind):
    r = np.random.default_rng(7)
    v = r.normal(0, 30, (5, 11, 3)).astype(np.float32)
    if kind == "flo":
        p = str(tmp_path / "x.flo")
        write_flo(p, v[:, :, :2])
    else:
        p = write_pfm(tmp_path / "x.pfm", v, big_endian=kind == "pfm-be")
    hdr = FI.flow_header(p)
    assert (hdr.width, hdr.height) == (11, 5)
    assert hdr.format == {"flo": F.FLOW_FLO, "pfm": F.FLOW_PFM, "pfm-be": F.FLOW_PFM_BE}[kind]
    buf = np.empty(hdr.nbytes + 8, np.uint8)
    FI.read_flow_payload(p, hdr, buf[4:4 + hdr.nbytes])
    raw = open(p, "rb").read()
    assert bytes(buf[4:4 + hdr.nbytes]) == raw[len(raw) - hdr.nbytes:]                 # the payload as stored
    if kind == "flo":
        want = np.fromfile(p, "<f4", offset=12).reshape(5, 11, 2)
    else:
        want = np.fromfile(p, ">f4" if kind == "pfm-be" else "<f4", offset=len(raw) - hdr.nbytes).reshape(5, 11, 3)[::-1, :, :2]
    assert np.array_equal(FI.read_flow(p), want) and np.array_equal(want, v[:, :, :2])


def test_uint16flow_restates_the_short_round_trip():
    v = np.array([0.0, -0.0, 1.0, -0.01, 0.03125, -0.03124, 1023.96875, 1023.97, 1024.0, -1024.0, -1024.03, -1024.04,
                  np.nan, np.inf, -np.inf, 3.3e38, 12.345678], np.float32)
    got = D.uint16flow(v)
    short = lambda x: int(np.trunc(np.float32(x) * np.float32(32)))
    for x, g in zip(v, got):
        if not abs(float(x)) < 2 ** 20 or not -32768 <= short(x) <= 32766:                 # NaN, inf, 3.3e38 included
            assert np.isnan(g), x
        else:
            assert g == np.float32(short(x) / 32.0) and (g != 0 or not np.signbit(g)), (x, g)     # zero is +0
    assert np.isnan(got[[7, 8, 11, 12, 13, 14, 15]]).all() and got[9] == -1024.0 and got[10] == -1024.0


# ---- ranks ----
def _rank_worker(rank, world, port, lst, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ds = D.FlowDataset(lst, 2)                                          # world and rank from the process group
        mine = [ds.keys(b) for b in range(6)]
        every = [None] * world
        dist.all_gather_object(every, mine)
        param = T.rank_params({"snapshot": 5, "snapshot_after_train": True}, dist.get_rank())
        q.put((rank, ds.world, ds.rank, every, ds.perm, bool(param["snapshot"])))
    finally:
        dist.destroy_process_group()


def test_two_ranks_partition_the_sequence(tmp_path):
    lst = make_list(tmp_path, 7)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_rank_worker, args=(r, 2, port, lst, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (r0, w0, k0, every, perm, snap0), (r1, w1, k1, every1, _, snap1) = res
    assert (w0, k0, w1, k1) == (2, 0, 2, 1) and every == every1
    assert snap0 and not snap1                                               # only rank 0 writes snapshots
    got = [k for b in range(6) for r in range(2) for k in every[r][b]]
    assert got == [perm[i % 7] for i in range(24)]                           # the ranks' batches partition world 1's sequence
