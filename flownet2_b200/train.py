"""Train a network from image and flow files: the reference's ``caffe train`` (tools/caffe.cpp) over a CustomData list.

    python -m flownet2_b200.train --solver solver.prototxt --model models/FlowNet2-C_train.prototxt.template \\
        --data train.txt --crop 448x320 --batch 8 [--weights c.caffemodel[:net1_] ...] [--snapshot x.solverstate] [--gpu N]

The model is a training prototxt whose first three Input tops are img0, img1 and the flow (models/*_train.prototxt.template).
A template gets $DATA_WIDTH$ / $DATA_HEIGHT$ from the list's frame size and $TARGET_*$ / $BATCH$ from --crop and --batch; a
filled prototxt is used as it is.  --weights takes weight files, each with an optional Net.copy_from prefix after a colon
(the stacked schedule's hand-over).  --snapshot resumes from a .solverstate, and the data continue where the interrupted run
stopped (flownet2_b200.data); as in Caffe, --weights and --snapshot exclude each other.  Without either, the parameters are
drawn from the prototxt's fillers by Net.fill_params(FN2_SEED), which also starts every DataAugmentation mean as already
computed.  The solver's max_iter, snapshot and snapshot_prefix govern the run, as in Caffe.  Every --display iterations
(default: the solver's display) rank 0 prints Caffe's iteration / loss and iteration / lr lines; the loss is the solver's
smoothed loss over the iterations since the last line.

The data flags mirror CustomData's data_param: permuted with seed 77 unless told otherwise; --flow-encoding float turns off
the reference's 16-bit quantisation of the ground truth.  --kitti reads every flow of the list as a KITTI 16-bit PNG (sparse
ground truth: its invalid pixels are NaN, which the NaN-aware losses leave out).  Under torchrun (WORLD_SIZE, RANK,
LOCAL_RANK) every rank builds the net, rank 0's parameters are broadcast, each rank takes its own batches and the gradients
are all-reduced before every update; only rank 0 writes snapshots.  Refused inputs exit with status 2 and a one-line message.

Validation (--val LIST --val-model TEMPLATE --val-interval N [--val-batch B] [--no-val-initial] [--val-occlusions LIST]
[--val-objects LIST] [--val-log FILE]): the weights are scored on a held-out list with the deploy net and evaluate's metrics
(flownet2_b200.evaluate.Validator), on Caffe's TestAll schedule (val_iters): at the start of every iteration k with
k % N == 0 (k = 0 unless --no-val-initial; the first iteration of a resumed run when it is due), and after the last iteration
when the run ends at a multiple of N.  Iteration k scores the weights after k updates, those of <prefix>_iter_k.caffemodel,
handed over as the same to_caffemodel() bytes, so it equals evaluate on that snapshot.  The list is probed before the net is
built and the hand-over is checked before iteration 0 (evaluate.check_handover).  Rank 0 prints Caffe's Solver::Test lines,
'Test net output #i: <score> = <value>' per score of the summary (nan when empty), and --val-log appends one JSON line per
validation; under torchrun each rank scores its share of the list and rank 0 gathers the records.  The validation only
reads the training net: the snapshots, the solver state, the data sequence and every training line are those of the same
run without --val.
"""
import argparse
import json
import os
import re
import sys
import time

from .files import RunError


def parse_size(text):
    m = re.fullmatch(r"(\d+)x(\d+)", text or "")
    if not m or int(m.group(1)) < 1 or int(m.group(2)) < 1:
        raise RunError("--crop must be WIDTHxHEIGHT, got %s" % text)
    return int(m.group(1)), int(m.group(2))


def parse_weights(items):
    """--weights values (space- or comma-separated) -> [(path, prefix)]; 'path:prefix' names a Net.copy_from prefix."""
    out = []
    for item in (w for it in items or [] for w in it.split(",") if w):
        path, prefix = item, ""
        if not os.path.isfile(item) and ":" in item:
            path, prefix = item.rsplit(":", 1)
        if not os.path.isfile(path):
            raise RunError("%s: no such weights file" % path)
        out.append((path, prefix))
    return out


def model_text(path, crop, data_size, batch):
    """The training prototxt: a template filled from the crop, the frames' size and the batch, or a filled file as it is."""
    import flownet2_b200 as F
    if not os.path.isfile(path):
        raise RunError("%s: no such model" % path)
    with open(path) as f:
        text = f.read()
    return F.fill_train_template(text, crop[0], crop[1], data_size[0], data_size[1], batch)


def solver_display(text):
    m = re.search(r"^\s*display\s*:\s*(\d+)", text, re.M)
    return int(m.group(1)) if m else 0


def rank_params(param, rank):
    """Solver parameters as rank `rank` runs them: only rank 0 snapshots."""
    if rank != 0:
        param["snapshot"], param["snapshot_after_train"] = 0, False
    return param


def val_iters(start, max_iter, interval, initial=True):
    """The iterations a run from `start` to `max_iter` validates at, Caffe's TestAll schedule (solver.cpp:205-208, 320-321):
    at the start of every iteration k in [start, max_iter) with k % interval == 0 (k = 0 only with `initial`), and once
    more after the last iteration when the run ends at a multiple of interval (a run resumed past max_iter ends at start)."""
    due = [k for k in range(start, max_iter) if k % interval == 0 and (k > 0 or initial)]
    end = max(start, max_iter)
    return due + [end] if end % interval == 0 else due


def score_keys(summary):
    """The scores of an evaluate summary, in its order: epe, epe_pair_mean, fl_percent, the speed bands and any region scores."""
    from .evaluate import BANDS, REGION_KEYS
    scores = {"epe", "epe_pair_mean", "fl_percent"} | {b[0] for b in BANDS} | {k[0] for v in REGION_KEYS.values() for k in v}
    return [k for k in summary if k in scores]


def val_lines(k, summary):
    """The lines of a validation at iteration k, in the shape of Caffe's Solver::Test: one 'Test net output' line per score
    (nan when a band or region is empty), then a line counting the pairs whose prediction is not finite, if any."""
    lines = ["Iteration %d, Testing net (#0)" % k]
    for i, key in enumerate(score_keys(summary)):
        v = summary[key]
        lines.append("    Test net output #%d: %s = %s" % (i, key, "nan" if v is None else "%.6g" % v))
    if summary["not_finite"]:
        lines.append("    %d validation pairs have a prediction that is not finite" % len(summary["not_finite"]))
    return lines


def val_record(k, summary, handover_s, wall_s):
    """A --val-log line: {"iter": k, ...summary, "handover_s", "wall_s"} as JSON; an empty band is null."""
    return json.dumps(dict({"iter": k}, **summary, handover_s=handover_s, wall_s=wall_s))


VAL_FLAGS = ("val_model", "val_interval", "val_occlusions", "val_objects", "val_log")


def validator(a, world, rank, device):
    """--val and its flags -> an evaluate.Validator over the list (probed here, before any training), or None without --val."""
    from .evaluate import Validator
    from .files import read_list
    if not a.val:
        given = [f for f in VAL_FLAGS if getattr(a, f) is not None] + (["val_batch"] if a.val_batch != 1 else []) + (
            ["no_val_initial"] if not a.val_initial else [])
        if given:
            raise RunError("--%s needs --val" % given[0].replace("_", "-"))
        return None
    if a.val_model is None:
        raise RunError("--val needs --val-model, the deploy template to score with")
    if a.val_interval is None:
        raise RunError("--val needs --val-interval")
    if a.val_interval < 1:
        raise RunError("--val-interval must be at least 1, got %d" % a.val_interval)
    if not os.path.isfile(a.val):
        raise RunError("%s: no such validation list" % a.val)
    return Validator(a.val_model, read_list(a.val), a.val_batch, device, None, a.kitti, a.val_occlusions, a.val_objects,
                     world, rank)


class Validation(object):
    """Scores the training net's weights at the iterations val_iters names: the weights go over as to_caffemodel() bytes,
    as a snapshot would write them, into the validator's kept deploy nets.  Rank 0 prints the lines and appends the log."""

    def __init__(self, val, net, due, rank, out, log):
        self.val, self.net, self.due, self.rank, self.out, self.log = val, net, set(due), rank, out, log

    def __call__(self, k):
        if k not in self.due:
            return
        self.due.discard(k)
        t0 = time.perf_counter()
        weights = self.net.to_caffemodel()
        t1 = time.perf_counter()
        summary, _ = self.val.score(weights)
        if self.rank != 0:
            return
        handover_s = t1 - t0 + summary["busy"]["build"]            # to_caffemodel, then copy_from into every kept net
        self.out.write("".join(l + "\n" for l in val_lines(k, summary)))
        self.out.flush()
        if self.log:
            with open(self.log, "a") as f:
                f.write(val_record(k, summary, handover_s, time.perf_counter() - t0) + "\n")


def train(a, world=1, rank=0, device=0, out=None):
    """Runs `caffe train` for parsed arguments `a` -> the Solver; progress goes to `out` (stdout).  Raises RunError on refused
    inputs."""
    out = out or sys.stdout
    import torch
    import flownet2_b200 as F
    from . import data as D, parallel as P
    crop = parse_size(a.crop)
    weights = parse_weights(a.weights)
    if a.snapshot and weights:                                              # tools/caffe.cpp refuses the pair as well
        raise RunError("give --snapshot to resume training or --weights to finetune, not both")
    if a.snapshot and not os.path.isfile(a.snapshot):
        raise RunError("%s: no such solverstate" % a.snapshot)
    if not os.path.isfile(a.solver):
        raise RunError("%s: no such solver" % a.solver)
    with open(a.solver) as f:
        solver_text = f.read()
    val = validator(a, world, rank, device)
    ds = D.FlowDataset(a.data, a.batch, rand_permute=a.rand_permute, rand_permute_seed=a.rand_permute_seed,
                       block_size=a.block_size, range_start=a.range_start, range_end=a.range_end,
                       rand_permute_order=a.rand_permute_order, flow_encoding=a.flow_encoding, world=world, rank=rank,
                       kitti=a.kitti)
    torch.cuda.set_device(device)
    net = F.Net(model_text(a.model, crop, ds.size, a.batch), None, F.TRAIN)
    if not weights and not a.snapshot:
        net.fill_params(int(os.environ.get("FN2_SEED", "1701")))
    for path, prefix in weights:
        net.copy_from(path, prefix)
    solver = F.Solver(solver_text, net)
    rank_params(solver.param, rank)
    if a.snapshot:
        solver.restore(a.snapshot)                                          # iter, history and the weights it names
    if world > 1:
        with torch.cuda.stream(torch.cuda.ExternalStream(net.stream)):     # ordered on the net's stream, like its own work
            P.broadcast_arena(P.arena_tensor(net))
        net.params_changed()
        grads = P.grad_arena_tensor(net, trainable_only=True)
        solver.add_callback(lambda: None, lambda: P.allreduce_gradients(grads))
    max_iter = int(solver.param["max_iter"])
    validate = lambda k: None
    if val is not None:
        val.check_handover(net)
        validate = Validation(val, net, val_iters(solver.iter, max_iter, a.val_interval, a.val_initial), rank, out,
                              a.val_log)
        solver.add_callback(lambda: validate(solver.iter), lambda: None)
    ds.seek(solver.iter * int(solver.param["iter_size"]))
    ds.bind(net)
    display = a.display if a.display is not None else solver_display(solver_text)
    try:
        while solver.iter < max_iter:
            it0, t0 = solver.iter, time.perf_counter()
            n = max_iter - it0 if display <= 0 else min(display - it0 % display, max_iter - it0)
            solver.step(n, ds)
            if display > 0 and rank == 0 and solver.iter % display == 0:
                dt = time.perf_counter() - t0
                out.write("Iteration %d (%.3g iter/s, %.3fs/%d iters), loss = %.6g\n" % (
                    solver.iter, n / dt, dt, n, solver.smoothed_loss))
                out.write("Iteration %d, lr = %.6g\n" % (solver.iter, solver.lr))
                out.flush()
        snap = solver.param["snapshot"]
        if solver.param["snapshot_after_train"] and (not snap or solver.iter % snap != 0):
            solver.snapshot()
        validate(solver.iter)                                              # after the last iteration, when it is due
    finally:
        ds.close()
    if rank == 0:
        out.write("Optimization Done.\n")
        out.flush()
    return solver


def parse_args(argv):
    ap = argparse.ArgumentParser(prog="python -m flownet2_b200.train", description=__doc__.split("\n\n")[0])
    ap.add_argument("--solver", required=True, help="solver prototxt (SGD or Adam)")
    ap.add_argument("--model", required=True, help="training prototxt or template (models/*_train.prototxt.template)")
    ap.add_argument("--data", required=True, help="list file of 'img0 img1 flow' lines")
    ap.add_argument("--crop", required=True, help="network input (augmentation crop) WIDTHxHEIGHT, e.g. 448x320")
    ap.add_argument("--batch", type=int, required=True, help="samples per iteration and rank")
    ap.add_argument("--weights", nargs="+", help="weights to start from: file.caffemodel[:prefix], several allowed")
    ap.add_argument("--snapshot", help="resume from this .solverstate")
    ap.add_argument("--gpu", type=int, default=0, help="device to use without torchrun")
    ap.add_argument("--display", type=int, help="print losses every N iterations (default: the solver's display)")
    ap.add_argument("--rand-permute", dest="rand_permute", action="store_true", default=True,
                    help="visit the samples in a seeded random order (default)")
    ap.add_argument("--no-rand-permute", dest="rand_permute", action="store_false", help="visit the samples in list order")
    ap.add_argument("--rand-permute-seed", type=int, default=77, help="std::srand seed (<= 0: glibc's initial state)")
    ap.add_argument("--rand-permute-order", default="FIRST_PERMUTE_THEN_RANGE", choices=("FIRST_PERMUTE_THEN_RANGE",
                                                                                        "FIRST_RANGE_THEN_PERMUTE"))
    ap.add_argument("--block-size", type=int, default=0, help="permute within blocks of this many samples")
    ap.add_argument("--range-start", type=int, default=0, help="first sample used (0-based list line among non-blank lines)")
    ap.add_argument("--range-end", type=int, default=-1, help="last sample used, inclusive (-1: the last)")
    ap.add_argument("--flow-encoding", default="uint16", choices=("uint16", "float"),
                    help="ground truth as the reference's LMDB holds it (uint16, default) or the files' floats")
    ap.add_argument("--kitti", action="store_true", help="the flows are KITTI 16-bit PNGs (KITTI 2012 / 2015 ground truth), "
                                                        "in --data and --val")
    ap.add_argument("--val", metavar="LIST", help="validate on this list of 'img0 img1 flow' lines (evaluate's metrics)")
    ap.add_argument("--val-model", metavar="TEMPLATE", help="deploy prototxt template to validate with (required with --val)")
    ap.add_argument("--val-interval", type=int, metavar="N", help="validate every N iterations (required with --val)")
    ap.add_argument("--val-batch", type=int, default=1, metavar="B",
                    help="validation pairs per forward (records reproduce single-pair runs only at 1)")
    ap.add_argument("--no-val-initial", dest="val_initial", action="store_false", help="do not validate at iteration 0")
    ap.add_argument("--val-occlusions", metavar="LIST", help="occlusion masks, one per --val line: the region scores")
    ap.add_argument("--val-objects", metavar="LIST", help="object maps, one per --val line: the region scores")
    ap.add_argument("--val-log", metavar="FILE", help="append one JSON line per validation")
    return ap.parse_args(argv)


def main(argv=None):
    a = parse_args(sys.argv[1:] if argv is None else argv)
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    device = int(os.environ.get("LOCAL_RANK", a.gpu)) if "WORLD_SIZE" in os.environ else a.gpu
    import flownet2_b200 as F
    dist = None
    try:
        if world > 1:
            import torch
            import torch.distributed as dist
            torch.cuda.set_device(device)
            dist.init_process_group("nccl")
        train(a, world, rank, device)
    except (RunError, F.Fn2Error) as e:
        sys.stderr.write("error: %s\n" % str(e).splitlines()[0])
        return 2
    finally:
        if dist is not None and dist.is_initialized():
            dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
