"""Score a net against ground-truth flow: end-point error, outlier rate and Sintel speed bands over an image-and-flow list.

    python -m flownet2_b200.evaluate weights.caffemodel models/FlowNet2_deploy.prototxt.template val.txt [--batch B]
                                     [--per-pair out.tsv] [--gpu G] [--kitti] [--occlusions LIST] [--objects LIST]
                                     [--visualize DIR [--max-flow F]] [--fb-check [--fb-alpha1 A] [--fb-alpha2 B]]

The list is the train command's: one ``img0 img1 flow`` line per pair (files.read_list; an occlusion field is refused), flows
as .flo or 'PF' PFM of either byte order.  Frame sizes may differ from line to line; a flow must have its frames' size
(files.probe checks every line before a net is built).  The pairs run through flownet2_b200.run's pipeline (one net per frame
size, the weights read once, reads and copies overlapped with the forwards); only what happens to each batch's flow differs.
The feeder's reader pool reads each ground-truth payload into a pinned slot beside the frames, the copy stream moves it to
the device, and on the net's stream it is converted (fn2_flow_to_tensor, the file's floats unquantised) and scored against
the prediction by fn2_flow_error (include/fn2_eval.h).  Only the per-pair records come back to the host; the padded pairs of
a size's last batch are dropped.

--kitti: every flow of the list is a KITTI 16-bit PNG (flownet2_b200.kitti), the ground truth of KITTI 2012 and 2015; sizes
may differ by line.  The reader pool inflates and unfilters each file into the slot, and fn2_flow_to_tensor (FLOW_KITTI)
turns the samples into the flow on the net's stream, unquantised, with NaN at the pixels the file marks invalid.

Metrics.  A ground-truth pixel is valid when both components are finite and at most 1e9 in absolute value.  EPE is the
float32 sqrt(du^2 + dv^2) of the prediction minus the ground truth; a valid pixel whose prediction is not finite is counted in
nonfinite_px and left out of every average.  Printed as one JSON line:
  epe            pooled over every counted pixel of the list (the Sintel and Middlebury convention);
  epe_pair_mean  the mean of the per-pair EPE over the pairs with a counted pixel (the per-image convention, e.g. KITTI's);
  fl_percent     counted pixels with EPE > 3 px and EPE > 5 % of |gt| (KITTI's Fl), in percent;
  s0-10, s10-40, s40+   pooled EPE over the pixels whose |gt| is in [0, 10), [10, 40), [40, inf) (null when a band is empty);
and pairs, valid_px, invalid_px, nonfinite_px, batch, ranks and wall (s).  --per-pair writes a TSV row per list line: where,
img0, img1, flow, valid pixels, EPE, Fl %.  A list with no valid pixel is refused (status 2).

Regions (include/fn2_eval.h defines them).  --occlusions LIST and --objects LIST each name a list of 8-bit one-channel masks,
one path per line for the pair list's lines in order (files.attach_masks, before any sharding; files.probe checks each mask's
size).  The feeder reads the masks into each pair's payload stride; on the net's stream fn2_occlusion_boundary_dist2 computes
the occlusion boundary distance and fn2_flow_error_regions scores the regions, and the records widen by FLOW_REGION_FIELDS.
Pooled over the list, null when empty:
  --occlusions   epe_matched, epe_unmatched (Sintel's matched / unmatched: the mask's zero / nonzero pixels), d0-10,
                 d10-60, d60-140 (EPE of the pixels closer than 10, 10 to 60, 60 to 140 pixels to the occlusion boundary;
                 this project's definition, see the header), matched_px, unmatched_px;
  --objects      fl_bg, fl_fg (KITTI 2015's Fl-bg / Fl-fg, in percent; fl_percent is Fl-all), epe_bg, epe_fg, bg_px, fg_px.
--per-pair appends the same scores per pair (NaN when empty), without the pixel counts.  Without either flag the output is
exactly the plain command's.  When a prediction is not finite
its pairs are named on stderr and the status is 1, as in run.

--fb-check [--fb-alpha1 A] [--fb-alpha2 B]: the net also runs on every pair with its frames exchanged (run --backward's two
forwards), and on the net's stream fn2_flow_fb_occlusion marks frame 0's pixels whose forward flow the backward flow does not
undo (the forward-backward check of Sundaram, Brox and Keutzer, ECCV 2010; include/fn2_flow.h, alpha1 = A, 0.01, and
alpha2 = B, 0.5).  fn2_flow_error_regions splits the EPE by that mask, and the summary gains, pooled over the list:
  epe_fb_visible, epe_fb_flagged   EPE of the counted pixels the check keeps / flags (null when empty);
  fb_visible_px, fb_flagged_px     their counts;
and with --occlusions the mask is scored against the ground-truth masks by fn2_mask_confusion, "occluded" the positive class
over all pixels: occ_tp, occ_fp, occ_fn, occ_precision, occ_recall, occ_f1 (null when undefined).  --per-pair gains the
same columns.  Without the flag nothing of the output changes.

--visualize DIR [--max-flow F]: for list line k (counting pairs from 0) DIR/<k, 6 digits>_pred.png and _gt.png, the
prediction and the ground truth colour-coded on the net's stream (fn2_flow_to_color_png_rows) at one scale, so that they can be
compared: F, else the ground truth's largest known flow (the prediction's when no ground-truth pixel is known).  The
scanlines come back with the records and the writer thread deflates them; under torchrun each rank writes its own pairs.
The summary and --per-pair are the same with and without it.

Under torchrun (WORLD_SIZE, RANK, LOCAL_RANK) rank r scores the lines i with i % WORLD_SIZE == r; rank 0 gathers every rank's
records, puts them back in list order (combine_shards) and prints the summary, so at --batch 1 it does not depend on the
number of ranks.  At larger batches a pair's flow, and so its record, can differ in the last bits (see run).
"""
import argparse
import json
import os
import sys
import time

import numpy as np

from . import FLOW_ERROR_FIELDS, FLOW_REGION_FIELDS, MASK_CONFUSION_FIELDS
from .feed import _align, mask_offset
from .files import RunError, attach_masks, probe, read_list
from .run import STAGES, _run_size, check_fb_alphas, check_inputs, check_max_flow, group_by_size, run_groups, shard

FIELD = {name: i for i, name in enumerate(FLOW_ERROR_FIELDS)}
REGION = {name: i for i, name in enumerate(FLOW_REGION_FIELDS)}
CONFUSION = {name: len(FLOW_REGION_FIELDS) + i for i, name in enumerate(MASK_CONFUSION_FIELDS)}     # in an --fb-check block
FB_FIELDS = len(FLOW_REGION_FIELDS) + len(MASK_CONFUSION_FIELDS)
BANDS = (("s0-10", "n_s0_10", "sum_s0_10"), ("s10-40", "n_s10_40", "sum_s10_40"), ("s40+", "n_s40", "sum_s40"))
# the region scores each mask adds to the summary and the per-pair file: (key, region, pooled EPE or Fl %)
REGION_KEYS = {"occlusions": (("epe_matched", "matched", "epe"), ("epe_unmatched", "unmatched", "epe"),
                              ("d0-10", "d0_10", "epe"), ("d10-60", "d10_60", "epe"), ("d60-140", "d60_140", "epe")),
               "objects": (("fl_bg", "bg", "fl"), ("fl_fg", "fg", "fl"), ("epe_bg", "bg", "epe"), ("epe_fg", "fg", "epe"))}


def record_width(masks, fb=False):
    """Fields of a pair's record: FLOW_ERROR_FIELDS, then FLOW_REGION_FIELDS when the pairs carry masks, then with fb (the
    --fb-check block) FLOW_REGION_FIELDS split by the predicted mask and MASK_CONFUSION_FIELDS."""
    return len(FLOW_ERROR_FIELDS) + (len(FLOW_REGION_FIELDS) if masks else 0) + (FB_FIELDS if fb else 0)


class Scores(object):
    """evaluate's per-batch sink for run._run_size (the interface is described at run.FlowFiles): the ground-truth payloads
    ride in the frames' slots, each pair's at a stride that holds any format's, are converted on the net's stream before the
    forward, and each batch's flow is scored on the net's stream; the records of the real pairs land in
    records[sample.index].

    masks: the kinds of mask each pair carries, in files.Pair.masks order ("occlusions", "objects" or both).  With masks the
    records widen by FLOW_REGION_FIELDS: stage() computes the occlusion boundary distance straight from the slot and copies
    the mask planes out of it (the slot is refilled while the forward runs), and score() adds fn2_flow_error_regions.

    visualize: a directory; score() also colour-codes the prediction and the ground truth at one scale per pair (max_flow,
    else the ground truth's largest known flow, else the prediction's) into PNG scanlines behind the records, and take() writes
    them as <visualize>/<sample.number, 6 digits>_pred.png and _gt.png.

    fb: (alpha1, alpha2) of the forward-backward check, or None.  With it _run_size also fills bwd_dev[s] with the flow of the
    exchanged frames, and score() computes frame 0's occlusion mask (fn2_flow_fb_occlusion), splits the EPE by it
    (fn2_flow_error_regions with the mask as the object map: BG visible, FG flagged) and, with occlusion masks, counts it
    against them (fn2_mask_confusion); the records widen by FB_FIELDS (the confusion counts stay 0 without occlusions)."""

    def __init__(self, n, masks=(), visualize=None, max_flow=None, fb=None):
        self.masks, self.fb, self.backward = tuple(masks), fb, fb is not None
        self.records = np.full((n, record_width(self.masks, self.backward)), np.nan)
        self.stats = {"collect": 0.0}
        self.visualize, self.max_flow = visualize, max_flow

    def item_bytes(self, H, W):
        return _align(mask_offset(H, W) + len(self.masks) * H * W)

    def bind(self, torch, batch, H, W, flow_dev, bwd_dev=None):
        from . import ops
        self.ops, self.batch = ops, batch
        nf, nr = len(FLOW_ERROR_FIELDS), record_width(self.masks) - len(FLOW_ERROR_FIELDS)
        # each block of a pair's record: the fields of fn2_flow_error, fn2_flow_error_regions and, with fb, the regions split
        # by the predicted mask and its confusion counts
        self.widths = (nf, nr) + ((len(FLOW_REGION_FIELDS), len(MASK_CONFUSION_FIELDS)) if self.fb else ())
        self.pred = [f.permute(0, 3, 1, 2) for f in flow_dev]                       # (B, 2, H, W) views of the NHWC flow
        self.gt = [torch.empty((batch, 2, H, W), device="cuda") for _ in range(2)]
        # each batch's records in one buffer: per block of widths, its (B, width) fields; then with visualize the
        # prediction's and the ground truth's colour scanlines
        self.rec_bytes = batch * sum(self.widths) * 8
        self.size, self.vis_bytes = (W, H), H * (1 + 3 * W)
        nb = self.rec_bytes + (2 * batch * self.vis_bytes if self.visualize else 0)
        self.dev = [torch.empty(nb, dtype=torch.uint8, device="cuda") for _ in range(2)]
        self.host = [torch.empty(nb, dtype=torch.uint8).pin_memory() for _ in range(2)]
        rec = [d[:self.rec_bytes].view(torch.float64) for d in self.dev]
        self.blocks = [[b.view(batch, w) for b, w in zip(r.split([batch * w for w in self.widths]), self.widths)] for r in rec]
        self.err = [b[0] for b in self.blocks]
        self.reg = [b[1] for b in self.blocks]
        if self.fb:
            self.bwd = [b.permute(0, 3, 1, 2) for b in bwd_dev]
            self.fbmask = [torch.empty((batch, H, W), dtype=torch.uint8, device="cuda") for _ in range(2)]
            for b in self.blocks:
                b[3].zero_()                                                        # the counts without occlusion masks
        if self.visualize:
            self.radius = [torch.empty((2, batch), device="cuda") for _ in range(2)]      # the ground truth's, the prediction's
        ws = ops.flow_error_workspace_bytes(batch, H, W)
        if self.masks or self.fb:
            ws = max(ws, ops.flow_error_regions_workspace_bytes(batch, H, W))
        if self.masks:
            self.planes = [torch.empty((len(self.masks), batch, H, W), dtype=torch.uint8, device="cuda") for _ in range(2)]
            if "occlusions" in self.masks:
                self.dist2 = [torch.empty((batch, H, W), dtype=torch.int32, device="cuda") for _ in range(2)]
        self.workspace = torch.empty(max(ws, 8), dtype=torch.uint8, device="cuda")

    def stage(self, pairs, s, payload, stride):
        """On the net's stream: pair i's payload, at payload[i * stride], into gt[s][i] (formats may differ per pair); its masks
        into planes[s][:, i] and, from its occlusion mask, the boundary distance into dist2[s][i]."""
        for i, p in enumerate(pairs):
            fh = p.flow_header
            self.ops.flow_to_tensor(payload[i * stride:i * stride + fh.nbytes], fh.format, 0, self.gt[s][i:i + 1])
        if not self.masks:
            return
        _, B, H, W = self.planes[s].shape
        items = payload[:B * stride].view(B, stride)
        for m, kind in enumerate(self.masks):
            off = mask_offset(H, W) + m * H * W
            if kind == "occlusions":
                self.ops.occlusion_boundary_dist2(payload[off:], out=self.dist2[s], pair_stride=stride)
            self.planes[s][m].view(B, H * W).copy_(items[:, off:off + H * W])

    def score(self, s):
        self.ops.flow_error(self.pred[s], self.gt[s], out=self.err[s], workspace=self.workspace)
        if self.masks:
            plane = {kind: self.planes[s][m] for m, kind in enumerate(self.masks)}
            self.ops.flow_error_regions(self.pred[s], self.gt[s], occ=plane.get("occlusions"), obj=plane.get("objects"),
                                        dist2=self.dist2[s] if "occlusions" in plane else None, out=self.reg[s],
                                        workspace=self.workspace)
        if self.fb:
            fbreg, conf = self.blocks[s][2:]
            self.ops.flow_fb_occlusion(self.pred[s], self.bwd[s], *self.fb, out=self.fbmask[s])
            self.ops.flow_error_regions(self.pred[s], self.gt[s], obj=self.fbmask[s], out=fbreg, workspace=self.workspace)
            if "occlusions" in self.masks:
                self.ops.mask_confusion(self.fbmask[s], self.planes[s][self.masks.index("occlusions")], out=conf)
        if self.visualize:
            gt_r = pred_r = None
            if self.max_flow is None:
                gt_r, pred_r = self.ops.flow_max_radius(self.gt[s], self.radius[s][0]), self.ops.flow_max_radius(
                    self.pred[s], self.radius[s][1])
            o, n = self.rec_bytes, self.batch * self.vis_bytes
            for k, flow in enumerate((self.pred[s], self.gt[s])):
                self.ops.flow_to_color_png_rows(flow, self.dev[s][o + k * n:o + (k + 1) * n], self.max_flow, max_radius=gt_r,
                                                fallback=pred_r)

    def take(self, pairs, s, n_real):
        t0 = time.perf_counter()
        raw = self.host[s].numpy()
        buf = raw[:self.rec_bytes].view(np.float64)
        ends = np.cumsum((0,) + self.widths) * self.batch
        blocks = [buf[a:b].reshape(self.batch, -1) for a, b in zip(ends[:-1], ends[1:])]
        for i, p in enumerate(pairs[:n_real]):
            self.records[p.index] = np.concatenate([b[i] for b in blocks])
            if self.visualize:
                from . import kitti
                o, n, m = self.rec_bytes, self.batch * self.vis_bytes, self.vis_bytes
                for k, tag in enumerate(("pred", "gt")):
                    kitti.write_png_rows(os.path.join(self.visualize, "%06d_%s.png" % (p.number, tag)),
                                         raw[o + k * n + i * m:o + k * n + (i + 1) * m], *self.size, 8)
        self.stats["collect"] += time.perf_counter() - t0


def combine_shards(shards):
    """Per-rank record arrays, rank r holding list lines r, r + world, ... in order (run.shard) -> one array in list order."""
    world = len(shards)
    out = np.empty((sum(len(s) for s in shards),) + tuple(np.shape(shards[0])[1:]), np.float64)
    for r, s in enumerate(shards):
        out[r::world] = s
    return out


def _ratio(num, den):
    return float(num / den) if den > 0 else None


def region_keys(occlusions, objects):
    """The region scores of the summary and the per-pair file, in order: (key, region, EPE or Fl %)."""
    return (REGION_KEYS["occlusions"] if occlusions else ()) + (REGION_KEYS["objects"] if objects else ())


def region_scores(region, occlusions, objects):
    """Region fields summed over some pairs (FLOW_REGION_FIELDS) -> [(key, pooled EPE or Fl %, None when the region is
    empty)] of the masks given."""
    at = lambda f: region[REGION[f]]
    return [(key, _ratio(at("sum_" + r), at("n_" + r)) if what == "epe" else _ratio(100.0 * at("out_" + r), at("n_" + r)))
            for key, r, what in region_keys(occlusions, objects)]


def fb_scores(block, occlusions):
    """An --fb-check block (FB_FIELDS) summed over some pairs -> [(key, value)]: the EPE and counted pixels the check keeps
    and flags and, with occlusions, the confusion counts against the ground-truth masks with precision, recall and F1
    (None when undefined)."""
    at = lambda f: block[REGION[f]]
    out = [("epe_fb_visible", _ratio(at("sum_bg"), at("n_bg"))), ("epe_fb_flagged", _ratio(at("sum_fg"), at("n_fg"))),
           ("fb_visible_px", int(at("n_bg"))), ("fb_flagged_px", int(at("n_fg")))]
    if occlusions:
        tp, fp, fn = (block[CONFUSION[f]] for f in ("tp", "fp", "fn"))
        out += [("occ_tp", int(tp)), ("occ_fp", int(fp)), ("occ_fn", int(fn)), ("occ_precision", _ratio(tp, tp + fp)),
                ("occ_recall", _ratio(tp, tp + fn)), ("occ_f1", _ratio(2 * tp, 2 * tp + fp + fn))]
    return out


def fb_keys(occlusions):
    return [k for k, _ in fb_scores(np.zeros(FB_FIELDS), occlusions)]


def summarize(records, pixels, name, occlusions=False, objects=False, fb=False):
    """The summary of per-pair records in list order ((n, FIELDS) float64, or FIELDS + REGION FIELDS with masks) and each
    pair's pixel count -> dict; with occlusions / objects, the pooled region scores and pixel counts of those masks are added;
    with fb (records ending in the --fb-check block), fb_scores of the block pooled over the list.
    Refuses a list with no valid pixel, naming it."""
    records = np.asarray(records, np.float64)
    col = lambda f: records[:, FIELD[f]]
    valid, nonfinite = col("valid"), col("nonfinite")
    if not len(records) or valid.sum() == 0:
        raise RunError("%s: no ground-truth pixel is valid in any of its %d pairs" % (name, len(records)))
    counted = valid - nonfinite
    has = counted > 0
    out = {"pairs": len(records), "valid_px": int(valid.sum()), "invalid_px": int(np.sum(pixels) - valid.sum()),
           "nonfinite_px": int(nonfinite.sum()),
           "epe": _ratio(col("epe_sum").sum(), counted.sum()),
           "epe_pair_mean": float(np.mean(col("epe_sum")[has] / counted[has])) if has.any() else None,
           "fl_percent": _ratio(100.0 * col("outliers").sum(), counted.sum())}
    for key, n, s in BANDS:
        out[key] = _ratio(col(s).sum(), col(n).sum())
    if occlusions or objects:
        region = records[:, len(FLOW_ERROR_FIELDS):].sum(axis=0)
        out.update(region_scores(region, occlusions, objects))
        for r in (("matched", "unmatched") if occlusions else ()) + (("bg", "fg") if objects else ()):
            out[r + "_px"] = int(region[REGION["n_" + r]])
    if fb:
        out.update(fb_scores(records[:, -FB_FIELDS:].sum(axis=0), occlusions))
    return out


def pair_rows(records, occlusions=False, objects=False, fb=False):
    """-> per pair (valid pixels, EPE, Fl %) followed by its region scores of the masks given and with fb its fb_scores, NaN
    where no pixel counts."""
    rows = []
    nan = lambda v: float("nan") if v is None else v
    for r in np.asarray(records, np.float64):
        counted = r[FIELD["valid"]] - r[FIELD["nonfinite"]]
        epe = r[FIELD["epe_sum"]] / counted if counted > 0 else float("nan")
        fl = 100.0 * r[FIELD["outliers"]] / counted if counted > 0 else float("nan")
        regions = region_scores(r[len(FLOW_ERROR_FIELDS):], occlusions, objects) if occlusions or objects else []
        regions += fb_scores(r[-FB_FIELDS:], occlusions) if fb else []
        rows.append((int(r[FIELD["valid"]]), epe, fl) + tuple(nan(v) for _, v in regions))
    return rows


def write_per_pair(path, samples, records, occlusions=False, objects=False, fb=False):
    extra = "".join("\t" + key for key, _, _ in region_keys(occlusions, objects))
    extra += "".join("\t" + key for key in fb_keys(occlusions)) if fb else ""
    with open(path, "w") as f:
        f.write("where\timg0\timg1\tflow\tvalid\tepe\tfl_percent%s\n" % extra)
        for s, (valid, epe, fl, *regions) in zip(samples, pair_rows(records, occlusions, objects, fb)):
            f.write("%s\t%s\t%s\t%s\t%d\t%.9g\t%.9g%s\n" % (s.where, s.img0, s.img1, s.flow, valid, epe, fl,
                                                          "".join("\t%.9g" % v for v in regions)))


def not_finite(samples, records):
    """The samples with a valid pixel whose prediction is not finite."""
    return [s for s, r in zip(samples, records) if r[FIELD["nonfinite"]] > 0]


def _list_name(samples):
    return samples[0].where.rsplit(":", 1)[0] if samples else "the list"


def _mask_kinds(occlusions, objects):
    """-> (mask kinds, their lists) of the mask lists given, in files.Pair.masks order."""
    given = [(k, l) for k, l in (("occlusions", occlusions), ("objects", objects)) if l]
    return tuple(k for k, _ in given), [l for _, l in given]


def _score(caffemodel, template, samples, batch, device, threads, kitti=False, masks=(), visualize=None, max_flow=None, fb=None):
    """-> (records in the samples' order, per-stage busy seconds, number of sizes).  masks: the kinds of the samples' masks.
    visualize, max_flow, fb: see Scores (each sample's number names its images)."""
    t0 = time.perf_counter()
    if fb is not None:
        check_fb_alphas(*fb)
    check_inputs(caffemodel, template, batch)
    check_max_flow(max_flow)
    probe(samples, ground_truth=True, kitti=kitti)
    for i, s in enumerate(samples):
        s.index = i
    if visualize:
        os.makedirs(visualize, exist_ok=True)
    sink = Scores(len(samples), masks, visualize, max_flow, fb)
    stats, sizes = run_groups(caffemodel, template, samples, batch, device, threads, sink, t0)
    return sink.records, stats, sizes


def number(samples):
    """Numbers the samples of a whole list, before any sharding, by their position: the names of evaluate --visualize."""
    for k, s in enumerate(samples):
        s.number = k


def evaluate(caffemodel, template, samples, batch=1, device=0, threads=None, kitti=False, occlusions=None, objects=None,
             visualize=None, max_flow=None, fb=None):
    """Scores the net on every files.Pair -> (summary dict, per-pair records): the summary of summarize() plus batch, sizes,
    wall (s), per-stage busy seconds and the samples whose prediction is not finite; the records are an (n, FIELDS) float64
    array in the samples' order (fields: flownet2_b200.FLOW_ERROR_FIELDS, then FLOW_REGION_FIELDS with a mask list).  kitti:
    the flows are KITTI PNGs.  occlusions, objects: mask lists (one path per sample, in order) of occlusion masks and object
    maps, either or both, for the region scores of summarize().  visualize: a directory for each pair's colour-coded
    prediction and ground truth (Scores), at the fixed scale max_flow if given.  fb: (alpha1, alpha2) of the forward-backward
    check, which adds fb_scores to the summary and the --fb-check block to the records, or None."""
    t0 = time.perf_counter()
    masks, lists = _mask_kinds(occlusions, objects)
    attach_masks(samples, lists)
    number(samples)
    records, stats, sizes = _score(caffemodel, template, samples, batch, device, threads, kitti, masks, visualize, max_flow, fb)
    summary = summarize(records, [s.size[0] * s.size[1] for s in samples], _list_name(samples), bool(occlusions), bool(objects),
                        fb is not None)
    summary.update({"batch": batch, "sizes": sizes, "wall": time.perf_counter() - t0, "busy": stats,
                    "not_finite": [s.where for s in not_finite(samples, records)]})
    return summary, records


def gather_records(local, n_total, world, rank):
    """Every rank's (n_r, cols) records -> the list-order array on rank 0 (None elsewhere): one gather of equal, zero-padded
    float64 tensors on the process group's device, then combine_shards."""
    import torch
    import torch.distributed as dist
    mx = (n_total + world - 1) // world
    dev = "cuda" if dist.get_backend() == "nccl" else "cpu"
    t = torch.zeros((mx, local.shape[1]), dtype=torch.float64, device=dev)
    t[:len(local)] = torch.from_numpy(local)
    got = [torch.empty_like(t) for _ in range(world)] if rank == 0 else None
    dist.gather(t, got, dst=0)
    if rank != 0:
        return None
    return combine_shards([g[:len(range(r, n_total, world))].cpu().numpy() for r, g in enumerate(got)])


def _squeeze(shape):
    """A blob shape without its leading ones: the shapes Net.copy_from treats as equal."""
    shape = tuple(shape)
    while len(shape) > 1 and shape[0] == 1:
        shape = shape[1:]
    return shape


def check_handover(train_layers, deploy_layers, deploy_name="the deploy net"):
    """Refuses a deploy net that cannot score the training net's weights (Net.param_layers of each), naming the first
    offending layer: a layer the training net trains (an lr_mult != 0) with no layer of that name and blob shapes in the
    deploy net, a layer of both whose blobs the copy would refuse, or a deploy layer with parameters that gets none from the
    training net and whose weights the template does not define (a diagonal filler)."""
    train = {name: (flags, shapes) for name, _, flags, shapes, _ in train_layers}
    deploy = {name: (flags, shapes) for name, _, flags, shapes, _ in deploy_layers}
    same = lambda a, b: [_squeeze(s) for s in a] == [_squeeze(s) for s in b]
    for name, _, flags, shapes, mults in train_layers:
        if name in deploy:
            if "c" not in flags and not same(shapes, deploy[name][1]):
                raise RunError("the training net's layer %s has blobs %s, its namesake in %s %s" % (
                    name, shapes, deploy_name, deploy[name][1]))
        elif any(m != 0 for m in mults):
            raise RunError("the training net trains layer %s, which %s lacks" % (name, deploy_name))
    for name, _, flags, _, _ in deploy_layers:
        if name not in train and "t" not in flags:
            raise RunError("layer %s of %s gets no weights from the training net" % (name, deploy_name))


class Validator(object):
    """Scores weights held in memory against a list, again and again: the train command's --val.

    At construction the list is read the way evaluate() reads it (files.probe, the mask lists attached, the pairs numbered),
    so a bad list is refused before anything runs on the device.  Under torchrun (world, rank) this rank scores the lines i
    with i % world == rank.  One deploy net per frame size (fill_template of `template`) is built on first use and kept;
    score(weights) loads caffemodel bytes into each kept net with Net.copy_from and runs its pairs through run._run_size into
    a Scores sink.  The summary and records are evaluate()'s for the same weights read from a file, bit for bit."""

    def __init__(self, template, samples, batch=1, device=0, threads=None, kitti=False, occlusions=None, objects=None,
                 world=1, rank=0):
        if batch < 1:
            raise RunError("--val-batch must be at least 1, got %d" % batch)
        if not os.path.isfile(template):
            raise RunError("%s: no such deploy prototxt template" % template)
        if not samples:
            raise RunError("the validation list holds no pairs")
        with open(template) as f:
            self.text = f.read()
        self.masks, lists = _mask_kinds(occlusions, objects)
        self.occlusions, self.objects = bool(occlusions), bool(objects)
        attach_masks(samples, lists)
        number(samples)
        probe(samples, ground_truth=True, kitti=kitti)
        self.samples, self.template, self.batch, self.device, self.threads = samples, template, batch, device, threads
        self.world, self.rank = world, rank
        self.mine = shard(samples, world, rank)
        for i, s in enumerate(self.mine):
            s.index = i
        self.groups = group_by_size(self.mine)
        self.nets = {}

    def net(self, size):
        """The kept deploy net of frame size (width, height), built on first use."""
        if size not in self.nets:
            import torch
            import flownet2_b200 as F
            torch.cuda.set_device(self.device)
            self.nets[size] = F.Net(F.fill_template(self.text, size[0], size[1]), None, F.TEST, batch=self.batch)
        return self.nets[size]

    def check_handover(self, train_net):
        """Refuses (check_handover) a training net whose weights this deploy template cannot score, before any validation."""
        size = self.groups[0][0] if self.groups else self.samples[0].size
        check_handover(train_net.param_layers(), self.net(size).param_layers(), self.template)

    def score(self, weights):
        """caffemodel bytes -> (summary, records) on rank 0, (None, None) elsewhere: evaluate()'s summary keys and records."""
        import torch
        t0 = time.perf_counter()
        torch.cuda.set_device(self.device)
        sink = Scores(len(self.mine), self.masks)
        stats = dict.fromkeys(STAGES, 0.0)
        stats.update(sink.stats)
        for size, group in self.groups:
            tb = time.perf_counter()
            net = self.net(size)
            net.copy_from(weights)
            stats["build"] += time.perf_counter() - tb
            _run_size(torch, net, size, group, self.batch, self.threads, stats, sink)
        stats.update(sink.stats)
        local = np.concatenate([sink.records, [[s.size[0] * s.size[1]] for s in self.mine]], axis=1) if self.mine \
            else np.empty((0, record_width(self.masks) + 1))
        full = gather_records(local, len(self.samples), self.world, self.rank) if self.world > 1 else local
        if self.rank != 0:
            return None, None
        records = full[:, :-1]
        summary = summarize(records, full[:, -1], _list_name(self.samples), self.occlusions, self.objects)
        summary.update({"batch": self.batch, "sizes": len(group_by_size(self.samples)), "wall": time.perf_counter() - t0,
                        "busy": stats, "not_finite": [s.where for s in not_finite(self.samples, records)]})
        return summary, records


def parse_args(argv):
    ap = argparse.ArgumentParser(prog="python -m flownet2_b200.evaluate", description=__doc__.split("\n\n")[0])
    ap.add_argument("caffemodel", help="weights: .caffemodel or .caffemodel.h5")
    ap.add_argument("deployproto", help="deploy prototxt template, e.g. models/FlowNet2_deploy.prototxt.template")
    ap.add_argument("listfile", help="list of 'img0 img1 flow' lines, flows as .flo or .pfm (KITTI .png with --kitti)")
    ap.add_argument("--batch", type=int, default=1, help="pairs per forward (records reproduce single-pair runs only at 1)")
    ap.add_argument("--per-pair", metavar="TSV", help="write one row per list line: where, img0, img1, flow, valid, EPE, Fl %%")
    ap.add_argument("--gpu", type=int, default=0, help="device to use without torchrun")
    ap.add_argument("--kitti", action="store_true", help="the flows are KITTI 16-bit PNGs (KITTI 2012 / 2015 ground truth)")
    ap.add_argument("--occlusions", metavar="LIST", help="occlusion masks, one per list line (Sintel's occlusions/*.png): "
                                                         "EPE matched / unmatched and by distance to the occlusion boundary")
    ap.add_argument("--objects", metavar="LIST", help="object maps, one per list line (KITTI 2015's obj_map/*.png): "
                                                      "Fl and EPE of the background and the foreground")
    ap.add_argument("--visualize", metavar="DIR", help="write each pair's colour-coded prediction and ground truth, at one "
                                                       "scale, as DIR/<list index>_pred.png and _gt.png")
    ap.add_argument("--max-flow", type=float, metavar="F", help="with --visualize: colour at this scale (pixels) instead of "
                                                                "each ground truth's largest flow")
    ap.add_argument("--fb-check", action="store_true", help="also run each pair backward and score the forward-backward "
                                                            "occlusion mask (against --occlusions when given)")
    ap.add_argument("--fb-alpha1", type=float, default=0.01, metavar="A", help="with --fb-check: the check's relative term "
                                                                               "(default 0.01)")
    ap.add_argument("--fb-alpha2", type=float, default=0.5, metavar="B", help="with --fb-check: the check's constant term, "
                                                                              "in squared pixels (default 0.5)")
    return ap.parse_args(argv)


def main(argv=None):
    a = parse_args(sys.argv[1:] if argv is None else argv)
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    device = int(os.environ.get("LOCAL_RANK", a.gpu)) if "WORLD_SIZE" in os.environ else a.gpu
    t0 = time.perf_counter()
    dist = None
    fb = (a.fb_alpha1, a.fb_alpha2) if a.fb_check else None
    try:
        check_max_flow(a.max_flow)
        check_fb_alphas(a.fb_alpha1, a.fb_alpha2)
        check_inputs(a.caffemodel, a.deployproto, a.batch)
        samples = read_list(a.listfile)
        if not samples:
            raise RunError("%s: the list holds no pairs" % a.listfile)
        masks, lists = _mask_kinds(a.occlusions, a.objects)
        attach_masks(samples, lists)                                    # before sharding: every rank sees the same lines
        number(samples)
        if world > 1:
            import torch
            import torch.distributed as dist
            torch.cuda.set_device(device)
            dist.init_process_group("nccl")
        mine = shard(samples, world, rank)
        local = np.empty((0, record_width(masks, a.fb_check) + 1))      # this rank's records, each pair's pixel count last
        if mine:
            records = _score(a.caffemodel, a.deployproto, mine, a.batch, device, None, a.kitti, masks, a.visualize,
                             a.max_flow, fb)[0]
            local = np.concatenate([records, [[s.size[0] * s.size[1]] for s in mine]], axis=1)
        full = gather_records(local, len(samples), world, rank) if world > 1 else local
        if rank != 0:
            return 1 if np.any(local[:, FIELD["nonfinite"]] > 0) else 0
        records, pixels = full[:, :-1], full[:, -1]
        summary = summarize(records, pixels, a.listfile, bool(a.occlusions), bool(a.objects), a.fb_check)
    except RunError as e:
        sys.stderr.write("error: %s\n" % e)
        return 2
    finally:
        if dist is not None and dist.is_initialized():
            dist.destroy_process_group()
    summary.update({"batch": a.batch, "ranks": world, "wall": time.perf_counter() - t0})
    if a.per_pair:
        write_per_pair(a.per_pair, samples, records, bool(a.occlusions), bool(a.objects), a.fb_check)
    bad = not_finite(samples, records)
    for s in bad:
        sys.stderr.write("%s: the flow of %s %s is not finite\n" % (s.where, s.img0, s.img1))
    print(json.dumps(summary), flush=True)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
