/*
 * fn2_eval.h -- C-ABI of libfn2.so for scoring a predicted flow against ground truth: end-point error, outlier rate and the
 * Sintel speed bands of every pair, reduced on the device.  A sibling of fn2_flow.h and fn2_lpq.h, with fn2.h's conventions:
 * status 0 or negative with the message in fn2_last_error().
 *
 * fn2_flow_error(pred, gt, out_dev, ...) -- pred and gt are float views of shape (N, 2, H, W), any strides (the NHWC buffer
 * fn2_net_get_blob_nhwc_device fills is one).  out_dev: N x FN2_FLOW_ERROR_FIELDS device doubles, one record per pair, the
 * fields at the FN2_FLOW_ERROR_* indices below:
 *   VALID      ground-truth pixels that count: both components finite and neither above 1e9 in absolute value (1e9 is
 *              Middlebury's UNKNOWN_FLOW_THRESH; NaN is the reference's marker of missing flow);
 *   EPE_SUM    sum of the EPE over the valid pixels whose prediction is finite;
 *   OUTLIERS   of those, the pixels with EPE > 3 and EPE > 0.05 |gt| (KITTI's Fl);
 *   NONFINITE  valid pixels whose prediction is not finite (NaN or Inf in either component); they are left out of every
 *              other field, so N_S0_10 + N_S10_40 + N_S40 = VALID - NONFINITE;
 *   N_S0_10 / SUM_S0_10, N_S10_40 / SUM_S10_40, N_S40 / SUM_S40: count and EPE sum per Sintel speed band, |gt| in [0, 10),
 *              [10, 40) and [40, inf).
 * EPE = sqrtf(du*du + dv*dv) with du = pred_u - gt_u, dv = pred_v - gt_v, in float32 with separately rounded products (the
 * plain benchmark EPE, not L1Loss's Power(0.5, shift = epsilon) form); |gt| = sqrtf(gt_u*gt_u + gt_v*gt_v) the same way.
 * Every per-pixel value, band and outlier decision is therefore reproduced exactly by a float32 restatement; the sums are
 * accumulated in double.
 *
 * Reduction: each block writes double partials of one pair, a second kernel adds each pair's partials in index order, so equal
 * inputs give bit-identical records.  workspace: at least fn2_flow_error_workspace_bytes(N, H, W) bytes, 8-byte aligned; a NULL,
 * smaller or misaligned one returns FN2_ERR_WORKSPACE.  FN2_ERR_INVALID when pred and gt differ in shape or have c != 2.
 *
 * Scoring by region: the columns of the Sintel table (EPE matched / unmatched, EPE by distance to the nearest occlusion
 * boundary) and KITTI 2015's Fl-bg / Fl-fg.
 *
 * Masks are 8-bit planes [H][W], one per pair, pair i's at byte i * pair_stride (pair_stride >= H * W, so a mask can be read
 * where it lies in a larger per-pair buffer).  An occlusion mask: a nonzero byte is occluded, zero is visible (the reference's
 * reading of an occlusion image, cv_occ.at<uchar>(y, x) > 0).  An object map (KITTI obj_map): zero is background, nonzero is
 * foreground.
 *
 * fn2_occlusion_boundary_dist2(masks_dev, pair_stride, N, H, W, dist2_dev, stream) -- the occlusion boundary is the set of
 * pixels with at least one 4-neighbour inside the image of the other occlusion label; dist2_dev (dense int32 [N][H][W]) gets
 * each pixel's exact squared Euclidean distance, centre to centre, to the nearest boundary pixel (0 on the boundary), or
 * FN2_DIST2_NONE at every pixel of a pair without a boundary (all clear or all occluded).  Two separable passes of an exact
 * distance transform, in integers.  FN2_ERR_INVALID for H or W above 16384 (so every distance squared fits in int32), N above
 * 65535 or pair_stride < H * W.
 *
 * fn2_flow_error_regions(pred, gt, occ_dev, obj_dev, mask_pair_stride, dist2_dev, out_dev, ...) -- pred and gt as for
 * fn2_flow_error; out_dev: N x FN2_FLOW_REGION_FIELDS device doubles, for each region a count (N_), an EPE sum (SUM_) and
 * the Fl outliers (OUT_) of its pixels, at the FN2_FLOW_REGION_* indices below.  A pixel counts exactly when it counts in
 * fn2_flow_error (valid ground truth, finite prediction), with fn2_flow_error's float32 EPE and outlier decision, so
 *   N_MATCHED + N_UNMATCHED = N_BG + N_FG = VALID - NONFINITE, and the D bands are a subset of the matched and unmatched pixels:
 *   MATCHED / UNMATCHED  occ_dev's byte is zero / nonzero;
 *   D0_10 / D10_60 / D60_140  dist2_dev's value in [0, 100), [100, 3600), [3600, 19600): distance to the nearest occlusion
 *              boundary in [0, 10), [10, 60), [60, 140) pixels.  A pixel 140 or more pixels away, or in a pair without a
 *              boundary, is in no band.  Sintel describes these columns only in prose ("closer than 0-10 pixels to the
 *              nearest occlusion boundary") and its server's code is not public: the boundary and the half-open bands are
 *              this project's definition, not checked against the leaderboard's numbers;
 *   BG / FG    obj_dev's byte is zero / nonzero.
 * occ_dev and obj_dev may each be NULL, which leaves that mask's fields 0; dist2_dev (dense int32 [N][H][W], as
 * fn2_occlusion_boundary_dist2 writes it) is required when occ_dev is given and refused when it is not.  Both masks are
 * read at mask_pair_stride.  The reduction, its bit-identical records and the workspace convention are fn2_flow_error's,
 * with its own size query.
 *
 * fn2_mask_confusion(pred_dev, gt_dev, pair_stride, N, H, W, out_dev, stream) -- a predicted occlusion mask (fn2_flow_fb_occlusion,
 * include/fn2_flow.h) against a ground-truth one, both 8-bit planes read as above (nonzero: occluded, the positive class), at
 * pair_stride.  out_dev: N x FN2_MASK_CONFUSION_FIELDS device doubles, 8-byte aligned, per pair the pixels that are TP
 * (occluded in both), FP (pred only), FN (gt only) and TN (neither), TP + FP + FN + TN = H * W.  Counted in integers and
 * stored as doubles (exact below 2^53), so equal inputs give bit-identical records; no workspace.  The EPE split by the
 * predicted mask is fn2_flow_error_regions with that mask as obj_dev (BG: visible, FG: occluded).  FN2_ERR_INVALID for N
 * above 65535, H * W above 2^30, pair_stride < H * W or a misaligned out_dev.
 */
#ifndef FN2_EVAL_H_
#define FN2_EVAL_H_

#include "fn2.h"

#define FN2_FLOW_ERROR_FIELDS 10
#define FN2_FLOW_ERROR_VALID 0
#define FN2_FLOW_ERROR_EPE_SUM 1
#define FN2_FLOW_ERROR_OUTLIERS 2
#define FN2_FLOW_ERROR_NONFINITE 3
#define FN2_FLOW_ERROR_N_S0_10 4
#define FN2_FLOW_ERROR_SUM_S0_10 5
#define FN2_FLOW_ERROR_N_S10_40 6
#define FN2_FLOW_ERROR_SUM_S10_40 7
#define FN2_FLOW_ERROR_N_S40 8
#define FN2_FLOW_ERROR_SUM_S40 9

#define FN2_FLOW_REGION_FIELDS 21
#define FN2_FLOW_REGION_N_MATCHED 0
#define FN2_FLOW_REGION_SUM_MATCHED 1
#define FN2_FLOW_REGION_OUT_MATCHED 2
#define FN2_FLOW_REGION_N_UNMATCHED 3
#define FN2_FLOW_REGION_SUM_UNMATCHED 4
#define FN2_FLOW_REGION_OUT_UNMATCHED 5
#define FN2_FLOW_REGION_N_D0_10 6
#define FN2_FLOW_REGION_SUM_D0_10 7
#define FN2_FLOW_REGION_OUT_D0_10 8
#define FN2_FLOW_REGION_N_D10_60 9
#define FN2_FLOW_REGION_SUM_D10_60 10
#define FN2_FLOW_REGION_OUT_D10_60 11
#define FN2_FLOW_REGION_N_D60_140 12
#define FN2_FLOW_REGION_SUM_D60_140 13
#define FN2_FLOW_REGION_OUT_D60_140 14
#define FN2_FLOW_REGION_N_BG 15
#define FN2_FLOW_REGION_SUM_BG 16
#define FN2_FLOW_REGION_OUT_BG 17
#define FN2_FLOW_REGION_N_FG 18
#define FN2_FLOW_REGION_SUM_FG 19
#define FN2_FLOW_REGION_OUT_FG 20

#define FN2_MASK_CONFUSION_FIELDS 4
#define FN2_MASK_CONFUSION_TP 0
#define FN2_MASK_CONFUSION_FP 1
#define FN2_MASK_CONFUSION_FN 2
#define FN2_MASK_CONFUSION_TN 3

/* dist2 of every pixel of a pair without an occlusion boundary: INT32_MAX */
#define FN2_DIST2_NONE 2147483647

#ifdef __cplusplus
extern "C" {
#endif

FN2_API int fn2_flow_error_workspace_bytes(int N, int H, int W, size_t* bytes);
FN2_API int fn2_flow_error(const fn2_tensor* pred, const fn2_tensor* gt, double* out_dev, void* workspace, size_t workspace_bytes,
                           void* stream);
FN2_API int fn2_occlusion_boundary_dist2(const void* masks_dev, size_t pair_stride, int N, int H, int W, int32_t* dist2_dev,
                                         void* stream);
FN2_API int fn2_flow_error_regions_workspace_bytes(int N, int H, int W, size_t* bytes);
FN2_API int fn2_flow_error_regions(const fn2_tensor* pred, const fn2_tensor* gt, const void* occ_dev, const void* obj_dev,
                                   size_t mask_pair_stride, const int32_t* dist2_dev, double* out_dev, void* workspace,
                                   size_t workspace_bytes, void* stream);
FN2_API int fn2_mask_confusion(const void* pred_dev, const void* gt_dev, size_t pair_stride, int N, int H, int W, double* out_dev,
                               void* stream);

/* Scoring a training net's weights with a deploy net (the train command's --val) needs the two to fit: every layer the
 * training net trains has a namesake in the deploy net with the same blob shapes, and every deploy layer with parameters gets
 * them from the training net or from its own template.  fn2_net_param_layers lists what that check reads.
 *
 * The layers that hold parameter blobs, in net order, as text: one line per layer,
 *   name TAB type TAB flags TAB shapes TAB lr_mults
 * flags: 'c' when the layer takes its blobs through its own copy (DataAugmentation: adjusted to this net's crop, so the
 * shapes need not match the source's), 't' when the template alone defines its weights (a diagonal filler, filled by
 * fn2_net_copy_trained_layers when the source leaves the layer out), '-' for neither; shapes: each blob's dims joined by 'x', the blobs separated by ','; lr_mults: each blob's
 * ParamSpec lr_mult, separated by ','.  The size-query convention of fn2_net_to_caffemodel (fn2.h); the text ends in a NUL. */
FN2_API int fn2_net_param_layers(fn2_net* net, char* out, size_t* bytes);

#ifdef __cplusplus
}
#endif

#endif /* FN2_EVAL_H_ */
