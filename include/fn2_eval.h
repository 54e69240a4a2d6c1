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

#ifdef __cplusplus
extern "C" {
#endif

FN2_API int fn2_flow_error_workspace_bytes(int N, int H, int W, size_t* bytes);
FN2_API int fn2_flow_error(const fn2_tensor* pred, const fn2_tensor* gt, double* out_dev, void* workspace, size_t workspace_bytes,
                           void* stream);

#ifdef __cplusplus
}
#endif

#endif /* FN2_EVAL_H_ */
