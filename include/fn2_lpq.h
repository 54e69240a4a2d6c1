/*
 * fn2_lpq.h -- C-ABI of libfn2.so for the robust flow loss LpqLoss (lpq_loss_layer.{cpp,cu}, LpqLossParameter at
 * caffe.proto:563-602), and the net iteration its p/q schedule follows.  A sibling of fn2_solver.h, fn2_frames.h and
 * fn2_flow.h, with fn2.h's conventions: status 0 or negative with the message in fn2_last_error().
 *
 * LpqLoss -- replaces LpqLossLayer::Forward_gpu / Backward_gpu (lpq_loss_layer.cu:96-245; the CPU paths are NOT_IMPLEMENTED
 * in the reference, lpq_loss_layer.cpp:175-188):
 *     loss = sum over (n, y, x) of Q(sum_c w * P(|d_c|)) / norm,   P(a) = (a + p_epsilon)^p,   Q(s) = (s + q_epsilon)^q,
 * d = bottom0 - bottom1 (or bottom0 alone when bottom1 is NULL), a NaN d_c counted as 0, w = 1 or 1/C
 * (l2_prescale_by_channels), norm = N or (not-NaN count) / C (normalize_by_num_entries).
 *
 * state_dev: FN2_LPQLOSS_STATE_FLOATS device floats {loss, normalize_coeff, loss sum, not-NaN count, p, q}.  The caller writes
 * p and q (state_dev[4], state_dev[5]) on the stream before the forward; they are not descriptor fields, so a forward
 * captured in a CUDA graph and the backward read the values current when they run.  The forward writes state_dev[0..3] and
 * loss_dev (may be NULL); the backward reads normalize_coeff, p and q.  workspace: at least fn2_lpqloss_workspace_bytes(N, H,
 * W) bytes, 4-byte aligned; a NULL or smaller one returns FN2_ERR_WORKSPACE.  The forward reduces its per-block partials in a
 * fixed order: equal inputs give bit-identical state.  top_diff_dev: device scalar (the loss weight).  The backward recomputes
 * the difference, the NaN mask, the signs, the per-location sum and both power derivatives from the bottoms; a NULL diff
 * pointer means "do not propagate to this bottom"; accumulate != 0 adds to the diff.
 */
#ifndef FN2_LPQ_H_
#define FN2_LPQ_H_

#include "fn2.h"

#define FN2_LPQLOSS_STATE_FLOATS 6

#ifdef __cplusplus
extern "C" {
#endif

typedef struct fn2_lpqloss_desc {
    float p_epsilon, q_epsilon;                                          /* LpqLossParameter, caffe.proto:563-602 */
    int32_t l2_prescale_by_channels, normalize_by_num_entries;
} fn2_lpqloss_desc;
FN2_API int fn2_lpqloss_workspace_bytes(int N, int H, int W, size_t* bytes);
FN2_API int fn2_lpqloss_forward(const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_lpqloss_desc* d, float* state_dev,
                                float* loss_dev, void* workspace, size_t workspace_bytes, void* stream);
FN2_API int fn2_lpqloss_backward(const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_lpqloss_desc* d,
                                 const float* state_dev, const float* top_diff_dev, const fn2_tensor* bottom0_diff,
                                 const fn2_tensor* bottom1_diff, int accumulate0, int accumulate1, void* stream);

/* Net::set_iter / iter (net.hpp:230-231): the iteration the net's layers see (LpqLoss picks its p/q schedule step by it).  A
 * net starts at 0; the Solver sets it at the start of every iteration, before the parameter diffs are cleared. */
FN2_API int fn2_net_set_iter(fn2_net* net, int iter);
FN2_API int fn2_net_iter(fn2_net* net, int* iter);

#ifdef __cplusplus
}
#endif

#endif /* FN2_LPQ_H_ */
