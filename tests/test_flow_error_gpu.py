"""GPU: fn2_flow_error (include/fn2_eval.h, ops.flow_error) against the float32 numpy restatement in tests/flow_error_ref.py:
counts exactly, sums within 1e-12 relative, bit-identical repeats; planted ground-truth and prediction edge cases, strided NHWC
views, and the argument refusals."""
import ctypes as C

import numpy as np
import pytest

from tests.flow_error_ref import assert_records_match, flow_error_ref

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")


def seeded_flows(n, h, w, seed):
    """gt spread over the three speed bands, pred = gt + noise wide enough to put pixels on both sides of the outlier rule,
    then the planted cases of plant()."""
    r = np.random.default_rng(seed)
    gt = (r.standard_normal((n, 2, h, w)) * r.choice([2.0, 15.0, 60.0], (n, 1, h, w))).astype(np.float32)
    pred = (gt + r.standard_normal((n, 2, h, w)) * r.choice([0.5, 3.0, 8.0], (n, 1, h, w))).astype(np.float32)
    plant(gt, pred)
    return pred, gt


# (gt_u, gt_v, pred_u, pred_v): invalid ground truth, the 1e9 limit, |gt| exactly 10 and 40, EPE exactly 3, both sides of 5 % of
# |gt| = 100 (EPE 4.5 and 5.5), and non-finite predictions on valid and on invalid pixels
CASES = [(NAN, 0.0, 1.0, 1.0), (0.0, NAN, 1.0, 1.0), (1e10, 0.0, 0.0, 0.0), (0.0, -1e10, 0.0, 0.0), (INF, 0.0, 0.0, 0.0),
         (1e9, 0.0, 1e9, 0.0), (-1e9, 1e9, -1e9, 1e9), (6.0, 8.0, 6.0, 8.0), (6.0, 8.0, 7.0, 8.0), (24.0, 32.0, 25.0, 32.0),
         (-24.0, 32.0, -24.0, 33.0), (9.999999, 0.0, 20.0, 0.0), (39.99999, 0.0, 40.0, 0.0), (0.0, 0.0, 3.0, 0.0),
         (0.0, 0.0, 3.0001, 0.0), (100.0, 0.0, 104.5, 0.0), (100.0, 0.0, 105.5, 0.0), (100.0, 0.0, 95.0, 0.0),
         (1.0, 1.0, NAN, 0.0), (1.0, 1.0, 0.0, INF), (50.0, 0.0, -INF, 0.0), (NAN, NAN, NAN, NAN), (1e10, 1e10, INF, 0.0)]


def plant(gt, pred):
    n, _, h, w = gt.shape
    for k, (gu, gv, pu, pv) in enumerate(CASES):
        i = k * 7919 % (n * h * w)                             # spread over pairs and rows
        b, y, x = i // (h * w), i // w % h, i % w
        gt[b, :, y, x] = gu, gv
        pred[b, :, y, x] = pu, pv


def run_op(pred, gt, nhwc_pred=False, sliced_gt=False):
    """The op on device copies of pred / gt: pred as the (B, 2, H, W) view of an NHWC buffer, gt as channels [1, 3) of a
    4-channel channels_last parent, when asked."""
    import torch
    from flownet2_b200 import ops
    if nhwc_pred:
        p = torch.from_numpy(np.ascontiguousarray(pred.transpose(0, 2, 3, 1))).cuda().permute(0, 3, 1, 2)
    else:
        p = torch.from_numpy(pred).cuda()
    if sliced_gt:
        parent = torch.full((gt.shape[0], 4) + gt.shape[2:], NAN, device="cuda").contiguous(memory_format=torch.channels_last)
        parent[:, 1:3] = torch.from_numpy(gt).cuda()
        g = parent[:, 1:3]
    else:
        g = torch.from_numpy(gt).cuda()
    out = ops.flow_error(p, g)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("shape", [(1, 7, 13), (3, 37, 61), (8, 436, 1024)])
def test_matches_float32_restatement(fn2, shape):
    n, h, w = shape
    pred, gt = seeded_flows(n, h, w, seed=h * w)
    want = flow_error_ref(pred, gt)
    got = run_op(pred, gt)
    assert_records_match(got, want)
    again = run_op(pred, gt)
    assert np.array_equal(got.view(np.uint64), again.view(np.uint64))               # bit-identical repeat
    strided = run_op(pred, gt, nhwc_pred=True, sliced_gt=True)
    assert np.array_equal(got.view(np.uint64), strided.view(np.uint64))             # the same pixels, the same order


def test_planted_cases_one_by_one(fn2):
    """Each planted pixel alone in a 1x1 pair: its record is what the header's definitions say."""
    F = fn2.FLOW_ERROR_FIELDS
    gt = np.array([[[[c[0]]], [[c[1]]]] for c in CASES], np.float32)
    pred = np.array([[[[c[2]]], [[c[3]]]] for c in CASES], np.float32)
    got = run_op(pred, gt)
    assert_records_match(got, flow_error_ref(pred, gt))
    rec = {k: dict(zip(F, got[k])) for k in range(len(CASES))}
    assert [rec[k]["valid"] for k in range(len(CASES))] == [0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0]
    assert rec[7]["n_s10_40"] == 1 and rec[7]["epe_sum"] == 0                          # |gt| = 10 is in [10, 40)
    assert rec[9]["n_s40"] == 1 and rec[9]["epe_sum"] == 1                             # |gt| = 40 is in [40, inf)
    assert rec[11]["n_s0_10"] == 1 and rec[12]["n_s10_40"] == 1
    assert rec[13]["outliers"] == 0 and rec[14]["outliers"] == 1                       # EPE 3 is not above 3
    assert rec[15]["outliers"] == 0 and rec[16]["outliers"] == 1 and rec[17]["outliers"] == 0   # 5 % of |gt| = 5
    for k in (18, 19, 20):                                                             # non-finite prediction, valid gt
        assert rec[k]["nonfinite"] == 1 and rec[k]["epe_sum"] == 0 and rec[k]["n_s0_10"] + rec[k]["n_s40"] == 0
    assert rec[22]["nonfinite"] == 0                                                   # on an invalid pixel it is not counted


def test_pair_without_valid_pixel(fn2):
    pred, gt = seeded_flows(3, 9, 17, seed=5)
    gt[1] = NAN
    gt[1, 0, 2, 3] = 1e10
    got = run_op(pred, gt, nhwc_pred=True)
    assert_records_match(got, flow_error_ref(pred, gt))
    assert np.all(got[1] == 0) and got[0, 0] > 0 and got[2, 0] > 0


def test_refusals(fn2):
    import torch
    from flownet2_b200 import ops
    lib = fn2.lib()
    p = torch.zeros((2, 2, 5, 7), device="cuda")
    out = torch.zeros((2, len(fn2.FLOW_ERROR_FIELDS)), dtype=torch.float64, device="cuda")
    optr = C.cast(out.data_ptr(), C.POINTER(C.c_double))
    n = ops.flow_error_workspace_bytes(2, 5, 7)
    ws = torch.zeros(n + 8, dtype=torch.uint8, device="cuda")
    call = lambda a, b, w, nb: lib.fn2_flow_error(ops.desc(a), ops.desc(b), optr, w, nb, None)
    assert call(p, p, ws.data_ptr(), n) == 0
    assert call(p, p, None, n) == -5 and "workspace" in lib.fn2_last_error().decode()
    assert call(p, p, ws.data_ptr(), n - 8) == -5
    assert call(p, p, ws.data_ptr() + 4, n) == -5 and "8-byte aligned" in lib.fn2_last_error().decode()
    assert call(p, torch.zeros((2, 2, 5, 8), device="cuda"), ws.data_ptr(), n) == -1
    assert "flow_error: pred is 2x2x5x7 but gt is 2x2x5x8" == lib.fn2_last_error().decode()
    assert call(p, torch.zeros((3, 2, 5, 7), device="cuda"), ws.data_ptr(), n) == -1
    three = torch.zeros((2, 3, 5, 7), device="cuda")
    assert call(three, three, ws.data_ptr(), n) == -1 and "2 channels, got 3" in lib.fn2_last_error().decode()
    assert lib.fn2_flow_error_workspace_bytes(0, 5, 7, C.byref(C.c_size_t())) == -1
    torch.cuda.synchronize()
