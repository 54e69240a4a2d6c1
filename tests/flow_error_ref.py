"""Float32 restatement of fn2_flow_error (include/fn2_eval.h) in numpy: every per-pixel value in float32 with separately rounded
operations, as the kernel computes them, and the sums in float64."""
import numpy as np

from flownet2_b200 import FLOW_ERROR_FIELDS

F32 = np.float32


def flow_error_ref(pred, gt):
    """pred, gt: float32 (N, 2, H, W) -> (N, FIELDS) float64 records."""
    pred, gt = np.asarray(pred, F32), np.asarray(gt, F32)
    out = np.zeros((pred.shape[0], len(FLOW_ERROR_FIELDS)))
    col = {f: i for i, f in enumerate(FLOW_ERROR_FIELDS)}
    with np.errstate(all="ignore"):
        for n in range(pred.shape[0]):
            gu, gv, pu, pv = gt[n, 0], gt[n, 1], pred[n, 0], pred[n, 1]
            valid = (np.abs(gu) <= F32(1e9)) & (np.abs(gv) <= F32(1e9))
            finite = np.isfinite(pu) & np.isfinite(pv)
            ok = valid & finite
            du, dv = pu - gu, pv - gv
            epe = np.sqrt(du * du + dv * dv)
            mag = np.sqrt(gu * gu + gv * gv)
            assert epe.dtype == F32 and mag.dtype == F32
            r = out[n]
            r[col["valid"]] = valid.sum()
            r[col["nonfinite"]] = (valid & ~finite).sum()
            r[col["epe_sum"]] = epe[ok].astype(np.float64).sum()
            r[col["outliers"]] = (ok & (epe > F32(3)) & (epe > F32(0.05) * mag)).sum()
            for band, sel in (("s0_10", mag < F32(10)), ("s10_40", (mag >= F32(10)) & (mag < F32(40))), ("s40", mag >= F32(40))):
                r[col["n_" + band]] = (ok & sel).sum()
                r[col["sum_" + band]] = epe[ok & sel].astype(np.float64).sum()
    return out


def assert_records_match(got, want, rtol=1e-12):
    """Counts exactly, sums within rtol relative (of the larger magnitude)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (got.shape, want.shape)
    for j, f in enumerate(FLOW_ERROR_FIELDS):
        if "sum" in f:
            tol = rtol * np.maximum(np.abs(want[:, j]), 1e-300)
            assert np.all(np.abs(got[:, j] - want[:, j]) <= tol), (f, got[:, j], want[:, j])
        else:
            assert np.array_equal(got[:, j], want[:, j]), (f, got[:, j], want[:, j])
