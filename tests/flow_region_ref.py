"""numpy restatement of fn2_occlusion_boundary_dist2 and fn2_flow_error_regions (include/fn2_eval.h): the boundary from the
mask's 4-neighbours, the distance from scipy's exact Euclidean distance transform with dist2 recomputed in integers from the
indices of the nearest boundary pixel, and the region records as tests/flow_error_ref.py states fn2_flow_error's (float32 per
pixel, float64 sums)."""
import numpy as np
from scipy import ndimage

from flownet2_b200 import DIST2_NONE, FLOW_REGION_FIELDS

F32 = np.float32
COL = {f: i for i, f in enumerate(FLOW_REGION_FIELDS)}


def boundary(mask):
    """(H, W) occlusion mask -> bool (H, W): the pixels with a 4-neighbour inside the image of the other label."""
    occ = np.asarray(mask) != 0
    b = np.zeros(occ.shape, bool)
    d = occ[1:, :] != occ[:-1, :]
    b[1:, :] |= d
    b[:-1, :] |= d
    d = occ[:, 1:] != occ[:, :-1]
    b[:, 1:] |= d
    b[:, :-1] |= d
    return b


def dist2_ref(masks):
    """(N, H, W) occlusion masks -> int64 (N, H, W) squared distance to the nearest boundary pixel, DIST2_NONE throughout a
    pair without one."""
    masks = np.asarray(masks)
    out = np.empty(masks.shape, np.int64)
    yy, xx = np.mgrid[:masks.shape[1], :masks.shape[2]]
    for n, m in enumerate(masks):
        b = boundary(m)
        if not b.any():
            out[n] = DIST2_NONE
            continue
        _, (iy, ix) = ndimage.distance_transform_edt(~b, return_indices=True)
        out[n] = (yy - iy.astype(np.int64)) ** 2 + (xx - ix.astype(np.int64)) ** 2
    return out


def flow_region_ref(pred, gt, occ=None, obj=None, dist2=None):
    """pred, gt: float32 (N, 2, H, W); occ, obj: (N, H, W) masks or None; dist2: the occlusion boundary distance (dist2_ref(occ)
    if None) -> (N, FLOW_REGION_FIELDS) float64 records."""
    pred, gt = np.asarray(pred, F32), np.asarray(gt, F32)
    if occ is not None and dist2 is None:
        dist2 = dist2_ref(occ)
    out = np.zeros((pred.shape[0], len(FLOW_REGION_FIELDS)))
    with np.errstate(all="ignore"):
        for n in range(pred.shape[0]):
            gu, gv, pu, pv = gt[n, 0], gt[n, 1], pred[n, 0], pred[n, 1]
            ok = (np.abs(gu) <= F32(1e9)) & (np.abs(gv) <= F32(1e9)) & np.isfinite(pu) & np.isfinite(pv)
            du, dv = pu - gu, pv - gv
            epe = np.sqrt(du * du + dv * dv)
            mag = np.sqrt(gu * gu + gv * gv)
            assert epe.dtype == F32 and mag.dtype == F32
            outlier = (epe > F32(3)) & (epe > F32(0.05) * mag)
            r = out[n]

            def add(region, sel):
                sel = ok & sel
                r[COL["n_" + region]] = sel.sum()
                r[COL["sum_" + region]] = epe[sel].astype(np.float64).sum()
                r[COL["out_" + region]] = (sel & outlier).sum()

            if occ is not None:
                o, d = np.asarray(occ[n]) != 0, dist2[n]
                add("matched", ~o)
                add("unmatched", o)
                add("d0_10", d < 100)
                add("d10_60", (d >= 100) & (d < 3600))
                add("d60_140", (d >= 3600) & (d < 19600))
            if obj is not None:
                f = np.asarray(obj[n]) != 0
                add("bg", ~f)
                add("fg", f)
    return out


def assert_region_match(got, want, rtol=1e-12):
    """Counts exactly, sums within rtol relative (of the larger magnitude)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (got.shape, want.shape)
    for j, f in enumerate(FLOW_REGION_FIELDS):
        if f.startswith("sum_"):
            tol = rtol * np.maximum(np.abs(want[:, j]), 1e-300)
            assert np.all(np.abs(got[:, j] - want[:, j]) <= tol), (f, got[:, j], want[:, j])
        else:
            assert np.array_equal(got[:, j], want[:, j]), (f, got[:, j], want[:, j])
