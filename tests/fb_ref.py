"""A numpy float32 restatement of the forward-backward occlusion check of include/fn2_flow.h (fn2_flow_fb_occlusion), in the
header's order, with a float32 restatement of FlowWarp's bilinear taps.  numpy rounds every float32 operation separately, as
the device does under -fmad=false, so the restatement reproduces every byte.

Flows are float32 (H, W, 2) arrays (one pair); the mask is uint8 (H, W), 255 occluded and 0 visible."""
import numpy as np

F1 = np.float32(1)


def landing(fwd):
    """-> (x2, y2, inside): the float32 point x + fu, y + fv of every pixel and FlowWarp's test of it lying in the image
    (false where the flow is not finite)."""
    H, W, _ = fwd.shape
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        x2 = xs + fwd[..., 0]
        y2 = ys + fwd[..., 1]
        inside = (x2 >= 0) & (y2 >= 0) & (x2 < np.float32(W)) & (y2 < np.float32(H))
    return x2, y2, inside


def warp(img, fwd):
    """img (H, W, C) sampled at every pixel's landing point with FlowWarp's taps and mix -> (sampled (H, W, C), inside);
    0 outside, as fn2_flow_warp_forward(fill_nan = 0) writes it."""
    H, W, _ = img.shape
    x2, y2, inside = landing(fwd)
    x2, y2 = np.where(inside, x2, 0).astype(np.float32), np.where(inside, y2, 0).astype(np.float32)
    ix, iy = x2.astype(np.int64), y2.astype(np.int64)                # (int) truncation; x2, y2 >= 0 inside
    ixr, iyb = np.minimum(ix + 1, W - 1), np.minimum(iy + 1, H - 1)
    a = x2 - ix.astype(np.float32)
    b = y2 - iy.astype(np.float32)
    cTL, cTR, cBL, cBR = (F1 - a) * (F1 - b), a * (F1 - b), (F1 - a) * b, a * b
    with np.errstate(invalid="ignore", over="ignore"):
        out = ((cTL[..., None] * img[iy, ix] + cTR[..., None] * img[iy, ixr]) + cBL[..., None] * img[iyb, ix]) \
            + cBR[..., None] * img[iyb, ixr]
    return np.where(inside[..., None], out, np.float32(0)).astype(np.float32), inside


def decide(fwd, sampled, inside, alpha1=0.01, alpha2=0.5):
    """The check from the forward flow, the backward flow sampled where it lands and FlowWarp's inside test -> uint8 mask."""
    fu, fv = fwd[..., 0], fwd[..., 1]
    bu, bv = sampled[..., 0], sampled[..., 1]
    with np.errstate(invalid="ignore", over="ignore"):
        du = fu + bu
        dv = fv + bv
        lhs = du * du + dv * dv
        mag = (fu * fu + fv * fv) + (bu * bu + bv * bv)
        fails = lhs > np.float32(alpha1) * mag + np.float32(alpha2)
    occ = ~(np.isfinite(fu) & np.isfinite(fv)) | ~inside | ~(np.isfinite(bu) & np.isfinite(bv)) | fails
    return np.where(occ, 255, 0).astype(np.uint8)


def fb_occlusion(fwd, bwd, alpha1=0.01, alpha2=0.5):
    """Frame 0's mask from the forward flow fwd and the backward flow bwd, both float32 (H, W, 2)."""
    fwd, bwd = np.asarray(fwd, np.float32), np.asarray(bwd, np.float32)
    sampled, inside = warp(bwd, fwd)
    return decide(fwd, sampled, inside, alpha1, alpha2)
