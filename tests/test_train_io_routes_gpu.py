"""The kernels that make every training input and every loss gradient of the FlowNet2-C training step, at its shapes (batch 8,
512x384 data, 448x320 crop), on every layout, against float64.

- L1Loss (fn2_loss.cu): the forward reduces one (loss, count) partial per block and sums the partials in a fixed order in
  l1loss_final_kernel (about 280 partials at the flow_loss2 bottom, several hundred at the fusion net's full-resolution one);
  the backward recomputes difference and masks.  Both modes (end-point error and L1), one and two bottoms, the normalisers and
  the plateau, NaN in the ground truth.
- FlowAugmentation (fn2_loss.cu, compiled with FMA contraction): nearest flow sample at the transformed position.  Where that
  position lies within MARGIN of a rounding tie either neighbouring sample is accepted; everywhere else the exact one.
- DataAugmentation (fn2_ops.cu, -fmad=false): spatial augmentation, the eigenspace statistics, chromatic-eigen and colour
  contrast, effects and noise, the running mean.  They write in place: the parent's other channels must keep their NaN.
- FlowWarp backward (fn2_ops.cu): the flow gradient has no atomics (bit-identical run to run), the image gradient is an atomic
  scatter into a zero-filled view.

Layouts (tests.util.device_view): dense NCHW and channels_last, the nets' padded pixel stride, and a channel slice of a wider
parent; channels outside the view hold NaN.  Outputs go into channel slices of sentinel-filled parents.  References are float64
numpy, pinned to the oracle on small cases.  Measured worst cases are recorded as test properties (`--junitxml` with
`-o junit_family=legacy`).
"""
import ctypes as C
import re
import zlib

import numpy as np
import pytest

from oracle import oracle as O
from tests.util import device_view, kernels_per_case, maxabs, net_losses, rng

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

SENTINEL = -7.25
LAYOUTS = ("nchw", "nhwc", "pad", "slice")
BATCH, DATA_H, DATA_W, CROP_H, CROP_W = 8, 384, 512, 320, 448
F32_EPS = 2.0 ** -23


@pytest.fixture(scope="module")
def ops(fn2):
    from flownet2_b200 import ops as _ops
    return _ops


def seed_of(*key):
    return zlib.crc32(repr(key).encode())


def host(t):
    return t.contiguous().cpu().numpy()


def out_view(shape, layout):
    """An output of shape at channel 1 of a sentinel-filled parent with 2 more channels, channels_last unless layout is nchw
    -> (view, parent, index of the view)."""
    n, c, h, w = shape
    p = torch.full((n, c + 2, h, w), SENTINEL, device="cuda")
    if layout != "nchw":
        p = p.contiguous(memory_format=torch.channels_last)
    idx = (slice(None), slice(1, 1 + c))
    return p[idx], p, idx


def outside_kept(p, idx):
    keep = np.ones(p.shape, bool)
    keep[idx] = False
    return bool((host(p)[keep] == SENTINEL).all())


def neighbours_nan(v):
    """True when every channel of v's channels_last parent outside v is still NaN (device_view's padded / slice layouts;
    a dense view has no such channels)."""
    n, c, h, w = v.shape
    width = v.stride(3)
    if v.stride(1) != 1 or width == c:
        return True
    off = v.storage_offset() % width
    parent = torch.as_strided(v, (n, width, h, w), (v.stride(0), 1, v.stride(2), width), v.storage_offset() - off)
    rest = host(parent)
    rest = np.concatenate([rest[:, :off], rest[:, off + c:]], axis=1)
    return bool(np.isnan(rest).all())


def rel(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return maxabs(got, want) / max(float(np.nanmax(np.abs(want))), 1e-30)


# ---- L1Loss -----------------------------------------------------------------------------------------------------------------
def largest_train_loss():
    """The largest L1Loss bottom of any models/*_train.prototxt.template at the config-5 crop and batch."""
    import glob
    import os
    from flownet2_b200 import fill_train_template, train_template
    best = None
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "models")
    for f in sorted(glob.glob(os.path.join(root, "*_train.prototxt.template"))):
        model = os.path.basename(f)[:-len("_train.prototxt.template")]
        for _, chw in net_losses(fill_train_template(train_template(model), CROP_W, CROP_H, DATA_W, DATA_H, BATCH)):
            if best is None or np.prod(chw) > np.prod(best):
                best = chw
    return (BATCH,) + tuple(best)


# the five losses of FlowNet2-C at 448x320 (flow_loss6 .. flow_loss2), then the fusion net's full-resolution flow_loss0
L1_SHAPES = [(BATCH, 2, 5, 7), (BATCH, 2, 10, 14), (BATCH, 2, 20, 28), (BATCH, 2, 40, 56), (BATCH, 2, 80, 112), largest_train_loss()]
L1_MODES = {
    "epe": dict(l2_per_location=True),                                    # the nets' mode
    "epe_all": dict(l2_per_location=True, l2_prescale_by_channels=True, normalize_by_num_entries=True, plateau=0.3),
    "l1": dict(),
    "l1_all": dict(normalize_by_num_entries=True, plateau=0.2, epsilon=0.0),
}
LOSS_TOL = 5e-7        # relative; measured on an H100 80GB HBM3 (700 W): loss 9.2e-8, gradients 2.1e-7
TOP_DIFF = 0.32                                                           # flow_loss6's loss weight


def l1_inputs(shape, mode, two, seed):
    """(bottom0, bottom1 or None) float32: differences of a few units, NaN blocks in the ground truth (or in the single
    bottom) and a whole NaN sample; no per-location sum or |difference| within 1e-4 (relative) of the plateau threshold."""
    kw = L1_MODES[mode]
    r = rng(seed)
    n, c, h, w = shape
    pred = (3 * r.standard_normal(shape)).astype(np.float32)
    d = (0.6 * r.standard_normal(shape)).astype(np.float32)
    p = np.float32(kw.get("plateau", 0.0))
    for _ in range(4):
        gt = (pred - d).astype(np.float32)
        e = np.asarray(pred - gt if two else d, np.float64)              # the difference the kernel forms
        if kw.get("l2_per_location"):
            wsum = 1.0 / c if kw.get("l2_prescale_by_channels") else 1.0
            s = (wsum * e * e).sum(1, keepdims=True)
            near = np.broadcast_to(np.abs(s - float(p * p)) <= 1e-4 * float(p * p), d.shape)
        else:
            near = np.abs(np.abs(e) - float(p)) <= 1e-4 * float(p)
        if not near.any():
            break
        d = np.where(near, 1.5 * d, d).astype(np.float32)
    assert not near.any()
    nanb = gt if two else d
    nanb[0, :, h // 4:h // 2 + 1, w // 3:w // 2 + 1] = np.nan
    if n > 2:
        nanb[2] = np.nan
    return (pred, gt) if two else (d, None)


def l1_ref(b0, b1, mode, top_diff=TOP_DIFF):
    """float64 L1Loss: -> (loss, norm (float32, exact), masked sum, not-NaN count, grad of bottom0)."""
    kw = L1_MODES[mode]
    eps, p = float(np.float32(kw.get("epsilon", 1e-2))), np.float32(kw.get("plateau", 0.0))
    d = np.asarray(b0, np.float64) - (np.asarray(b1, np.float64) if b1 is not None else 0.0)
    n, c = d.shape[:2]
    ok = ~np.isnan(d)
    cnt = int(ok.sum())
    norm = np.float32(np.float32(cnt) / np.float32(c)) if kw.get("normalize_by_num_entries") else np.float32(n)
    alpha = float(np.float32(top_diff)) / float(norm) if norm else np.inf
    dz = np.where(ok, d, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        if kw.get("l2_per_location"):
            wsum = 1.0 / c if kw.get("l2_prescale_by_channels") else 1.0
            s = (wsum * dz * dz).sum(1)
            kill = (s < float(p * p)) if p > 0 else np.zeros(s.shape, bool)
            s = np.where(kill, 0.0, s)
            root = np.sqrt(s + eps)
            masked = root.sum()
            gs = np.where(kill, 0.0, 0.5 / root * alpha)
            g = np.where(ok, 2.0 * dz * wsum * gs[:, None], 0.0)
        else:
            keep = ok & ~(np.abs(dz) < float(p)) if p > 0 else ok
            masked = np.abs(np.where(keep, dz, 0.0)).sum()
            g = np.where(keep, alpha * np.where(dz > 0, 1.0, -1.0), 0.0)
        loss = masked / float(norm)
    return loss, norm, masked, cnt, g


@pytest.mark.parametrize("mode", list(L1_MODES))
@pytest.mark.parametrize("two", [True, False])
def test_l1_reference_matches_oracle(mode, two):
    b0, b1 = l1_inputs((3, 2, 9, 13), mode, two, seed_of("l1ref", mode, two))
    loss, norm, _, _, g = l1_ref(b0, b1, mode, 1.7)
    oloss, onorm = O.l1loss_fwd(b0, b1, **L1_MODES[mode])
    og, og1 = O.l1loss_bwd(b0, b1, 1.7, **L1_MODES[mode])
    assert norm == onorm
    assert abs(loss - float(oloss)) <= 4 * F32_EPS * abs(loss)
    assert rel(og, g) <= 4 * F32_EPS and np.array_equal(og1, -og)


L1_CASES = ([(shape, mode, "pad", True) for shape in L1_SHAPES for mode in L1_MODES] +
            [(L1_SHAPES[4], mode, lay, two) for mode in L1_MODES for lay in LAYOUTS for two in (True, False)
             if (lay, two) != ("pad", True)])


def l1_id(c):
    shape, mode, lay, two = c
    return "%dx%d-%s-%s-%s" % (shape[2], shape[3], mode, lay, "two" if two else "one")


def l1_run(ops, b0, b1, mode, lay):
    v0 = device_view(b0, lay)
    v1 = device_view(b1, lay) if b1 is not None else None
    return v0, v1, (lambda: ops.l1loss(v0, v1, **L1_MODES[mode]))


@pytest.mark.parametrize("c", L1_CASES, ids=l1_id)
def test_l1loss(ops, c, record_property):
    """Forward: state[1] and state[3] exact, loss and masked sum within LOSS_TOL of float64, two calls bit-identical.
    Backward into sentinel-guarded slices, the loss weight a device scalar, within LOSS_TOL of the largest gradient."""
    shape, mode, lay, two = c
    b0, b1 = l1_inputs(shape, mode, two, seed_of("l1", c))
    loss, norm, masked, cnt, g = l1_ref(b0, b1, mode)
    v0, v1, run = l1_run(ops, b0, b1, mode, lay)
    dloss, dstate = run()
    st, ls = host(dstate), host(dloss)
    assert st[1] == norm and st[3] == cnt
    assert ls[0] == st[0]
    el, em = abs(st[0] - loss) / abs(loss), abs(st[2] - masked) / abs(masked)
    assert el <= LOSS_TOL and em <= LOSS_TOL, (el, em)
    dloss2, dstate2 = run()
    assert np.array_equal(host(dstate2), st) and np.array_equal(host(dloss2), ls)
    top = torch.tensor([TOP_DIFF], device="cuda")
    o0 = out_view(shape, lay)
    o1 = out_view(shape, lay) if two else (None, None, None)
    ops.l1loss_backward(v0, v1, state=dstate, top_diff=top, out0=o0[0], out1=o1[0], **L1_MODES[mode])
    eg = rel(host(o0[0]), g)
    assert eg <= LOSS_TOL, eg
    assert outside_kept(o0[1], o0[2])
    if two:
        assert np.array_equal(host(o1[0]), -host(o0[0])) and outside_kept(o1[1], o1[2])
    assert neighbours_nan(v0) and (v1 is None or neighbours_nan(v1))
    record_property("loss_rel", max(el, em))
    record_property("grad_rel", eg)


@pytest.mark.parametrize("lay", LAYOUTS)
@pytest.mark.parametrize("mode", ["epe", "l1_all"])
def test_l1loss_backward_accumulate_and_null(ops, lay, mode, record_property):
    """accumulate into non-zero priors (bottom0 adds g, bottom1 adds -g); each diff NULL in turn leaves the other one right."""
    shape = L1_SHAPES[4]
    b0, b1 = l1_inputs(shape, mode, True, seed_of("acc", lay, mode))
    _, _, _, _, g = l1_ref(b0, b1, mode)
    v0, v1, run = l1_run(ops, b0, b1, mode, lay)
    _, state = run()
    top = torch.tensor([TOP_DIFF], device="cuda")
    r = rng(seed_of("prior", lay, mode))
    p0, p1 = r.standard_normal(shape).astype(np.float32), r.standard_normal(shape).astype(np.float32)
    o0, o1 = out_view(shape, lay), out_view(shape, lay)
    o0[0].copy_(torch.from_numpy(p0))
    o1[0].copy_(torch.from_numpy(p1))
    ops.l1loss_backward(v0, v1, state=state, top_diff=top, out0=o0[0], out1=o1[0], accumulate0=True, accumulate1=True,
                        **L1_MODES[mode])
    e = 0.0
    for got, want in ((host(o0[0]), p0 + g), (host(o1[0]), p1 - g)):
        # beyond the float32 rounding of the sum, which can exceed the gradient when the entries normalise it
        beyond = np.abs(got - want) - np.spacing(np.abs(want).astype(np.float32))
        e = max(e, float(beyond.max()) / np.abs(g).max())
    assert e <= LOSS_TOL, e
    record_property("acc_rel", e)
    for which in (0, 1):
        o = out_view(shape, lay)
        kw = dict(out0=o[0]) if which == 0 else dict(out1=o[0])
        ops.l1loss_backward(v0, v1, state=state, top_diff=top, **kw, **L1_MODES[mode])
        assert rel(host(o[0]), g if which == 0 else -g) <= LOSS_TOL
        assert outside_kept(o[1], o[2])


@pytest.mark.parametrize("mode", list(L1_MODES))
def test_l1loss_all_nan_bottom(ops, mode):
    """An all-NaN ground truth: the not-NaN count is 0, loss and normaliser as the oracle gives them (normalising by the
    entries divides by 0), and every gradient is 0."""
    shape = (BATCH, 2, 10, 14)
    b0 = rng(5).standard_normal(shape).astype(np.float32)
    b1 = np.full(shape, np.nan, np.float32)
    oloss, onorm = O.l1loss_fwd(b0, b1, **L1_MODES[mode])
    loss, state = ops.l1loss(device_view(b0, "pad"), device_view(b1, "pad"), **L1_MODES[mode])
    st = host(state)
    assert st[3] == 0 and st[1] == onorm
    assert np.array_equal(st[:1], np.array([oloss], np.float32), equal_nan=True)
    o0, o1 = torch.full(shape, 5.0, device="cuda"), torch.full(shape, 5.0, device="cuda")
    ops.l1loss_backward(device_view(b0, "pad"), device_view(b1, "pad"), state=state, top_diff=torch.tensor([1.0], device="cuda"),
                        out0=o0, out1=o1, **L1_MODES[mode])
    assert (host(o0) == 0).all() and (host(o1) == 0).all()


def test_l1loss_errors(ops, fn2):
    """A workspace one float short (or none) is FN2_ERR_WORKSPACE; the exact size works; a shape mismatch and a diff for a
    missing bottom are FN2_ERR_INVALID."""
    l = fn2.lib()
    shape = L1_SHAPES[4]
    b0 = torch.zeros(shape, device="cuda")
    b1 = torch.zeros(shape, device="cuda")
    n = C.c_size_t()
    assert l.fn2_l1loss_workspace_bytes(shape[0], shape[2], shape[3], C.byref(n)) == 0
    ws = torch.zeros(n.value, dtype=torch.uint8, device="cuda")
    state = torch.zeros(4, device="cuda")
    d = fn2.fn2_l1loss_desc(1, 0, 0, 0.01, 0.0)
    fwd = lambda a, b, nb, w=ws: l.fn2_l1loss_forward(ops.desc(a), ops.desc(b) if b is not None else None, d, state.data_ptr(),
                                                      None, w.data_ptr() if w is not None else None, nb, None)
    assert fwd(b0, b1, n.value) == 0
    torch.cuda.synchronize()
    assert fwd(b0, b1, n.value - 4) == -5 and fwd(b0, b1, 0, None) == -5 and fwd(b0, b1, n.value, None) == -5
    assert fwd(b0, torch.zeros((shape[0], 2, shape[2], shape[3] + 1), device="cuda"), n.value) == -1
    top = torch.ones(1, device="cuda")
    assert l.fn2_l1loss_backward(ops.desc(b0), None, d, state.data_ptr(), top.data_ptr(), None, ops.desc(b1), 0, 0, None) == -1
    assert l.fn2_l1loss_backward(ops.desc(b0), ops.desc(b1), d, state.data_ptr(), top.data_ptr(),
                                 ops.desc(torch.zeros((shape[0], 2, shape[2] + 1, shape[3]), device="cuda")), None, 0, 0, None) == -1


# ---- augmentation transforms ------------------------------------------------------------------------------------------------
def sampled_coeffs(fn2, seed, num_iter=1e9):
    """Coefficient records of the FlowNet2-C training template's first DataAugmentation layer (img0s_aug) at num_iter (1e9:
    the discount schedule at full strength), -> (BATCH, 42) in value form."""
    from flownet2_b200 import fill_train_template, train_template
    text = fill_train_template(train_template("FlowNet2-C"), CROP_W, CROP_H, DATA_W, DATA_H, BATCH)
    layer = re.search(r'layer \{\n  name: "img0s_aug".*?\n\}\n', text, re.S).group(0)
    out = np.zeros((BATCH, 42), np.float32)
    rc = fn2.lib().fn2_aug_sample(layer.encode(), seed, BATCH, DATA_W, DATA_H, C.c_float(num_iter),
                                  out.ctypes.data_as(C.POINTER(C.c_float)))
    assert rc == 0
    return O.aug_array_to_values(out)


def spatial_mats(v):
    """NAME-ordered transforms of the value records v (the order of oracle.flow_augmentation)."""
    return np.stack([O.transmat_from_coeff(CROP_W, CROP_H, DATA_W, DATA_H, *[float(r[i]) for i in (0, 3, 1, 2, 4, 5)]) for r in v])


IDENTITY = np.tile(np.array([1, 0, 0, 1, 0, 0], np.float32), (BATCH, 1))
# x' ~ 1.3 x - 0.2 y - 150, y' ~ 0.1 x + 1.2 y - 60 and a mirror: sample positions left of, right of, above and below the
# image (coefficients off round decimals, which would put whole columns on rounding ties)
OUTSIDE = np.tile(np.array([1.2917, 0.1063, -0.2141, 1.1874, -150.37, -60.21], np.float32), (BATCH, 1))
OUTSIDE[1::2] = [-1.3127, 0.0971, 0.2033, 1.2461, 600.13, -20.29]


def flow_transforms(fn2, kind):
    if kind == "sampled":
        return spatial_mats(sampled_coeffs(fn2, 3)), np.stack([O.transmat_inverse(m) for m in spatial_mats(sampled_coeffs(fn2, 4))])
    if kind == "identity":
        return IDENTITY, IDENTITY
    return OUTSIDE, np.stack([O.transmat_inverse(m) for m in spatial_mats(sampled_coeffs(fn2, 5))])


# ---- FlowAugmentation ---------------------------------------------------------------------------------------------------------
MARGIN = 1e-3          # |x1 + 0.5 - k| below this: the kernel's contracted x1 may round to either side of the tie


def flow_aug_ref(flow, m1, m2, oh, ow):
    """float64 -> (out for the low / high candidate sample of each axis: 4 arrays (N, 2, oh, ow), ambiguous-pixel mask)."""
    flow = np.asarray(flow, np.float64)
    N, _, H, W = flow.shape
    flat = flow.reshape(-1)
    ys, xs = np.mgrid[0:oh, 0:ow].astype(np.float64)
    outs = np.empty((4, N, 2, oh, ow))
    amb = np.zeros((N, oh, ow), bool)
    for n in range(N):
        a, b = np.asarray(m1[n], np.float64), np.asarray(m2[n], np.float64)
        x1, y1 = xs * a[0] + ys * a[2] + a[4], xs * a[1] + ys * a[3] + a[5]
        cx = [np.trunc(x1 + 0.5 - MARGIN), np.trunc(x1 + 0.5 + MARGIN)]
        cy = [np.trunc(y1 + 0.5 - MARGIN), np.trunc(y1 + 0.5 + MARGIN)]
        amb[n] = (cx[0] != cx[1]) | (cy[0] != cy[1])
        for k, (sx, sy) in enumerate((cx[i], cy[j]) for i in (0, 1) for j in (0, 1)):
            iu = np.clip(W * (H * (2 * n) + sy) + sx, 0, flat.size - 1).astype(np.int64)
            iv = np.clip(W * (H * (2 * n + 1) + sy) + sx, 0, flat.size - 1).astype(np.int64)
            x2, y2 = x1 + flat[iu], y1 + flat[iv]
            outs[k, n, 0] = x2 * b[0] + y2 * b[2] + b[4] - xs
            outs[k, n, 1] = x2 * b[1] + y2 * b[3] + b[5] - ys
    return outs, amb


def flow_aug_input(seed, shape=(BATCH, 2, DATA_H, DATA_W)):
    r = rng(seed)
    flow = (5 * r.standard_normal(shape)).astype(np.float32)       # white noise: a wrong sample is off by several units
    flow[1, :, 100:140, 200:260] = np.nan                              # invalid ground truth
    return flow


FLOW_AUG_TOL = 5e-4    # absolute, on positions up to ~1000 (float32 ulp 6e-5); measured 2.2e-4


def test_flow_aug_reference_matches_oracle():
    """flow_aug_ref's unambiguous pixels against oracle.flow_augmentation (float32, uncontracted)."""
    n = 2
    flow = flow_aug_input(9, (n, 2, 48, 64))
    p1, p2 = np.zeros((n, 42), np.float32), np.zeros((n, 42), np.float32)
    p1[:, 3], p1[:, 1], p2[:, 3], p2[:, 4] = 0.1, 0.05, -0.05, np.log(1.1)     # angle, dx; angle, log zoom_x
    p1[1, 0] = 1.0                                                     # mirror
    want = O.flow_augmentation(flow, p1, p2, 56, 40)
    v1, v2 = O.aug_array_to_values(p1), O.aug_array_to_values(p2)
    m1 = np.stack([O.transmat_from_coeff(56, 40, 64, 48, *[float(v1[k, i]) for i in (0, 3, 1, 2, 4, 5)]) for k in range(n)])
    m2 = np.stack([O.transmat_inverse(O.transmat_from_coeff(56, 40, 64, 48, *[float(v2[k, i]) for i in (0, 3, 1, 2, 4, 5)]))
                   for k in range(n)])
    outs, amb = flow_aug_ref(flow, m1, m2, 40, 56)
    sel = ~np.broadcast_to(amb[:, None], want.shape)
    assert maxabs(np.where(sel, want, 0), np.where(sel, outs[0], 0)) <= FLOW_AUG_TOL


@pytest.mark.parametrize("kind", ["sampled", "identity", "outside"])
@pytest.mark.parametrize("lay", LAYOUTS)
def test_flow_augmentation(ops, fn2, kind, lay, record_property):
    flow = flow_aug_input(seed_of("flowaug", kind))
    m1, m2 = flow_transforms(fn2, kind)
    vf = device_view(flow, lay)
    out = out_view((BATCH, 2, CROP_H, CROP_W), lay)
    ops.flow_augmentation(vf, torch.from_numpy(m1).cuda(), torch.from_numpy(m2).cuda(), CROP_H, CROP_W, out=out[0])
    got = host(out[0]).astype(np.float64)
    outs, amb = flow_aug_ref(flow, m1, m2, CROP_H, CROP_W)
    assert kind != "identity" or np.isnan(got).any()                  # the NaN block of the ground truth was sampled
    with np.errstate(invalid="ignore"):
        err = np.abs(got[None] - outs)
    both_nan = np.isnan(got)[None] & np.isnan(outs)
    err = np.where(both_nan, 0.0, np.where(np.isnan(err), np.inf, err))
    best = err.min(0)
    exact = np.broadcast_to(~amb[:, None], got.shape)
    e_exact = float(err[0][exact].max())
    assert e_exact <= FLOW_AUG_TOL, e_exact                           # the exact index away from ties
    assert float(best.max()) <= FLOW_AUG_TOL                          # one of the neighbours at a tie
    assert amb.mean() < 1e-2 if kind != "identity" else not amb.any()
    assert outside_kept(out[1], out[2]) and neighbours_nan(vf)
    record_property("flow_aug_abs", e_exact)
    record_property("ambiguous", float(amb.mean()))


# ---- DataAugmentation -------------------------------------------------------------------------------------------------------
EIGVEC = [0.51, 0.56, 0.65, 0.79, 0.01, -0.62, 0.35, -0.83, 0.44]


def images(seed, shape=(BATCH, 3, DATA_H, DATA_W)):
    """Frames scaled to [0, 1] as the nets feed them (Eltwise 1/255), with smooth structure and a few saturated pixels."""
    r = rng(seed)
    x = r.uniform(0.05, 0.95, shape).astype(np.float32)
    x[:, :, :4] = 1.0
    x[:, :, -4:, :8] = 0.0
    return x


@pytest.mark.parametrize("lay", LAYOUTS)
def test_spatial_augmentation_config5(ops, fn2, lay):
    """8x3x384x512 -> 320x448 with the sampled transforms, bit-exact to the oracle."""
    x = images(seed_of("spatial", lay))
    mats = spatial_mats(sampled_coeffs(fn2, 11))
    vx = device_view(x, lay)
    out = out_view((BATCH, 3, CROP_H, CROP_W), lay)
    ops.spatial_augmentation(vx, torch.from_numpy(mats).cuda(), CROP_H, CROP_W, out=out[0])
    assert np.array_equal(host(out[0]), O.spatial_augmentation(x, mats, CROP_H, CROP_W))
    assert outside_kept(out[1], out[2]) and neighbours_nan(vx)


def crop_images(seed):
    return images(seed, (BATCH, 3, CROP_H, CROP_W))


@pytest.mark.parametrize("lay", LAYOUTS)
def test_chromatic_eigenspace_config5(ops, lay, record_property):
    """The grid-wide reduction over 8x320x448 pixels: max / min (and the max |eigen| products) exact, the means within the
    float32 rounding of the float64 means."""
    x = crop_images(seed_of("eig", lay))
    vx = device_view(x, lay)
    space = host(ops.chromatic_eigenspace(vx, EIGVEC))[:25]
    want = O.chromatic_eigenspace(x, EIGVEC)
    assert np.array_equal(space[6:16], want[6:16]) and np.array_equal(space[16:25], want[16:25])
    assert np.array_equal(space[9:12], x.max((0, 2, 3))) and np.array_equal(space[12:15], x.min((0, 2, 3)))
    mean64 = np.asarray(x, np.float64).mean((0, 2, 3))
    e = np.abs(space[3:6] - mean64) / mean64
    assert (e <= 2 * F32_EPS).all(), e
    ev = np.asarray(EIGVEC, np.float64).reshape(3, 3)
    me64 = ev @ mean64 / np.asarray(want[6:9], np.float64)
    assert np.abs(space[0:3] - me64).max() <= 8 * F32_EPS * np.abs(me64).max()
    assert neighbours_nan(vx)
    record_property("mean_rel", float(e.max()))


def eigen_coeffs(seed):
    r = rng(seed)
    c = np.tile(np.array([1, 1, 1, 0, 0, 0, 1, 1, 1, 1, 1, 1, 0, 0, 0, 1, 1, 1, 1, 0, 1, 0], np.float32), (BATCH, 1))
    return (c + r.uniform(-0.2, 0.2, c.shape)).astype(np.float32)


# powf / cosf / sinf differ by a few ulps between the device and libm; absolute, on values in [0, 1]; measured 1.8e-6 and 1.8e-7
EIGEN_TOL, CONTRAST_TOL = 4e-6, 4e-7


@pytest.mark.parametrize("lay", LAYOUTS)
def test_colour_augmentations_config5(ops, lay, record_property):
    """chromatic-eigen and colour contrast against the oracle within POW_TOL; apply_effects (shadow and clamp) exact."""
    x = crop_images(seed_of("colour", lay))
    space = O.chromatic_eigenspace(x, EIGVEC)
    coeffs = eigen_coeffs(seed_of("coeffs", lay))
    dspace = torch.zeros(32, device="cuda")
    dspace[:25] = torch.from_numpy(space)
    r = rng(seed_of("chroma", lay))
    chroma = np.stack([r.uniform(0.8, 1.2, BATCH), r.uniform(-0.05, 0.05, BATCH), r.uniform(0.8, 1.2, BATCH),
                       r.uniform(0.9, 1.1, BATCH), r.uniform(0.9, 1.1, BATCH), r.uniform(0.9, 1.1, BATCH)], 1).astype(np.float32)
    eff = np.zeros((BATCH, 9), np.float32)
    ang = r.uniform(0, 6.28, BATCH)
    eff[:, 4], eff[:, 5], eff[:, 6], eff[:, 7] = np.cos(ang), np.sin(ang), r.uniform(-50, 50, BATCH), r.uniform(0.1, 0.4, BATCH)
    dcoeffs, dchroma, deff = (torch.from_numpy(a).cuda() for a in (coeffs, chroma, eff))
    v = in_place(x, lay, "fn2_chromatic_eigen_augmentation", dcoeffs.data_ptr(), dspace.data_ptr(), 1.0)
    e1 = maxabs(host(v), O.chromatic_eigen_augmentation(x, coeffs, space, 1.0))
    assert neighbours_nan(v)
    v = in_place(x, lay, "fn2_color_contrast_augmentation", dchroma.data_ptr(), 1.0)
    e2 = maxabs(host(v), O.color_contrast_augmentation(x, chroma, 1.0))
    assert neighbours_nan(v)
    v = in_place(x, lay, "fn2_apply_effects", deff.data_ptr(), 1.0, 0, 0)
    assert np.array_equal(host(v), O.apply_effects(x, eff, 1.0))
    assert neighbours_nan(v)
    assert e1 <= EIGEN_TOL and e2 <= CONTRAST_TOL, (e1, e2)
    record_property("eigen_abs", e1)
    record_property("contrast_abs", e2)


def in_place(x, lay, entry, *args):
    """x placed in layout lay, then the in-place augmentation `entry` run on that view itself (the ops wrappers work on a
    clone, which is dense) -> the view."""
    from flownet2_b200 import lib
    from flownet2_b200 import ops as _ops
    v = device_view(x, lay)
    assert getattr(lib(), entry)(_ops.desc(v), *args, torch.cuda.current_stream().cuda_stream) == 0
    return v


@pytest.mark.parametrize("lay", ["nchw", "pad"])
def test_gaussian_noise_config5(ops, fn2, lay, record_property):
    """The sampled per-sample sigma: same seed, same noise; another seed, other noise; mean and standard deviation of each
    sample's noise within 1 % of sigma (about 8 standard errors for 430,080 draws)."""
    sigma = sampled_coeffs(fn2, 13)[:, 41]
    sigma[0] = 0.0
    base = np.full((BATCH, 3, CROP_H, CROP_W), 0.5, np.float32)
    eff = np.zeros((BATCH, 9), np.float32)
    eff[:, 8] = sigma
    deff = torch.from_numpy(eff).cuda()
    run = lambda seed: host(in_place(base, lay, "fn2_apply_effects", deff.data_ptr(), 10.0, seed, 1))
    a, b, c = run(1234), run(1234), run(99)
    assert np.array_equal(a, b) and not np.array_equal(a, c)
    assert (a[0] == 0.5).all()
    worst = 0.0
    for n in range(1, BATCH):
        d = a[n].astype(np.float64) - 0.5
        e = max(abs(d.std() / sigma[n] - 1), abs(d.mean()) / sigma[n])
        worst = max(worst, e)
        assert e < 0.01, (n, sigma[n], d.mean(), d.std())
    record_property("noise_rel", worst)


@pytest.mark.parametrize("num_iter", [1, 1000])
@pytest.mark.parametrize("lay", LAYOUTS)
def test_mean_update_config5(ops, lay, num_iter, record_property):
    """The running mean over the batch (bit-exact to the oracle) and its per-channel average of 143,360 pixels against float64."""
    x = crop_images(seed_of("mean", lay, num_iter))
    prior = rng(seed_of("mpp", lay)).uniform(0.3, 0.5, (1, 3, CROP_H, CROP_W)).astype(np.float32)
    vx, vm = device_view(x, lay), device_view(prior, lay)
    pc = torch.zeros(3, device="cuda")
    ops.mean_update(vx, vm, pc, num_iter)
    _, wpp, _ = O.mean_subtract(x, 0, num_iter=float(num_iter), recompute_mean=1000, mean_pp=prior[0])
    mpp = host(vm)[0]
    assert np.array_equal(mpp, wpp)
    pp64 = (np.asarray(prior[0], np.float64) * (num_iter - 1) + np.asarray(x, np.float64).mean(0)) / num_iter
    assert np.abs(mpp - pp64).max() <= 4 * F32_EPS * np.abs(pp64).max()
    pc64 = np.asarray(mpp, np.float64).mean((1, 2))
    e = np.abs(host(pc) - pc64) / pc64
    assert (e <= F32_EPS).all(), e                                     # one float32 rounding of the float64 mean
    assert neighbours_nan(vx) and neighbours_nan(vm)
    record_property("mean_pc_rel", float(e.max()))


# ---- FlowWarp backward ------------------------------------------------------------------------------------------------------
WARP_SHAPES = [(BATCH, 3, CROP_H, CROP_W), (3, 3, 23, 31)]


def warp_inputs(shape, seed):
    """image, flow, warped diff; the flow lands on the last column and row (integer and half-way: the R == L / B == T clamp),
    outside the image, on exact grid points, and is NaN in places."""
    n, c, h, w = shape
    r = rng(seed)
    img = r.standard_normal(shape).astype(np.float32)
    wd = r.standard_normal(shape).astype(np.float32)
    flow = r.uniform(-6, 6, (n, 2, h, w)).astype(np.float32)
    xs, ys = np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32)
    # every 9th / 11th pixel only: the image gradient's atomic sums stay short enough for WARP_GI_TOL
    flow[:, 0, 1::5, ::9] = ((w - 1) - xs)[::9]                           # exactly on the last column
    flow[:, 0, 2::5, 4::9] = ((w - 1) - xs + 0.5)[4::9]                   # in [W-1, W): R clamped to L
    flow[:, 1, ::11, 3::7] = ((h - 1) - ys + 0.25)[::11, None]            # in [H-1, H): B clamped to T
    flow[:, 1, 5::11, 4::7] = ((h - 1) - ys)[5::11, None]
    flow[:, :, 3::5, 5::6] = np.round(flow[:, :, 3::5, 5::6])             # grid points
    flow[0, 0, :, :3] = -1000.0                                           # outside
    flow[-1, 1, 0, :] = h + 0.0                                           # just below the image
    flow[0, :, 5, 7] = np.nan
    flow[-1, 0, h - 2, w - 3] = np.nan
    return img, flow, wd


def warp_bwd_ref(img, flow, wd):
    """float64 -> (image diff, flow diff); x + u and y + v are formed in float32 as the kernel does."""
    n, c, h, w = img.shape
    xs = np.arange(w, dtype=np.float32)[None, None, :]
    ys = np.arange(h, dtype=np.float32)[None, :, None]
    x2 = (xs + flow[:, 0]).astype(np.float64)
    y2 = (ys + flow[:, 1]).astype(np.float64)
    with np.errstate(invalid="ignore"):
        inside = (x2 >= 0) & (y2 >= 0) & (x2 < w) & (y2 < h)
    x2, y2 = np.where(inside, x2, 0), np.where(inside, y2, 0)
    L, T = np.floor(x2).astype(np.int64), np.floor(y2).astype(np.int64)
    R, B = np.minimum(L + 1, w - 1), np.minimum(T + 1, h - 1)
    a, b = x2 - L, y2 - T
    gy, gx = B - y2, R - x2
    im, wdd = np.asarray(img, np.float64), np.asarray(wd, np.float64) * inside[:, None]
    ni = np.arange(n)[:, None, None]
    gi = np.zeros((n, c, h, w))
    du, dv = np.zeros((n, h, w)), np.zeros((n, h, w))
    for ch in range(c):
        W = wdd[:, ch]
        for (yy, xx, wt) in ((T, L, (1 - a) * (1 - b)), (T, R, a * (1 - b)), (B, L, (1 - a) * b), (B, R, a * b)):
            np.add.at(gi[:, ch], (np.broadcast_to(ni, yy.shape), yy, xx), W * wt)
        TL, TR, BL, BR = (im[:, ch][ni, T, L], im[:, ch][ni, T, R], im[:, ch][ni, B, L], im[:, ch][ni, B, R])
        du += W * (gy * (TR - TL) + (1 - gy) * (BR - BL))
        dv += W * (gx * (BL - TL) + (1 - gx) * (BR - TR))
    return gi, np.stack([du, dv], 1)


def test_warp_bwd_reference_matches_oracle():
    img, flow, wd = warp_inputs((2, 3, 13, 17), 3)
    wi, wf = O.flow_warp_bwd(img, flow, wd)
    gi, gf = warp_bwd_ref(img, flow, wd)
    assert rel(wi, gi) <= 1e-6 and rel(wf, gf) <= 1e-6


WARP_GF_TOL, WARP_GI_TOL = 5e-7, 1e-5   # relative to the largest entry; measured 1.4e-7 and 5.7e-6 (float32 atomics)


@pytest.mark.parametrize("lay", LAYOUTS)
@pytest.mark.parametrize("shape", WARP_SHAPES, ids=lambda s: "%dx%dx%dx%d" % s)
def test_flow_warp_backward(ops, shape, lay, record_property):
    img, flow, wd = warp_inputs(shape, seed_of("warpbwd", shape, lay))
    gi64, gf64 = warp_bwd_ref(img, flow, wd)
    vi, vw = device_view(img, lay), device_view(wd, lay)
    vf = device_view(flow, "nchw" if lay == "nchw" else "nhwc")
    runs = []
    for _ in range(2):
        oi, of = out_view(img.shape, lay), out_view(flow.shape, lay)
        oi[0].fill_(3.0)                                                  # the entry point zero-fills the image diff
        ops.flow_warp_backward(vi, vf, vw, out=(oi[0], of[0]))
        runs.append((host(oi[0]), host(of[0])))
        assert outside_kept(oi[1], oi[2]) and outside_kept(of[1], of[2])
    assert np.array_equal(runs[0][1], runs[1][1])                        # no atomics in the flow gradient
    eg, ei = rel(runs[0][1], gf64), rel(runs[0][0], gi64)
    assert eg <= WARP_GF_TOL and ei <= WARP_GI_TOL, (eg, ei)
    assert neighbours_nan(vi) and neighbours_nan(vw)
    record_property("warp_gf_rel", eg)
    record_property("warp_gi_rel", ei)


# ---- routes -----------------------------------------------------------------------------------------------------------------
def test_train_io_route_kernels(ops, fn2):
    """Each case launches its kernels and none of a sibling's."""
    cases = []
    shape = L1_SHAPES[4]
    for mode, l2 in (("epe", "true"), ("l1", "false")):
        b0, b1 = l1_inputs(shape, mode, True, 1)
        v0, v1, run = l1_run(ops, b0, b1, mode, "pad")
        _, state = run()
        o = torch.empty(shape, device="cuda")
        top = torch.ones(1, device="cuda")
        cases.append((run, ["l1loss_fwd_kernel<%s>" % l2, "l1loss_final_kernel"], ["l1loss_bwd", "l1loss_fwd_kernel<%s>" % ("false" if l2 == "true" else "true")]))
        cases.append((lambda v0=v0, v1=v1, state=state, o=o, top=top, mode=mode:
                      ops.l1loss_backward(v0, v1, state=state, top_diff=top, out0=o, **L1_MODES[mode]),
                      ["l1loss_bwd_kernel<%s>" % l2], ["l1loss_fwd", "l1loss_final", "l1loss_bwd_kernel<%s>" % ("false" if l2 == "true" else "true")]))
    flow = device_view(flow_aug_input(1), "pad")
    m = torch.from_numpy(IDENTITY).cuda()
    cases.append((lambda: ops.flow_augmentation(flow, m, m, CROP_H, CROP_W), ["flow_aug_kernel"], ["spatial_aug", "l1loss"]))
    x = device_view(crop_images(1), "pad")
    cases.append((lambda: ops.chromatic_eigenspace(x, EIGVEC),
                  ["eigenspace_init_kernel", "eigenspace_stats_kernel", "eigenspace_finish_kernel"], ["chromatic_eigen_kernel"]))
    mpp, pc = torch.zeros((1, 3, CROP_H, CROP_W), device="cuda"), torch.zeros(3, device="cuda")
    cases.append((lambda: ops.mean_update(x, mpp, pc, 2), ["mean_update_kernel", "mean_per_channel_kernel"], ["mean_subtract"]))
    img, fl, wd = warp_inputs(WARP_SHAPES[1], 1)
    vi, vf, vw = device_view(img, "pad"), device_view(fl, "nhwc"), device_view(wd, "pad")
    cases.append((lambda: ops.flow_warp_backward(vi, vf, vw), ["flow_warp_bwd_kernel"], ["flow_warp_fwd"]))
    names = kernels_per_case([run for run, _, _ in cases])
    bad = []
    for (_, want, sibling), got in zip(cases, names):
        if not all(any(w in n for n in got) for w in want) or any(s in n for s in sibling for n in got):
            bad.append((want, sorted(got)))
    assert not bad, bad
