"""Case list of LpqLoss (lpq_loss_layer.{cpp,cu}), shared by tests/golden/make_lpq_golden.py (runs the REFERENCE's LpqLossLayer,
oracle/_ref, on a GPU -- the reference has no CPU path, lpq_loss_layer.cpp:175-188 -- and writes tests/golden/lpq_golden.npz) and
by the tests that compare the oracle (CPU) and the CUDA kernels (GPU) with those vectors.  Each case has a constant (p, q): the
reference layer runs without a Net, so it stays at its first schedule step.  Inputs are regenerated from the seeds; only the
reference's outputs are stored."""
import numpy as np

from ref_cases import rng_for


def _pair(r, N, C, H, W, nan_blocks=True, zeros=True):
    a = (3 * r.standard_normal((N, C, H, W))).astype(np.float32)
    b = (3 * r.standard_normal((N, C, H, W))).astype(np.float32)
    if nan_blocks:                                   # invalid ground truth: every channel NaN, and single-channel NaNs
        b[0, :, 1:4, 2:7] = np.nan
        b[-1, 0, H - 2, W - 3] = np.nan
        b[-1, C - 1, 2, 3:5] = np.nan
    if zeros:                                        # exact zero differences: one whole location, and single channels
        a[0, :, 5, 5] = b[0, :, 5, 5]
        a[0, 0, 6, 1:4] = b[0, 0, 6, 1:4]
        a[-1, C - 1, 7, 8] = b[-1, C - 1, 7, 8]
    return a, b


def _lpq(name, p, q, N=2, C=2, H=12, W=16, single=False, nan_blocks=True, zeros=True, deviation=False, **kw):
    fields = " ".join("%s: %s" % (k, str(v).lower() if isinstance(v, bool) else v) for k, v in kw.items())
    bots = 'bottom: "a"' if single else 'bottom: "a" bottom: "b"'
    text = 'name: "%s" type: "LpqLoss" %s top: "loss" lpq_loss_param { p: %r q: %r %s }' % (name, bots, p, q, fields)

    def inputs(r):
        a, b = _pair(r, N, C, H, W, nan_blocks=nan_blocks and not single, zeros=zeros)
        if single:
            a = (a - b).astype(np.float32)
            a[0, :, 1:3, 2:5] = np.nan
            a[-1, 0, 4, 4] = np.nan
            return [a]
        return [a, b]
    args = dict(p=p, q=q, p_epsilon=kw.get("p_epsilon", 0.0), q_epsilon=kw.get("q_epsilon", 1e-2),
                l2_prescale_by_channels=kw.get("l2_prescale_by_channels", False),
                normalize_by_num_entries=kw.get("normalize_by_num_entries", False))
    return dict(text=text, inputs=inputs, args=args, top_diff=1.7, deviation=deviation)


LPQ_CASES = {
    "lpq_1_1": _lpq("lpq_1_1", 1.0, 1.0),
    "lpq_2_05": _lpq("lpq_2_05", 2.0, 0.5),                                         # the end-point error with q_epsilon
    "lpq_1_04": _lpq("lpq_1_04", 1.0, 0.4),                                         # the fine-tuning loss
    "lpq_08_04_eps": _lpq("lpq_08_04_eps", 0.8, 0.4, p_epsilon=0.01),               # zero differences away from the kink
    "lpq_2_1": _lpq("lpq_2_1", 2.0, 1.0),
    "lpq_2_2": _lpq("lpq_2_2", 2.0, 2.0),
    "lpq_1_1_q0": _lpq("lpq_1_1_q0", 1.0, 1.0, q_epsilon=0.0),
    "lpq_2_05_prescale": _lpq("lpq_2_05_prescale", 2.0, 0.5, l2_prescale_by_channels=True),
    "lpq_1_04_norm": _lpq("lpq_1_04_norm", 1.0, 0.4, normalize_by_num_entries=True),
    "lpq_single": _lpq("lpq_single", 1.0, 0.4, single=True, normalize_by_num_entries=True),
    "lpq_c3": _lpq("lpq_c3", 0.8, 0.5, C=3, p_epsilon=0.01, q_epsilon=0.001, l2_prescale_by_channels=True),
    # p_epsilon 0 and p not in {1, 2}: the reference's Power backward divides 0 / 0 at the exact-zero differences
    "lpq_kink": _lpq("lpq_kink", 0.8, 0.4, deviation=True),
}


def lpq_inputs(name):
    """-> bottoms of a case, deterministic."""
    return LPQ_CASES[name]["inputs"](rng_for(name))
