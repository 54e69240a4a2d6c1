"""Float32 restatement of LpqLoss (lpq_loss_layer.cpp:13-138, lpq_loss_layer.cu:96-245) for the tests: the forward and backward
chain step by step, the p/q schedule of LayerSetUp, and LpqOracleNet, an OracleNet that also runs LpqLoss layers.  Pinned by
tests/test_lpqloss_cpu.py against the reference layer's recorded outputs (tests/golden/lpq_golden.npz)."""
import numpy as np

from oracle.net import OracleNet, get, getall


def lpq_schedule(p, q, starts=()):
    """LpqLossLayer::LayerSetUp's schedule (lpq_loss_layer.cpp:19-82) -> [(start_iter, p, q)], raising ValueError with the
    reference's messages: one p and one q without start iterations are constant values; otherwise equal, non-zero sizes,
    strictly increasing start iterations, the first one 0."""
    p, q, starts = list(p), list(q), [int(s) for s in starts]
    if not starts and len(p) == 1 and len(q) == 1:
        return [(0, float(p[0]), float(q[0]))]
    if len(starts) != len(p) or len(p) != len(q):
        raise ValueError("Incompatible sizes: (pq_episode_starts_at_iter -> %d, p -> %d, q -> %d)" % (len(starts), len(p), len(q)))
    if not starts:
        raise ValueError("Lpq schedule parameters must not be empty")
    if any(a >= b for a, b in zip(starts, starts[1:])):
        raise ValueError("pq_episode_starts_at_frame is not ordered or contains duplicates:" + "".join(" %d" % s for s in starts))
    if starts[0] != 0:
        raise ValueError("First entry in pq_episode_starts_at_frame is not 0, this is probably a mistake.")
    return [(s, float(a), float(b)) for s, a, b in zip(starts, p, q)]


def lpq_step(schedule, iteration):
    """(p, q) at `iteration`: the last step whose start_iter <= iteration (the engine's lookup; equal to the reference's pop queue,
    lpq_loss_layer.cu:100-135, while the iteration only grows)."""
    cur = schedule[0]
    for st in schedule:
        if st[0] <= iteration:
            cur = st
    return cur[1], cur[2]


def _power(x, power, shift):
    """PowerLayer::Forward_gpu (power_layer.cu:8-30), scale 1, float32: power 0 -> 1; + shift when shift != 0; pow when power != 1."""
    f = np.float32
    if power == 0:
        return np.ones_like(x)
    t = (x + f(shift)).astype(f) if shift != 0 else x
    return np.power(t, f(power)).astype(f) if power != 1 else t


def _dpower(x, y, power, shift, zero_at_kink):
    """PowerLayer::Backward_gpu (power_layer.cu:32-84) before the product with the top diff: power 0 -> 0, 1 -> 1, 2 -> 2x + 2 shift,
    shift 0 -> power * y / x, else power * y / (x + shift).  zero_at_kink: 0 instead of the reference's 0 / 0 where shift == 0 and
    x == 0 (the engine's rule)."""
    f = np.float32
    if power == 0:
        return np.zeros_like(x)
    if power == 1:
        return np.ones_like(x)
    if power == 2:
        g = (f(2) * x).astype(f)
        return (g + f(2) * f(shift)).astype(f) if shift != 0 else g
    with np.errstate(divide="ignore", invalid="ignore"):
        if shift == 0:
            g = ((y / x).astype(f) * f(power)).astype(f)
            return np.where(x == 0, f(0), g).astype(f) if zero_at_kink else g
        return ((y / (x + f(shift)).astype(f)).astype(f) * f(power)).astype(f)


def _chain(b0, b1, p, q, p_epsilon, q_epsilon, l2_prescale_by_channels, normalize_by_num_entries):
    f = np.float32
    d = np.asarray(b0, f) if b1 is None else (np.asarray(b0, f) - np.asarray(b1, f))     # Eltwise SUM, coeffs 1, -1
    ok = d == d                                                                           # FindNotNaNs
    N, Cc = d.shape[0], d.shape[1]
    norm = f(ok.sum(dtype=np.float64)) / f(Cc) if normalize_by_num_entries else f(N)
    dz = np.where(ok, d, f(0))                                                            # KillMasked
    sign = np.where(dz > 0, f(1), f(-1))                                                  # ComputeSign: 0 -> -1
    a = (dz * sign).astype(f)                                                             # EltwiseMult
    P = _power(a, p, p_epsilon)                                                           # Power(p, shift p_epsilon)
    w = f(1) / f(Cc) if l2_prescale_by_channels else f(1)
    s = np.zeros((N,) + d.shape[2:], f)
    for c in range(Cc):                                                                   # 1x1 sum convolution, weight w
        s = (s + w * P[:, c]).astype(f)
    Qv = _power(s, q, q_epsilon)                                                          # Power(q, shift q_epsilon)
    return ok, norm, sign, a, P, w, s, Qv


def lpqloss_fwd(b0, b1=None, p=1.0, q=1.0, p_epsilon=0.0, q_epsilon=1e-2, l2_prescale_by_channels=False,
                normalize_by_num_entries=False):
    """LpqLossLayer::Forward_gpu (lpq_loss_layer.cu:96-198) at a given (p, q): float32 element operations in the reference's
    order, the dot product accumulated in float64.  -> (loss, normalize_coeff)."""
    f = np.float32
    _, norm, _, _, _, _, _, Qv = _chain(b0, b1, p, q, p_epsilon, q_epsilon, l2_prescale_by_channels, normalize_by_num_entries)
    return f(f(Qv.sum(dtype=np.float64)) / norm), norm


def lpqloss_bwd(b0, b1=None, top_diff=1.0, p=1.0, q=1.0, p_epsilon=0.0, q_epsilon=1e-2, l2_prescale_by_channels=False,
                normalize_by_num_entries=False, zero_at_kink=True):
    """LpqLossLayer::Backward_gpu (lpq_loss_layer.cu:204-245) -> (bottom0 diff, bottom1 diff).  zero_at_kink=False keeps the
    reference's NaN where a zero-shift power is differentiated at 0 (the engine writes 0 there)."""
    f = np.float32
    ok, norm, sign, a, P, w, s, Qv = _chain(b0, b1, p, q, p_epsilon, q_epsilon, l2_prescale_by_channels, normalize_by_num_entries)
    alpha = f(top_diff) / norm
    dq = (alpha * _dpower(s, Qv, q, q_epsilon, zero_at_kink)).astype(f)                  # Power(q) backward
    dp = (w * dq).astype(f)                                                               # sum convolution backward
    g = (dp[:, None] * _dpower(a, P, p, p_epsilon, zero_at_kink)).astype(f)              # Power(p) backward
    g = np.where(ok, (g * sign).astype(f), f(0)).astype(f)                                # sign, then KillMasked
    return g, (-g).astype(f)


def lpq_args(layer, pq=None):
    """lpqloss_fwd / lpqloss_bwd arguments of a parsed LpqLoss layer block, at its first schedule step or at pq = (p, q)."""
    lp = get(layer, "lpq_loss_param", [])
    tf = lambda k: get(lp, k, "false") == "true"
    sched = lpq_schedule([float(v) for v in getall(lp, "p")], [float(v) for v in getall(lp, "q")],
                         [int(v) for v in getall(lp, "pq_episode_starts_at_iter")])
    p, q = pq or sched[0][1:]
    return dict(p=p, q=q, p_epsilon=float(get(lp, "p_epsilon", 0)), q_epsilon=float(get(lp, "q_epsilon", 1e-2)),
                l2_prescale_by_channels=tf("l2_prescale_by_channels"), normalize_by_num_entries=tf("normalize_by_num_entries"))


class LpqOracleNet(OracleNet):
    """OracleNet with LpqLoss layers, forward and backward.  The oracle has no iteration: every LpqLoss layer runs at its first
    schedule step, or at self.lpq_pq = (p, q) when that is set."""
    lpq_pq = None

    def run_layer(self, l, bots):
        if get(l, "type") == "LpqLoss":
            loss, _ = lpqloss_fwd(bots[0], bots[1] if len(bots) > 1 else None, **lpq_args(l, self.lpq_pq))
            return [np.array([loss], np.float32)]
        return super().run_layer(l, bots)

    def backward_layer(self, l, bots, tops, tds, P):
        if get(l, "type") == "LpqLoss":
            g0, g1 = lpqloss_bwd(bots[0], bots[1] if len(bots) > 1 else None, float(np.asarray(tds[0]).reshape(-1)[0]),
                                 **lpq_args(l, self.lpq_pq))
            return [g0, g1][:len(bots)]
        return super().backward_layer(l, bots, tops, tds, P)
