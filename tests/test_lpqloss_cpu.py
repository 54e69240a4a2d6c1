"""CPU: LpqLoss's oracle restatement (tests/lpq_oracle.py: lpqloss_fwd / lpqloss_bwd) against the outputs of the REFERENCE's own LpqLossLayer
(tests/golden/lpq_golden.npz, written on a GPU by tests/golden/make_lpq_golden.py), its gradient against finite differences, the
p/q schedule against the reference's pop queue, and the prototxt parser on the repeated schedule fields.  No GPU needed."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import lpq_cases as LC  # noqa: E402
from tests import lpq_oracle as O  # noqa: E402
from tests.refcheck import TRAIN_TOL  # noqa: E402
from tests.test_host_cpu import canonical  # noqa: E402
from tests.util import maxabs  # noqa: E402

GOLD = os.path.join(HERE, "golden", "lpq_golden.npz")
TOL = TRAIN_TOL["l1loss"]         # the same chain of float32 element operations, cuBLAS orders and powf


@pytest.fixture(scope="module")
def gold():
    if not os.path.exists(GOLD):
        pytest.fail("tests/golden/lpq_golden.npz is missing: run tests/golden/make_lpq_golden.py on a GPU")
    return np.load(GOLD)


def oracle_eval(name, zero_at_kink):
    c = LC.LPQ_CASES[name]
    bots = LC.lpq_inputs(name)
    b1 = bots[1] if len(bots) > 1 else None
    loss, _ = O.lpqloss_fwd(bots[0], b1, **c["args"])
    g0, g1 = O.lpqloss_bwd(bots[0], b1, c["top_diff"], zero_at_kink=zero_at_kink, **c["args"])
    out = {"top0": np.array([loss], np.float32), "bdiff0": g0}
    if b1 is not None:
        out["bdiff1"] = g1
    return out


def kinks(name):
    """Entries where the reference differentiates a zero-shift power at 0: not-NaN exact-zero differences."""
    bots = LC.lpq_inputs(name)
    d = bots[0] - bots[1] if len(bots) > 1 else bots[0]
    return d == 0


@pytest.mark.parametrize("name", list(LC.LPQ_CASES))
def test_oracle_matches_reference(gold, name):
    out = oracle_eval(name, zero_at_kink=False)
    keys = [k[len("L/%s/" % name):] for k in gold.files if k.startswith("L/%s/" % name)]
    assert keys and set(out) == set(keys), (sorted(out), sorted(keys))
    for k in keys:
        want = gold["L/%s/%s" % (name, k)]
        got = np.asarray(out[k]).reshape(want.shape)
        scale = max(float(np.nanmax(np.abs(want))), 1e-6)
        assert maxabs(got, want) <= TOL * scale, (name, k, maxabs(got, want), scale)


def test_reference_is_nan_exactly_at_the_kinks(gold):
    """lpq_kink (p_epsilon 0, p = 0.8): the reference's gradient is NaN at the exact-zero differences and finite elsewhere; the
    oracle with the engine's rule writes 0 there and agrees everywhere else."""
    k = kinks("lpq_kink")
    assert k.sum() >= 5
    mine = oracle_eval("lpq_kink", zero_at_kink=True)
    for i in (0, 1):
        want = gold["L/lpq_kink/bdiff%d" % i]
        assert np.array_equal(np.isnan(want), k)
        assert np.all(mine["bdiff%d" % i][k] == 0)
        scale = float(np.nanmax(np.abs(want)))
        assert maxabs(np.where(k, 0, mine["bdiff%d" % i]), np.where(k, 0, want)) <= TOL * scale
    for name in LC.LPQ_CASES:                        # no other case reaches the deviation
        if name != "lpq_kink":
            assert not np.isnan(gold["L/%s/bdiff0" % name]).any(), name


@pytest.mark.parametrize("p,q,pe,qe,prescale", [(1.0, 0.4, 0.0, 0.01, False), (2.0, 0.5, 0.0, 0.01, True),
                                                 (0.8, 0.4, 0.01, 0.01, False), (1.3, 1.7, 0.0, 0.001, False)])
def test_gradient_is_the_derivative_of_the_loss(p, q, pe, qe, prescale):
    """Central differences of the forward in float64 against the backward, away from the kinks (no zero differences)."""
    r = np.random.default_rng(7)
    a = r.uniform(0.3, 2.0, (1, 2, 3, 4)) * r.choice([-1.0, 1.0], (1, 2, 3, 4))
    b = np.zeros_like(a)
    b[0, :, 0, 0] = np.nan
    kw = dict(p=p, q=q, p_epsilon=pe, q_epsilon=qe, l2_prescale_by_channels=prescale)
    g0, g1 = O.lpqloss_bwd(a.astype(np.float32), b.astype(np.float32), 1.5, **kw)
    assert np.array_equal(g1, -g0) and np.all(g0[0, :, 0, 0] == 0)
    eps = 1e-2
    for idx in [(0, 0, 1, 2), (0, 1, 2, 3), (0, 0, 2, 0), (0, 1, 0, 1)]:
        ap, am = a.copy(), a.copy()
        ap[idx] += eps
        am[idx] -= eps
        fwd = lambda x: float(O.lpqloss_fwd(x.astype(np.float32), b.astype(np.float32), **kw)[0])
        fd = 1.5 * (fwd(ap) - fwd(am)) / (2 * eps)
        assert abs(fd - float(g0[idx])) <= 2e-3 * max(1.0, abs(fd)), (idx, fd, float(g0[idx]))


def pop_queue(schedule, iterations):
    """LpqLossLayer's own schedule (lpq_loss_layer.cpp:84-136 pops the first step at setup; .cu:100-135 pops every step whose
    start_iter <= the current iteration before each forward) -> (p, q) per forward, iterations visited in order."""
    queue = list(schedule)
    p, q = queue.pop(0)[1:]
    out = []
    for it in iterations:
        step = None
        while queue and it >= queue[0][0]:
            step = queue.pop(0)
        if step:
            p, q = step[1:]
        out.append((p, q))
    return out


def test_schedule_lookup_equals_the_pop_queue():
    sched = O.lpq_schedule([1.0, 2.0, 2.0, 0.5], [1.0, 1.0, 2.0, 0.4], [0, 3, 10, 11])
    its = list(range(0, 16))
    assert [O.lpq_step(sched, i) for i in its] == pop_queue(sched, its)
    for start, p, q in sched:                        # at and around every boundary
        assert O.lpq_step(sched, start) == (p, q)
        assert O.lpq_step(sched, start + 1) == (p, q) or start + 1 in (s for s, _, _ in sched)
    assert O.lpq_step(sched, 2) == (1.0, 1.0) and O.lpq_step(sched, 9) == (2.0, 1.0) and O.lpq_step(sched, 10 ** 6) == (0.5, 0.4)
    # iterations that skip boundaries (iter_size, or a resumed run) still land on the last step that started
    its = [0, 2, 5, 12]
    assert [O.lpq_step(sched, i) for i in its] == pop_queue(sched, its) == [(1.0, 1.0), (1.0, 1.0), (2.0, 1.0), (0.5, 0.4)]
    assert O.lpq_schedule([0.8], [0.4]) == [(0, 0.8, 0.4)]                  # constant values need no start iteration


@pytest.mark.parametrize("p,q,starts,msg", [
    ([1, 2], [1, 2], [0], r"Incompatible sizes: \(pq_episode_starts_at_iter -> 1, p -> 2, q -> 2\)"),
    ([], [], [], "Lpq schedule parameters must not be empty"),
    ([1, 2, 3], [1, 1, 1], [0, 5, 5], "pq_episode_starts_at_frame is not ordered or contains duplicates: 0 5 5"),
    ([1, 2], [1, 1], [1, 5], "First entry in pq_episode_starts_at_frame is not 0, this is probably a mistake."),
])
def test_schedule_checks(p, q, starts, msg):
    with pytest.raises(ValueError, match=msg):
        O.lpq_schedule(p, q, starts)


def test_parser_reads_the_repeated_schedule_fields(fn2):
    text = ('layer { name: "l" type: "LpqLoss" bottom: "a" bottom: "b" top: "loss" lpq_loss_param { '
            'pq_episode_starts_at_iter: 0 pq_episode_starts_at_iter: 3000 p: 1 p: 2 q: [0.4, 1] p_epsilon: 0.01 q_epsilon: 0.001 '
            'normalize_by_num_entries: true } }')
    lines = [l.strip() for l in canonical(fn2, text).splitlines()]
    i = lines.index("lpq_loss_param {")
    assert lines[i + 1:i + 10] == ["pq_episode_starts_at_iter: 0", "pq_episode_starts_at_iter: 3000", "p: 1", "p: 2", "q: 0.4",
                                   "q: 1", "p_epsilon: 0.01", "q_epsilon: 0.001", "normalize_by_num_entries: true"]
    from oracle.net import parse_prototxt, get, getall
    lp = get(get(parse_prototxt(text), "layer"), "lpq_loss_param")
    sched = O.lpq_schedule([float(v) for v in getall(lp, "p")], [float(v) for v in getall(lp, "q")],
                           [int(v) for v in getall(lp, "pq_episode_starts_at_iter")])
    assert sched == [(0, 1.0, 0.4), (3000, 2.0, 1.0)]
