"""Solver parameters, the learning-rate schedule and the solver's C-ABI, without a GPU.

The parameter fixtures were written by the reference's own caffe_pb2 (tests/golden/make_solver_golden.py); the schedule is
compared with the restatement in tests/solver_oracle.py."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

from tests import solver_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
with open(os.path.join(GOLD, "ref_pb2_solver.json")) as _f:
    FIX = json.load(_f)
UPGRADED = {0: "SGD", 1: "Nesterov", 2: "AdaGrad", 3: "RMSProp", 4: "AdaDelta", 5: "Adam"}


@pytest.mark.parametrize("name", sorted(FIX["solvers"]))
def test_resolved_parameters_match_caffe_pb2(fn2, name):
    case = FIX["solvers"][name]
    got = fn2.solver_params(case["text"])
    want = dict(case["fields"])
    if case["solver_type"] is not None:
        want["type"] = UPGRADED[case["solver_type"]]
    assert sorted(got) == sorted(want)
    for k, v in want.items():
        if isinstance(v, float):
            assert np.float32(got[k]) == np.float32(v), (k, got[k], v)
        else:
            assert got[k] == v, (k, got[k], v)


@pytest.mark.parametrize("i", range(6))
def test_solver_type_upgrade_pairs(fn2, i):
    """SolverTypeUpgradeTest.TestSimple (test_upgrade_proto.cpp:2929-2990): the upgraded input reads like the expected output."""
    pair = FIX["upgrade_pairs"][i]
    got, want = fn2.solver_params(pair["input"]), fn2.solver_params(pair["expected"])
    assert got == want and got["type"] == pair["type"]


def test_solver_type_and_type_together_are_refused(fn2):
    with pytest.raises(fn2.Fn2Error, match="old solver_type field .enum. and new type field .string. cannot be both specified"):
        fn2.solver_params('type: "Adam"\nsolver_type: ADAM\n')


OK = 'base_lr: 0.01\nlr_policy: "fixed"\n'
REFUSED = [
    ('type: "Nesterov"\n', "type: solver type Nesterov is not supported"),
    ('solver_type: ADAGRAD\n', "type: solver type AdaGrad is not supported"),
    ('type: "RMSProp"\n', "type: solver type RMSProp is not supported"),
    ('type: "AdaDelta"\n', "type: solver type AdaDelta is not supported"),
    ('test_iter: 100\n', "test_iter: test nets are not supported"),
    ('test_net: "t.prototxt"\n', "test_net: test nets are not supported"),
    ('test_interval: 500\n', "test_interval: test nets are not supported"),
    ('snapshot_format: HDF5\n', "snapshot_format: HDF5 snapshots are not supported"),
    ('snapshot_diff: true\n', "snapshot_diff: diff snapshots are not supported"),
    ('solver_mode: CPU\n', "solver_mode: CPU is not supported"),
    ('regularization_type: "L3"\n', "Unknown regularization type: L3"),
    ('train_state { phase: TRAIN }\n', "train_state is not supported"),
]


@pytest.mark.parametrize("extra,message", REFUSED)
def test_refused_fields_name_themselves(fn2, extra, message):
    with pytest.raises(fn2.Fn2Error, match=re.escape(message)):
        fn2.learning_rate(OK + extra, 0)


def test_unknown_policy_uses_the_reference_message(fn2):
    with pytest.raises(fn2.Fn2Error, match="Unknown learning rate policy: cosine"):
        fn2.learning_rate('base_lr: 0.1\nlr_policy: "cosine"\n', 0)


def test_accepted_fields_have_no_effect(fn2):
    extra = ('net: "n.prototxt"\ntrain_net: "t.prototxt"\ndisplay: 20\ndebug_info: true\nsolver_mode: GPU\ndevice_id: 3\n'
             'random_seed: 7\ntest_interval: 0\nsnapshot_format: BINARYPROTO\nsnapshot_diff: false\n')
    assert fn2.learning_rate(OK + extra, 5) == fn2.learning_rate(OK, 5)


SCHEDULES = {
    "fixed": 'base_lr: 0.01\nlr_policy: "fixed"\n',
    "step": 'base_lr: 0.01\nlr_policy: "step"\ngamma: 0.1\nstepsize: 7\n',
    "exp": 'base_lr: 0.1\nlr_policy: "exp"\ngamma: 0.999\n',
    "inv": 'base_lr: 0.01\nlr_policy: "inv"\ngamma: 0.0001\npower: 0.75\n',
    "multistep": 'base_lr: 1e-4\nlr_policy: "multistep"\ngamma: 0.5\nstepvalue: 3\nstepvalue: 10\nstepvalue: 11\nstepvalue: 30\n',
    "poly": 'base_lr: 0.02\nlr_policy: "poly"\npower: 2\nmax_iter: 50\n',
    "sigmoid": 'base_lr: 0.5\nlr_policy: "sigmoid"\ngamma: -0.3\nstepsize: 20\n',
}


@pytest.mark.parametrize("policy", sorted(SCHEDULES))
def test_learning_rate_equals_the_restatement(fn2, policy):
    text = SCHEDULES[policy]
    p = fn2.solver_params(text)
    cs_engine = cs_oracle = 0
    for it in range(60):
        rate, cs_engine = fn2.learning_rate(text, it, cs_engine)
        want, cs_oracle = SO.learning_rate(p, it, cs_oracle)
        assert np.float32(rate).tobytes() == want.tobytes() and cs_engine == cs_oracle, (it, rate, want, cs_engine, cs_oracle)


def test_multistep_resumed_past_two_steps(fn2):
    """A solver restored at iteration 12 with current_step 0 catches up one step per iteration, as the reference's does."""
    text = SCHEDULES["multistep"]
    p = fn2.solver_params(text)
    cs, seen = 0, []
    for it in range(12, 16):
        rate, cs = fn2.learning_rate(text, it, cs)
        want, _ = SO.learning_rate(p, it, len(seen))
        seen.append(cs)
        assert np.float32(rate) == want
    assert seen == [1, 2, 3, 3]
    # resumed with the current_step the state recorded: no catching up
    rate, cs = fn2.learning_rate(text, 12, 3)
    assert cs == 3 and np.float32(rate) == np.float32(1e-4 * 0.5 ** 3)


def test_flownet2_schedule(fn2):
    text = FIX["solvers"]["flownet2_adam_multistep"]["text"]
    cs, rates = 0, {}
    for it in (0, 399999, 400000, 600000, 800000, 1000000):
        if it == 400000:
            cs = 0
        rates[it], cs = fn2.learning_rate(text, it, cs)
    assert rates[0] == rates[399999] == np.float32(1e-4)
    assert rates[400000] == np.float32(float(np.float32(1e-4)) * 0.5)


def _header_arity(name):
    text = re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", name)).read(), flags=re.S)
    return {n: (" ".join(r.split()), 0 if a.strip() == "void" else a.count(",") + 1)
            for r, n, a in re.findall(r"FN2_API\s+([\w\s\*]+?)\s*\b(fn2_\w+)\s*\(([^)]*)\)", text)}


def test_every_solver_declaration_has_a_prototype(fn2):
    lib = fn2.lib()
    arity = _header_arity("fn2_solver.h")
    assert len(arity) == 10 and not set(arity) & set(_header_arity("fn2.h"))
    restypes = {"int": C.c_int, "void": None}
    for name, (ret, n) in arity.items():
        f = getattr(lib, name)
        assert f.argtypes is not None and len(f.argtypes) == n and f.restype is restypes[ret], name
    assert lib.fn2_solver_create.argtypes[2] is C.POINTER(C.c_void_p)
    assert lib.fn2_solver_learning_rate.argtypes[2] is C.POINTER(C.c_int)
    assert lib.fn2_solver_learning_rate.argtypes[3] is C.c_void_p          # float* is a data pointer
    assert lib.fn2_solver_destroy.restype is None


def test_solver_null_arguments(fn2):
    lib = fn2.lib()
    n, it, cs = C.c_size_t(), C.c_int(), C.c_int()
    h = C.c_void_p()
    assert lib.fn2_solver_create(OK.encode(), None, C.byref(h)) == -1
    assert lib.fn2_last_error().decode() == "solver_create: null argument"
    assert lib.fn2_solver_apply_update(None) == -1 and lib.fn2_solver_iter(None, C.byref(it), C.byref(cs)) == -1
    assert lib.fn2_solver_state(None, b"", None, C.byref(n)) == -1
    lib.fn2_solver_destroy(None)


def test_solverstate_fixture_reads(fn2):
    raw = open(os.path.join(GOLD, "ref_pb2_solverstate.bin"), "rb").read()
    meta = json.load(open(os.path.join(GOLD, "ref_pb2_solverstate.json")))
    buf = (C.c_char * len(raw)).from_buffer_copy(raw)
    assert fn2.sized_output(fn2.lib().fn2_solverstate_learned_net, buf, len(raw))[:-1].decode() == meta["learned_net"]
    st = SO.parse_state(raw)
    assert st["iter"] == meta["iter"] and st["current_step"] == meta["current_step"]
    assert [s for s, _ in st["history"]] == meta["shapes"]
    for (_, h), want in zip(st["history"], meta["history"]):
        assert np.array_equal(h, np.asarray(want, np.float32))
    # the test's own writer produces what caffe_pb2 wrote
    assert SO.write_state(st["iter"], st["current_step"], st["learned_net"], st["history"]) == raw


def test_float_policies_use_the_float_functions(fn2):
    """inv, poly and sigmoid call pow(float, float) / exp(float), which resolve to the float functions in the reference build
    (<math.h> is in scope through mkl_alternate.hpp): the rate is powf / expf of float arguments, not a double evaluation."""
    import math
    for policy in ("inv", "poly", "sigmoid"):
        text = SCHEDULES[policy] if policy != "inv" else FIX["solvers"]["sgd_defaults_inv"]["text"]
        p = fn2.solver_params(text)
        differs = 0
        for it in {"inv": range(0, 3000, 7), "poly": range(0, 51), "sigmoid": range(0, 150)}[policy]:
            rate, _ = fn2.learning_rate(text, it, 0)
            want, _ = SO.learning_rate(p, it, 0)
            assert np.float32(rate) == want, (policy, it)
            base, gamma, power = (float(np.float32(p[k])) for k in ("base_lr", "gamma", "power"))
            if policy == "inv":
                dbl = base * math.pow(float(np.float32(1) + np.float32(gamma) * np.float32(it)), -power)
            elif policy == "poly":
                dbl = base * math.pow(float(np.float32(1) - np.float32(it) / np.float32(p["max_iter"])), power)
            else:
                dbl = base * (1.0 / (1.0 + math.exp(float(-np.float32(gamma) * (np.float32(it) - np.float32(p["stepsize"]))))))
            differs += np.float32(dbl) != np.float32(rate)
        assert policy == "poly" or differs > 0, policy


def test_restatement_equals_the_reference_update_kernels(fn2):
    """tests/solver_oracle.update, which the engine's update equals bit for bit, reproduces the outputs of the reference's own
    SGDUpdate / AdamUpdate kernels (tests/golden/ref_solver_update.npz) bit for bit."""
    from tests.golden import make_solver_ref_golden as G
    gold = np.load(os.path.join(GOLD, "ref_solver_update.npz"))
    for k, (name, text, it) in enumerate(G.CASES):
        w, g, h, v = G.inputs(100 + k)
        p = fn2.solver_params(text + "weight_decay: 0\n")
        rate, _ = SO.learning_rate(p, it, 0)
        _, diff, hist, v1 = SO.update(p, rate, it, w, g, h, v if p["type"] == "Adam" else None, 1, 1)
        assert diff.tobytes() == gold[name + "_diff"].tobytes() and hist.tobytes() == gold[name + "_hist"].tobytes(), name
        if v1 is not None:
            assert v1.tobytes() == gold[name + "_v"].tobytes(), name
