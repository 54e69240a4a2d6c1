"""Solver fixtures written by the REFERENCE's own caffe_pb2 (python/caffe/proto/caffe_pb2.py), against which the engine's solver
parameters and SolverState bytes are checked:

  ref_pb2_solver.json      solver prototxts, the fields caffe_pb2 reads from each (defaults filled), and the SolverTypeUpgradeTest
                           pairs (src/caffe/test/test_upgrade_proto.cpp:2929-2990) as caffe_pb2 parses both sides
  ref_pb2_solverstate.bin  a SolverState (caffe.proto:247-252) with known iter, current_step, learned_net and history
  ref_pb2_solverstate.json what it holds

Run in the container that has /root/reference:  PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION=python python tests/golden/make_solver_golden.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, "/root/reference/python/caffe/proto")

FIELDS = ["type", "base_lr", "lr_policy", "gamma", "power", "stepsize", "stepvalue", "max_iter", "momentum", "momentum2", "delta",
          "weight_decay", "regularization_type", "clip_gradients", "iter_size", "average_loss", "snapshot", "snapshot_prefix",
          "snapshot_after_train"]

SOLVERS = {
    # the FlowNet2 schedule (Ilg et al. 2017, S_long): Adam, multistep halving, weight decay, snapshots
    "flownet2_adam_multistep": (
        'net: "train.prototxt"\n'
        'base_lr: 1e-4\nlr_policy: "multistep"\ngamma: 0.5\n'
        'stepvalue: 400000\nstepvalue: 600000\nstepvalue: 800000\nstepvalue: 1000000\n'
        'max_iter: 1200000\nmomentum: 0.9\nmomentum2: 0.999\nweight_decay: 0.0004\ntype: "Adam"\n'
        'display: 100\nsnapshot: 20000\nsnapshot_prefix: "flow"\nsolver_mode: GPU\ndevice_id: 0\nrandom_seed: 1\n'),
    "solver_type_adam": (
        'base_lr: 0.001\nlr_policy: "fixed"\nmomentum: 0.9\nmomentum2: 0.999\ndelta: 1e-8\nsolver_type: ADAM\nmax_iter: 100\n'),
    "sgd_step_l1_clip": (
        'train_net: "t.prototxt"\nbase_lr: 0.01\nlr_policy: "step"\ngamma: 0.1\nstepsize: 1000\nmomentum: 0.9\n'
        'weight_decay: 0.0005\nregularization_type: "L1"\nclip_gradients: 10\niter_size: 3\naverage_loss: 20\n'
        'snapshot_after_train: false\n'),
    "sgd_defaults_inv": 'base_lr: 0.01\nlr_policy: "inv"\ngamma: 0.0001\npower: 0.75\n',
    "poly": 'base_lr: 0.02\nlr_policy: "poly"\npower: 2\nmax_iter: 5000\ntype: "SGD"\n',
    "sigmoid": 'base_lr: 0.5\nlr_policy: "sigmoid"\ngamma: -0.01\nstepsize: 300\n',
    "exp": 'base_lr: 0.1\nlr_policy: "exp"\ngamma: 0.999\n',
}


def fields(sp):
    out = {}
    for f in FIELDS:
        v = getattr(sp, f)
        if f == "type" and sp.HasField("solver_type"):
            v = None                                   # set by the upgrade, compared separately
        out[f] = list(v) if f == "stepvalue" else (float(v) if isinstance(v, float) else v)
    return out


def main():
    import caffe_pb2
    from google.protobuf import text_format
    solvers = {}
    for name, text in SOLVERS.items():
        sp = caffe_pb2.SolverParameter()
        text_format.Merge(text, sp)
        solvers[name] = {"text": text, "fields": fields(sp), "solver_type": sp.solver_type if sp.HasField("solver_type") else None}
    # SolverTypeUpgradeTest.TestSimple
    body = ("net: 'examples/mnist/lenet_train_test.prototxt' test_iter: 100 test_interval: 500 base_lr: 0.01 momentum: 0.0 "
            "weight_decay: 0.0005 lr_policy: 'inv' gamma: 0.0001 power: 0.75 display: 100 max_iter: 10000 snapshot: 5000 "
            "snapshot_prefix: 'examples/mnist/lenet_rmsprop' solver_mode: GPU ")
    pairs = []
    for old, new in zip(["SGD", "ADAGRAD", "NESTEROV", "RMSPROP", "ADADELTA", "ADAM"],
                        ["SGD", "AdaGrad", "Nesterov", "RMSProp", "AdaDelta", "Adam"]):
        a, b = caffe_pb2.SolverParameter(), caffe_pb2.SolverParameter()
        text_format.Merge(body + "solver_type: " + old + " ", a)
        text_format.Merge(body + "type: '" + new + "' ", b)
        assert a.solver_type == getattr(caffe_pb2.SolverParameter, old) and b.type == new
        pairs.append({"input": body + "solver_type: " + old + " ", "expected": body + "type: '" + new + "' ", "type": b.type})
    with open(os.path.join(HERE, "ref_pb2_solver.json"), "w") as f:
        json.dump({"solvers": solvers, "upgrade_pairs": pairs}, f, indent=1, sort_keys=True)

    r = np.random.default_rng(2024)
    shapes = [[4, 3, 3, 3], [4], [2, 4, 1, 1], [2]]
    history = [r.standard_normal(int(np.prod(s))).astype(np.float32) for s in shapes * 2]    # Adam: m of each, then v of each
    history[len(shapes):] = [np.abs(h) for h in history[len(shapes):]]
    st = caffe_pb2.SolverState()
    st.iter = 1234
    st.current_step = 2
    st.learned_net = "snap/flow_iter_1234.caffemodel"
    for s, h in zip(shapes * 2, history):
        b = st.history.add()
        b.shape.dim.extend(s)
        b.data.extend(h.tolist())
    with open(os.path.join(HERE, "ref_pb2_solverstate.bin"), "wb") as f:
        f.write(st.SerializeToString())
    with open(os.path.join(HERE, "ref_pb2_solverstate.json"), "w") as f:
        json.dump({"iter": st.iter, "current_step": st.current_step, "learned_net": st.learned_net, "shapes": shapes * 2,
                   "history": [h.tolist() for h in history]}, f)


if __name__ == "__main__":
    main()
