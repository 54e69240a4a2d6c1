"""The engine's fused update against the REFERENCE's own SGDUpdate / AdamUpdate kernels (sgd_solver.cu:6-12, adam_solver.cu:6-16),
whose outputs on seeded cases tests/golden/make_solver_ref_golden.py stored in ref_solver_update.npz: within 2 ulp per element
of data, diff and history.  The engine fuses the same multiply-adds the reference's nvcc build does, so in practice the two
agree bit for bit; a failure names the largest distance per array."""
import os

import numpy as np
import pytest

from tests import solver_oracle as SO
from tests.golden import make_solver_ref_golden as G

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_solver_update.npz"))
NET = ('layer { name: "in" type: "Input" top: "x" input_param { shape { dim: 1 dim: 3 dim: 8 dim: 8 } } }\n'
       'layer { name: "a" type: "Convolution" bottom: "x" top: "y" convolution_param { num_output: 16 kernel_size: 3 } }\n'
       'layer { name: "b" type: "Convolution" bottom: "y" top: "z" convolution_param { num_output: 37 kernel_size: 3 } }\n')


def ulps(a, b):
    """Distance in units in the last place between float32 arrays (ordered integer images of the bit patterns)."""
    def key(x):
        i = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(key(a) - key(b))


@pytest.mark.parametrize("case", range(len(G.CASES)))
def test_update_within_2_ulp_of_the_reference_kernels(fn2, case):
    from flownet2_b200 import parallel
    from tests.test_solver_gpu import learnable
    name, text, it = G.CASES[case]
    adam = name.startswith("adam")
    net = fn2.Net(NET, None, fn2.TRAIN)
    net.fill_params(1)
    params = learnable(fn2, net)
    assert sum(n for _, _, n, _ in params) == G.COUNT
    w, g, h, v = G.inputs(100 + case)
    data, grads = parallel.arena_tensor(net), parallel.grad_arena_tensor(net)
    k = 0
    for _, _, n, off in params:                       # the learnable blobs, in order, hold the case's concatenated arrays
        data[off:off + n].copy_(torch.from_numpy(w[k:k + n]))
        grads[off:off + n].copy_(torch.from_numpy(g[k:k + n]))
        k += n
    torch.cuda.synchronize()
    net.params_changed()
    solver = fn2.get_solver(text + "weight_decay: 0\n", net)
    split = lambda a: [a[sum(p[2] for p in params[:i]):][:n] for i, (_, _, n, _) in enumerate(params)]
    hist = split(h) + (split(v) if adam else [])
    solver.restore(SO.write_state(it, 0, "", [([len(x)], x) for x in hist]))
    fn2.check(fn2.lib().fn2_solver_apply_update(solver._h))
    net.sync()
    wa, ga = parallel.arena_tensor(net).cpu().numpy(), parallel.grad_arena_tensor(net).cpu().numpy()
    st = SO.parse_state(solver.state())
    eng = {"diff": np.concatenate([ga[off:off + n] for _, _, n, off in params]),
           "data": np.concatenate([wa[off:off + n] for _, _, n, off in params]),
           "hist": np.concatenate([d for _, d in st["history"][:len(params)]])}
    ref = {"diff": GOLD[name + "_diff"], "hist": GOLD[name + "_hist"]}
    ref["data"] = w - ref["diff"]                     # Net::Update: caffe_gpu_axpy(-1, diff, data), one rounding
    if adam:
        eng["v"] = np.concatenate([d for _, d in st["history"][len(params):]])
        ref["v"] = GOLD[name + "_v"]
    worst = {key: int(ulps(eng[key], ref[key]).max()) for key in ref}
    assert all(u <= 2 for u in worst.values()), worst
    assert np.all(np.isfinite(eng["data"]))
