"""End-to-end flow error of the engine vs the float64-accumulating oracle (same prototxt, same weights).
Usage: [FN2_CONV_ENGINE=simt] python tools/net_err.py [model] [width] [height]
FN2_CONV_ENGINE=simt runs every convolution on the exact-FP32 SIMT engine instead of the tensor cores."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import flownet2_b200 as fn2
from oracle.net import OracleNet
from tests.util import maxabs, rng, smooth_images
model = sys.argv[1] if len(sys.argv) > 1 else "FlowNet2"
w = int(sys.argv[2]) if len(sys.argv) > 2 else 256
h = int(sys.argv[3]) if len(sys.argv) > 3 else 128
proto = fn2.fill_template(fn2.model_template(model), w, h)
cache = "/tmp/net_err_%s_%d_%d.npz" % (model, w, h)
net = fn2.Net(proto, None, fn2.TEST, batch=1)
net.fill_params(1701)
img0, img1 = smooth_images(rng(1701), 1, h, w)
got = net.forward(img0=img0, img1=img1)["predict_flow_final"].copy()
if os.path.exists(cache):
    want = np.load(cache)["want"]
else:
    t = time.time()
    want = OracleNet(proto, net.to_caffemodel(), batch=1, f64acc=True).forward(img0=img0, img1=img1)["predict_flow_final"]
    np.savez(cache, want=want)
    print("oracle %.1f s" % (time.time() - t))
print("conv engine %s, %s %dx%d: flow max-abs err %.3e  (|flow| max %.2f, mean abs err %.3e)" % (
    os.environ.get("FN2_CONV_ENGINE", "default"), model, w, h, maxabs(got, want), np.abs(want).max(),
    float(np.abs(got - want).mean())), flush=True)
