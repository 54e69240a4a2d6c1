"""flownet2_b200 -- Hopper-native FlowNet2 forward path.

Python here is only a ctypes front end over the C-ABI in include/fn2.h, fn2_solver.h, fn2_frames.h, fn2_flow.h, fn2_lpq.h and
fn2_eval.h (libfn2.so: hand-written sm_90a CUDA + the Caffe-surface C++ host).  It mirrors the slice of pycaffe that the reference's
driver uses (scripts/run-flownet.py:64-98): ``Net(prototxt, weights, phase)``, ``net.inputs``,
``net.forward(img0=..., img1=...)``, ``net.blobs[name].data``.

There is NO CPU fallback: importing works anywhere (so the CPU test-suite can check symbols), but
any compute call without the built library or without a GPU raises.
"""
import ctypes as C
import math
import os

import numpy as np

from ._abi import read_defines, read_header

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
TRAIN, TEST = 0, 1

_STRUCTS, _PROTOTYPES, _DEFINES = {}, {}, {}
for _name in ("fn2.h", "fn2_solver.h", "fn2_frames.h", "fn2_flow.h", "fn2_lpq.h", "fn2_eval.h"):
    with open(os.path.join(os.path.dirname(_HERE), "include", _name)) as _f:
        _text = _f.read()
    _s, _p = read_header(_text, _STRUCTS)
    _STRUCTS.update(_s)
    _PROTOTYPES.update(_p)
    _DEFINES.update(read_defines(_text))
fn2_tensor, fn2_conv_desc, fn2_l1loss_desc, fn2_lpqloss_desc = (_STRUCTS[n] for n in ("fn2_tensor", "fn2_conv_desc", "fn2_l1loss_desc",
                                                                                     "fn2_lpqloss_desc"))
LPQLOSS_STATE_FLOATS = _DEFINES["FN2_LPQLOSS_STATE_FLOATS"]            # device floats of an LpqLoss state (include/fn2_lpq.h)
# flow payload formats and flags of fn2_flow_to_tensor (include/fn2_flow.h)
FLOW_FLO, FLOW_PFM, FLOW_PFM_BE, FLOW_KITTI, FLOW_UINT16FLOW = (_DEFINES[n] for n in (
    "FN2_FLOW_FLO", "FN2_FLOW_PFM", "FN2_FLOW_PFM_BE", "FN2_FLOW_KITTI", "FN2_FLOW_UINT16FLOW"))
# the per-pair record of fn2_flow_error (include/fn2_eval.h): its field names, lower case, in record order
FLOW_ERROR_FIELDS = tuple(sorted((k[len("FN2_FLOW_ERROR_"):].lower() for k in _DEFINES
                                 if k.startswith("FN2_FLOW_ERROR_") and k != "FN2_FLOW_ERROR_FIELDS"),
                                key=lambda f: _DEFINES["FN2_FLOW_ERROR_" + f.upper()]))
assert len(FLOW_ERROR_FIELDS) == _DEFINES["FN2_FLOW_ERROR_FIELDS"]
# the per-pair record of fn2_flow_error_regions, the same way; and fn2_occlusion_boundary_dist2's value for a pair without boundary
FLOW_REGION_FIELDS = tuple(sorted((k[len("FN2_FLOW_REGION_"):].lower() for k in _DEFINES
                                  if k.startswith("FN2_FLOW_REGION_") and k != "FN2_FLOW_REGION_FIELDS"),
                                 key=lambda f: _DEFINES["FN2_FLOW_REGION_" + f.upper()]))
assert len(FLOW_REGION_FIELDS) == _DEFINES["FN2_FLOW_REGION_FIELDS"]
# the per-pair record of fn2_mask_confusion, the same way
MASK_CONFUSION_FIELDS = tuple(sorted((k[len("FN2_MASK_CONFUSION_"):].lower() for k in _DEFINES
                                     if k.startswith("FN2_MASK_CONFUSION_") and k != "FN2_MASK_CONFUSION_FIELDS"),
                                    key=lambda f: _DEFINES["FN2_MASK_CONFUSION_" + f.upper()]))
assert len(MASK_CONFUSION_FIELDS) == _DEFINES["FN2_MASK_CONFUSION_FIELDS"]
DIST2_NONE = _DEFINES["FN2_DIST2_NONE"]


class Fn2Error(RuntimeError):
    pass


def lib_path():
    return os.environ.get("FN2_LIB") or os.path.join(_HERE, "libfn2.so")      # FN2_LIB: A/B a differently built library


def lib():
    """Load libfn2.so (built in-tree by flownet2_b200.build).  Fails loudly if it is missing."""
    global _LIB
    if _LIB is None:
        p = lib_path()
        if not os.path.exists(p):
            raise Fn2Error("libfn2.so is not built (%s); run `python -m flownet2_b200.build` -- there is no "
                           "CPU/PyTorch fallback" % p)
        l = C.CDLL(p)
        for name, (restype, argtypes) in _PROTOTYPES.items():
            f = getattr(l, name)
            f.restype, f.argtypes = restype, argtypes
        _LIB = l
    return _LIB


def check(rc):
    if rc != 0:
        raise Fn2Error("fn2 error %d: %s" % (rc, lib().fn2_last_error().decode("utf-8", "replace")))


def sized_output(fn, *args):
    """The size-query convention: fn(*args, NULL, &bytes) reports the size, fn(*args, buf, &bytes) fills buf -> its bytes
    (a text output's bytes include the terminating NUL)."""
    n = C.c_size_t(0)
    check(fn(*args, None, C.byref(n)))
    buf = C.create_string_buffer(n.value)
    check(fn(*args, buf, C.byref(n)))
    return buf.raw[:n.value]


def out_span(fn, *args):
    """fn(*args, &dev_ptr, &bytes) -> (dev_ptr, bytes): the parameter and gradient arenas."""
    p, n = C.c_void_p(), C.c_size_t()
    check(fn(*args, C.byref(p), C.byref(n)))
    return p.value, n.value


def launch_count():
    return int(lib().fn2_launch_count())


def device_allocations():
    """(allocations made so far, bytes held now) by the net host's device and pinned-host buffers."""
    live = C.c_uint64()
    n = lib().fn2_device_allocations(C.byref(live))
    return int(n), int(live.value)


def _read_text(text_or_path):
    """A prototxt given as text or as a path -> its text."""
    if "\n" not in text_or_path and os.path.exists(text_or_path):
        with open(text_or_path) as f:
            return f.read()
    return text_or_path


# ------------------------------------------------------------------------------------------------
# Template handling of scripts/run-flownet.py:39-60
# ------------------------------------------------------------------------------------------------
def template_vars(width, height, divisor=64.0):
    v = {"TARGET_WIDTH": width, "TARGET_HEIGHT": height}
    v["ADAPTED_WIDTH"] = int(math.ceil(width / divisor) * divisor)
    v["ADAPTED_HEIGHT"] = int(math.ceil(height / divisor) * divisor)
    v["SCALE_WIDTH"] = width / float(v["ADAPTED_WIDTH"])
    v["SCALE_HEIGHT"] = height / float(v["ADAPTED_HEIGHT"])
    return v


def fill_template(text, width, height):
    for key, value in template_vars(width, height).items():
        text = text.replace("$%s$" % key, str(value))
    return text


def train_template(name="FlowNet2-C"):
    """Text of models/<name>_train.prototxt.template: the authored training graphs of the FlowNet2 schedule, FlowNet2-C
    (BASELINE config 5), FlowNet2-CS, FlowNet2-CSS, FlowNet2-SD and FlowNet2 (the fusion stage)."""
    p = os.path.join(os.path.dirname(_HERE), "models", "%s_train.prototxt.template" % name)
    with open(p) as f:
        return f.read()


def fill_train_template(text, crop_width, crop_height, data_width, data_height, batch):
    """Training template variables: $TARGET_*$ = the augmentation crop (network input), $DATA_*$ = the frames read, $BATCH$."""
    for key, value in (("TARGET_WIDTH", crop_width), ("TARGET_HEIGHT", crop_height), ("DATA_WIDTH", data_width),
                       ("DATA_HEIGHT", data_height), ("BATCH", batch)):
        text = text.replace("$%s$" % key, str(value))
    return text


def model_template(name):
    """Text of models/<name>_deploy.prototxt.template (FlowNet2, FlowNet2-C, -S, -CS, -CSS, -SD)."""
    p = os.path.join(os.path.dirname(_HERE), "models", "%s_deploy.prototxt.template" % name)
    with open(p) as f:
        return f.read()


# ------------------------------------------------------------------------------------------------
# Net (pycaffe-like)
# ------------------------------------------------------------------------------------------------
class _BlobView(object):
    def __init__(self, net, name):
        self._net, self._name = net, name

    @property
    def shape(self):
        s = (C.c_int * 4)()
        check(lib().fn2_net_blob_shape(self._net._h, self._name.encode(), s))
        return tuple(s)

    @property
    def data(self):
        out = np.empty(self.shape, np.float32)
        check(lib().fn2_net_get_blob(self._net._h, self._name.encode(), out.ctypes.data_as(C.c_void_p)))
        return out


class _Blobs(object):
    def __init__(self, net):
        self._net = net

    def __getitem__(self, name):
        if name not in self._net.blob_names:
            raise KeyError(name)
        return _BlobView(self._net, name)

    def __iter__(self):
        return iter(self._net.blob_names)

    def __contains__(self, name):
        return name in self._net.blob_names


class Net(object):
    """caffe.Net(prototxt, weights, phase) look-alike (python/caffe/pycaffe.py:78-124).

    prototxt: path or text (``$VARS$`` already substituted, see fill_template).  weights: path or
    bytes of a .caffemodel, or None (then call fill_params for synthetic weights).  batch > 0
    overrides dim 0 of the Input shapes.
    """

    def __init__(self, prototxt, weights=None, phase=TEST, batch=0):
        l = lib()
        prototxt = _read_text(prototxt)
        h = C.c_void_p()
        check(l.fn2_net_create_batch(prototxt.encode(), int(phase), int(batch), C.byref(h)))
        self._h = h
        self.inputs = [l.fn2_net_input_name(h, i).decode() for i in range(l.fn2_net_num_inputs(h))]
        self.outputs = [l.fn2_net_output_name(h, i).decode() for i in range(l.fn2_net_num_outputs(h))]
        self.blob_names = [l.fn2_net_blob_name(h, i).decode() for i in range(l.fn2_net_num_blobs(h))]
        self.layer_names = [l.fn2_net_layer_name(h, i).decode() for i in range(l.fn2_net_num_layers(h))]
        self.layer_types = [l.fn2_net_layer_type(h, i).decode() for i in range(l.fn2_net_num_layers(h))]
        self.blobs = _Blobs(self)
        if weights is not None:
            self.copy_from(weights)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().fn2_net_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def copy_from(self, weights, prefix=""):
        """Load a .caffemodel (path or bytes).  Source layer X fills layer prefix + X; source layers with no target are ignored
        (the FlowNet2 stage hand-over: FlowNet2-C_train into FlowNet2-CS_train with prefix="net1_")."""
        if isinstance(weights, str):
            with open(weights, "rb") as f:
                weights = f.read()
        buf = (C.c_char * len(weights)).from_buffer_copy(weights)
        check(lib().fn2_net_copy_trained_layers_prefixed(self._h, buf, len(weights), prefix.encode()))

    def fill_params(self, seed=1701):
        check(lib().fn2_net_fill_params(self._h, int(seed)))

    def to_caffemodel(self):
        return sized_output(lib().fn2_net_to_caffemodel, self._h)

    def param_layers(self):
        """The layers that hold parameter blobs, in net order -> [(name, type, flags, blob shapes, lr_mults)]: flags "c" when
        the layer takes its blobs through its own copy (DataAugmentation, adjusted to this net's crop), "t" when the template
        alone defines its weights (a diagonal filler), "" otherwise (include/fn2_eval.h fn2_net_param_layers)."""
        out = []
        for line in sized_output(lib().fn2_net_param_layers, self._h)[:-1].decode().splitlines():
            name, typ, flags, shapes, mults = line.split("\t")
            out.append((name, typ, flags.strip("-"), [tuple(int(d) for d in s.split("x")) for s in shapes.split(",")],
                        [float(m) for m in mults.split(",")]))
        return out

    def to_hdf5(self):
        """Net::ToHDF5 (net.cpp:905-960): the weights as the bytes of a .caffemodel.h5 file."""
        return sized_output(lib().fn2_net_to_hdf5, self._h)

    def param_arena(self):
        return out_span(lib().fn2_net_param_arena, self._h)

    def params_changed(self):
        check(lib().fn2_net_params_changed(self._h))

    def set_input(self, name, array):
        a = np.ascontiguousarray(array, dtype=np.float32)
        if tuple(a.shape) != self.blobs[name].shape:
            raise Fn2Error("input %s has shape %s, net expects %s" % (name, a.shape, self.blobs[name].shape))
        self._keep = getattr(self, "_keep", {})
        self._keep[name] = a       # must outlive the async H2D copy
        check(lib().fn2_net_set_input(self._h, name.encode(), a.ctypes.data_as(C.c_void_p)))

    def set_input_ptr(self, name, host_ptr):
        """host_ptr: address of a (pinned) float32 NCHW buffer of the blob's size."""
        check(lib().fn2_net_set_input(self._h, name.encode(), C.c_void_p(host_ptr)))

    def set_input_device(self, name, dev_ptr):
        check(lib().fn2_net_set_input_device(self._h, name.encode(), C.c_void_p(dev_ptr)))

    def get_blob_ptr(self, name, host_ptr):
        check(lib().fn2_net_get_blob(self._h, name.encode(), C.c_void_p(host_ptr)))

    def get_blob_device(self, name, dev_ptr):
        check(lib().fn2_net_get_blob_device(self._h, name.encode(), C.c_void_p(dev_ptr)))

    def set_input_image(self, name, frames):
        """8-bit frames -> input blob (N, 3, H, W) as BGR floats, converted on the device (include/fn2_frames.h).  frames: uint8
        (N, H, W, K) with K = 1 (gray), 3 (RGB) or 4 (RGBA, alpha ignored), or (H, W, K) / (H, W) for N = 1.  The blob equals
        set_input of image_to_blob(frame) (a gray frame broadcast to the three channels)."""
        a = np.asarray(frames)
        if a.dtype != np.uint8:
            raise Fn2Error("input %s: frames must be uint8, got %s" % (name, a.dtype))
        a = a[np.newaxis, :, :, np.newaxis] if a.ndim == 2 else a[np.newaxis] if a.ndim == 3 else a
        n, c, h, w = self.blobs[name].shape
        if a.ndim != 4 or a.shape[:3] != (n, h, w):
            raise Fn2Error("input %s: frames of shape %s, net expects (%d, %d, %d, K)" % (name, np.shape(frames), n, h, w))
        a = np.ascontiguousarray(a)
        self._keep = getattr(self, "_keep", {})
        self._keep[name] = a       # must outlive the async H2D copy
        check(lib().fn2_net_set_input_frames(self._h, name.encode(), a.ctypes.data_as(C.c_void_p), a.shape[3]))

    def set_input_image_device(self, name, dev_ptr, channels):
        """dev_ptr: device address of dense uint8 frames (N, H, W, channels) for the (N, 3, H, W) input blob `name`."""
        check(lib().fn2_net_set_input_frames_device(self._h, name.encode(), C.c_void_p(dev_ptr), int(channels)))

    def set_input_flow_device(self, name, dev_ptr, format, flags=0):
        """dev_ptr: device address of the payloads of N flow files (FLOW_FLO, FLOW_PFM or FLOW_PFM_BE, 4-byte aligned; FLOW_KITTI,
        2-byte aligned) for the (N, 2, H, W) input blob `name`; flags FLOW_UINT16FLOW quantises as the reference's training data
        (include/fn2_flow.h)."""
        check(lib().fn2_net_set_input_flow_device(self._h, name.encode(), C.c_void_p(dev_ptr), int(format), int(flags)))

    def get_blob_nhwc(self, name):
        """The blob as an (N, H, W, C) array; for the flow, (N, H, W, 2) is the payload of a .flo file per pair."""
        n, c, h, w = self.blobs[name].shape
        out = np.empty((n, h, w, c), np.float32)
        check(lib().fn2_net_get_blob_nhwc(self._h, name.encode(), out.ctypes.data_as(C.c_void_p)))
        return out

    def get_blob_nhwc_device(self, name, dev_ptr):
        check(lib().fn2_net_get_blob_nhwc_device(self._h, name.encode(), C.c_void_p(dev_ptr)))

    def forward_async(self):
        check(lib().fn2_net_forward(self._h))

    # ---- gradients (pycaffe.py:127-175 Net.backward; net.cpp:640-655) ----
    def backward_async(self):
        check(lib().fn2_net_backward(self._h))

    def clear_param_diffs(self):
        check(lib().fn2_net_clear_param_diffs(self._h))

    @property
    def iter(self):
        """Net::iter: the iteration the layers see (LpqLoss picks its p/q schedule step by it); 0 until set."""
        it = C.c_int()
        check(lib().fn2_net_iter(self._h, C.byref(it)))
        return it.value

    def set_iter(self, iteration):
        """Net::set_iter.  Solver.step sets it at the start of every iteration."""
        check(lib().fn2_net_set_iter(self._h, int(iteration)))

    def set_diff(self, name, array):
        a = np.ascontiguousarray(array, dtype=np.float32)
        if tuple(a.shape) != self.blobs[name].shape:
            raise Fn2Error("diff of %s has shape %s, net expects %s" % (name, a.shape, self.blobs[name].shape))
        check(lib().fn2_net_set_diff(self._h, name.encode(), a.ctypes.data_as(C.c_void_p)))

    def get_diff(self, name):
        out = np.empty(self.blobs[name].shape, np.float32)
        self.sync()
        check(lib().fn2_net_get_diff(self._h, name.encode(), out.ctypes.data_as(C.c_void_p)))
        return out

    def backward(self, **kwargs):
        """net.backward(flow=top_diff) -> {input blob name: gradient}; parameter gradients through net.param(layer, i, diff=True)."""
        for k, v in kwargs.items():
            self.set_diff(k, v)
        self.backward_async()
        self.sync()
        return {}

    def param(self, layer, index=0, diff=False):
        shp = (C.c_int * 4)()
        check(lib().fn2_net_param_shape(self._h, layer.encode(), int(index), shp))
        out = np.empty(tuple(int(x) for x in shp), np.float32)
        check(lib().fn2_net_get_param(self._h, layer.encode(), int(index), 1 if diff else 0, out.ctypes.data_as(C.c_void_p)))
        return out

    def param_diff_arena(self):
        return out_span(lib().fn2_net_param_diff_arena, self._h)

    def trainable_diff_span(self):
        """(device pointer, bytes): the range of param_diff_arena() that holds every gradient the backward pass writes."""
        return out_span(lib().fn2_net_trainable_diff_span, self._h)

    def layer_need_backward(self):
        return [bool(lib().fn2_net_layer_need_backward(self._h, i)) for i in range(len(self.layer_names))]

    @property
    def launches_per_backward(self):
        return int(lib().fn2_net_launches_per_backward(self._h))

    def sync(self):
        check(lib().fn2_net_sync(self._h))

    def forward(self, **kwargs):
        """net.forward(img0=..., img1=...) -> {output blob name: ndarray} (pycaffe.py:78-124)."""
        for k, v in kwargs.items():
            if k not in self.inputs:
                raise Fn2Error("Input blob arguments do not match net inputs.")
            self.set_input(k, v)
        self.forward_async()
        return {o: self.blobs[o].data for o in self.outputs}

    @property
    def stream(self):
        return lib().fn2_net_stream(self._h)

    def time_layers(self):
        ms = (C.c_float * len(self.layer_names))()
        check(lib().fn2_net_time_layers(self._h, ms))
        return list(zip(self.layer_names, self.layer_types, [float(x) for x in ms]))

    def layer_work(self):
        """[(name, type, algorithmic flops, algorithmic bytes)] per layer."""
        out = []
        for i, (n, t) in enumerate(zip(self.layer_names, self.layer_types)):
            f, b = C.c_double(), C.c_double()
            check(lib().fn2_net_layer_work(self._h, i, C.byref(f), C.byref(b)))
            out.append((n, t, f.value, b.value))
        return out

    @property
    def graph_active(self):
        return bool(lib().fn2_net_graph_active(self._h))

    @property
    def launches_per_forward(self):
        return int(lib().fn2_net_launches_per_forward(self._h))


# ------------------------------------------------------------------------------------------------
# Solver (pycaffe-like: python/caffe/_caffe.cpp:338-371; the loop of src/caffe/solver.cpp:194-481)
# ------------------------------------------------------------------------------------------------
def solver_params(solver):
    """Resolved parameters of a solver prototxt (text or path): {field: value}, defaults filled in, solver_type upgraded to
    type; stepvalue is a list."""
    out = {"stepvalue": []}
    text = sized_output(lib().fn2_solver_params, _read_text(solver).encode())[:-1].decode()
    for line in text.splitlines():
        k, v = line.split(": ", 1)
        if v.startswith('"'):
            v = v[1:-1]
        elif v in ("true", "false"):
            v = v == "true"
        else:
            v = float(v) if any(c in v for c in ".eEna") else int(v)
        if k == "stepvalue":
            out[k].append(v)
        else:
            out[k] = v
    return out


def learning_rate(solver, iteration, current_step=0):
    """SGDSolver::GetLearningRate at `iteration` -> (rate, current_step after the call); multistep advances at most one step."""
    cs, rate = C.c_int(int(current_step)), C.c_float()
    check(lib().fn2_solver_learning_rate(_read_text(solver).encode(), int(iteration), C.byref(cs), C.byref(rate)))
    return rate.value, cs.value


def get_solver(solver, net):
    """caffe.get_solver look-alike: solver prototxt (text or path) over a TRAIN Net."""
    return Solver(solver, net)


class Solver(object):
    """Caffe's SGD / Adam solver over a TRAIN Net (src/caffe/solver.cpp:194-481, solvers/sgd_solver.cpp, adam_solver.cpp).

    ``step(n, feed)`` runs n iterations: Net.set_iter(iter), ClearParamDiffs, the on_start callbacks, iter_size x (feed, forward, backward), the
    on_gradients_ready callbacks, the update on the device, iter += 1, and a snapshot when one is due.  ``feed()`` returns
    {input name: ndarray or CUDA tensor} and is called before every forward.  Within an iteration the only host
    synchronisation is the read of the loss outputs, after the update has been enqueued.  Data-parallel training all-reduces
    the gradients in ``on_gradients_ready`` (parallel.allreduce_gradients(parallel.grad_arena_tensor(net,
    trainable_only=True))); every rank then applies the same update.
    """

    def __init__(self, solver, net):
        self._text = _read_text(solver)
        self.net = net
        self.param = solver_params(self._text)
        h = C.c_void_p()
        check(lib().fn2_solver_create(self._text.encode(), net._h, C.byref(h)))
        self._h = h
        self._callbacks = []
        w = (C.c_float * len(net.outputs))()
        check(lib().fn2_solver_output_loss_weights(h, w, len(net.outputs)))
        self._loss_outputs = [(o, float(x)) for o, x in zip(net.outputs, w) if x != 0]
        for o, _ in self._loss_outputs:
            if int(np.prod(net.blobs[o].shape)) != 1:
                raise Fn2Error("loss output %s is not a scalar: %s" % (o, net.blobs[o].shape))
        self._loss_buf = None
        self._losses = []
        self.smoothed_loss = 0.0

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().fn2_solver_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def _status(self):
        it, cs = C.c_int(), C.c_int()
        check(lib().fn2_solver_iter(self._h, C.byref(it), C.byref(cs)))
        return it.value, cs.value

    @property
    def iter(self):
        return self._status()[0]

    @property
    def lr(self):
        """The learning rate the next update uses."""
        it, cs = self._status()
        return learning_rate(self._text, it, cs)[0]

    def add_callback(self, on_start, on_gradients_ready):
        self._callbacks.append((on_start, on_gradients_ready))

    def _feed(self, inputs):
        import torch
        for name, value in inputs.items():
            if isinstance(value, torch.Tensor):
                t = value.detach().to(torch.float32).contiguous()
                if tuple(t.shape) != self.net.blobs[name].shape or not t.is_cuda:
                    raise Fn2Error("input %s: a CUDA tensor of shape %s is expected" % (name, self.net.blobs[name].shape))
                ready = torch.cuda.Event()
                ready.record()
                torch.cuda.ExternalStream(self.net.stream).wait_event(ready)       # the net reads it after torch wrote it
                self._keep.append(t)
                self.net.set_input_device(name, t.data_ptr())
            else:
                self.net.set_input(name, value)

    def step(self, iters, feed=None):
        import torch
        it0 = self.iter
        iter_size = int(self.param["iter_size"])
        self._losses, self.smoothed_loss = [], 0.0
        if self._loss_outputs and (self._loss_buf is None or self._loss_buf.shape[0] != iter_size):
            self._loss_buf = torch.empty((iter_size, len(self._loss_outputs)), dtype=torch.float32, device="cuda")
        weights = [wt for _, wt in self._loss_outputs]
        net_stream = torch.cuda.ExternalStream(self.net.stream)
        for _ in range(int(iters)):
            self._keep = []
            self.net.set_iter(self.iter)                                   # solver.cpp:202, before ClearParamDiffs
            self.net.clear_param_diffs()
            for on_start, _ in self._callbacks:
                on_start()
            for i in range(iter_size):
                if feed is not None:
                    self._feed(feed())
                self.net.forward_async()
                self.net.backward_async()
                for j, (name, _) in enumerate(self._loss_outputs):
                    self.net.get_blob_device(name, self._loss_buf[i, j].data_ptr())
            if self._callbacks:
                # the callbacks' work (an all-reduce of the gradient arena) runs on torch's current stream after the backward,
                # and the update on the net's stream after the callbacks' work: ordered on the device, no host wait
                done = torch.cuda.Event()
                done.record(net_stream)
                torch.cuda.current_stream().wait_event(done)
                for _, on_gradients_ready in self._callbacks:
                    on_gradients_ready()
                reduced = torch.cuda.Event()
                reduced.record()
                net_stream.wait_event(reduced)
            check(lib().fn2_solver_apply_update(self._h))
            self.net.sync()
            if self._loss_outputs:
                per_pass = self._loss_buf.cpu().numpy().astype(np.float64) @ np.asarray(weights, np.float64)
                self._update_smoothed_loss(float(per_pass.sum()) / iter_size, it0)
            it = self.iter
            if self.param["snapshot"] and it % self.param["snapshot"] == 0:
                self.snapshot()
        self._keep = []

    def _update_smoothed_loss(self, loss, start_iter):
        """Solver::UpdateSmoothedLoss (solver.cpp:484-495)."""
        average = int(self.param["average_loss"])
        if len(self._losses) < average:
            self._losses.append(loss)
            self.smoothed_loss = (self.smoothed_loss * (len(self._losses) - 1) + loss) / len(self._losses)
        else:
            idx = (self.iter - 1 - start_iter) % average
            self.smoothed_loss += (loss - self._losses[idx]) / average
            self._losses[idx] = loss

    def solve(self, feed=None, resume=None):
        """Solver::Solve (solver.cpp:277-330): optionally restore, step to max_iter, and snapshot at the end unless that
        iteration was just snapshotted or snapshot_after_train is false."""
        if resume is not None:
            self.restore(resume)
        self.step(int(self.param["max_iter"]) - self.iter, feed)
        snap = self.param["snapshot"]
        if self.param["snapshot_after_train"] and (not snap or self.iter % snap != 0):
            self.snapshot()

    def state(self, learned_net=""):
        """The SolverState message as bytes (history in Net::learnable_params order; Adam: every m, then every v)."""
        return sized_output(lib().fn2_solver_state, self._h, learned_net.encode())

    def snapshot(self):
        """Solver::Snapshot (solver.cpp:447-469): <prefix>_iter_<N>.caffemodel and <prefix>_iter_<N>.solverstate.
        Returns (caffemodel path, solverstate path)."""
        prefix = self.param["snapshot_prefix"]
        if not prefix:
            raise Fn2Error("snapshot: snapshot_prefix is not set")
        base = "%s_iter_%d" % (prefix, self.iter)
        model, state = base + ".caffemodel", base + ".solverstate"
        with open(model, "wb") as f:
            f.write(self.net.to_caffemodel())
        with open(state, "wb") as f:
            f.write(self.state(model))
        return model, state

    def restore(self, state):
        """Solver::Restore (sgd_solver.cpp:305-322): a .solverstate path or its bytes.  Restores iter, current_step and the
        history, and loads the weights of learned_net through Net.copy_from when the state names one."""
        if isinstance(state, str):
            with open(state, "rb") as f:
                state = f.read()
        buf = (C.c_char * len(state)).from_buffer_copy(state)
        learned = sized_output(lib().fn2_solverstate_learned_net, buf, len(state))[:-1].decode()
        check(lib().fn2_solver_restore(self._h, buf, len(state)))
        if learned:
            self.net.copy_from(learned)


# ------------------------------------------------------------------------------------------------
# .flo IO (src/caffe/util/output.cpp:16-64, scripts/run-flownet.py:100-126)
# ------------------------------------------------------------------------------------------------
def write_flo(path, flow_2hw):
    a = np.ascontiguousarray(flow_2hw, np.float32)
    assert a.ndim == 3 and a.shape[0] == 2
    check(lib().fn2_write_flo(path.encode(), a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[2]))


def read_flo(path):
    h, w = C.c_int(), C.c_int()
    check(lib().fn2_read_flo(path.encode(), None, C.byref(h), C.byref(w), 0))
    out = np.empty((2, h.value, w.value), np.float32)
    check(lib().fn2_read_flo(path.encode(), out.ctypes.data_as(C.c_void_p), C.byref(h), C.byref(w), out.size))
    return out


def image_to_blob(img_hwc_rgb_uint8):
    """HWC RGB uint8 -> (1,3,H,W) BGR float 0..255, scripts/run-flownet.py:30-35."""
    a = np.asarray(img_hwc_rgb_uint8)
    if a.ndim < 3:
        return a[np.newaxis, np.newaxis, :, :].astype(np.float32)
    return a[np.newaxis, :, :, :].transpose(0, 3, 1, 2)[:, [2, 1, 0], :, :].astype(np.float32)
