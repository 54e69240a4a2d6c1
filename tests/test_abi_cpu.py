"""The Python binding of libfn2.so is derived from include/fn2.h: every declared entry point gets a prototype with the
header's arity, the structs have the header's layout, and the status / message of the error paths stay put."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests.test_host_cpu import GOLD, ROOT, canonical, declared_symbols

# C return types as the header spells them -> the restype ctypes must use
RESTYPES = {"int": C.c_int, "void": None, "const char*": C.c_char_p, "void*": C.c_void_p, "uint64_t": C.c_uint64}


def header_arity():
    text = re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", "fn2.h")).read(), flags=re.S)
    out = {}
    for ret, name, params in re.findall(r"FN2_API\s+([\w\s\*]+?)\s*\b(fn2_\w+)\s*\(([^)]*)\)", text):
        out[name] = (" ".join(ret.split()), 0 if params.strip() == "void" else params.count(",") + 1)
    return out


def test_every_declaration_has_a_prototype(fn2):
    lib = fn2.lib()
    arity = header_arity()
    assert sorted(arity) == declared_symbols() and len(arity) == 95
    bad = []
    for name, (ret, n) in arity.items():
        f = getattr(lib, name)
        if f.argtypes is None or len(f.argtypes) != n or f.restype is not RESTYPES[ret]:
            bad.append((name, n, f.argtypes and len(f.argtypes), ret, f.restype))
    assert not bad, bad


def test_pinned_prototypes(fn2):
    lib = fn2.lib()
    T = C.POINTER(fn2.fn2_tensor)
    assert lib.fn2_correlation_backward.argtypes == [T] * 5 + [C.c_int] * 6 + [C.c_void_p, C.c_size_t, C.c_void_p]
    assert lib.fn2_eltwise_sum.argtypes[0] is C.POINTER(T)
    assert lib.fn2_conv_forward.argtypes[0] is C.POINTER(fn2.fn2_conv_desc)
    assert lib.fn2_l1loss_forward.argtypes[2] is C.POINTER(fn2.fn2_l1loss_desc)
    assert lib.fn2_net_create_batch.argtypes[3] is C.POINTER(C.c_void_p)
    assert lib.fn2_net_blob_shape.argtypes[2] is C.POINTER(C.c_int)
    assert lib.fn2_apply_effects.argtypes[3] is C.c_ulonglong and lib.fn2_aug_sample.argtypes[1] is C.c_uint
    assert lib.fn2_net_destroy.restype is None
    assert lib.fn2_net_stream.restype is C.c_void_p
    assert lib.fn2_launch_count.restype is C.c_uint64


def test_struct_layouts(fn2):
    assert [C.sizeof(s) for s in (fn2.fn2_tensor, fn2.fn2_conv_desc, fn2.fn2_l1loss_desc)] == [56, 64, 20]
    assert [f[0] for f in fn2.fn2_tensor._fields_] == ["data", "n", "c", "h", "w", "sn", "sc", "sh", "sw"]
    assert [f[0] for f in fn2.fn2_conv_desc._fields_] == [
        "ci", "co", "kh", "kw", "stride_h", "stride_w", "pad_h", "pad_w", "deconv", "has_bias", "relu", "negative_slope", "engine",
        "input_guard_bytes", "out_pad_h", "out_pad_w"]
    assert [f[0] for f in fn2.fn2_l1loss_desc._fields_] == [
        "l2_per_location", "l2_prescale_by_channels", "normalize_by_num_entries", "epsilon", "plateau"]
    assert fn2.fn2_conv_desc.negative_slope.offset == 44 and fn2.fn2_tensor.sn.offset == 24


def test_header_reader_rejects_an_unknown_type():
    from flownet2_b200 import _abi
    structs, protos = _abi.read_header("typedef struct s { int32_t a; float b; } s;\nFN2_API int fn2_x(const s* p, size_t* n);")
    assert C.sizeof(structs["s"]) == 8 and protos["fn2_x"] == (C.c_int, [C.POINTER(structs["s"]), C.POINTER(C.c_size_t)])
    with pytest.raises(ValueError, match="long double"):
        _abi.read_header("FN2_API int fn2_x(long double v);")
    with pytest.raises(ValueError, match="fn2_y"):
        _abi.read_header("FN2_API int fn2_y(void (*callback)(int));")


# ---- error paths: the status and message a caller sees ----
def last_error(fn2):
    return fn2.lib().fn2_last_error().decode()


def test_null_net_arguments(fn2):
    lib = fn2.lib()
    n, p, f, b = C.c_size_t(), C.c_void_p(), C.c_double(), C.c_double()
    assert lib.fn2_net_forward(None) == -1 and last_error(fn2).startswith("forward: null")
    assert lib.fn2_net_to_caffemodel(None, None, C.byref(n)) == -1 and last_error(fn2) == "to_caffemodel: null argument"
    assert lib.fn2_net_param_arena(None, C.byref(p), C.byref(n)) == -1 and last_error(fn2) == "param_arena: null argument"
    assert lib.fn2_net_layer_work(None, 0, C.byref(f), C.byref(b)) == -1 and last_error(fn2).startswith("layer_work: ")


def test_size_query_buffer_too_small(fn2):
    lib = fn2.lib()
    text = 'layer { name: "a" type: "Input" top: "x" }'
    n = C.c_size_t()
    assert lib.fn2_proto_canonical(text.encode(), None, C.byref(n)) == 0
    assert n.value == len(canonical(fn2, text)) + 1                       # text outputs report the NUL
    short = C.c_size_t(n.value - 1)
    assert lib.fn2_proto_canonical(text.encode(), C.create_string_buffer(n.value), C.byref(short)) == -1
    assert last_error(fn2).endswith("buffer too small")
    raw = open(os.path.join(GOLD, "ref_pb2_caffemodel.bin"), "rb").read()
    assert lib.fn2_caffemodel_to_hdf5(raw, len(raw), None, C.byref(n)) == 0
    short = C.c_size_t(n.value - 1)
    assert lib.fn2_caffemodel_to_hdf5(raw, len(raw), C.create_string_buffer(n.value), C.byref(short)) == -1
    assert last_error(fn2) == "caffemodel_to_hdf5: buffer too small"
    assert lib.fn2_caffemodel_to_hdf5(raw[:100], 100, None, C.byref(n)) == -3    # every exception is a parse error


TINY = ('layer { name: "in" type: "Input" top: "x" input_param { shape { dim: 1 dim: 3 dim: 8 dim: 8 } } }\n'
        'layer { name: "conv" type: "Convolution" bottom: "x" top: "y" convolution_param { num_output: 4 kernel_size: 3 } }\n')


@pytest.mark.gpu
def test_net_error_paths(fn2):
    lib = fn2.lib()
    net = fn2.Net(TINY, None, fn2.TEST)
    net.fill_params(3)
    shape = (C.c_int * 4)()
    assert lib.fn2_net_blob_shape(net._h, b"nope", shape) == -4 and "Unknown blob name nope" in last_error(fn2)
    assert lib.fn2_net_param_shape(net._h, b"conv", 2, shape) == -1 and last_error(fn2) == "param_shape: no parameter blob conv[2]"
    assert lib.fn2_net_param_shape(net._h, b"conv", 1, shape) == 0 and list(shape) == [4, 1, 1, 1]
    for name in ("fn2_net_to_caffemodel", "fn2_net_to_hdf5"):
        call = getattr(lib, name)
        n = C.c_size_t()
        assert call(net._h, None, C.byref(n)) == 0 and n.value > 0
        short = C.c_size_t(n.value - 1)
        assert call(net._h, C.create_string_buffer(n.value), C.byref(short)) == -1 and last_error(fn2).endswith("buffer too small")
    # the refused call leaves the net able to serialise; a caffemodel round-trips
    cm = net.to_caffemodel()
    other = fn2.Net(TINY, cm, fn2.TEST)
    assert np.array_equal(other.param("conv", 0), net.param("conv", 0)) and other.to_caffemodel() == cm
    assert len(net.to_hdf5()) > 0
