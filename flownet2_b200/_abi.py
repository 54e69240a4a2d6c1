"""ctypes structs, prototypes and integer constants of libfn2.so, read from include/fn2.h, fn2_solver.h, fn2_frames.h and
fn2_flow.h: the headers are the only statement of the ABI.

Types map through one table; a type it does not know raises, so a new header entry cannot go undeclared."""
import ctypes as C
import re

SCALARS = {"int": C.c_int, "unsigned int": C.c_uint, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint64_t": C.c_uint64,
           "unsigned long long": C.c_ulonglong, "size_t": C.c_size_t, "float": C.c_float, "double": C.c_double}
# data pointers and the opaque net and solver handles: c_void_p takes ints from data_ptr(), numpy / ctypes pointers, arrays and None
OPAQUE = ("void", "float", "fn2_net", "fn2_solver")


def ctype(t, known):
    """ctypes type of a C type as the header spells it ('const fn2_tensor* const*', 'int[4]', 'void')."""
    t = " ".join(re.sub(r"\bconst\b", " ", t).split())
    t = re.sub(r"\s*\[\d*\]$", "*", t)                                   # an array parameter is a pointer
    if t.endswith("*"):
        base = t[:-1].strip()
        if base == "char":
            return C.c_char_p
        return C.c_void_p if base in OPAQUE else C.POINTER(ctype(base, known))
    if t == "void":
        return None
    if t not in known:
        raise ValueError("fn2.h: no ctypes type for %r" % t)
    return known[t]


def _split(decl):
    """'const fn2_tensor* bottom0' -> 'const fn2_tensor*'; 'int shape[4]' -> 'int[4]'."""
    m = re.fullmatch(r"(.*?)\s*\b\w+\s*(\[\d*\])?", decl.strip(), re.S)
    return m.group(1) + (m.group(2) or "")


def read_defines(text):
    """-> {name: int} of the header's integer constants (#define FN2_... <integer>)."""
    return {k: int(v, 0) for k, v in re.findall(r"^\s*#define\s+(FN2_\w+)\s+(-?(?:0x[0-9a-fA-F]+|\d+))\s*$", text, re.M)}


def read_header(text, included=None):
    """-> ({struct name: ctypes.Structure}, {function: (restype, argtypes)}) of every typedef'd struct and FN2_API declaration.
    included: the structs of headers this one includes (fn2.h's fn2_tensor for fn2_frames.h)."""
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    text = re.sub(r"^\s*#.*$", "", text, flags=re.M)
    known, structs = dict(SCALARS, **(included or {})), {}
    for name, body in re.findall(r"typedef struct (\w+) \{(.*?)\} \1;", text, re.S):
        fields = []
        for member in filter(None, (m.strip() for m in body.split(";"))):
            ty, names = re.fullmatch(r"(.*?)\s*\b(\w+(?:\s*,\s*\w+)*)", member, re.S).groups()
            fields += [(n.strip(), ctype(ty, known)) for n in names.split(",")]
        structs[name] = known[name] = type(name, (C.Structure,), {"_fields_": fields})
    protos = {}
    for decl in re.findall(r"\bFN2_API\b([^;]*);", text):
        m = re.fullmatch(r"\s*(.+?)\s*\b(fn2_\w+)\s*\(([^()]*)\)\s*", decl, re.S)
        if not m:
            raise ValueError("fn2.h: cannot read the declaration %r" % " ".join(decl.split()))
        ret, name, params = m.groups()
        params = [] if params.strip() == "void" else params.split(",")
        protos[name] = (ctype(ret, known), [ctype(_split(p), known) for p in params])
    return structs, protos
