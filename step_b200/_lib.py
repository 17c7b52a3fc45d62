"""ctypes binding of libstep_b200.so, read from the C ABI in include/step_b200.h.

PyTorch only supplies device memory and the current CUDA stream; every compute call below goes
through the C ABI.  There is no fallback: if the library is missing or a tensor is not on a CUDA
device the call raises (north_star: "no CPU fallback").

The header is the one declaration of the ABI.  At import, `read_header` turns it into the enum constants (exposed here
with the STEP_ prefix dropped: STEP_F16 -> F16, STEP_E_ARG -> E_ARG), one ctypes.Structure per struct typedef (exposed
under its C name: step_conv_params, ...) and the argtypes / restype of every entry point, which `lib()` sets.  A
declaration the reader does not know raises at import, so a header edit it cannot follow fails on the host instead of
shifting the arguments of a launch.
"""
import ctypes
import os
import re

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libstep_b200.so")
HEADER = os.path.join(os.path.dirname(HERE), "include", "step_b200.h")

_lib = None

c_void_p = ctypes.c_void_p


class Struct(ctypes.Structure):
    """Base of the header's structs.  Every pointer parameter and step_stream_t binds as c_void_p, which takes an int
    address, c_void_p, ctypes.byref(...), a ctypes array or None in C; an instance of one of these structs passes by
    reference through `_as_parameter_`.  (A Python-level from_param would run on every pointer argument of every call.)"""

    @property
    def _as_parameter_(self):
        return ctypes.byref(self)


_SCALARS = {"int": ctypes.c_int, "int32_t": ctypes.c_int32, "float": ctypes.c_float, "long long": ctypes.c_longlong,
            "size_t": ctypes.c_size_t, "uint64_t": ctypes.c_uint64}
_STATEMENT = re.compile(r"\s*(?:enum\s*\{(?P<enum>[^{}]*)\}|typedef\s+struct\s*\{(?P<fields>[^{}]*)\}\s*(?P<struct>\w+)"
                        r"|typedef\s+struct\s+\w+\s*\*\s*(?P<handle>\w+)"
                        r"|(?P<ret>[\w\s*]+?)\s*\b(?P<fn>step_\w+)\s*\((?P<params>[^;{}()]*)\))\s*;")
_DECLARATOR = re.compile(r"(?:const\s+)?(?P<type>\w+(?:\s+\w+)*?)\s*(?P<ptr>\*?)\s*(?P<name>\w+)(?:\[(?P<len>\w+)\])?")


def read_header(text):
    """(constants, structs, functions) of a header written in the C subset of include/step_b200.h: enums of integer
    literals and `1 << n`; `typedef struct { ... } name;` with scalar, pointer (c_void_p), fixed-array and struct fields,
    several declarators per line allowed; opaque handles `typedef struct X* name;`; `step_*` prototypes of scalars and
    pointers (every pointer and handle binds as c_void_p, a `const char*` result as c_char_p).  Anything else raises
    ValueError naming the declaration."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"#ifdef __cplusplus.*?#endif|#[^\n]*", " ", text, flags=re.S)
    consts, structs, functions, handles = {}, {}, {}, set()

    def fail(declaration):
        raise ValueError("step_b200.h: cannot bind %r" % " ".join(declaration.split()))

    def bind(decl, field=False):
        """(name, ctypes type) of one declarator `[const] type [*]name[[len]]`."""
        d = _DECLARATOR.fullmatch(decl.strip())
        if d is None or (d["len"] and not field):
            fail(stmt)
        pointer = d["ptr"] or d["type"] in handles
        t = ctypes.c_void_p if pointer else _SCALARS.get(d["type"]) or field and structs.get(d["type"])
        if d["len"]:
            n = int(d["len"]) if d["len"].isdigit() else consts.get(d["len"])
            t = t and n and t * n
        return d["name"], t or fail(stmt)

    pos = 0
    while text[pos:].strip():
        m = _STATEMENT.match(text, pos)
        stmt = m.group(0) if m else text[pos:text.find(";", pos) + 1 or len(text)]
        if m is None:
            fail(stmt)
        pos = m.end()
        if m["enum"] is not None:
            for item in filter(str.strip, m["enum"].split(",")):
                e = re.fullmatch(r"\s*(\w+)\s*=\s*(\d+)(?:\s*<<\s*(\d+))?\s*", item) or fail(stmt)
                consts[e[1]] = int(e[2]) << int(e[3] or 0)
        elif m["struct"]:
            fields = []
            for line in filter(str.strip, m["fields"].split(";")):
                first, *more = line.split(",")
                base = (_DECLARATOR.fullmatch(first.strip()) or fail(stmt))["type"]
                fields += [bind(d, field=True) for d in [first] + [base + " " + d for d in more]]
            structs[m["struct"]] = type(m["struct"], (Struct,), {"_fields_": fields})
        elif m["handle"]:
            handles.add(m["handle"])
        else:
            ret = m["ret"].strip()
            restype = ctypes.c_char_p if re.fullmatch(r"const char\s*\*", ret) else bind(ret + " " + m["fn"])[1]
            params = [] if m["params"].strip() == "void" else m["params"].split(",")
            functions[m["fn"]] = ([bind(p)[1] for p in params], restype)
    return consts, structs, functions


with open(HEADER) as _f:
    CONSTANTS, STRUCTS, FUNCTIONS = read_header(_f.read())
globals().update({name.removeprefix("STEP_"): value for name, value in CONSTANTS.items()})
globals().update(STRUCTS)
# The names these structs had before they were read from the header; existing callers keep them (select.py and
# evaluation.py keep theirs likewise).
ConvParams, OptimTensor, OptimBlock, FrameSrc, ClipAug, AugErase = (STRUCTS[n] for n in (
    "step_conv_params", "step_optim_tensor", "step_optim_block", "step_frame_src", "step_clip_aug", "step_aug_erase"))


def lib():
    """Load (once) and return the shared library.  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("step_b200: %s not found -- run `python -m step_b200.build` (there is no "
                               "CPU / PyTorch fallback for the hot path)" % LIB_PATH)
        l = ctypes.CDLL(LIB_PATH)
        for name, (argtypes, restype) in FUNCTIONS.items():
            fn = getattr(l, name)  # AttributeError here == header / library mismatch
            fn.argtypes, fn.restype = argtypes, restype
        _lib = l
    return _lib


def exported_symbols():
    """Every entry point the header declares; lib() has checked that the library exports each."""
    lib()
    return sorted(FUNCTIONS)


def check(rc):
    if rc != 0:
        raise RuntimeError("step_b200 [%d]: %s" % (rc, lib().step_last_error().decode("utf-8", "replace")))


def stream(device=None):
    """The launch stream: torch's current stream of `device` (default: the current device).  Callers working on
    tensors of another GPU wrap their launches in `torch.cuda.device(dev)` (kernels must run on the device that owns
    their pointers; test.py:85-87 places det_net i on cuda:(i+1) % gpu_count)."""
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)


def same_device(*tensors):
    """All CUDA tensors of one launch must live on one device; returns it."""
    dev = None
    for t in tensors:
        if t is None:
            continue
        need_cuda(t)
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise RuntimeError("step_b200: tensors of one launch on different devices (%s vs %s)" % (dev, t.device))
    return dev


def ptr(t):
    return c_void_p(t.data_ptr()) if t is not None else c_void_p(0)


def need_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("step_b200: expected a CUDA tensor (no CPU fallback on the hot path), got device %s"
                               % t.device)


def dt(t):
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.float16:
        return F16
    raise RuntimeError("step_b200: unsupported dtype %s (float32 / float16 only)" % t.dtype)


def launch_count():
    return int(lib().step_launch_count())
