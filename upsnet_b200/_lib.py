"""ctypes binding of libupsnet_b200.so (the C ABI declared in include/upsnet_b200.h).

There is deliberately NO fallback: if the CUDA library cannot be loaded, or a tensor is not a
CUDA tensor, the ops raise.  (The reference does the same for non-CUDA tensors:
operators/functions/deform_conv.py:40-41, functions/roialign.py:34-35.)
"""
import ctypes as C
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libupsnet_b200.so")
HEADER_PATH = os.path.join(_HERE, "..", "include", "upsnet_b200.h")
_lib = None

LAYOUT_NCHW, LAYOUT_NHWC = 0, 1
EPI_RELU = 1
EPI_RES_UP2 = 2
EPI_NO_TMA = 4
EPI_STEM_PAIR = 8
EPI_RES_BILINEAR = 16


def EPI_SIGMOID_FROM(c):
    return ((int(c) + 1) & 0x3ff) << 20
PREC_FP32_SIMT, PREC_BF16X3, PREC_BF16 = 0, 1, 2
DTYPE_F32, DTYPE_BF16, DTYPE_PAIR = 0, 1, 2
LAYOUT_FLAT_PAIR = 2
GRAD_RELU, GRAD_RES_UP2, GRAD_UNSHUFFLE2, GRAD_DY_NHWC = 1, 2, 4, 8

E_UNSUPPORTED = -2
_ERR = {-1: "bad argument", E_UNSUPPORTED: "unsupported configuration", -3: "workspace too small"}


class UpsnetError(RuntimeError):
    pass


_CTYPES = {"int": C.c_int, "float": C.c_float, "double": C.c_double, "size_t": C.c_size_t,
           "long long": C.c_longlong, "int64_t": C.c_longlong,
           "unsigned long long": C.c_ulonglong, "uint64_t": C.c_ulonglong}


def declarations(header=HEADER_PATH):
    """[(name, argtypes)] of every `int upsnet_*(...)` declared in the header.  A pointer or array parameter is a c_void_p
    (which takes a device address, None, a ctypes array or byref()); scalars map through _CTYPES, and any other type
    raises, so a new kind of parameter cannot be bound wrongly without notice."""
    with open(header) as f:
        text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", f.read(), flags=re.S)
    decls = []
    for name, params in re.findall(r"\bint\s+(upsnet_\w+)\s*\(([^)]*)\)\s*;", text):
        types = []
        for p in params.split(","):
            if "*" in p or "[" in p:
                types.append(C.c_void_p)
                continue
            words = [w for w in p.split() if w != "const"]
            t = _CTYPES.get(" ".join(words[:-1]))
            if t is None:
                raise UpsnetError("%s: parameter %r of %s has no ctypes mapping" % (header, p.strip(), name))
            types.append(t)
        decls.append((name, types))
    return decls


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            from . import build as _build  # in-tree nvcc build; raises if nvcc is missing
            _build.build()
        L = C.CDLL(LIB_PATH)
        for name, types in declarations():
            getattr(L, name).argtypes = types
        _lib = L
    return _lib


def check(rc, what):
    if rc == 0:
        return
    if rc < 0:
        raise UpsnetError("%s: %s (%d)" % (what, _ERR.get(rc, "error"), rc))
    raise UpsnetError("%s: CUDA error %d" % (what, rc))


def try_call(name, device, *args):
    """Enqueues the entry point upsnet_<name> on the current stream of `device`, which is appended as the last argument.
    A tensor argument is passed as its data_ptr(), None as NULL, anything else as it is.  Returns 0, or
    UPSNET_E_UNSUPPORTED for a caller that then takes another path; raises UpsnetError on any other failure."""
    with torch.cuda.device(device):
        rc = getattr(lib(), "upsnet_" + name)(*[a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args],
                                               torch.cuda.current_stream(device).cuda_stream)
    if rc != E_UNSUPPORTED:
        check(rc, "upsnet_" + name)
    return rc


def call(name, device, *args):
    """try_call() that raises on UPSNET_E_UNSUPPORTED too."""
    check(try_call(name, device, *args), "upsnet_" + name)


def query_bytes(name, *args, unsupported=False):
    """The size_t that the host-only query upsnet_<name>(..., size_t* bytes) writes: a workspace or packed-weight size.
    With unsupported=True, None when the query answers UPSNET_E_UNSUPPORTED."""
    n = C.c_size_t(0)
    rc = getattr(lib(), "upsnet_" + name)(*args, C.byref(n))
    if unsupported and rc == E_UNSUPPORTED:
        return None
    check(rc, "upsnet_" + name)
    return n.value


# for code that calls lib().upsnet_* directly instead of through call()
def stream_ptr(device=None):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(None)


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise UpsnetError("upsnet_b200 ops are CUDA-only (sm_90a); got a %s tensor" % t.device)


def f32c(t):
    """fp32 + contiguous (NCHW), no copy when already so."""
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()
