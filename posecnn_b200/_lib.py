"""ctypes binding of libposecnn_b200.so (include/posecnn_b200.h).

The Python side binds from the header: when the library is loaded, every `pcnn_*` prototype of include/posecnn_b200.h
sets the `argtypes` / `restype` of its entry point, so a call with the wrong number of arguments, or a tensor where a pointer
belongs, raises in Python before C is entered, and plain Python numbers reach C as the declared int / float / size_t.
Pointers travel as ints (`ptr(t)`, `stream()`); ctypes values (c_void_p, c_float, c_size_t, byref, host arrays) are accepted too.

There is NO fallback: if the shared object is missing or a call fails, the ops raise.
PyTorch is used only for device memory and streams.
"""
from __future__ import annotations

import ctypes
import os
import re

import torch

from .build import HEADER, LIB

_lib = None
_ws = {}

_SCALARS = {"int": ctypes.c_int, "float": ctypes.c_float, "double": ctypes.c_double, "size_t": ctypes.c_size_t,
            "int8_t": ctypes.c_int8, "uint8_t": ctypes.c_uint8, "int16_t": ctypes.c_int16, "uint16_t": ctypes.c_uint16,
            "int32_t": ctypes.c_int32, "uint32_t": ctypes.c_uint32, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64}
_RETURNS = {"int": ctypes.c_int, "const char*": ctypes.c_char_p}


def prototypes(text: str) -> dict:
    """{name: (restype, [argtypes])} for every `pcnn_*` prototype of a C header; any pointer is c_void_p.  A return or
    parameter type outside the table raises, naming the function, so no entry point is ever bound in a wrong way."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"^[ \t]*#[^\n]*", " ", text, flags=re.M)          # preprocessor lines
    protos = {}
    for ret, name, params in re.findall(r"([^;{}]*?)\b(pcnn_\w+)\s*\(([^)]*)\)\s*;", text):
        ret = re.sub(r"\s*\*", "*", " ".join(ret.split()))
        if ret not in _RETURNS:
            raise TypeError(f"{name}: return type {ret!r} has no ctypes binding")
        argtypes = []
        for p in params.split(","):
            p = " ".join(p.split())
            if "*" in p:
                argtypes.append(ctypes.c_void_p)
            elif p not in ("", "void"):
                t = re.sub(r"^const ", "", p).rsplit(" ", 1)[0]
                if t not in _SCALARS:
                    raise TypeError(f"{name}: parameter {p!r} has no ctypes binding")
                argtypes.append(_SCALARS[t])
        protos[name] = (_RETURNS[ret], argtypes)
    return protos


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            raise RuntimeError(
                f"{LIB} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(posecnn_b200 has no CPU or PyTorch fallback)")
        handle = ctypes.CDLL(LIB)
        with open(HEADER) as f:
            for name, (restype, argtypes) in prototypes(f.read()).items():
                fn = getattr(handle, name)
                fn.restype, fn.argtypes = restype, argtypes
        _lib = handle
    return _lib


def check(rc: int):
    if rc != 0:
        raise RuntimeError(f"posecnn_b200 native call failed ({rc}): {lib().pcnn_last_error().decode()}")


def ptr(t):
    return None if t is None else t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def f32(x: float):
    """A float argument as ctypes.c_float.  Not needed with the header binding (a plain number converts the same way), and
    kept so that callers written against the untyped binding keep working: the bound entry points accept it unchanged."""
    return ctypes.c_float(float(x))


def workspace(tag: str, nbytes: int, device, zero: bool = False) -> torch.Tensor:
    """Scratch buffer for one native call, stream-ordered on the current stream.

    Eager calls: grow-only cache keyed by (tag, device, stream) — two streams never share a scratch buffer, and a
    buffer is only ever replaced by a larger one for the SAME stream (the old one returns to the caching allocator,
    which is stream-ordered for that stream).  Under CUDA-graph capture the buffer is allocated fresh from the graph's
    private memory pool and NOT cached: it belongs to the graph for the graph's lifetime, so a later eager call that
    needs a larger scratch can never free (or scribble over) memory a captured graph still replays into.
    `zero=True`: the buffer is zero-filled when it is created (kernels that re-arm their own tickets)."""
    device = torch.device(device)
    n = max(int(nbytes), 256)
    make = torch.zeros if zero else torch.empty
    if torch.cuda.is_current_stream_capturing():
        return make(n, dtype=torch.uint8, device=device)
    key = (tag, device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = _ws.get(key)
    if buf is None or buf.numel() < n:
        buf = make(n, dtype=torch.uint8, device=device)
        _ws[key] = buf
    return buf


def require_cuda(name: str, t: torch.Tensor, dtype, ndim=None):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (posecnn_b200 has no CPU path)")
    if t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")
    if ndim is not None and t.dim() not in (ndim if isinstance(ndim, (tuple, list)) else (ndim,)):
        raise ValueError(f"{name} must be {ndim}-dimensional")  # OP_REQUIRES rank checks of the reference
    return t.contiguous()
