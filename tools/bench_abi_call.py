"""Host cost of one call into libposecnn_b200.so through ctypes: the training step's loss-gradient adjoint, pcnn_up8_heads_bwd
(27 arguments), on a path its argument check rejects before any CUDA work (C = 7), so it runs on a machine without a GPU.

  typed    the package's binding: argtypes from include/posecnn_b200.h, ptr(t) as a plain int, plain Python scalars
  untyped  a second handle of the same library without argtypes, every argument wrapped in Python (c_void_p / c_float /
           c_size_t), the way the package called it before it bound from the header

The two run alternately, --repeats times --calls calls each; the median microseconds per call is printed as one JSON line.
The numbers are host CPU time and depend on the machine's CPU, not on the GPU.

    python tools/bench_abi_call.py [--calls 20000] [--repeats 7]
"""
import argparse
import ctypes
import json
import os
import platform
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from posecnn_b200 import _lib                                    # noqa: E402
from posecnn_b200.build import LIB, build_native                 # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20000)
    ap.add_argument("--repeats", type=int, default=7)
    a = ap.parse_args()
    build_native()
    B, h, w, C = 1, 8, 8, 7
    t = {k: torch.zeros(16) for k in ("prob", "score", "gt", "cls", "lowres", "bv", "centers", "vtx", "d_sc", "d_vt", "dbias", "ws")}
    lib, plain = _lib.lib, ctypes.CDLL(LIB)
    ptr = _lib.ptr

    def old_ptr(x):                                              # the helpers of the untyped binding
        return ctypes.c_void_p(0) if x is None else ctypes.c_void_p(x.data_ptr())

    def old_f32(x):
        return ctypes.c_float(float(x))

    def call_typed():
        return lib().pcnn_up8_heads_bwd(ptr(t["prob"]), ptr(t["score"]), ptr(t["gt"]), ptr(t["cls"]), 1.0, 0.7, ptr(t["lowres"]),
                                        ptr(t["bv"]), ptr(t["centers"]), ptr(None), ptr(None), ptr(t["vtx"]), 2.0, 10.0, 1.0, B, h, w, C, 64,
                                        160, ptr(t["d_sc"]), ptr(t["d_vt"]), ptr(t["dbias"]), ptr(t["ws"]), t["ws"].numel(), 0)

    def call_untyped():
        p, f = old_ptr, old_f32
        return plain.pcnn_up8_heads_bwd(p(t["prob"]), p(t["score"]), p(t["gt"]), p(t["cls"]), f(1.0), f(0.7), p(t["lowres"]), p(t["bv"]),
                                        p(t["centers"]), p(None), p(None), p(t["vtx"]), f(2.0), f(10.0), f(1.0), B, h, w, C, 64, 160,
                                        p(t["d_sc"]), p(t["d_vt"]), p(t["dbias"]), p(t["ws"]), ctypes.c_size_t(t["ws"].numel()),
                                        ctypes.c_void_p(0))

    res = {"typed": [], "untyped": []}
    for _ in range(a.repeats):
        for name, fn in (("typed", call_typed), ("untyped", call_untyped)):
            assert fn() == -1 and b"(C = 7)" in lib().pcnn_last_error()
            t0 = time.perf_counter()
            for _ in range(a.calls):
                fn()
            res[name].append((time.perf_counter() - t0) / a.calls * 1e6)
    out = dict(metric="host microseconds per pcnn_up8_heads_bwd call (27 arguments, rejected before CUDA work)",
               cpu=platform.processor() or platform.machine(), python=platform.python_version(), calls=a.calls, repeats=a.repeats)
    out.update({f"{k}_us": statistics.median(v) for k, v in res.items()})
    out["typed_over_untyped"] = out["typed_us"] / out["untyped_us"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
