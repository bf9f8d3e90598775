"""Build libposecnn_b200.so (hand-written sm_90a CUDA + C ABI) in-tree with nvcc.

The shared object lands in posecnn_b200/_build/ (git-ignored) next to the sources, so the
package is importable from the repository tree.  nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "_build")
LIB = os.path.join(OUT_DIR, "libposecnn_b200.so")
HEADER = os.path.join(os.path.dirname(HERE), "include", "posecnn_b200.h")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "-shared", "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; cannot build libposecnn_b200.so")


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [HEADER, os.path.abspath(__file__)]  # the flags live here
    return any(os.path.getmtime(d) > t for d in deps)


def build_native(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    os.makedirs(OUT_DIR, exist_ok=True)
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(OUT_DIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [_nvcc()] + [f for f in NVCC_FLAGS if f != "-shared"] + ["-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{out}")
        if verbose and out:
            print(out)
    cmd = [_nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build_native(force=True, verbose=True))
