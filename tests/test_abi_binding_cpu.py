"""The ctypes binding of libposecnn_b200.so is the header's: every `pcnn_*` prototype of include/posecnn_b200.h sets the
argtypes / restype of its entry point (posecnn_b200/_lib.py), every call site in the repository passes exactly the declared
number of arguments, a mismatch raises in Python before C is entered, and plain Python scalars reach C with their values.
Every native call here is one the library's argument checks reject before any CUDA work, so no GPU is needed."""
import ast
import ctypes
import os
import re
import subprocess

import pytest
import torch

from posecnn_b200 import _lib
from posecnn_b200.build import HEADER

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_prototypes():
    with open(HEADER) as f:
        return _lib.prototypes(f.read())


def python_files():
    """The tracked .py files; outside a git checkout, every .py file except those under hidden or build directories."""
    try:
        return subprocess.run(["git", "ls-files", "*.py"], cwd=ROOT, capture_output=True, text=True, check=True).stdout.split()
    except (OSError, subprocess.CalledProcessError):
        files = []
        for d, dirs, names in os.walk(ROOT):
            dirs[:] = [x for x in dirs if not x.startswith(".") and x != "_build"]
            files += [os.path.relpath(os.path.join(d, n), ROOT) for n in names if n.endswith(".py")]
        return files


def test_binding_is_complete(native_lib):
    with open(HEADER) as f:
        declared = set(re.findall(r"\b(pcnn_[a-z0-9_]+)\s*\(", f.read()))
    protos = header_prototypes()
    assert set(protos) == declared and len(protos) >= 70
    for name, (restype, argtypes) in protos.items():
        fn = getattr(native_lib, name)
        assert fn.restype is restype and fn.argtypes == argtypes, name
    assert protos["pcnn_last_error"] == (ctypes.c_char_p, [])
    assert protos["pcnn_hough_vote_workspace_bytes"][1] == [ctypes.c_int] * 5 + [ctypes.c_float, ctypes.c_void_p]
    assert protos["pcnn_sgd_momentum"][1][3] is ctypes.c_size_t and protos["pcnn_augment_color_fwd"][1][5] is ctypes.c_void_p


def test_unknown_types_are_refused():
    assert _lib.prototypes("/* int pcnn_gone(int); */ const char* pcnn_a(void);\nint pcnn_b(const uint64_t* k, double x, size_t n);") == \
        {"pcnn_a": (ctypes.c_char_p, []), "pcnn_b": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_double, ctypes.c_size_t])}
    with pytest.raises(TypeError, match="pcnn_half"):
        _lib.prototypes("int pcnn_ok(int n);\nint pcnn_half(__half h);")
    with pytest.raises(TypeError, match="pcnn_void"):
        _lib.prototypes("void pcnn_void(int n);")


def test_every_call_site_matches_the_header():
    """ctypes passes surplus arguments through silently even with argtypes set, so the count is checked here, exactly."""
    arity = {name: len(argtypes) for name, (_, argtypes) in header_prototypes().items()}
    bad, seen = [], 0
    for path in python_files():
        with open(os.path.join(ROOT, path)) as f:
            tree = ast.parse(f.read(), path)
        for node in ast.walk(tree):
            if not (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr in arity):
                continue
            if any(isinstance(a, ast.Starred) for a in node.args):
                continue
            seen += 1
            if len(node.args) != arity[node.func.attr] or node.keywords:
                bad.append(f"{path}:{node.lineno}: {node.func.attr} takes {arity[node.func.attr]} arguments, the call passes "
                           f"{len(node.args)}" + (f" and {len(node.keywords)} keywords" if node.keywords else ""))
    assert seen >= 150
    assert not bad, "\n".join(bad)


def test_mismatches_raise_before_c_is_entered(native_lib):
    assert native_lib.pcnn_hard_label_bwd(1, 1, 1, 1, None, None, None) == -1              # leaves a known error message
    err = native_lib.pcnn_last_error()
    with pytest.raises(TypeError):
        native_lib.pcnn_hard_label_bwd(*(1, 1, 1, 1, None, None))                           # one argument short (starred: not a call site)
    with pytest.raises(ctypes.ArgumentError):
        native_lib.pcnn_hard_label_bwd(1, 1, 1, 1, 1.5, None, None)                         # a float where a pointer belongs
    with pytest.raises(ctypes.ArgumentError):
        native_lib.pcnn_hard_label_bwd(1, 1, 1, 1, torch.zeros(4), None, None)              # a tensor without ptr()
    with pytest.raises(ctypes.ArgumentError):
        native_lib.pcnn_hard_label_bwd(1, 1, 1.0, 1, None, None, None)                      # a float where an int belongs
    assert native_lib.pcnn_last_error() == err


def test_plain_scalars_reach_c(native_lib):
    buf = ctypes.create_string_buffer(64)                      # any non-NULL host address: the checks fail before it is read

    def up8(C, h, w, ws):
        return native_lib.pcnn_up8_heads_bwd_ex(buf, buf, buf, buf, 1.0, 0.7, buf, None, None, buf, buf, 2.0, 10.0, 1.0, 1, h, w, C,
                                                64, 160, buf, buf, buf, buf, ws, None)
    assert up8(7, 8, 8, 1 << 20) == -1 and b"(C = 7)" in native_lib.pcnn_last_error()                       # int
    assert up8(2, 60, 80, 16) == -1 and b"workspace too small (16 < 640)" in native_lib.pcnn_last_error()   # size_t
    assert native_lib.pcnn_average_distance_fwd(None, None, None, None, None, 1, 22, 100, -0.25, None, None, None, 0, None) == -1
    assert b"got -0.250000" in native_lib.pcnn_last_error()                                                  # float
    # the wrapped values of the untyped binding still convert the same way
    assert up8(2, 60, 80, ctypes.c_size_t(16)) == -1 and b"workspace too small (16 < 640)" in native_lib.pcnn_last_error()
    assert native_lib.pcnn_average_distance_fwd(None, None, None, None, None, 1, 22, 100, _lib.f32(-0.5), None, None, None, 0, None) == -1
    assert b"got -0.500000" in native_lib.pcnn_last_error()
