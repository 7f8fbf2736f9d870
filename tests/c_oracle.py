"""Compiles the plain-C oracles of tests/ (each includes the pinned oracle/splashsurf_oracle.c) with the pinned oracle's compiler flags:
single precision and un-contracted, so every operation is one f32 rounding in the order written.  Not a test module."""
import ctypes as C
import os
import subprocess
import tempfile

_LIBS = {}


def build(source, bindings):
    """The library of tests/<source>, compiled into a temporary directory once per session, with the ctypes signatures of `bindings`
    ({name: (restype, argtypes)}) applied."""
    if source not in _LIBS:
        name = os.path.splitext(source)[0]
        so = os.path.join(tempfile.mkdtemp(prefix=name + "_"), "lib" + name + ".so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-std=c11", "-ffp-contract=off", "-fno-fast-math",
                               "-mfma", "-mavx2", "-o", so, os.path.join(os.path.dirname(os.path.abspath(__file__)), source), "-lm", "-lpthread"])
        _LIBS[source] = C.CDLL(so)
    L = _LIBS[source]
    for fn, (restype, argtypes) in bindings.items():
        getattr(L, fn).restype = restype
        getattr(L, fn).argtypes = argtypes
    return L
