"""ctypes front-end of the host emulation of the batched DARE core (tests only): the SeqTeam build of
pympc_b200/csrc/bmpc_dare.cuh, with the argument layout of bmpc_dare (include/bmpc.h)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libdareemu.so")
_CSRC = os.path.join(_HERE, "..", "..", "pympc_b200", "csrc")


def build():
    src = os.path.join(_HERE, "dare_emu.cpp")
    deps = [src, os.path.join(_CSRC, "bmpc_core.cuh"), os.path.join(_CSRC, "bmpc_dare.cuh"),
            os.path.join(_HERE, "..", "..", "include", "bmpc.h")]
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-x", "c++", src, "-o", _SO + ".tmp"])
        os.replace(_SO + ".tmp", _SO)
    L = ctypes.CDLL(_SO)
    L.emu_dare.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 9
    L.emu_dare.restype = None
    return L


def dare(A, B, Q, R, S=None):
    """Batched inputs A [b,n,n], B [b,n,m], Q [b,n,n], R [b,m,m], S [b,n,m] or None -> (X, G, status, iters)."""
    c = lambda a: np.ascontiguousarray(a, float)
    A, B, Q, R = c(A), c(B), c(Q), c(R)
    S = None if S is None else c(S)
    b, n, m = B.shape
    X = np.zeros((b, n, n)); G = np.zeros((b, m, n)); st = np.zeros(b, np.int32); it = np.zeros(b, np.int32)
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)
    build().emu_dare(n, m, b, p(A), p(B), p(Q), p(R), p(S), p(X), p(G), p(st), p(it))
    return X, G, st, it
