"""ctypes front-end of the host emulation of the batched Kalman filter step (tests only): the host build of
pympc_b200/csrc/bmpc_kf.cuh run over a batch with the library's layouts (see kf_emu.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libkfemu.so")
_CSRC = os.path.join(_HERE, "..", "..", "pympc_b200", "csrc")
_lib = None


def build():
    global _lib
    src = os.path.join(_HERE, "kf_emu.cpp")
    deps = [src, os.path.join(_CSRC, "bmpc_core.cuh"), os.path.join(_CSRC, "bmpc_kf.cuh"),
            os.path.join(_HERE, "..", "..", "include", "bmpc.h")]
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-x", "c++", src, "-o", _SO + ".tmp"])
        os.replace(_SO + ".tmp", _SO)
        _lib = None
    if _lib is None:
        L = ctypes.CDLL(_SO)
        L.emu_kf_layout.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p]
        L.emu_kf_step.argtypes = [ctypes.c_int] * 6 + [ctypes.c_void_p] * 7
        L.emu_kf_step.restype = None
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _pk(n):
    """(rows, cols) of the packed upper triangle, in the library's order"""
    return np.triu_indices(n)


class KalmanFilter:
    """B filters in the library's layout.  Model arrays 2-D (shared: packed, n_sys = 1) or 3-D (per instance: field-major)."""

    def __init__(self, x0, A, B, C, Qn, Rn, P0):
        self.L = build()
        mats = [np.asarray(a, float) for a in (A, B, C, Qn, Rn)]
        self.per = mats[0].ndim == 3
        self.nx, self.nu, self.ny = mats[0].shape[-1], mats[1].shape[-1], mats[2].shape[-2]
        x0 = np.asarray(x0, float)
        self.B = x0.shape[0]
        sz = np.zeros(3, np.int32); self.L.emu_kf_layout(self.nx, self.nu, self.ny, _p(sz))
        self.nmodel, self.nP, self.nws = (int(v) for v in sz)
        self.x = np.ascontiguousarray(x0.copy())
        self.mats = None
        self.set_model(*mats)
        C = mats[2]
        self.y = np.einsum("...ij,bj->bi", C, self.x) if C.ndim == 2 else np.einsum("bij,bj->bi", C, self.x)
        self.y = np.ascontiguousarray(self.y)
        r, c = _pk(self.nx)
        self.P = np.ascontiguousarray(np.asarray(P0, float)[:, r, c].T)                   # [nP, B]
        self.ws = np.zeros((self.nws, self.B))
        self.status = np.ones(self.B, np.int32)

    def set_model(self, A=None, B=None, C=None, Qn=None, Rn=None):
        n = self.B if self.per else 1
        fields = []
        cur = self.fields() if self.mats is not None else None
        for k, a in enumerate((A, B, C, Qn, Rn)):
            fields.append(np.broadcast_to(np.asarray(a, float), (n,) + np.shape(a)[-2:]).reshape(n, -1) if a is not None
                          else cur[k])
        flat = np.concatenate(fields, axis=1)                                            # [n, model]
        self.mats = np.ascontiguousarray(flat.T if self.per else flat[0])

    def fields(self):
        """the model's fields as [n_sys, count] arrays"""
        flat = self.mats.T if self.per else self.mats[None]
        nx, nu, ny = self.nx, self.nu, self.ny
        cuts = np.cumsum([nx * nx, nx * nu, ny * nx, nx * nx])
        return np.split(flat, cuts, axis=1)

    def predict(self, u):
        u = np.ascontiguousarray(np.broadcast_to(np.asarray(u, float), (self.B, self.nu)))
        self._step(0, u)

    def update(self, ym):
        ym = np.ascontiguousarray(np.broadcast_to(np.asarray(ym, float), (self.B, self.ny)))
        self._step(1, ym)

    def _step(self, mode, a):
        self.L.emu_kf_step(self.nx, self.nu, self.ny, self.B, self.B if self.per else 1, mode, _p(self.mats), _p(a), _p(self.x),
                           _p(self.y), _p(self.P), _p(self.ws), _p(self.status))

    def cov(self):
        """P [B, nx, nx]"""
        r, c = _pk(self.nx)
        P = np.zeros((self.B, self.nx, self.nx))
        P[:, r, c] = self.P.T; P[:, c, r] = self.P.T
        return P

    def gain(self):
        """the gain K [B, nx, ny] of the last successful update (the workspace after it)"""
        off = 2 * self.nx * self.nx
        return self.ws[off:off + self.nx * self.ny].T.reshape(self.B, self.nx, self.ny)
