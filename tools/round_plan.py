"""The solver's round policy (pympc_b200/csrc/bmpc_rounds.cuh::bmpc_plan_round) from Python, for the host-emulation studies and the
schedule test: round_plan.cpp compiled with g++ (once, under tools/build/), loaded with ctypes."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = [os.path.join(_HERE, "round_plan.cpp"), os.path.join(_HERE, "..", "pympc_b200", "csrc", "bmpc_rounds.cuh")]
_SO = os.path.join(_HERE, "build", "libround_plan.so")
_LIB = None

# names of the enums of bmpc_rounds.cuh, in their order
FAMILIES = ("tpi", "tpi_view", "tpm", "team")
ADMM = ("none", "tpi", "team")
POLISH = ("tpi", "tpm", "schur", "check")
WS = {-1: "record", 0: "stored", 1: "shifted", 2: "from_v"}


def _lib():
    global _LIB
    if _LIB is None:
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(p) for p in _SRC):
            subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", _SRC[0], "-o", _SO + ".tmp"])
            os.replace(_SO + ".tmp", _SO)
        _LIB = ctypes.CDLL(_SO)
        _LIB.round_plan.argtypes = [ctypes.c_int] * 11 + [ctypes.c_void_p]
    return _LIB


def plan_round(family, round, total, cold, codes_valid=False, polish=1, first_iters=0, cold_iters=0, max_iter=4000, pdas_steps=10,
               shift_warm=1):
    """The library's plan of the next round for a handle of `family` (FAMILIES) with these options, after `round` rounds and
    `total` ADMM iterations of a solve that started cold or warm: a dict of the plan's fields (kinds by name; ws None for the
    polishes that take no working sets), or None when the iteration budget is spent."""
    out = np.zeros(10, np.int32)
    if not _lib().round_plan(FAMILIES.index(family), polish, first_iters, cold_iters, max_iter, pdas_steps, shift_warm, round, total,
                             int(cold), int(codes_valid), out.ctypes.data_as(ctypes.c_void_p)):
        return None
    p = dict(zip(("admm", "chunk", "polish", "ws", "capA", "capB", "cap", "exchange", "reset", "infeas"), out.tolist()))
    p["admm"], p["polish"] = ADMM[p["admm"]], POLISH[p["polish"]]
    p["ws"] = WS[p["ws"]] if p["polish"] in ("tpi", "tpm") else None
    return p
