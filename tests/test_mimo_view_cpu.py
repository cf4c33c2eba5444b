"""CPU tests of the multi-input fast path on per-instance systems (bmpc_tpm.cuh): tpm_fill reads only raw fields, so a block whose
condensed part is stale gives bit for bit the parameters of a freshly condensed block, and the sweeps compiled against the
field-major per-instance view (TpmPolView) give bit for bit what they give against the shared parameter block (TpmParams).
tests/hostemu/tpm_view_emu.cpp compiles both for the CPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from emu import EmuSystem
from pympc_b200.workloads import mimo

ENTRIES = {0: (8, 4, 40, 40), 1: (8, 4, 40, 40), 2: (8, 4, 12, 5)}     # csrc/tpm_shapes.inc: governor pattern, dense, dense
RAW = ("Ad", "Bd", "Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "uref")


@pytest.fixture(scope="module")
def view_lib(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "hostemu", "tpm_view_emu.cpp")
    so = str(tmp_path_factory.mktemp("tpm_view_emu") / "libtpm_view_emu.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-x", "c++", src, "-o", so])
    L = ctypes.CDLL(so)
    L.emu_tpm_fill.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    L.emu_tpm_view_step.argtypes = ([ctypes.c_int] * 4 + [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
                                    + [ctypes.c_void_p] * 2 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p])
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _fill(L, entry, sys):
    out = np.zeros(8192); diag = ctypes.c_int(-1)
    n = L.emu_tpm_fill(entry, _p(sys), _p(out), out.size, ctypes.byref(diag))
    assert n > 0, n
    return out[:n].copy(), diag.value


def _rand_cfg(rng, shape, nondiag=False):
    nx, nu, Np, Nc = shape
    A = np.eye(nx) + 0.1 * rng.standard_normal((nx, nx)); Bm = rng.standard_normal((nx, nu))

    def bounds(n, scale):
        lo = -scale * rng.uniform(0.5, 2, n); hi = scale * rng.uniform(0.5, 2, n)
        lo[rng.random(n) < 0.3] = -np.inf; hi[rng.random(n) < 0.3] = np.inf
        return lo, hi
    xmin, xmax = bounds(nx, 1.0); umin, umax = bounds(nu, 3.0); Dumin, Dumax = bounds(nu, 0.5)
    Qd = np.diag(rng.uniform(0.0, 2.0, nx))
    QDu = np.diag(rng.uniform(0.01, 1, nu))
    if nondiag:
        QDu[0, 1] = QDu[1, 0] = 0.1 * QDu[0, 0]
    return dict(Ad=A, Bd=Bm, Np=Np, Nc=Nc, Qx=Qd, QxN=Qd * rng.uniform(1, 3), Qu=np.diag(rng.uniform(0, 1, nu)), QDu=QDu,
                xmin=xmin, xmax=xmax, umin=umin, umax=umax, Dumin=Dumin, Dumax=Dumax, uref=rng.standard_normal(nu),
                eps_feas=float(rng.choice([1e3, 1e6])))


@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_tpm_fill_on_a_stale_block_equals_a_fresh_condense_bit_for_bit(entry, view_lib):
    """k_fill_view after an update fills from the raw inputs of a block whose condensed part predates them: over random bounds
    (with +-inf rows, so that rows change between free and bounded), weights and uref it equals, bit for bit, the fill of the
    same block condensed afresh with the rho the setup chose.  "QDu diagonal" is reported the same way on both"""
    shape = ENTRIES[entry]
    rng = np.random.default_rng(100 + entry)
    for trial in range(10):
        old, new = _rand_cfg(rng, shape), _rand_cfg(rng, shape, nondiag=(trial % 4 == 3))
        new["eps_feas"] = old["eps_feas"]
        E = EmuSystem(old)
        rho = float(E.get("scal", (8,))[0])
        stale = E.sys.copy()
        F = EmuSystem(new, rho=rho)
        for name in RAW:
            o = E.off[name]; n = np.size(new[name])
            stale[o:o + n] = F.sys[o:o + n]
        a, da = _fill(view_lib, entry, stale); b, db = _fill(view_lib, entry, F.sys)
        assert a.tobytes() == b.tobytes(), (trial, np.flatnonzero(a != b))
        assert da == db == (0 if trial % 4 == 3 else 1), (trial, da, db)
        if not np.array_equal(E.get("lo0", (E.mc,)), F.get("lo0", (F.mc,))):
            assert not np.array_equal(stale[E.off["lo0"]:E.off["lo0"] + E.mc], F.sys[F.off["lo0"]:F.off["lo0"] + F.mc])


def _step(L, entry, view, E, state, x, um1, xref, mode, max_ref, exchange_from, B=37, idx=23):
    codes, v, U, mm = (a.copy() for a in state)
    col = np.zeros(L.emu_tpm_slots(entry) + 8)
    xref = np.ascontiguousarray(xref, float)
    ps = L.emu_tpm_view_step(entry, view, B, idx, _p(E.sys), _p(np.ascontiguousarray(x, float)), _p(np.ascontiguousarray(um1, float)),
                             _p(xref), 0 if xref.ndim == 1 else 1, _p(codes), mode, _p(v), _p(U), max_ref, _p(mm), exchange_from, _p(col))
    return ps, (codes, v, U, mm), col


def _same(a, b):
    return all(np.asarray(p).tobytes() == np.asarray(q).tobytes() for p, q in zip(a, b))


@pytest.mark.parametrize("entry,tv", [(0, False), (1, False), (1, True), (2, False), (2, True)])
def test_sweeps_on_the_view_equal_the_sweeps_on_the_parameter_block(entry, tv, view_lib):
    """the closed loop of the host emulation's MIMO steps, each solved twice — the sweeps reading TpmParams and reading a TpmPolView
    of a 37-instance field-major array (the instance at index 23, every other instance NaN): the same U, working sets, v*, multiplier
    scale, gain column and verdict, bit for bit.  Default refinements from the stored and shifted working sets, and the straggler
    rounds' exchange mode from the team path's iterate; optionally a time-varying xref"""
    nx, nu, Np, Nc = ENTRIES[entry]
    cfg = dict(mimo(), Np=Np, Nc=Nc)
    E = EmuSystem(cfg)
    NU = Nc * nu
    state = (np.zeros(Np, np.uint64), np.zeros(E.mc), np.zeros(NU), np.zeros(1))
    x = 0.4 * np.ones(nx); um1 = np.zeros(nu)
    n_ver = n_ex = 0
    for t in range(10):
        xref = (cfg["xref"] + 0.2 * np.sin(0.3 * (np.arange(Np + 1)[:, None] + t) + np.arange(nx)[None, :])) if tv else cfg["xref"]
        mode = 0 if t == 0 else 1
        r0, s0, c0 = _step(view_lib, entry, 0, E, state, x, um1, xref, mode, 14, -1)
        r1, s1, c1 = _step(view_lib, entry, 1, E, state, x, um1, xref, mode, 14, -1)
        assert r0 == r1 and _same(s0, s1) and c0.tobytes() == c1.tobytes(), (t, r0, r1)
        # exchange mode from the team path's iterate (the straggler rounds)
        U, st, *_ = E.solve(x, um1, xref)
        assert st in (1, 2)
        vs = (state[0], E.v.copy(), state[2], state[3])
        e0, t0, d0 = _step(view_lib, entry, 0, E, vs, x, um1, xref, 2, 12, 0)
        e1, t1, d1 = _step(view_lib, entry, 1, E, vs, x, um1, xref, 2, 12, 0)
        assert e0 == e1 and _same(t0, t1) and d0.tobytes() == d1.tobytes(), (t, e0, e1)
        n_ex += e0 > 0
        if r0 > 0:
            n_ver += 1; state = s0; U = s0[2]
        else:
            state = t0 if e0 > 0 else (state[0], E.v.copy(), U.copy(), state[3])
        x = cfg["Ad"] @ x + cfg["Bd"] @ U[:nu]; um1 = U[:nu].copy()
    assert n_ver >= 5 and n_ex >= 5, (n_ver, n_ex)
