"""CPU tests of time-varying weights, bounds and uref (MPCController.update_system keywords / bmpc_update_problem): the C entry point
is declared and exported next to an unchanged bmpc_update_system, the arguments are validated before any library call with the
constructor's messages, and the fast path's per-instance parameter fill reads only raw fields, so that a block whose condensed part
is stale gives bit for bit the parameters of a freshly condensed block."""
import ctypes
import os

import numpy as np
import pytest

from conftest import ROOT
from pympc_b200 import _lib
from pympc_b200.workloads import pendulum

KEYS = ("Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "eps_feas")


def test_update_problem_is_declared_and_exported(bmpc_lib):
    header = open(os.path.join(ROOT, "include", "bmpc.h")).read()
    flat = " ".join(header.split())
    assert ("int bmpc_update_problem(bmpc_handle* h, const double* Ad, const double* Bd, const double* Qx, const double* QxN, "
            "const double* Qu, const double* QDu, const double* xmin, const double* xmax, const double* umin, "
            "const double* umax, const double* Dumin, const double* Dumax, const double* uref, int on_device);") in flat
    assert "int bmpc_update_system(bmpc_handle* h, const double* Ad, const double* Bd, int on_device);" in header
    assert "bmpc_update_problem" in _lib.EXPORTS and hasattr(bmpc_lib, "bmpc_update_problem")
    assert len(bmpc_lib.bmpc_update_problem.argtypes) == 15
    assert len(bmpc_lib.bmpc_update_system.argtypes) == 4


def _controllers(B=6):
    from pympc_b200 import MPCController
    c = pendulum()
    kw = {k: c[k] for k in KEYS}
    shared = MPCController(c["Ad"], c["Bd"], Np=20, batch=B, x0=np.zeros((B, 4)), **kw)
    per = MPCController(np.broadcast_to(c["Ad"], (B, 4, 4)).copy(), np.broadcast_to(c["Bd"], (B, 4, 1)).copy(), Np=20, batch=B,
                        x0=np.zeros((B, 4)), **kw)
    return c, B, shared, per


@pytest.mark.parametrize("name,bad,msg", [
    ("Qx", np.eye(3), "Qx should be a matrix of shape"), ("QxN", np.eye(5), "QxN should be a square matrix"),
    ("Qu", np.eye(2), "Qu should be a square matrix"), ("QDu", np.zeros((1, 2)), "QDu should be a square matrix"),
    ("xmin", np.zeros(3), "xmin should be a vector"), ("xmax", np.zeros((2, 2)), "xmax should be a vector"),
    ("umin", np.zeros(2), "umin should be a vector"), ("umax", np.zeros((4, 1)), "umax should be a vector"),
    ("Dumin", np.zeros(0), "Dumin should be a vector"), ("Dumax", np.zeros(3), "Dumax should be a vector"),
    ("uref", np.zeros(2), "uref should be a vector")])
def test_update_system_validates_every_array_before_any_library_call(bmpc_lib, name, bad, msg):
    """a wrong shape raises the constructor's ValueError, on shared and per-instance controllers, before the not-set-up check"""
    c, B, shared, per = _controllers()
    for K in (shared, per):
        with pytest.raises(ValueError, match=msg):
            K.update_system(**{name: bad})
    with pytest.raises(ValueError, match=msg):
        per.update_system(**{name: np.zeros((B + 1,) + np.shape(c[name] if name in c else np.zeros(1)))})


@pytest.mark.parametrize("name", ["Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "uref"])
def test_per_instance_arrays_need_a_per_instance_controller(bmpc_lib, name):
    c, B, shared, per = _controllers()
    base = np.atleast_1d(np.asarray(c.get(name, np.zeros(1)), float))
    if name == "uref":
        base = np.zeros(1)
    batched = np.broadcast_to(base, (B,) + base.shape).copy()
    with pytest.raises(ValueError, match=f"per-instance {name} of shape \\(batch, ...\\) needs a controller set up with per-instance"):
        shared.update_system(**{name: batched})
    # the same array on a per-instance controller passes validation and stops at the missing setup()
    from pympc_b200 import BmpcError
    with pytest.raises(BmpcError, match="before setup"):
        per.update_system(**{name: batched})


def test_update_system_accepts_the_reference_forms_and_keeps_attributes_until_a_valid_call(bmpc_lib):
    """dense or scipy.sparse weights (quirk Q16), vectors in the reference's __is_vector__ sense ((n,), (1, n)); a failing call
    changes no attribute; assigning an attribute keeps the reference meaning (no effect until setup())"""
    import scipy.sparse as sp
    from pympc_b200 import BmpcError
    c, B, shared, per = _controllers()
    for K in (shared, per):
        with pytest.raises(BmpcError, match="before setup"):
            K.update_system(Qx=sp.csc_matrix(2 * c["Qx"]), QDu=np.eye(1), umax=np.array([[3.0]]), xmin=-np.ones((1, 4)),
                            uref=[0.5])
        assert np.array_equal(K.umax, c["umax"]) and np.array_equal(K.uref, np.zeros(1))
        with pytest.raises(BmpcError, match="before setup"):
            K.update_system_from_device(umax=0)
    shared.xmin = -2 * np.ones(4)
    assert shared._h is None and np.array_equal(shared.xmin, -2 * np.ones(4))


@pytest.fixture(scope="module")
def fill_lib(tmp_path_factory):
    """tests/hostemu/tpi_fill_emu.cpp (tpi_fill_pol compiled for the CPU), built with g++ into a temporary directory"""
    import subprocess
    src = os.path.join(ROOT, "tests", "hostemu", "tpi_fill_emu.cpp")
    so = str(tmp_path_factory.mktemp("tpi_fill_emu") / "libtpi_fill_emu.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-x", "c++", src, "-o", so])
    return ctypes.CDLL(so)


def _emu_fill(L, shape, sys):
    nx, nu, Np, Nc = shape
    out = np.zeros(4096)
    f = L.emu_tpi_fill_pol
    f.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    n = f(nx, nu, Np, Nc, sys.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p), out.size)
    assert n > 0, n
    return out[:n].copy()


@pytest.mark.parametrize("shape", [(4, 1, 20, 20), (2, 1, 20, 20), (4, 1, 10, 10), (4, 1, 20, 10)])
def test_fast_path_fill_on_a_stale_block_equals_a_fresh_condense_bit_for_bit(shape, fill_lib):
    """the per-instance parameter view after an update is built from the raw inputs of a block whose condensed part predates them:
    over random bounds (with +-inf rows, so that rows change between free and bounded), weights and uref it equals, bit for bit,
    the fill of the same block condensed afresh with the rho the setup chose (what k_condense_list does later)"""
    from emu import EmuSystem
    nx, nu, Np, Nc = shape
    rng = np.random.default_rng(sum(shape))
    inf = np.inf

    def rand_cfg():
        A = np.eye(nx) + 0.1 * rng.standard_normal((nx, nx)); Bm = rng.standard_normal((nx, 1))
        def bounds(n, scale):
            lo = -scale * rng.uniform(0.5, 2, n); hi = scale * rng.uniform(0.5, 2, n)
            lo[rng.random(n) < 0.3] = -inf; hi[rng.random(n) < 0.3] = inf
            return lo, hi
        xmin, xmax = bounds(nx, 1.0); umin, umax = bounds(1, 3.0); Dumin, Dumax = bounds(1, 0.5)
        Qd = np.diag(rng.uniform(0.0, 2.0, nx))
        return dict(Ad=A, Bd=Bm, Np=Np, Nc=Nc, Qx=Qd, QxN=Qd * rng.uniform(1, 3), Qu=np.array([[rng.uniform(0, 1)]]),
                    QDu=np.array([[rng.uniform(0.01, 1)]]), xmin=xmin, xmax=xmax, umin=umin, umax=umax, Dumin=Dumin, Dumax=Dumax,
                    uref=rng.standard_normal(1), eps_feas=float(rng.choice([1e3, 1e6])))

    raw = ("Ad", "Bd", "Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "uref")
    for trial in range(12):
        old, new = rand_cfg(), rand_cfg()
        new["eps_feas"] = old["eps_feas"]                  # setup-time (rho_e)
        E = EmuSystem(old)
        rho = float(E.get("scal", (8,))[0])
        stale = E.sys.copy()
        F = EmuSystem(new, rho=rho)                         # condensed afresh with the kept rho
        for name in raw:                                    # the update: raw inputs only, condensed part untouched
            o = E.off[name]; n = np.size(new[name])
            stale[o:o + n] = F.sys[o:o + n]
        assert np.array_equal(stale[E.off["scal"]:E.off["scal"] + 4], F.sys[F.off["scal"]:F.off["scal"] + 4]), trial
        a = _emu_fill(fill_lib, shape, stale); b = _emu_fill(fill_lib, shape, F.sys)
        assert a.tobytes() == b.tobytes(), (trial, np.flatnonzero(a != b))
        # and the stale block's condensed rows really are stale when a row changed between free and bounded
        lo_o, lo_n = E.get("lo0", (E.mc,)), F.get("lo0", (F.mc,))
        if not np.array_equal(lo_o, lo_n):
            assert not np.array_equal(stale[E.off["lo0"]:E.off["lo0"] + E.mc], lo_n)
