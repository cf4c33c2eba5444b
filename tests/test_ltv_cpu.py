"""CPU tests of time-varying system matrices: the C entry point is declared and exported, MPCController.update_system validates its
arguments before any library call, and the batched cart-pole linearisation used by successive-linearisation loops is the
pendulum model at the upright equilibrium and the exact Jacobian elsewhere."""
import os

import numpy as np
import pytest

from conftest import ROOT
from pympc_b200 import _lib
from pympc_b200.workloads import pendulum, cartpole_rhs, cartpole_linearised


def test_update_system_is_declared_and_exported(bmpc_lib):
    header = open(os.path.join(ROOT, "include", "bmpc.h")).read()
    assert "int bmpc_update_system(bmpc_handle* h, const double* Ad, const double* Bd, int on_device);" in header
    assert "bmpc_update_system" in _lib.EXPORTS and hasattr(bmpc_lib, "bmpc_update_system")
    assert "recondensed" in [f for f, _ in _lib.BmpcStats._fields_][-1:]       # appended: the earlier fields keep their offsets


def _controllers():
    from pympc_b200 import MPCController
    c = pendulum(); B = 6
    kw = {k: c[k] for k in ("Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "eps_feas")}
    shared = MPCController(c["Ad"], c["Bd"], Np=20, batch=B, x0=np.zeros((B, 4)), **kw)
    per = MPCController(np.broadcast_to(c["Ad"], (B, 4, 4)).copy(), np.broadcast_to(c["Bd"], (B, 4, 1)).copy(), Np=20, batch=B,
                        x0=np.zeros((B, 4)), **kw)
    return c, B, shared, per


def test_update_system_validates_before_any_library_call(bmpc_lib):
    """shapes are checked first (ValueError, like the constructor); a valid call before setup() raises BmpcError"""
    from pympc_b200 import BmpcError
    import scipy.sparse as sp
    c, B, shared, per = _controllers()
    for K in (shared, per):
        with pytest.raises(ValueError, match="Ad should be a square matrix"):
            K.update_system(Ad=np.zeros((4, 3)))
        with pytest.raises(ValueError, match="Bd should be a matrix"):
            K.update_system(Bd=np.zeros((3, 1)))
        with pytest.raises(BmpcError, match="before setup"):
            K.update_system(Ad=sp.csc_matrix(c["Ad"]))
        with pytest.raises(BmpcError, match="before setup"):
            K.update_system_from_device(0, 0)
    with pytest.raises(ValueError, match="Ad should be a square matrix"):
        per.update_system(Ad=np.zeros((B + 1, 4, 4)))
    with pytest.raises(ValueError, match="Bd should be a matrix"):
        per.update_system(Bd=np.zeros((B, 4, 2)))
    with pytest.raises(ValueError, match="per-instance Ad"):
        shared.update_system(Ad=np.zeros((B, 4, 4)))
    with pytest.raises(ValueError, match="per-instance Bd"):
        shared.update_system(Bd=np.zeros((B, 4, 1)))
    # nothing reached the attributes: the reference-form view still describes the constructed system
    assert np.array_equal(shared.Ad, c["Ad"]) and np.array_equal(per.Ad, c["Ad"])


def test_assigning_Ad_keeps_the_reference_meaning(bmpc_lib):
    """K.Ad = ... is a plain attribute (the reference reads it in setup()); only update_system reaches a set-up controller"""
    c, B, shared, per = _controllers()
    shared.Ad = 2 * c["Ad"]
    assert shared._h is None and np.array_equal(shared.Ad, 2 * c["Ad"])


def test_cartpole_linearisation_at_the_equilibrium_is_the_pendulum_model():
    c = pendulum()
    Ad, Bd = cartpole_linearised(np.zeros((5, 4)), np.zeros((5, 1)))
    assert Ad.shape == (5, 4, 4) and Bd.shape == (5, 4, 1)
    assert np.max(np.abs(Ad - c["Ad"])) < 1e-12 and np.max(np.abs(Bd - c["Bd"])) < 1e-12
    assert np.array_equal(cartpole_rhs(np.zeros((2, 4)), np.zeros(2)), np.zeros((2, 4)))


def test_cartpole_linearisation_matches_finite_differences():
    rng = np.random.default_rng(3); B, Ts, h = 64, 0.05, 1e-6
    X = np.column_stack([rng.uniform(-1, 1, B), rng.uniform(-2, 2, B), rng.uniform(-0.8, 0.8, B), rng.uniform(-3, 3, B)])
    U = rng.uniform(-10, 10, (B, 1))
    Ad, Bd = cartpole_linearised(X, U, Ts=Ts)
    J = np.zeros((B, 4, 4))
    for j in range(4):
        e = np.zeros(4); e[j] = h
        J[:, :, j] = (cartpole_rhs(X + e, U) - cartpole_rhs(X - e, U)) / (2 * h)
    Jb = (cartpole_rhs(X, U + h) - cartpole_rhs(X, U - h)) / (2 * h)
    assert np.max(np.abs(Ad - (np.eye(4) + Ts * J))) < 1e-6
    assert np.max(np.abs(Bd[:, :, 0] - Ts * Jb)) < 1e-6
    # the upright pole falls: d(omega)/d(theta) > 0 near theta = 0
    assert (Ad[np.abs(X[:, 2]) < 0.2, 3, 2] > 0).all()


def test_cartpole_functions_accept_torch_tensors():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(4)
    X = rng.standard_normal((8, 4)); U = rng.standard_normal((8, 1))
    Ad, Bd = cartpole_linearised(X, U)
    At, Bt = cartpole_linearised(torch.from_numpy(X), torch.from_numpy(U))
    assert isinstance(At, torch.Tensor) and At.is_contiguous() and Bt.is_contiguous()
    assert np.max(np.abs(At.numpy() - Ad)) < 1e-15 and np.max(np.abs(Bt.numpy() - Bd)) < 1e-15
    assert np.max(np.abs(cartpole_rhs(torch.from_numpy(X), torch.from_numpy(U)).numpy() - cartpole_rhs(X, U))) < 1e-15
