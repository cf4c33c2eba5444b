"""CPU tests of the batched Kalman filter (csrc/bmpc_kf.cuh): the per-instance step that k_kf / k_kf_pi run, built for the host
(tests/hostemu/kf_emu.cpp) with the library's layouts, against the numpy filter of tests/kf_oracle.py (plain covariance update,
independent of the Joseph form); failure isolation; the fixed point of the recursion against kalman_design_simple's gain; and
the argument checks of pympc_b200.kalman.KalmanFilter and the update_system methods.  No GPU needed."""
import numpy as np
import pytest

import kf_emu
from kf_oracle import KalmanFilter as Ref
from oracle.kalman_design import kalman_design_simple as okds
from pympc_b200 import BmpcError, kalman
from pympc_b200.workloads import mimo
from test_kalman_cpu import pendulum_5ms, point_mass_example

SHAPES = [(1, 1, 1), (2, 1, 1), (3, 2, 2), (4, 1, 2), (8, 4, 4), (5, 3, 7), (16, 2, 8), (32, 3, 1), (32, 1, 32)]


def spd(rng, b, n, lo=0.5):
    Z = rng.standard_normal((b, n, n))
    return Z @ Z.transpose(0, 2, 1) / n + lo * np.eye(n)


def random_models(rng, b, nx, nu, ny):
    """b random models, spectral radius of A in [0.5, 1.2] (half of them unstable when b is even)"""
    A = rng.standard_normal((b, nx, nx))
    rho = np.where(np.arange(b) % 2 == 0, rng.uniform(0.5, 0.95, b), rng.uniform(1.02, 1.2, b))
    A *= (rho / np.abs(np.linalg.eigvals(A)).max(-1))[:, None, None]
    return (A, rng.standard_normal((b, nx, nu)), rng.standard_normal((b, ny, nx)), 0.1 * spd(rng, b, nx), spd(rng, b, ny))


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("nx,nu,ny", SHAPES)
def test_emulated_step_matches_oracle(nx, nu, ny):
    """50 predict/update steps of 6 per-instance filters (3 stable, 3 unstable): every step within 1e-12 (relative) of the numpy
    filter's step from the same x and P, and the whole run within 1e-9 of the free-running numpy filter (the two recursions
    round differently, and the difference is carried from step to step); P exactly symmetric and positive definite.  The same
    models as one shared model per filter give bit-identical results (k_kf and k_kf_pi differ only in how a model element is
    addressed)."""
    rng = np.random.default_rng(100 * nx + 10 * nu + ny)
    b = 6
    A, Bm, C, Qn, Rn = random_models(rng, b, nx, nu, ny)
    X0 = rng.standard_normal((b, nx)); P0 = spd(rng, b, nx)
    E = kf_emu.KalmanFilter(X0, A, Bm, C, Qn, Rn, P0)
    refs = [Ref(X0[i], A[i], Bm[i], C[i], Qn[i], Rn[i], P0[i]) for i in range(b)]
    free = [Ref(X0[i], A[i], Bm[i], C[i], Qn[i], Rn[i], P0[i]) for i in range(b)]
    shared = [kf_emu.KalmanFilter(X0[i:i + 1], A[i], Bm[i], C[i], Qn[i], Rn[i], P0[i:i + 1]) for i in range(b)]
    for t in range(50):
        U = rng.standard_normal((b, nu)); Y = rng.standard_normal((b, ny))
        for i in range(b):
            refs[i].x, refs[i].P, refs[i].y = E.x[i].copy(), E.cov()[i], E.y[i].copy()
        E.predict(U); E.update(Y)
        for i in range(b):
            refs[i].predict(U[i]); refs[i].update(Y[i])
            free[i].predict(U[i]); free[i].update(Y[i])
            shared[i].predict(U[i:i + 1]); shared[i].update(Y[i:i + 1])
        P = E.cov()
        assert (E.status == 1).all()
        for i in range(b):
            assert rel(E.x[i], refs[i].x) < 1e-12 and rel(P[i], refs[i].P) < 1e-12, (t, i)
            assert rel(E.x[i], free[i].x) < 1e-9 and rel(P[i], free[i].P) < 1e-9, (t, i)
            assert np.array_equal(shared[i].x[0], E.x[i]) and np.array_equal(shared[i].P[:, 0], E.P[:, i])
    assert np.array_equal(P, P.transpose(0, 2, 1))
    assert (np.linalg.eigvalsh(P) > 0).all()


@pytest.mark.parametrize("nx,nu,ny", [(1, 1, 1), (4, 1, 2), (8, 4, 4), (32, 2, 32)])
def test_emulated_step_with_a_model_that_changes_every_step(nx, nu, ny):
    """every step a new (A, B, C, Qn, Rn) per instance, set between update and predict as bmpc_est_set_model does: each step
    within 1e-12 (relative) of the numpy filter's step with the new model from the same x and P"""
    rng = np.random.default_rng(7 + nx)
    b = 4
    models = random_models(rng, b, nx, nu, ny)
    X0 = rng.standard_normal((b, nx)); P0 = spd(rng, b, nx)
    E = kf_emu.KalmanFilter(X0, *models, P0)
    refs = [Ref(X0[i], *(m[i] for m in models), P0[i]) for i in range(b)]
    for t in range(50):
        A, Bm, C, Qn, Rn = random_models(rng, b, nx, nu, ny)
        E.set_model(A, Bm, C, Qn, Rn)
        x_prev, P_prev = E.x.copy(), E.cov()
        U = rng.standard_normal((b, nu)); Y = rng.standard_normal((b, ny))
        E.predict(U); E.update(Y)
        for i in range(b):
            r = refs[i]
            r.A, r.B, r.C, r.Qn, r.Rn = A[i], Bm[i], C[i], Qn[i], Rn[i]
            r.x, r.P = x_prev[i], P_prev[i]
            r.predict(U[i]); r.update(Y[i])
            assert rel(E.x[i], r.x) < 1e-12 and rel(E.cov()[i], r.P) < 1e-12, (t, i)


def test_failure_isolation():
    """an indefinite Rn on two instances: status -2 there, x and P of those instances unchanged by the update; every other
    instance bit-for-bit what it is without them"""
    rng = np.random.default_rng(3)
    b, nx, nu, ny = 9, 4, 1, 2
    A, Bm, C, Qn, Rn = random_models(rng, b, nx, nu, ny)
    X0 = rng.standard_normal((b, nx)); P0 = spd(rng, b, nx)
    clean = kf_emu.KalmanFilter(X0, A, Bm, C, Qn, Rn, P0)
    Rbad = Rn.copy(); Rbad[2] = [[1.0, 2.0], [2.0, 1.0]]; Rbad[7] = -np.eye(ny) * 1e6
    E = kf_emu.KalmanFilter(X0, A, Bm, C, Qn, Rbad, P0)
    keep = np.setdiff1d(np.arange(b), [2, 7])
    for t in range(5):
        U = rng.standard_normal((b, nu)); Y = rng.standard_normal((b, ny))
        clean.predict(U); E.predict(U)
        x_before, P_before = E.x.copy(), E.P.copy()
        clean.update(Y); E.update(Y)
        assert list(E.status) == [1, 1, -2, 1, 1, 1, 1, -2, 1]
        assert np.array_equal(E.x[[2, 7]], x_before[[2, 7]]) and np.array_equal(E.P[:, [2, 7]], P_before[:, [2, 7]])
        assert np.array_equal(E.x[keep], clean.x[keep]) and np.array_equal(E.P[:, keep], clean.P[:, keep])
    # a non-finite Rn is a failure too
    Rnan = Rn.copy(); Rnan[4, 0, 0] = np.nan
    F = kf_emu.KalmanFilter(X0, A, Bm, C, Qn, Rnan, P0)
    F.predict(np.zeros((b, nu))); F.update(np.zeros((b, ny)))
    assert F.status[4] == -2 and (np.delete(F.status, 4) == 1).all()


def _governor():
    c = mimo()
    ny = 4
    C = np.zeros((ny, 8))
    for i in range(ny):
        C[i, 2 * i + 1] = 1.0
    return c["Ad"], c["Bd"], C, 0.1 * np.eye(8), 0.5 * np.eye(ny)


@pytest.mark.parametrize("model", ["pendulum", "governor"])
def test_fixed_point_is_the_designed_filter_gain(model):
    """constant model, P0 = the a-priori DARE solution: the gain of every one of 50 steps equals kalman_design_simple's filter
    gain to 1e-10 (the pendulum filter of test_gpu_kalman.py; the MIMO governor model of workloads.mimo with 4 outputs)"""
    if model == "pendulum":
        A, C = pendulum_5ms(); Bm = np.array([[0.0], [0.1], [0.0], [-0.3]]); Qn, Rn = 10 * np.eye(4), np.eye(2)
    else:
        A, Bm, C, Qn, Rn = _governor()
    L, P, _ = okds(A, Bm, C, None, Qn, Rn, type='filter')
    rng = np.random.default_rng(11)
    b = 3
    E = kf_emu.KalmanFilter(rng.standard_normal((b, A.shape[0])), A, Bm, C, Qn, Rn, np.stack([P] * b))
    for t in range(50):
        E.update(rng.standard_normal((b, C.shape[0])))
        assert np.abs(E.gain() - L).max() <= 1e-10 * np.abs(L).max(), t
        E.predict(rng.standard_normal((b, Bm.shape[1])))
    assert rel(E.cov()[0], P) < 1e-10


def test_argument_validation():
    Ad, Bd, Cd, Dd = point_mass_example()
    Q, R = np.eye(2), np.eye(1)
    with pytest.raises(ValueError, match="Qn should have shape"):
        kalman.KalmanFilter(np.zeros(2), Ad, Bd, Cd, Dd, np.eye(3), R)
    with pytest.raises(ValueError, match="Rn should have shape"):
        kalman.KalmanFilter(np.zeros(2), Ad, Bd, Cd, Dd, Q, np.eye(2))
    with pytest.raises(ValueError, match="C should have shape"):
        kalman.KalmanFilter(np.zeros(2), Ad, Bd, np.ones((1, 3)), Dd, Q, R)
    with pytest.raises(ValueError, match="batch size"):
        kalman.KalmanFilter(np.zeros(2), np.stack([Ad] * 3), np.stack([Bd] * 2), Cd, Dd, Q, R)
    with pytest.raises(ValueError, match="batch = 5"):
        kalman.KalmanFilter(np.zeros(2), np.stack([Ad] * 3), Bd, Cd, Dd, Q, R, batch=5)
    with pytest.raises(ValueError, match="1 <= nx, ny <= 32"):
        kalman.KalmanFilter(np.zeros(33), np.eye(33), np.ones((33, 1)), np.ones((1, 33)), None, np.eye(33), R, P0=np.eye(33))
    with pytest.raises(ValueError, match="P0 should have shape"):
        kalman.KalmanFilter(np.zeros(2), Ad, Bd, Cd, Dd, Q, R, P0=np.eye(3))
    with pytest.raises(ValueError, match="matrix"):
        kalman.KalmanFilter(np.zeros(2), Ad, Bd, Cd, Dd, Q, np.ones(1))


class _Shell(kalman._DeviceEstimator):
    """the update_system checks without a device: an estimator object that never reaches the library"""
    def __init__(self, per, B=3):
        self._per, self._B, self.nx, self.nu, self.ny, self.device = per, B, 2, 1, 1, 0
        self.calls = []

    def _set_model(self, vals, on_device):
        self.calls.append((sorted(vals), on_device))


def test_update_system_validation():
    for per in (False, True):
        E = _Shell(per)
        with pytest.raises(ValueError, match="A should have shape"):
            E._update_system(A=np.eye(3))
        with pytest.raises(ValueError, match="Rn should have shape"):
            E._update_system(Rn=np.eye(2))
        E._update_system(A=np.eye(2), Qn=np.eye(2))
        assert E.calls[-1] == (["A", "Qn"], 0)
        E._update_system()
        assert len(E.calls) == 1
    with pytest.raises(ValueError, match="one shared model"):
        _Shell(False)._update_system(A=np.stack([np.eye(2)] * 3))
    with pytest.raises(ValueError, match=r"or \(3, 2, 2\)"):
        _Shell(True)._update_system(A=np.stack([np.eye(2)] * 4))
    E = _Shell(True); E._update_system(C=np.ones((3, 1, 2)))
    assert E.C.shape == (3, 1, 2)
    with pytest.raises(ValueError, match="contiguous float64 CUDA tensor"):
        _Shell(True)._update_system_from_device(A=np.eye(2))
    E = _Shell(True); E._update_system_from_device(A=12345, B=None)
    assert E.calls == [(["A", "B"], 1)]


def test_kalman_filter_without_device_raises(bmpc_lib):
    if bmpc_lib.bmpc_device_count() > 0:
        pytest.skip("a GPU is visible here")
    Ad, Bd, Cd, Dd = point_mass_example()
    with pytest.raises(BmpcError, match="no CUDA device"):
        kalman.KalmanFilter(np.zeros(2), Ad, Bd, Cd, Dd, np.eye(2), np.eye(1))
    with pytest.raises(BmpcError, match="no CUDA device"):
        kalman.KalmanFilter(np.zeros(2), np.stack([Ad] * 3), Bd, Cd, Dd, np.eye(2), np.eye(1), P0=np.eye(2))
