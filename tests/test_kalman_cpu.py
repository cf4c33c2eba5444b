"""CPU tests of the Kalman design (pympc_b200.kalman.dare / kalman_design / kalman_design_simple): the scipy oracle, the
structured-doubling core of csrc/bmpc_dare.cuh built for the host (tests/hostemu/dare_emu.cpp) against it, the acceptance rule
that rejects non-stabilising solutions, and the argument checks of the Python layer.  No GPU needed."""
import numpy as np
import pytest

import dare_emu
from oracle.kalman_design import dare as odare, kalman_design as okd, kalman_design_simple as okds
from pympc_b200 import BmpcError, kalman

SHAPES = [(n, m) for n in (1, 2, 3, 4, 8, 16, 32) for m in sorted({1, min(n, 2), min(n, 4), min(n, 8)})]


def dare_residual(A, B, Q, R, S, X):
    """relative residual of the DARE (control form with cross term)"""
    S = np.zeros(B.shape) if S is None else S
    M = A.T @ X @ B + S
    F = A.T @ X @ A - M @ np.linalg.solve(R + B.T @ X @ B, M.T) + Q - X
    return np.abs(F).max() / max(np.abs(X).max(), 1e-300)


def random_problems(rng, b, n, m, with_s):
    """b random instances: spectral radius of A in [0.3, 1.5], (Q, S, R) the blocks of one positive definite weight"""
    A = rng.standard_normal((b, n, n))
    A *= (rng.uniform(0.3, 1.5, b) / np.abs(np.linalg.eigvals(A)).max(-1))[:, None, None]
    B = rng.standard_normal((b, n, m))
    Z = rng.standard_normal((b, n + m, n + m))
    W = Z @ Z.transpose(0, 2, 1) / (n + m) + 0.5 * np.eye(n + m)
    return A, B, W[:, :n, :n].copy(), W[:, n:, n:].copy(), (W[:, :n, n:].copy() if with_s else None)


def point_mass_example():
    """the model of the reference module's own example (point mass, Ts = 0.2 s, kalman.py:155-175)"""
    Ts, M, b = 0.2, 2.0, 0.3
    Ad = np.array([[1.0, Ts], [0.0, 1.0 - b / M * Ts]])
    Bd = np.array([[0.0], [Ts / M]])
    return Ad, Bd, np.array([[1.0, 0.0]]), np.array([[0.0]])


def test_oracle_satisfies_its_riccati_equation():
    rng = np.random.default_rng(0)
    for n, m in ((2, 1), (4, 2), (8, 4), (16, 3)):
        for with_s in (False, True):
            A, B, Q, R, S = random_problems(rng, 4, n, m, with_s)
            for i in range(4):
                Si = None if S is None else S[i]
                X, W, G = odare(A[i], B[i], Q[i], R[i], Si)
                assert dare_residual(A[i], B[i], Q[i], R[i], Si, X) < 1e-12
                assert np.max(np.abs(W)) < 1.0
                assert np.allclose(np.sort_complex(W), np.sort_complex(np.linalg.eigvals(A[i] - B[i] @ G)))


def test_general_form_equals_simple_predictor_on_reference_example():
    """kalman.py:189-196: with Bw = I, Dw = 0, Nn = 0 the general design reduces to the simple one; the general form's gain is
    the PREDICTOR gain (L = A P C' (C P C' + R)^-1, the transpose of dare's G)"""
    Ad, Bd, Cd, Dd = point_mass_example()
    nx, ny = 2, 1
    Qn, Rn = 10 * np.eye(nx), np.eye(ny)
    Lg, Pg, Wg = okd(Ad, np.hstack([Bd, np.eye(nx)]), Cd, np.hstack([Dd, np.zeros((ny, nx))]), Qn, Rn)
    Ls, Ps, Ws = okds(Ad, Bd, Cd, Dd, Qn, Rn, type='predictor')
    assert np.allclose(Lg, Ls, rtol=1e-12, atol=1e-14) and np.allclose(Pg, Ps, rtol=1e-12)
    assert np.allclose(np.sort_complex(Wg), np.sort_complex(Ws))
    Lf, Pf, _ = okds(Ad, Bd, Cd, Dd, Qn, Rn, type='filter')
    assert np.allclose(Pf, Ps) and np.allclose(Ad @ Lf, Ls)


@pytest.mark.parametrize("with_s", [False, True])
@pytest.mark.parametrize("n,m", SHAPES)
def test_emulated_doubling_core_matches_scipy(n, m, with_s):
    """the SeqTeam build of the device core on random batches: every instance solved, X and G within 1e-9 (relative) of
    scipy's QZ solver where the problem is well conditioned (cond X <= 1e5: both methods leave a residual of about cond(X) * eps,
    so ill-conditioned instances are compared through their residual instead)"""
    rng = np.random.default_rng(1000 * n + 10 * m + with_s)
    b = 24
    A, B, Q, R, S = random_problems(rng, b, n, m, with_s)
    X, G, st, it = dare_emu.dare(A, B, Q, R, S)
    assert (st == 1).all() and (it >= 1).all() and (it <= 64).all()
    compared = 0
    for i in range(b):
        Si = None if S is None else S[i]
        Xr, _, Gr = odare(A[i], B[i], Q[i], R[i], Si)
        assert dare_residual(A[i], B[i], Q[i], R[i], Si, X[i]) < max(1e-12 * np.linalg.cond(Xr), 1e-12)
        if np.linalg.cond(Xr) <= 1e5:
            compared += 1
            assert np.abs(X[i] - Xr).max() <= 1e-9 * np.abs(Xr).max()
            assert np.abs(G[i] - Gr).max() <= 1e-9 * max(1.0, np.abs(Gr).max())
    assert compared >= b // 2


def _one(A, B, Q, R, S=None):
    f = lambda a: np.asarray(a, float)[None]
    X, G, st, it = dare_emu.dare(f(A), f(B), f(Q), f(R), None if S is None else f(S))
    assert (st[0] == 1) == np.isfinite(X).all() == np.isfinite(G).all()       # a failed instance returns NaN, not an iterate
    return int(st[0]), int(it[0])


def test_emulated_core_rejects_non_stabilising_and_indefinite_cases():
    B = [[0.0], [1.0]]
    # uncontrollable unstable mode that Q sees: no solution at all
    assert _one(np.diag([1.2, 0.5]), B, np.diag([1.0, 1.0]), [[1.0]])[0] == -1
    # the same mode hidden from Q: SDA's X converges in a few steps, but to a NON-stabilising solution (A_k does not decay)
    assert _one(np.diag([1.2, 0.5]), B, np.diag([0.0, 1.0]), [[1.0]])[0] == -1
    # uncontrollable mode on the unit circle: no stabilising solution
    assert _one(np.diag([1.0, 0.5]), B, np.diag([1.0, 1.0]), [[1.0]]) == (-1, 64)
    # R indefinite
    assert _one(np.diag([0.9, 0.5]), B, np.eye(2), [[-1.0]]) == (-2, 0)
    assert _one(np.diag([0.9, 0.5]), [[1.0, 0.0], [0.0, 1.0]], np.eye(2), [[1.0, 2.0], [2.0, 1.0]])[0] == -2
    # the stable twin of the first case is solved
    assert _one(np.diag([0.9, 0.5]), B, np.diag([1.0, 1.0]), [[1.0]])[0] == 1


def test_emulated_core_on_the_reference_pendulum_example_converges_in_13_steps():
    """the reference's Kalman example (inverted pendulum, Ts = 5 ms, Q = 10 I, R = I): filter DARE dare(A', C', Q, R)"""
    Ad, Cd = pendulum_5ms()
    X, G, st, it = dare_emu.dare(Ad.T[None], Cd.T[None], 10 * np.eye(4)[None], np.eye(2)[None])
    Xr, _, Gr = odare(Ad.T, Cd.T, 10 * np.eye(4), np.eye(2))
    assert st[0] == 1 and it[0] == 13
    assert np.abs(X[0] - Xr).max() <= 1e-10 * np.abs(Xr).max() and np.abs(G[0] - Gr).max() <= 1e-10 * np.abs(Gr).max()


def pendulum_5ms():
    """the inverted pendulum of the reference's Kalman example (forward Euler, Ts = 5 ms) and its output matrix"""
    M, m, b, ftheta, l, g, Ts = 0.5, 0.2, 0.1, 0.1, 0.3, 9.81, 5e-3
    Ac = np.array([[0, 1, 0, 0],
                   [0, -b / M, -(g * m) / M, (ftheta * m) / M],
                   [0, 0, 0, 1],
                   [0, b / (M * l), (M * g + g * m) / (M * l), -(M * ftheta + ftheta * m) / (M * l)]])
    return np.eye(4) + Ac * Ts, np.array([[1.0, 0, 0, 0], [0, 0, 1.0, 0]])


def test_argument_validation():
    Ad, Bd, Cd, Dd = point_mass_example()
    with pytest.raises(ValueError, match="Unknown Kalman design type"):
        kalman.kalman_design_simple(Ad, Bd, Cd, Dd, np.eye(2), np.eye(1), type='smoother')
    with pytest.raises(ValueError, match="1 <= n, m <= 32"):
        kalman.dare(np.eye(33), np.ones((33, 1)), np.eye(33), np.eye(1))
    with pytest.raises(ValueError, match="1 <= n, m <= 32"):
        kalman.kalman_design_simple(np.eye(33), None, np.ones((1, 33)), None, np.eye(33), np.eye(1))
    with pytest.raises(ValueError, match="Q should have shape"):
        kalman.dare(Ad, Bd, np.eye(3), np.eye(1))
    with pytest.raises(ValueError, match="S should have shape"):
        kalman.dare(Ad, Bd, np.eye(2), np.eye(1), S=np.zeros((2, 2)))
    with pytest.raises(ValueError, match="batch size"):
        kalman.dare(np.stack([Ad] * 3), np.stack([Bd] * 2), np.eye(2), np.eye(1))
    with pytest.raises(ValueError, match="E = I"):
        kalman.dare(Ad, Bd, np.eye(2), np.eye(1), E=2 * np.eye(2))
    with pytest.raises(ValueError, match="noise inputs last"):
        kalman.kalman_design(Ad, Bd, Cd, Dd, np.eye(2), np.eye(1))          # nw = 2 > columns of B
    with pytest.raises(ValueError, match="batch = 5"):
        kalman.LinearStateEstimator(np.zeros(2), np.stack([Ad] * 3), Bd, Cd, Dd, np.zeros((2, 1)), batch=5)


def test_kalman_design_without_device_raises(bmpc_lib):
    if bmpc_lib.bmpc_device_count() > 0:
        pytest.skip("a GPU is visible here")
    Ad, Bd, Cd, Dd = point_mass_example()
    with pytest.raises(BmpcError, match="no CUDA device"):
        kalman.kalman_design(Ad, np.hstack([Bd, Bd]), Cd, np.zeros((1, 2)), np.array([[100.0]]), np.eye(1))
    with pytest.raises(BmpcError, match="no CUDA device"):
        kalman.LinearStateEstimator(np.zeros(2), np.stack([Ad] * 3), Bd, Cd, Dd, np.zeros((2, 1)))
