"""-m gpu tests of the Kalman design on the device (bmpc_dare: structured doubling, csrc/bmpc_dare.cuh) and of the per-instance
state estimator (k_est_pi), against the scipy oracle (oracle/kalman_design.py) and the numpy estimator (oracle/estimator.py)."""
import ctypes

import numpy as np
import pytest

from oracle.kalman_design import dare as odare, kalman_design as okd, kalman_design_simple as okds
from pympc_b200.workloads import pendulum, pendulum_random
from test_kalman_cpu import SHAPES, dare_residual, pendulum_5ms, random_problems

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib(bmpc_lib):
    assert bmpc_lib.bmpc_device_count() > 0, "GPU tests need a CUDA device; the product has no CPU fallback"
    return bmpc_lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _dare(lib, A, B, Q, R, S=None):
    b, n, m = B.shape
    X = np.empty((b, n, n)); G = np.empty((b, m, n)); st = np.empty(b, np.int32); it = np.empty(b, np.int32)
    c = lambda a: None if a is None else np.ascontiguousarray(a, float)
    A, B, Q, R, S = c(A), c(B), c(Q), c(R), c(S)
    assert lib.bmpc_dare(n, m, b, 0, _p(A), _p(B), _p(Q), _p(R), _p(S), _p(X), _p(G), _p(st), _p(it)) == 0
    return X, G, st, it


def perturbed_pendulums(rng, b, Ad, Bd):
    """the perturbation of test_per_instance_systems_vs_oracle: the non-zeros of Ad by 1 %, Bd scaled by 1 + 10 % noise"""
    A = np.stack([Ad + 0.01 * rng.standard_normal((4, 4)) * (Ad != 0) for _ in range(b)])
    B = np.stack([Bd * (1 + 0.1 * rng.standard_normal()) for _ in range(b)])
    return A, B


def test_bmpc_dare_matches_scipy_and_isolates_failing_instances(lib):
    """4096 random per-instance problems over the shapes of the CPU test (n up to 32, m up to 8, with and without S): every
    instance solved, X and G within 1e-9 of scipy where cond(X) <= 1e5, the residual small everywhere.  Then the (2, 1) batch
    again with the four failure cases injected at known indices: their status comes back, every other instance is bit-identical."""
    rng = np.random.default_rng(42)
    per = 4096 // (2 * len(SHAPES))
    total = compared = 0
    for n, m in SHAPES:
        for with_s in (False, True):
            A, B, Q, R, S = random_problems(rng, per, n, m, with_s)
            X, G, st, it = _dare(lib, A, B, Q, R, S)
            assert (st == 1).all(), (n, m, with_s, np.flatnonzero(st != 1))
            assert (it >= 1).all() and (it <= 64).all()
            for i in range(per):
                Si = None if S is None else S[i]
                Xr, _, Gr = odare(A[i], B[i], Q[i], R[i], Si)
                c = np.linalg.cond(Xr)
                assert dare_residual(A[i], B[i], Q[i], R[i], Si, X[i]) < max(1e-12 * c, 1e-12), (n, m, i)
                if c <= 1e5:
                    compared += 1
                    assert np.abs(X[i] - Xr).max() <= 1e-9 * np.abs(Xr).max(), (n, m, with_s, i)
                    assert np.abs(G[i] - Gr).max() <= 1e-9 * max(1.0, np.abs(Gr).max()), (n, m, with_s, i)
            total += per
    assert total >= 4000 and compared >= total // 2
    # failure injection on the (2, 1) shape
    A, B, Q, R, S = random_problems(np.random.default_rng(7), 512, 2, 1, False)
    clean = _dare(lib, A, B, Q, R)
    bad = {17: (np.diag([1.2, 0.5]), np.diag([1.0, 1.0]), [[1.0]], -1),      # uncontrollable unstable mode Q sees
           100: (np.diag([1.2, 0.5]), np.diag([0.0, 1.0]), [[1.0]], -1),     # ... that Q does not see (non-stabilising fixed point)
           255: (np.diag([1.0, 0.5]), np.diag([1.0, 1.0]), [[1.0]], -1),     # uncontrollable mode on the unit circle
           511: (np.diag([0.9, 0.5]), np.diag([1.0, 1.0]), [[-1.0]], -2)}    # R indefinite
    A2, B2, Q2, R2 = A.copy(), B.copy(), Q.copy(), R.copy()
    for i, (a, q, r, _) in bad.items():
        A2[i], B2[i], Q2[i], R2[i] = a, [[0.0], [1.0]], q, r
    X, G, st, it = _dare(lib, A2, B2, Q2, R2)
    keep = np.setdiff1d(np.arange(512), list(bad))
    for i, (_, _, _, want) in bad.items():
        assert st[i] == want, (i, st[i])
        assert np.isnan(X[i]).all() and np.isnan(G[i]).all()
    assert (st[keep] == 1).all()
    assert np.array_equal(X[keep], clean[0][keep]) and np.array_equal(G[keep], clean[1][keep]) and np.array_equal(it[keep], clean[3][keep])


@pytest.mark.parametrize("type", ["filter", "predictor"])
def test_reference_pendulum_example(lib, type):
    """the reference's Kalman example (examples/example_inverted_pendulum_kalman.py: Ts = 5 ms, Q = 10 I, R = I)"""
    from pympc_b200.kalman import kalman_design_simple
    Ad, Cd = pendulum_5ms()
    Bd = pendulum()["Bd"] / 10; Dd = np.zeros((2, 1))
    L, P, W = kalman_design_simple(Ad, Bd, Cd, Dd, 10 * np.eye(4), np.eye(2), type=type)
    Lr, Pr, Wr = okds(Ad, Bd, Cd, Dd, 10 * np.eye(4), np.eye(2), type=type)
    assert L.shape == (4, 2) and P.shape == (4, 4) and W.shape == (4,)
    assert np.abs(L - Lr).max() <= 1e-10 * np.abs(Lr).max() and np.abs(P - Pr).max() <= 1e-10 * np.abs(Pr).max()
    assert np.abs(np.sort_complex(W) - np.sort_complex(Wr)).max() <= 1e-10


def test_general_design_batched(lib):
    """kalman_design on 1024 per-instance plants with per-instance (Qn, Rn, Nn) and a noise feed-through Dw != 0"""
    from pympc_b200.kalman import kalman_design
    rng = np.random.default_rng(3)
    b, nw, ny = 1024, 2, 2
    Ad, Cd = pendulum_5ms()
    A, Bu = perturbed_pendulums(rng, b, Ad, pendulum()["Bd"] / 10)
    Bw = 0.01 * rng.standard_normal((b, 4, nw))
    Bk = np.concatenate([Bu, Bw], axis=2)
    Dk = np.concatenate([np.zeros((b, ny, 1)), 0.1 * rng.standard_normal((b, ny, nw))], axis=2)
    Z = rng.standard_normal((b, nw + ny, nw + ny)); J = Z @ Z.transpose(0, 2, 1) / 4 + 0.5 * np.eye(nw + ny)
    Qn, Nn, Rn = J[:, :nw, :nw], J[:, :nw, nw:], J[:, nw:, nw:]
    L, P, W = kalman_design(A, Bk, Cd, Dk, Qn, Rn, Nn)
    assert L.shape == (b, 4, ny) and P.shape == (b, 4, 4) and W.shape == (b, 4)
    for i in range(b):
        Lr, Pr, Wr = okd(A[i], Bk[i], Cd, Dk[i], Qn[i], Rn[i], Nn[i])
        assert np.abs(L[i] - Lr).max() <= 1e-9 * np.abs(Lr).max(), i
        assert np.abs(P[i] - Pr).max() <= 1e-9 * np.abs(Pr).max(), i
        assert np.abs(np.sort_complex(W[i]) - np.sort_complex(Wr)).max() <= 1e-9, i


def test_per_instance_estimator_vs_oracle_and_shared_path_unchanged(lib):
    """257 per-instance (A, B, C, L) x 5 predict/update steps vs the numpy estimator; n_sys = 1 through bmpc_est_create_ex is
    bit-identical to bmpc_est_create"""
    from pympc_b200.kalman import LinearStateEstimator
    from oracle.estimator import LinearStateEstimator as Ref
    cfg = pendulum(); rng = np.random.default_rng(8); b = 257
    A, Bm = perturbed_pendulums(rng, b, cfg["Ad"], cfg["Bd"])
    C = np.array([[1.0, 0, 0, 0], [0, 0, 1.0, 0]]) + 0.01 * rng.standard_normal((b, 2, 4))
    D = np.zeros((2, 1)); Lg = 0.1 * rng.standard_normal((b, 4, 2))
    X0 = 0.1 * rng.standard_normal((b, 4))
    E = LinearStateEstimator(X0, A, Bm, C, D, Lg)
    assert E.batch == b
    refs = [Ref(X0[i], A[i], Bm[i], C[i], D, Lg[i]) for i in range(b)]
    for t in range(5):
        U = rng.standard_normal((b, 1)); Y = rng.standard_normal((b, 2))
        xp = E.predict(U); yp = E.y; xu = E.update(Y)
        for i in range(b):
            assert np.max(np.abs(refs[i].predict(U[i]) - xp[i])) < 1e-12
            assert np.max(np.abs(refs[i].y - yp[i])) < 1e-12
            assert np.max(np.abs(refs[i].update(Y[i]) - xu[i])) < 1e-12
    E.close()
    # shared system: create vs create_ex(n_sys = 1)
    L0 = np.ascontiguousarray(Lg[0]); A0, B0, C0 = (np.ascontiguousarray(a[0]) for a in (A, Bm, C))
    out = []
    for ex in (False, True):
        h = ctypes.c_void_p()
        args = (_p(A0), _p(B0), _p(C0), _p(L0), _p(X0), ctypes.byref(h))
        rc = lib.bmpc_est_create_ex(4, 1, 2, b, 1, 0, *args) if ex else lib.bmpc_est_create(4, 1, 2, b, 0, *args)
        assert rc == 0
        r = np.random.default_rng(9)
        for t in range(5):
            U = r.standard_normal((b, 1)); Y = r.standard_normal((b, 2))
            assert lib.bmpc_est_predict(h, _p(U), 0) == 0 and lib.bmpc_est_update(h, _p(Y), 0) == 0
        x = np.empty((b, 4)); y = np.empty((b, 2))
        assert lib.bmpc_est_get(h, _p(x), _p(y)) == 0
        lib.bmpc_est_destroy(h)
        out.append((x, y))
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])
    h = ctypes.c_void_p()
    assert lib.bmpc_est_create_ex(4, 1, 2, b, 3, 0, _p(A0), _p(B0), _p(C0), _p(L0), _p(X0), ctypes.byref(h)) == -1   # n_sys must be 1 or batch


def test_heterogeneous_closed_loop_on_device(lib):
    """per-instance pendulums: MPCController (fast path, one system per instance) + per-instance estimator whose gains come from
    the batched kalman_design on the GPU, chained on the device for 6 steps (estimate -> update_from_device -> u0 ->
    predict_device -> update_device) without host reads; equals the host-driven chain with the oracle's gains"""
    import torch
    from pympc_b200 import MPCController
    from pympc_b200.kalman import LinearStateEstimator, kalman_design
    cfg = pendulum(); rng = np.random.default_rng(21); b = 1024
    A, Bm = perturbed_pendulums(rng, b, cfg["Ad"], cfg["Bd"])
    C = np.array([[1.0, 0, 0, 0], [0, 0, 1.0, 0]]); D = np.zeros((2, 1))
    Bk = np.concatenate([Bm, np.broadcast_to(np.eye(4), (b, 4, 4))], axis=2); Dk = np.zeros((2, 5))
    Qn, Rn = 10 * np.eye(4), np.eye(2)
    Lgpu, _, _ = kalman_design(A, Bk, C, Dk, Qn, Rn)
    Lref = np.stack([okd(A[i], Bk[i], C, Dk, Qn, Rn)[0] for i in range(b)])
    assert np.abs(Lgpu - Lref).max() <= 1e-9 * np.abs(Lref).max()
    X0, Xref = pendulum_random(b, seed=4)
    Ys = 0.05 * rng.standard_normal((6, b, 2))
    kw = {k: cfg[k] for k in ("Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "eps_feas")}
    mk = lambda: MPCController(A, Bm, Np=20, x0=X0, xref=Xref, uminus1=np.zeros(1), batch=b, fast_path=1, **kw)
    # host-driven chain, oracle gains
    Eh = LinearStateEstimator(X0, A, Bm, C, D, Lref)
    Kh = mk(); Kh.setup(); U = Kh.output()
    for t in range(6):
        Eh.predict(U); x = Eh.update(Ys[t] + Eh.y)
        Kh.update(x); U = Kh.output()
    # device chain, GPU gains
    Ed = LinearStateEstimator(X0, A, Bm, C, D, Lgpu)
    Kd = mk(); Kd.setup(); Kd.output()
    Ed.attach(Kd)
    Ud = torch.zeros(b, 1, dtype=torch.float64, device="cuda")
    Yd = torch.zeros(b, 2, dtype=torch.float64, device="cuda")
    Ud.copy_(torch.from_numpy(Kd._u0.copy()))
    torch.cuda.synchronize()
    Lb, h = Kd._L, Kd.handle
    assert Lb.bmpc_bind_output(h, Ud.data_ptr()) == 0
    Yhost = np.empty((b, 2))
    for t in range(6):
        assert Ed.predict_device(Ud.data_ptr()) == 0
        Lb.bmpc_est_get(Ed._h, None, _p(Yhost))          # only to build the synthetic measurement of this test
        Yd.copy_(torch.from_numpy(Ys[t] + Yhost)); torch.cuda.synchronize()
        assert Ed.update_device(Yd.data_ptr()) == 0
        assert Lb.bmpc_update(h, Ed.device_state(), None, None, 1, 1) == 0
        assert Lb.bmpc_solve(h) == 0
        assert Lb.bmpc_output(h, None, None, 1, 1) == 0
    torch.cuda.synchronize()
    assert np.max(np.abs(Ud.cpu().numpy() - U)) < 1e-9
    assert np.max(np.abs(Ed.x - Eh.x)) < 1e-10
    for o in (Eh, Ed, Kh, Kd):
        o.close()
