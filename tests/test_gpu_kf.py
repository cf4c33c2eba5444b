"""-m gpu tests of the batched Kalman filter (k_kf: shared model, k_kf_pi: one model per instance; csrc/bmpc_kf.cuh) and of model
updates between steps for both estimator kinds (bmpc_est_set_model), against the numpy filter (tests/kf_oracle.py) and the numpy
estimator (oracle/estimator.py)."""
import ctypes

import numpy as np
import pytest

from kf_oracle import KalmanFilter as Ref
from oracle.estimator import LinearStateEstimator as RefLSE
from oracle.kalman_design import kalman_design_simple as okds
from pympc_b200.workloads import cartpole_linearised, pendulum, pendulum_random
from test_gpu_kalman import perturbed_pendulums
from test_kalman_cpu import pendulum_5ms

pytestmark = pytest.mark.gpu

C2 = np.array([[1.0, 0, 0, 0], [0, 0, 1.0, 0]])


@pytest.fixture(scope="module")
def lib(bmpc_lib):
    assert bmpc_lib.bmpc_device_count() > 0, "GPU tests need a CUDA device; the product has no CPU fallback"
    return bmpc_lib


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def test_filters_at_65536_against_oracle_and_shared_equals_per_instance(lib):
    """65 536 per-instance cart-pole filters over 30 steps: 64 sampled instances, each step within 1e-12 (relative) of the numpy
    filter's step from the same x and P, the whole run within 1e-9 of the free-running numpy filter.  A shared filter and a
    per-instance filter that holds the same model on every instance (k_kf against k_kf_pi) are bit-identical."""
    from pympc_b200.kalman import KalmanFilter
    rng = np.random.default_rng(5); b = 65536
    cfg = pendulum()
    A, Bm = perturbed_pendulums(rng, b, cfg["Ad"], cfg["Bd"])
    C = C2 + 0.01 * rng.standard_normal((b, 2, 4))
    Qn, Rn = 1e-3 * np.eye(4), 1e-2 * np.eye(2)
    X0 = 0.1 * rng.standard_normal((b, 4)); P0 = np.eye(4) * 0.05
    F = KalmanFilter(X0, A, Bm, C, None, Qn, Rn, P0=P0)
    assert F.batch == b and F.P.shape == (b, 4, 4)
    pick = rng.choice(b, 64, replace=False)
    free = {i: Ref(X0[i], A[i], Bm[i], C[i], Qn, Rn, P0) for i in pick}
    for t in range(30):
        U = rng.standard_normal((b, 1)); Y = 0.1 * rng.standard_normal((b, 2))
        x0, P0t, y0 = F.x, F.P, F.y
        F.predict(U); F.update(Y)
        x1, P1 = F.x, F.P
        for i in pick:
            r = Ref(x0[i], A[i], Bm[i], C[i], Qn, Rn, P0t[i]); r.y = y0[i]
            r.predict(U[i]); r.update(Y[i])
            assert rel(x1[i], r.x) < 1e-12 and rel(P1[i], r.P) < 1e-12, (t, i)
            free[i].predict(U[i]); free[i].update(Y[i])
            assert rel(x1[i], free[i].x) < 1e-9 and rel(P1[i], free[i].P) < 1e-9, (t, i)
    assert (F.status == 1).all()
    F.close()
    # k_kf against k_kf_pi on the same system
    out = []
    for per in (False, True):
        mk = (lambda a: np.stack([a] * b)) if per else (lambda a: a)
        G = KalmanFilter(X0, mk(cfg["Ad"]), mk(cfg["Bd"]), mk(C2), None, mk(Qn), mk(Rn), P0=P0, batch=b)
        r = np.random.default_rng(9)
        for t in range(10):
            G.predict(r.standard_normal((b, 1))); G.update(0.1 * r.standard_normal((b, 2)))
        out.append((G.x, G.P, G.y)); G.close()
    for a, c in zip(*out):
        assert np.array_equal(a, c)


def test_governor_filters_against_oracle(lib):
    """16 384 MIMO governor filters (nx = 8, nu = 4, ny = 4), shared model, against the numpy filter step by step"""
    from pympc_b200.kalman import KalmanFilter
    from test_kf_cpu import _governor
    A, Bm, C, Qn, Rn = _governor()
    b = 16384; rng = np.random.default_rng(6)
    X0 = rng.standard_normal((b, 8))
    F = KalmanFilter(X0, A, Bm, C, None, Qn, Rn, batch=b)
    for t in range(10):
        U = rng.standard_normal((b, 4)); Y = rng.standard_normal((b, 4))
        x0, P0, y0 = F.x, F.P, F.y
        F.predict(U); F.update(Y)
        x1, P1 = F.x, F.P
        for i in (0, 77, b - 1):
            r = Ref(x0[i], A, Bm, C, Qn, Rn, P0[i]); r.y = y0[i]
            r.predict(U[i]); r.update(Y[i])
            assert rel(x1[i], r.x) < 1e-12 and rel(P1[i], r.P) < 1e-12, (t, i)
    F.close()


def test_default_filter_reproduces_the_designed_estimator(lib):
    """a constant-model KalmanFilter with the default P0 tracks LinearStateEstimator built with kalman_design_simple's filter gain
    (the oracle's) to 1e-10 over 100 steps"""
    from pympc_b200.kalman import KalmanFilter, LinearStateEstimator
    Ad, Cd = pendulum_5ms(); Bd = pendulum()["Bd"] / 10; Dd = np.zeros((2, 1))
    Qn, Rn = 10 * np.eye(4), np.eye(2)
    L, P, _ = okds(Ad, Bd, Cd, Dd, Qn, Rn, type='filter')
    b = 1024; rng = np.random.default_rng(2)
    X0 = rng.standard_normal((b, 4))
    F = KalmanFilter(X0, Ad, Bd, Cd, Dd, Qn, Rn, batch=b)
    assert rel(F.P[0], P) < 1e-10
    E = LinearStateEstimator(X0, Ad, Bd, Cd, Dd, L, batch=b)
    for t in range(100):                        # both start at x[0|-1]: update, then predict
        U = rng.standard_normal((b, 1)); Y = rng.standard_normal((b, 2))
        xf = F.update(Y); xe = E.update(Y)
        assert np.abs(xf - xe).max() <= 1e-10 * max(1.0, np.abs(xe).max()), t
        xf = F.predict(U); xe = E.predict(U)
        assert np.abs(xf - xe).max() <= 1e-10 * max(1.0, np.abs(xe).max()), t
    F.close(); E.close()


def _new_models(rng, b):
    cfg = pendulum()
    A, Bm = perturbed_pendulums(rng, b, cfg["Ad"], cfg["Bd"])
    C = C2 + 0.01 * rng.standard_normal((b, 2, 4))
    return A, Bm, C


@pytest.mark.parametrize("per", [False, True])
def test_update_system_from_host_and_device_agree_with_oracle(lib, per):
    """update_system (host arrays) and update_system_from_device (torch tensors) give the same filter, equal to the numpy filter
    with the same matrices assigned, for a shared and a per-instance KalmanFilter and LinearStateEstimator.  A
    LinearStateEstimator after update_system is bit-identical to a fresh one built from the new matrices."""
    import torch
    from pympc_b200.kalman import KalmanFilter, LinearStateEstimator
    rng = np.random.default_rng(31 + per); b = 512
    cfg = pendulum(); Qn, Rn = 1e-3 * np.eye(4), 1e-2 * np.eye(2)
    X0 = 0.1 * rng.standard_normal((b, 4))
    dev = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda")
    pick = lambda a, i: a[i] if a.ndim == 3 else a
    # --- Kalman filter
    kf = []
    for mode in ("host", "device"):
        r = np.random.default_rng(1)
        A0, B0, C0 = (m if per else m[0] for m in _new_models(r, b))
        F = KalmanFilter(X0, A0, B0, C0, None, Qn, Rn, P0=0.05 * np.eye(4), batch=b)
        refs = [Ref(X0[i], pick(A0, i), pick(B0, i), pick(C0, i), Qn, Rn, 0.05 * np.eye(4)) for i in (0, 100, b - 1)]
        for t in range(5):
            A, Bm, C = (m if per else m[0] for m in _new_models(r, b))
            Qt, Rt = Qn * (1 + t), Rn * (1 + 0.5 * t)
            if mode == "host":
                F.update_system(A=A, B=Bm, C=C, Qn=Qt, Rn=Rt)
            else:
                full = lambda a: np.broadcast_to(a, (b,) + a.shape) if per else a
                keep = [dev(A), dev(Bm), dev(C), dev(full(Qt)), dev(full(Rt))]
                torch.cuda.synchronize()
                F.update_system_from_device(*keep)
            U = r.standard_normal((b, 1)); Y = 0.1 * r.standard_normal((b, 2))
            F.predict(U); F.update(Y)
            for ref, i in zip(refs, (0, 100, b - 1)):
                ref.A, ref.B, ref.C, ref.Qn, ref.Rn = pick(A, i), pick(Bm, i), pick(C, i), Qt, Rt
                ref.predict(U[i]); ref.update(Y[i])
        x, P = F.x, F.P
        for ref, i in zip(refs, (0, 100, b - 1)):
            assert rel(x[i], ref.x) < 1e-10 and rel(P[i], ref.P) < 1e-10
        kf.append((x, P)); F.close()
    assert np.array_equal(kf[0][0], kf[1][0]) and np.array_equal(kf[0][1], kf[1][1])
    # --- fixed-gain estimator
    lse = []
    for mode in ("host", "device"):
        r = np.random.default_rng(2)
        A0, B0, C0 = (m if per else m[0] for m in _new_models(r, b))
        L0 = 0.1 * r.standard_normal((b, 4, 2)) if per else 0.1 * r.standard_normal((4, 2))
        E = LinearStateEstimator(X0, A0, B0, C0, None, L0, batch=b)
        refs = [RefLSE(X0[i], pick(A0, i), pick(B0, i), pick(C0, i), None, pick(L0, i)) for i in (0, 100, b - 1)]
        for t in range(5):
            A, Bm, C = (m if per else m[0] for m in _new_models(r, b))
            L = 0.1 * r.standard_normal(L0.shape)
            if mode == "host":
                E.update_system(A=A, B=Bm, C=C, L=L)
            else:
                keep = [dev(A), dev(Bm), dev(C), dev(L)]
                torch.cuda.synchronize()
                E.update_system_from_device(*keep)
            U = r.standard_normal((b, 1)); Y = 0.1 * r.standard_normal((b, 2))
            E.predict(U); E.update(Y)
            for ref, i in zip(refs, (0, 100, b - 1)):
                ref.A, ref.B, ref.C, ref.L = pick(A, i), pick(Bm, i), pick(C, i), pick(L, i)
                ref.predict(U[i]); ref.update(Y[i])
        x = E.x
        for ref, i in zip(refs, (0, 100, b - 1)):
            assert rel(x[i], ref.x) < 1e-12
        lse.append(x)
        # a fresh estimator from the last matrices, started where E is, runs the same as E from here on
        G = LinearStateEstimator(x, A, Bm, C, None, L, batch=b)
        for t in range(3):
            U = r.standard_normal((b, 1)); Y = 0.1 * r.standard_normal((b, 2))
            assert np.array_equal(E.predict(U), G.predict(U)) and np.array_equal(E.y, G.y)
            assert np.array_equal(E.update(Y), G.update(Y))
        E.close(); G.close()
    assert np.array_equal(lse[0], lse[1])


def test_model_arguments_of_the_wrong_kind_are_refused(lib):
    from pympc_b200.kalman import KalmanFilter, LinearStateEstimator
    cfg = pendulum()
    F = KalmanFilter(np.zeros(4), cfg["Ad"], cfg["Bd"], C2, None, np.eye(4), np.eye(2))
    E = LinearStateEstimator(np.zeros(4), cfg["Ad"], cfg["Bd"], C2, None, np.zeros((4, 2)))
    Q = np.eye(4); Lg = np.zeros((4, 2))
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    assert lib.bmpc_est_set_model(F._h, None, None, None, p(Lg), None, None, 0) == -1
    assert lib.bmpc_est_set_model(E._h, None, None, None, None, p(Q), None, 0) == -1
    assert lib.bmpc_est_get_cov(E._h, None, None) == -1
    with pytest.raises(ValueError, match="one shared model"):
        F.update_system(A=np.stack([cfg["Ad"]] * 2))
    F.close(); E.close()


def test_failure_isolation_on_device(lib):
    """an indefinite Rn on three of 4 096 per-instance filters: status -2 there, x and P of those kept, every other instance
    bit-identical to the run without them"""
    from pympc_b200.kalman import KalmanFilter
    rng = np.random.default_rng(12); b = 4096
    A, Bm, C = _new_models(rng, b)
    Rn = np.stack([1e-2 * np.eye(2)] * b); bad = [5, 1000, b - 1]
    Rbad = Rn.copy(); Rbad[5] = [[1.0, 2.0], [2.0, 1.0]]; Rbad[1000] = -np.eye(2); Rbad[b - 1, 1, 1] = 0.0
    Rbad[b - 1] -= np.array([[0, 0], [0, 1e6]])
    X0 = 0.1 * rng.standard_normal((b, 4)); P0 = 0.05 * np.eye(4)
    clean = KalmanFilter(X0, A, Bm, C, None, 1e-3 * np.eye(4), Rn, P0=P0)
    F = KalmanFilter(X0, A, Bm, C, None, 1e-3 * np.eye(4), Rbad, P0=P0)
    keep = np.setdiff1d(np.arange(b), bad)
    for t in range(4):
        U = rng.standard_normal((b, 1)); Y = 0.1 * rng.standard_normal((b, 2))
        clean.predict(U); F.predict(U)
        xb, Pb = F.x, F.P
        clean.update(Y); F.update(Y)
        st = F.status
        assert (st[bad] == -2).all() and (st[keep] == 1).all()
        assert np.array_equal(F.x[bad], xb[bad]) and np.array_equal(F.P[bad], Pb[bad])
        assert np.array_equal(F.x[keep], clean.x[keep]) and np.array_equal(F.P[keep], clean.P[keep])
    clean.close(); F.close()


def test_device_side_successive_linearisation_with_filter(lib):
    """1 024 per-instance cart-poles, 10 steps with no host reads: re-linearise with cartpole_linearised on torch tensors about an
    operating-point trajectory and the last u*, hand the model to MPCController.update_system_from_device and
    KalmanFilter.update_system_from_device, predict_device(u*), update_device(y) on seeded noisy measurements, then
    update_from_device, solve and output into a device buffer.  Equals a host-driven chain of numpy oracle filters and a
    controller fed host arrays: u* to 1e-9, the estimates to 1e-10."""
    import torch
    from pympc_b200 import MPCController
    from pympc_b200.kalman import KalmanFilter
    cfg = pendulum(); b = 1024; T = 10
    X0, Xref = pendulum_random(b, seed=8)
    rng = np.random.default_rng(40)
    Xop = X0[None] * np.linspace(1.0, 0.5, T)[:, None, None]               # operating points of the linearisation
    Ys = (Xop @ C2.T) + 0.01 * rng.standard_normal((T, b, 2))              # seeded noisy measurements
    Qn, Rn = 1e-4 * np.eye(4), 1e-4 * np.eye(2)
    kw = {k: cfg[k] for k in ("Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "eps_feas")}
    A0, B0 = cartpole_linearised(X0, np.zeros((b, 1)))
    mk = lambda: MPCController(A0, B0, Np=20, x0=X0, xref=Xref, uminus1=np.zeros(1), batch=b, **kw)
    dev = torch.device("cuda", 0)
    # the models of the host chain: the same torch computation, read back
    Ah, Bh = [], []
    # --- device chain
    stream = torch.cuda.Stream(dev)
    Kd = mk(); Kd.setup(); Kd.output()
    Fd = KalmanFilter(X0, A0, B0, C2, None, Qn, Rn)
    P0 = Fd.P
    Lb, h = Kd._L, Kd.handle
    assert Lb.bmpc_set_stream(h, stream.cuda_stream) == 0
    Fd.attach(Kd)
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        Ud = torch.tensor(Kd._u0.copy(), device=dev)
        Xop_d = torch.tensor(Xop, device=dev); Ys_d = torch.tensor(Ys, device=dev)
        stream.synchronize()
        assert Lb.bmpc_bind_output(h, Ud.data_ptr()) == 0
        keep = []
        for t in range(T):
            Ad, Bd = cartpole_linearised(Xop_d[t], Ud)
            Ad, Bd = Ad.contiguous(), Bd.contiguous()
            keep.append((Ad, Bd))
            Kd.update_system_from_device(Ad, Bd)
            Fd.update_system_from_device(A=Ad, B=Bd)
            assert Fd.predict_device(Ud.data_ptr()) == 0
            assert Fd.update_device(Ys_d[t].data_ptr()) == 0
            assert Lb.bmpc_update(h, Fd.device_state(), None, None, 1, 1) == 0
            assert Lb.bmpc_solve(h) == 0
            assert Lb.bmpc_output(h, None, None, 1, 1) == 0
        stream.synchronize()
    Ud_final, Xd_final = Ud.cpu().numpy(), Fd.x
    # --- host chain: numpy filters, controller fed host arrays (the models recomputed from the host chain's own u*)
    Kh = mk(); Kh.setup(); U = Kh.output().copy()
    refs = [Ref(X0[i], A0[i], B0[i], C2, Qn, Rn, P0[i]) for i in range(b)]
    for t in range(T):
        Ad, Bd = [a.cpu().numpy() for a in cartpole_linearised(torch.tensor(Xop[t], device=dev), torch.tensor(U, device=dev))]
        Kh.update_system(Ad, Bd)
        x = np.empty((b, 4))
        for i, r in enumerate(refs):
            r.A, r.B = Ad[i], Bd[i]
            r.predict(U[i]); x[i] = r.update(Ys[t, i])
        Kh.update(x); U = Kh.output().copy()
    assert np.abs(Ud_final - U).max() < 1e-9
    assert np.abs(Xd_final - x).max() < 1e-10
    for o in (Kd, Kh, Fd):
        o.close()
