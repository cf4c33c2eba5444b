"""-m gpu tests of time-varying system matrices (MPCController.update_system / bmpc_update_system): after a model change the next
update() is a warm solve of the QP the reference assembles with the new (Ad, Bd) — checked against a controller set up from scratch
with those matrices and against the CPU oracle on each sampled instance's own QP, in every kernel family."""
import numpy as np
import pytest

from pympc_b200.workloads import pendulum, pendulum_random, mimo, cartpole_rhs, cartpole_linearised, CARTPOLE

pytestmark = pytest.mark.gpu
TOL = 1e-6
KEYS = ("Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "eps_feas")


@pytest.fixture(scope="module")
def MPC(bmpc_lib):
    assert bmpc_lib.bmpc_device_count() > 0, "GPU tests need a CUDA device; the product has no CPU fallback"
    from pympc_b200 import MPCController
    return MPCController


def _oracle(cfg):
    """exact minimiser of the reference-assembled QP: (U*, QPData, z)"""
    from oracle.qp_assembly import QPData
    from oracle.kkt import solve_exact
    Q = QPData(**cfg)
    z, y, r = solve_exact(Q.P, Q.q, Q.A, Q.l, Q.u)
    return z[Q.NX:Q.NX + Q.NU], Q, z


def _generic():
    Ad = np.array([[1.0, 0.1, 0, 0], [-0.2, 0.95, 0.05, 0], [0, 0, 1.0, 0.1], [0.03, 0, -0.3, 0.9]])
    Bd = np.array([[0.0, 0.0], [0.1, 0.02], [0.0, 0.0], [0.0, 0.1]])
    return dict(Ad=Ad, Bd=Bd, Np=30, Nc=24, Qx=np.diag([1.0, 0.1, 1.0, 0.1]), QxN=np.diag([2.0, 0.1, 2.0, 0.1]), Qu=0.01 * np.eye(2),
                QDu=0.1 * np.eye(2), xmin=-np.array([2.0, 5, 2, 5]), xmax=np.array([0.8, 5, 2, 5]), umin=-np.ones(2), umax=np.ones(2),
                Dumin=-0.3 * np.ones(2), Dumax=0.3 * np.ones(2), eps_feas=1e4)


def _step(Ad, Bd, X, U):
    """x+ = Ad x + Bd u for a shared (2-D) or per-instance (3-D) model"""
    if np.ndim(Ad) == 3:
        return np.einsum("bij,bj->bi", Ad, X) + np.einsum("bij,bj->bi", Bd, U)
    return X @ Ad.T + U @ Bd.T


def _family(name, rng):
    """-> (base cfg, B, controller options, per-instance flag, X0, Xref, new Ad, new Bd)"""
    if name in ("pi_tpi", "shared_tpi", "team"):
        c = pendulum(); c["Np"] = 20
        B = {"pi_tpi": 2048, "shared_tpi": 1024, "team": 256}[name]
        X0, Xref = pendulum_random(B, seed=5)
        opts = {"fast_path": 0} if name == "team" else {}
        if name == "pi_tpi":                                   # every instance re-linearised about its own state
            Ad2, Bd2 = cartpole_linearised(X0, np.zeros((B, 1)))
        else:
            Ad2, Bd2 = cartpole_linearised(np.array([[0.1, 0.3, 0.2, -0.4]]), np.array([[1.5]]))
            Ad2, Bd2 = Ad2[0], Bd2[0]
        return c, B, opts, name == "pi_tpi", X0, Xref, Ad2, Bd2
    if name == "mimo":
        c = mimo(); c.setdefault("eps_feas", 1e6); B = 256
        X0 = 0.3 * rng.standard_normal((B, 8)); Xref = np.tile(c["xref"], (B, 1))
        Ad2 = c["Ad"] * (1 + 0.02 * rng.standard_normal(c["Ad"].shape))          # same sparsity pattern: k_tpm_pol's entry stays
        Bd2 = c["Bd"] * 1.1
        return c, B, {}, False, X0, Xref, Ad2, Bd2
    c = _generic(); B = 600
    X0 = 0.4 * rng.standard_normal((B, 4)); Xref = np.tile(np.array([0.7, 0, -0.5, 0]), (B, 1))
    Ad2 = c["Ad"] + 0.02 * rng.standard_normal((4, 4)) * (c["Ad"] != 0); Bd2 = c["Bd"] * 0.9
    return c, B, {}, False, X0, Xref, Ad2, Bd2


@pytest.mark.parametrize("name", ["pi_tpi", "shared_tpi", "team", "mimo", "generic"])
def test_update_system_equals_a_fresh_setup(MPC, name):
    """a few warm steps with (Ad1, Bd1), update_system(Ad2, Bd2), update(x, u): the plan equals that of a controller set up from
    scratch with (Ad2, Bd2) and the same x0, u_-1 (instances verified by both), and the oracle on sampled instances' own QPs.
    Families: per-instance pendulum and shared pendulum on k_tpi_pol, fast_path=0 team kernels, the MIMO shape on k_tpm_pol + the
    tile kernel, a generic 2-input shape on the tile kernel."""
    rng = np.random.default_rng(11)
    c, B, opts, per, X0, Xref, Ad2, Bd2 = _family(name, rng)
    nu = c["Bd"].shape[1]
    kw = dict({k: c[k] for k in KEYS}, Np=c["Np"], Nc=c.get("Nc"), batch=B, xref=Xref, **opts)
    Ad1 = np.broadcast_to(c["Ad"], (B,) + c["Ad"].shape).copy() if per else c["Ad"]
    Bd1 = np.broadcast_to(c["Bd"], (B,) + c["Bd"].shape).copy() if per else c["Bd"]
    K = MPC(Ad1, Bd1, x0=X0, uminus1=np.zeros(nu), **kw); K.setup()
    X = X0.copy(); U = K.output()
    for t in range(3):
        X = _step(Ad1, Bd1, X, U)
        K.update(X, U); U = K.output()
    K.update_system(Ad2, Bd2)
    K.update(X, U)
    Un, info = K.output(return_u_seq=True); u1 = info["u_seq"].reshape(B, -1); s1 = np.array(K.res.info.status_val)
    warm_iters = K.stats()["admm_iters"]
    F = MPC(Ad2, Bd2, x0=X, uminus1=U, **kw); F.setup()
    _, info = F.output(return_u_seq=True); u2 = info["u_seq"].reshape(B, -1); s2 = np.array(F.res.info.status_val)
    cold_iters = F.stats()["admm_iters"]
    both = (s1 == 1) & (s2 == 1)
    assert both.mean() > 0.95 and (s1 > 0).all(), (name, both.mean())
    assert np.max(np.abs(u1[both] - u2[both])) < 1e-7, name
    for b in np.flatnonzero(both)[:: max(1, both.sum() // 4)][:4]:
        cb = dict(c, Ad=Ad2[b] if per else Ad2, Bd=Bd2[b] if per else Bd2, x0=X[b], xref=Xref[b], uminus1=U[b])
        ref, Q, z = _oracle(cb)
        assert np.max(np.abs(u1[b] - ref)) < TOL, (name, b)
    if name != "mimo":
        # the step after the change stayed warm.  (MIMO shape: the shifted working sets of most instances fail after the change and
        # the straggler rounds cost more ADMM iterations than a cold solve's 25 + polish — DESIGN.md §4 (v))
        assert warm_iters < cold_iters, (name, warm_iters, cold_iters)
    # the reference-form attributes describe the new QP
    assert np.array_equal(K.Ad, Ad2[0] if per else Ad2)
    K.close(); F.close()


def test_successive_linearisation_closed_loop(MPC):
    """8 192 per-instance pendulums driven by the nonlinear cart-pole (RK4), re-linearised about each instance's state at every
    step on the device (torch) and handed over with update_system_from_device: every step >= 99.9 % verified, sampled instances
    equal the oracle on their own QP with the new matrices, and from the second step on the solves stay far below a cold solve's
    ADMM iterations (the warm start survives the model change).  Starts: pendulum_random scaled by 1/2 — from the full spread
    about 1 % of the poles leave the region where the state-linearised model holds them, and their QPs (soft state rows violated
    by metres) end unverified on a fresh setup too (tools/bench_ltv.py)."""
    torch = pytest.importorskip("torch")
    c = pendulum(); B = 8192; Ts = CARTPOLE[6]; dev = torch.device("cuda", 0)
    X0, Xref = pendulum_random(B, seed=9)
    X0 = 0.5 * X0
    Ad0, Bd0 = cartpole_linearised(X0, np.zeros((B, 1)))
    K = MPC(Ad0, Bd0, Np=20, x0=X0, xref=Xref, uminus1=np.zeros(1), batch=B, **{k: c[k] for k in KEYS})
    K.setup()
    cold = K.stats()["admm_iters"]
    U = K.output().copy()
    X = torch.tensor(X0, device=dev)

    def rk4(x, u):
        k1 = cartpole_rhs(x, u); k2 = cartpole_rhs(x + 0.5 * Ts * k1, u)
        k3 = cartpole_rhs(x + 0.5 * Ts * k2, u); k4 = cartpole_rhs(x + Ts * k3, u)
        return x + Ts / 6.0 * (k1 + 2 * k2 + 2 * k3 + k4)
    rng = np.random.default_rng(1); warm = []
    for t in range(30):
        Ut = torch.tensor(U, device=dev)
        X = rk4(X, Ut)
        Ad_t, Bd_t = cartpole_linearised(X, Ut)
        torch.cuda.synchronize()                    # torch's stream wrote them; the controller reads them on its own stream
        K.update_system_from_device(Ad_t, Bd_t)
        Xh = X.cpu().numpy()
        K.update(Xh, U)
        Un, info = K.output(return_u_seq=True)
        st = np.array(K.res.info.status_val)
        assert (st == 1).mean() >= 0.999, (t, np.unique(st, return_counts=True))
        warm.append(K.stats()["admm_iters"])
        Ah, Bh = Ad_t.cpu().numpy(), Bd_t.cpu().numpy()
        useq = info["u_seq"].reshape(B, -1)
        for b in rng.choice(np.flatnonzero(st == 1), 2, replace=False):
            ref, Q, z = _oracle(dict(c, Ad=Ah[b], Bd=Bh[b], x0=Xh[b], xref=Xref[b], uminus1=U[b]))
            assert np.max(np.abs(useq[b] - ref)) < TOL, (t, b)
        U = Un.copy()
    print("closed loop: cold", cold, "warm", warm)
    assert max(warm[1:]) < 0.2 * cold, (cold, warm)
    K.close()


def test_lazy_refresh_consumers_see_the_new_system(MPC):
    """per-instance fast path after update_system + a warm solve that k_tpi_pol finishes alone: x_seq is the roll-out of the NEW
    (Ad, Bd) under u_seq, obj_val the oracle's objective, condensed('H') the oracle algebra of the new system 0; a solve with
    straggler rounds (64 instances jump) runs its ADMM rounds on re-condensed blocks and still equals the oracle; a warm solve that
    verifies every instance in the first launch re-condenses nothing"""
    from oracle.qp_assembly import QPData
    c = pendulum(); B = 1024; rng = np.random.default_rng(6)
    X0, Xref = pendulum_random(B, seed=12)
    Ad1 = np.broadcast_to(c["Ad"], (B, 4, 4)).copy(); Bd1 = np.broadcast_to(c["Bd"], (B, 4, 1)).copy()
    K = MPC(Ad1, Bd1, Np=20, x0=X0, xref=Xref, uminus1=np.zeros(1), batch=B, **{k: c[k] for k in KEYS}); K.setup()
    X = X0.copy(); U = K.output()
    for t in range(4):
        X = np.einsum("bij,bj->bi", Ad1, X) + np.einsum("bij,bj->bi", Bd1, U)
        K.update(X, U); U = K.output()
    # (a) the settled loop, every step with the same matrices again: a solve that k_tpi_pol finishes in its one launch re-condenses
    # nothing (every instance is stale after each update_system)
    one_launch = 0
    for t in range(6):
        K.update_system(Ad1, Bd1)
        X = _step(Ad1, Bd1, X, U)
        K.update(X, U); U = K.output()
        s = K.stats()
        if s["rounds"] == 1:
            one_launch += 1
            assert s["recondensed"] == 0 and s["admm_iters"] == 0, s
        else:
            assert s["recondensed"] > 0, s
    assert one_launch > 0
    # (b) a new model per instance; warm solve; the lazily refreshed consumers
    Ad2, Bd2 = cartpole_linearised(X, U)
    K.update_system(Ad2, Bd2)
    X = np.einsum("bij,bj->bi", Ad1, X) + np.einsum("bij,bj->bi", Bd1, U)
    K.update(X, U)
    Un, info = K.output(return_u_seq=True, return_x_seq=True, return_obj_val=True)
    st = np.array(K.res.info.status_val); assert (st == 1).mean() > 0.999
    useq = info["u_seq"][:, :, 0]; xseq = info["x_seq"]
    roll = np.empty_like(xseq); roll[:, 0] = X
    for k in range(20):
        roll[:, k + 1] = np.einsum("bij,bj->bi", Ad2, roll[:, k]) + Bd2[:, :, 0] * useq[:, k:k + 1]
    assert np.max(np.abs(xseq - roll)) < 1e-9
    for b in (0, B // 2, B - 1):
        if st[b] != 1:
            continue
        ref, Q, z = _oracle(dict(c, Ad=Ad2[b], Bd=Bd2[b], x0=X[b], xref=Xref[b], uminus1=U[b]))
        obj = 0.5 * z @ (Q.P @ z) + Q.q @ z + np.atleast_1d(K.J_CNST)[b]
        assert abs(info["obj_val"][b] - obj) < 1e-6 * max(1.0, abs(obj)), b
    Q0 = QPData(**dict(c, Ad=Ad2[0], Bd=Bd2[0], x0=X[0], xref=Xref[0], uminus1=U[0]))
    NX, NU = Q0.NX, Q0.NU
    Bcal = -np.linalg.solve(Q0.A[:NX, :NX], Q0.A[:NX, NX:NX + NU])
    H = Bcal.T @ Q0.P[:NX, :NX] @ Bcal + Q0.P[NX:NX + NU, NX:NX + NU]
    assert np.max(np.abs(K.condensed("H") - H)) / max(1.0, np.max(np.abs(H))) < 1e-12
    U = Un
    # (c) straggler rounds on re-condensed blocks
    Ad3, Bd3 = cartpole_linearised(X + 0.05 * rng.standard_normal(X.shape), U)
    K.update_system(Ad3, Bd3)
    X = np.einsum("bij,bj->bi", Ad2, X) + np.einsum("bij,bj->bi", Bd2, U)
    jump = rng.choice(B, 64, replace=False)
    X[jump] = pendulum_random(64, seed=78)[0]
    K.update(X, U)
    Un, info = K.output(return_u_seq=True)
    s = K.stats(); st = np.array(K.res.info.status_val)
    assert s["rounds"] > 1 and 0 < s["recondensed"] < B, s
    assert (st > 0).all()
    for b in [j for j in jump if st[j] == 1][:4]:
        ref, Q, z = _oracle(dict(c, Ad=Ad3[b], Bd=Bd3[b], x0=X[b], xref=Xref[b], uminus1=U[b]))
        assert np.max(np.abs(info["u_seq"][b, :, 0] - ref)) < TOL, b
    K.close()


@pytest.mark.parametrize("per", [False, True])
def test_update_system_with_the_current_matrices_is_a_no_op(MPC, per):
    c = pendulum(); B = 512
    X0, Xref = pendulum_random(B, seed=14)
    Ad = np.broadcast_to(c["Ad"], (B, 4, 4)).copy() if per else c["Ad"]
    Bd = np.broadcast_to(c["Bd"], (B, 4, 1)).copy() if per else c["Bd"]
    Ks = [MPC(Ad, Bd, Np=20, x0=X0, xref=Xref, uminus1=np.zeros(1), batch=B, **{k: c[k] for k in KEYS}) for _ in range(2)]
    for K in Ks:
        K.setup()
    X = X0.copy(); U = Ks[0].output().copy(); Ks[1].output()
    for t in range(4):
        X = _step(Ad, Bd, X, U)
        Ks[1].update_system(Ad, Bd)
        outs = []
        for K in Ks:
            K.update(X, U); outs.append(K.output().copy())
        assert np.array_equal(outs[0], outs[1]), t
        U = outs[0]
    for K in Ks:
        K.close()


def test_multi_input_pattern_change_is_answered_correctly(MPC):
    """the MIMO controller runs on the sparse-pattern instantiation of k_tpm_pol; a dense Ad leaves that pattern, so the entry is
    chosen again (the dense instantiation) — never a kernel that skips the new non-zeros"""
    c = mimo(); c.setdefault("eps_feas", 1e6); B = 128; rng = np.random.default_rng(7)
    X0 = 0.3 * rng.standard_normal((B, 8))
    kw = dict({k: c[k] for k in KEYS}, Np=40, batch=B, xref=c["xref"])
    K = MPC(c["Ad"], c["Bd"], x0=X0, uminus1=np.zeros(4), **kw); K.setup()
    X = X0.copy(); U = K.output()
    for t in range(2):
        X = X @ c["Ad"].T + U @ c["Bd"].T
        K.update(X, U); U = K.output()
    Ad2 = c["Ad"] + 0.01 * rng.standard_normal((8, 8))
    Ad2 *= 0.95 / max(abs(np.linalg.eigvals(Ad2)))
    K.update_system(Ad=Ad2)
    K.update(X, U); _, info = K.output(return_u_seq=True); u1 = info["u_seq"].reshape(B, -1); s1 = np.array(K.res.info.status_val)
    F = MPC(Ad2, c["Bd"], x0=X, uminus1=U, **kw); F.setup()
    _, info = F.output(return_u_seq=True); u2 = info["u_seq"].reshape(B, -1); s2 = np.array(F.res.info.status_val)
    both = (s1 == 1) & (s2 == 1)
    assert both.mean() > 0.9 and (s1 > 0).all()
    assert np.max(np.abs(u1[both] - u2[both])) < 1e-7
    for b in np.flatnonzero(both)[:3]:
        ref, Q, z = _oracle(dict(c, Ad=Ad2, x0=X[b], uminus1=U[b]))
        assert np.max(np.abs(u1[b] - ref)) < TOL, b
    K.close(); F.close()


@pytest.mark.parametrize("per", [False, True])
def test_singular_hessian_is_refused_until_a_valid_update(MPC, per):
    """Qu = QDu = 0: H = B'P_X B depends on Bd and is singular for Bd = 0 -> BmpcError, the next solve raises, and a valid
    update_system makes the controller usable again (per-instance systems condense eagerly here: P_U is not definite)"""
    from pympc_b200 import BmpcError
    c = pendulum(); B = 64
    X0, Xref = pendulum_random(B, seed=15)
    kw = dict({k: c[k] for k in KEYS}, Qx=np.eye(4), QxN=np.eye(4), Qu=np.zeros((1, 1)), QDu=np.zeros((1, 1)))
    Ad = np.broadcast_to(c["Ad"], (B, 4, 4)).copy() if per else c["Ad"]
    Bd = np.broadcast_to(c["Bd"], (B, 4, 1)).copy() if per else c["Bd"]
    K = MPC(Ad, Bd, Np=20, x0=X0, xref=Xref, uminus1=np.zeros(1), batch=B, **kw); K.setup()
    U = K.output().copy()
    with pytest.raises(BmpcError, match="not positive definite"):
        K.update_system(Bd=np.zeros_like(Bd))
    with pytest.raises(BmpcError, match="update_system"):
        K.update(X0, U)
    K.update_system(Bd=Bd)
    K.update(X0, U)
    u = K.output()
    st = np.array(K.res.info.status_val); assert (st > 0).all() and (st == 1).mean() > 0.9
    for b in np.flatnonzero(st == 1)[:2]:
        ref, Q, z = _oracle(dict(c, **{k: kw[k] for k in ("Qx", "QxN", "Qu", "QDu")}, x0=X0[b], xref=Xref[b], uminus1=U[b]))
        assert abs(u[b, 0] - ref[0]) < TOL
    K.close()
