"""-m gpu tests of time-varying weights, bounds and uref (MPCController.update_system keywords / bmpc_update_problem): after an
update the next update() is a warm solve of the QP the reference assembles with the new arrays — checked against a controller set
up from scratch with them and against the CPU oracle on each sampled instance's own QP, in every kernel family."""
import numpy as np
import pytest

from pympc_b200.workloads import pendulum, pendulum_random, mimo, cartpole_linearised

pytestmark = pytest.mark.gpu
TOL = 1e-6
KEYS = ("Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "eps_feas")
PROBLEM = ("Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "uref")


@pytest.fixture(scope="module")
def MPC(bmpc_lib):
    assert bmpc_lib.bmpc_device_count() > 0, "GPU tests need a CUDA device; the product has no CPU fallback"
    from pympc_b200 import MPCController
    return MPCController


def _oracle(cfg):
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
    if np.ndim(Ad) == 3:
        return np.einsum("bij,bj->bi", Ad, X) + np.einsum("bij,bj->bi", Bd, U)
    return X @ Ad.T + U @ Bd.T


def _family(name, rng):
    """-> (cfg, B, options, per-instance, SOFT_ON, X0, Xref)"""
    if name in ("pi_tpi", "shared_tpi", "team", "hard"):
        c = pendulum(); c["uref"] = np.zeros(1)
        B = {"pi_tpi": 2048, "shared_tpi": 1024, "team": 256, "hard": 256}[name]
        X0, Xref = pendulum_random(B, seed=5)
        if name == "hard":                      # hard state rows: keep the starts inside the box
            X0 = 0.3 * X0; c["xmin"] = np.array([-2.0, -100, -100, -100]); c["xmax"] = np.array([2.0, 100, 100, 100])
        opts = {"fast_path": 0} if name == "team" else {}
        return c, B, opts, name == "pi_tpi", name != "hard", X0, Xref
    if name == "mimo":
        c = mimo(); c.setdefault("eps_feas", 1e6); c["uref"] = np.zeros(4); B = 256
        X0 = 0.3 * rng.standard_normal((B, 8)); Xref = np.tile(c["xref"], (B, 1))
        return c, B, {}, False, True, X0, Xref
    c = _generic(); c["uref"] = np.zeros(2); B = 600
    X0 = 0.4 * rng.standard_normal((B, 4)); Xref = np.tile(np.array([0.7, 0, -0.5, 0]), (B, 1))
    return c, B, {}, False, True, X0, Xref


def _change(c, kind, B, per, rng):
    """new arrays for an update of `kind` (bounds, uref, weights, all): small changes (bounds by +-5 %, uref by a small offset);
    per-instance controllers get one set per instance"""
    nx, nu = c["Bd"].shape
    s = (lambda n: 1.0 + 0.05 * rng.uniform(-1, 1, (B, n))) if per else (lambda n: 1.0 + 0.05 * rng.uniform(-1, 1, n))
    new = {}
    if kind in ("bounds", "all"):
        for k, n in (("xmin", nx), ("xmax", nx), ("umin", nu), ("umax", nu), ("Dumin", nu), ("Dumax", nu)):
            new[k] = c[k] * s(n)
    if kind in ("uref", "all"):
        new["uref"] = 0.02 * (rng.standard_normal((B, nu)) if per else rng.standard_normal(nu))
    if kind in ("weights", "all"):
        for k, n in (("Qx", nx), ("QxN", nx), ("Qu", nu), ("QDu", nu)):
            base = c[k] + (1e-3 * np.eye(n) if k == "Qu" else 0.0)
            new[k] = np.einsum("bi,ij->bij", s(n), base) if per else np.diag(s(n)) @ base
    return new


def _inst(new, b, per):
    return {k: (v[b] if per and np.ndim(v) > (2 if k in ("Qx", "QxN", "Qu", "QDu", "Ad", "Bd") else 1) else v) for k, v in new.items()}


def _fresh(MPC, c, new, kw, per, soft, X, U):
    """a controller set up from scratch with the new arrays at (X, U): cold solve"""
    args = dict(kw); args.update({k: v for k, v in new.items() if k not in ("uref", "Ad", "Bd")})
    uref = new.get("uref", c["uref"])
    Ad, Bd = new.get("Ad", c["Ad"]), new.get("Bd", c["Bd"])
    if per:
        B = X.shape[0]
        Ad = np.broadcast_to(Ad, (B,) + np.shape(c["Ad"])).copy(); Bd = np.broadcast_to(Bd, (B,) + np.shape(c["Bd"])).copy()
    F = MPC(Ad, Bd, x0=X, uminus1=U, uref=None if np.ndim(uref) == 2 else uref, **args)
    F.SOFT_ON = soft
    F.setup(solve=False)
    if np.ndim(uref) == 2:                               # per-instance uref: set before the first (cold) solve
        F.update_system(uref=uref)
    F.solve()
    return F


@pytest.mark.parametrize("kind", ["bounds", "uref", "weights", "all"])
@pytest.mark.parametrize("name", ["pi_tpi", "shared_tpi", "team", "mimo", "generic", "hard"])
def test_update_equals_a_fresh_setup(MPC, name, kind):
    """three warm steps, the update, one warm step: the plan equals a fresh setup's at the same x0, u_-1 (instances verified by
    both) and the oracle on sampled instances; every status > 0; on the pendulum families the warm step is cheaper than a cold
    solve"""
    rng = np.random.default_rng(21)
    c, B, opts, per, soft, X0, Xref = _family(name, rng)
    nx, nu = c["Bd"].shape
    kw = dict({k: c[k] for k in KEYS}, Np=c["Np"], Nc=c.get("Nc"), batch=B, xref=Xref, **opts)
    Ad = np.broadcast_to(c["Ad"], (B, nx, nx)).copy() if per else c["Ad"]
    Bd = np.broadcast_to(c["Bd"], (B, nx, nu)).copy() if per else c["Bd"]
    K = MPC(Ad, Bd, x0=X0, uminus1=np.zeros(nu), uref=c["uref"], **kw); K.SOFT_ON = soft; K.setup()
    X = X0.copy(); U = K.output()
    for t in range(3):
        X = _step(Ad, Bd, X, U)
        K.update(X, U); U = K.output()
    new = _change(c, kind, B, per, rng)
    if kind == "all":
        if name == "pi_tpi":
            new["Ad"], new["Bd"] = cartpole_linearised(0.1 * X, np.zeros((B, 1)))
        elif name == "mimo":
            new["Ad"] = c["Ad"] * (1 + 0.02 * rng.standard_normal(c["Ad"].shape)); new["Bd"] = c["Bd"] * 1.1
        else:
            new["Ad"] = c["Ad"] + 0.01 * rng.standard_normal((nx, nx)) * (c["Ad"] != 0); new["Bd"] = c["Bd"] * 0.95
    X = _step(Ad, Bd, X, U)
    K.update_system(**new)
    K.update(X, U)
    _, info = K.output(return_u_seq=True); u1 = info["u_seq"].reshape(B, -1); s1 = np.array(K.res.info.status_val)
    warm_iters = K.stats()["admm_iters"]
    F = _fresh(MPC, c, new, kw, per, soft, X, U)
    _, info = F.output(return_u_seq=True); u2 = info["u_seq"].reshape(B, -1); s2 = np.array(F.res.info.status_val)
    cold_iters = F.stats()["admm_iters"]
    both = (s1 == 1) & (s2 == 1)
    assert (s1 > 0).all() and both.mean() > 0.9, (name, kind, both.mean(), np.unique(s1, return_counts=True))
    assert np.max(np.abs(u1[both] - u2[both])) < 1e-7, (name, kind)
    for b in np.flatnonzero(both)[:: max(1, both.sum() // 3)][:3]:
        cb = dict(c, **_inst(new, b, per), x0=X[b], xref=Xref[b], uminus1=U[b])
        ref, Q, z = _oracle(dict(cb, soft=soft))
        assert np.max(np.abs(u1[b] - ref)) < TOL, (name, kind, b)
    if name in ("pi_tpi", "shared_tpi") and kind != "all":
        assert warm_iters < cold_iters, (name, kind, warm_iters, cold_iters)
    K.close(); F.close()


@pytest.mark.parametrize("name", ["pi_tpi", "shared_tpi", "team"])
def test_rows_between_free_and_bounded(MPC, name):
    """umax from +inf to finite and back, xmin from finite to -inf: each row changes its rho and the fast path's row parameters;
    every step equals a fresh setup"""
    rng = np.random.default_rng(3)
    c, B, opts, per, soft, X0, Xref = _family(name, rng)
    kw = dict({k: c[k] for k in KEYS}, Np=20, batch=B, xref=Xref, **opts)
    kw["umax"] = np.array([np.inf])
    Ad = np.broadcast_to(c["Ad"], (B, 4, 4)).copy() if per else c["Ad"]
    Bd = np.broadcast_to(c["Bd"], (B, 4, 1)).copy() if per else c["Bd"]
    K = MPC(Ad, Bd, x0=X0, uminus1=np.zeros(1), **kw); K.setup()
    X = X0.copy(); U = K.output()
    cur = dict(umax=np.array([np.inf]), xmin=c["xmin"])
    for t, upd in enumerate([dict(umax=np.array([15.0])), dict(xmin=np.array([-np.inf, -100, -100, -100])), dict(umax=np.array([np.inf])),
                             dict(xmin=c["xmin"])]):
        X = _step(Ad, Bd, X, U)
        K.update_system(**upd); cur.update(upd)
        K.update(X, U)
        Un, info = K.output(return_u_seq=True); u1 = info["u_seq"].reshape(B, -1); s1 = np.array(K.res.info.status_val)
        F = MPC(Ad, Bd, x0=X, uminus1=U, **dict(kw, **cur)); F.setup()
        _, info = F.output(return_u_seq=True); u2 = info["u_seq"].reshape(B, -1); s2 = np.array(F.res.info.status_val)
        both = (s1 == 1) & (s2 == 1)
        assert (s1 > 0).all() and both.mean() > 0.9, (name, t, both.mean())
        assert np.max(np.abs(u1[both] - u2[both])) < 1e-7, (name, t)
        b = int(np.flatnonzero(both)[0])
        ref, Q, z = _oracle(dict(c, **cur, x0=X[b], xref=Xref[b], uminus1=U[b]))
        assert np.max(np.abs(u1[b] - ref)) < TOL, (name, t)
        F.close(); U = Un
    K.close()


@pytest.mark.parametrize("from_device", [False, True])
def test_per_instance_closed_loop_with_changing_limits(MPC, from_device):
    """8 192 pendulums, each with its own umax, Dumax and uref schedule, changed at every step (host arrays or device tensors):
    every step >= 99.9 % verified, sampled instances equal the oracle, a step that one launch finishes condenses nothing and runs
    no ADMM, and a step with jumped states condenses only its stragglers and stays exact"""
    c = pendulum(); B = 8192; rng = np.random.default_rng(17)
    X0, Xref = pendulum_random(B, seed=19)
    X0 = 0.5 * X0
    Ad = np.broadcast_to(c["Ad"], (B, 4, 4)).copy(); Bd = np.broadcast_to(c["Bd"], (B, 4, 1)).copy()
    K = MPC(Ad, Bd, Np=20, x0=X0, xref=Xref, uminus1=np.zeros(1), batch=B, **{k: c[k] for k in KEYS}); K.setup()
    X = X0.copy(); U = K.output().copy()
    lim = rng.uniform(8.0, 20.0, (B, 1)); rate = rng.uniform(2.0, 5.0, (B, 1)); off = rng.uniform(-0.05, 0.05, (B, 1))
    torch = pytest.importorskip("torch") if from_device else None
    one_round = 0
    for t in range(12):
        umax = lim * (1.0 - 0.02 * t / 12); Dumax = rate * (1.0 + 0.1 * np.sin(t)); uref = off * np.cos(0.3 * t)
        if t == 11:
            jump = rng.choice(B, 64, replace=False); X[jump] = pendulum_random(64, seed=80)[0]
        if from_device:
            dev = torch.device("cuda", K.device)
            T = {k: torch.tensor(np.ascontiguousarray(v), device=dev) for k, v in (("umax", umax), ("Dumax", Dumax), ("uref", uref))}
            torch.cuda.synchronize()
            K.update_system_from_device(**T)
        else:
            K.update_system(umax=umax, Dumax=Dumax, uref=uref)
        K.update(X, U)
        Un, info = K.output(return_u_seq=True)
        st = np.array(K.res.info.status_val); s = K.stats()
        assert (st == 1).mean() >= 0.999, (t, np.unique(st, return_counts=True))
        if s["rounds"] == 1:
            one_round += 1
            assert s["recondensed"] == 0 and s["admm_iters"] == 0, (t, s)
        if t == 11:
            assert s["rounds"] > 1 and 0 < s["recondensed"] < B, s
        useq = info["u_seq"][:, :, 0]
        pick = list(rng.choice(np.flatnonzero(st == 1), 2, replace=False)) + ([int(j) for j in jump if st[j] == 1][:2] if t == 11 else [])
        for b in pick:
            ref, Q, z = _oracle(dict(c, umax=umax[b], Dumax=Dumax[b], uref=uref[b], x0=X[b], xref=Xref[b], uminus1=U[b]))
            assert np.max(np.abs(useq[b] - ref)) < TOL, (t, b)
        U = Un.copy(); X = _step(Ad, Bd, X, U)
        if t == 11:
            break
    assert one_round > 0
    K.close()


@pytest.mark.parametrize("per", [False, True])
def test_singular_weights_are_refused_until_a_valid_update(MPC, per):
    """Qu = QDu = Qx = QxN = 0 makes H singular: BmpcError, the next update() raises, a valid weight update restores the
    controller (host weights; per-instance device weights take the eager condense-and-check path)"""
    from pympc_b200 import BmpcError
    c = pendulum(); B = 64
    X0, Xref = pendulum_random(B, seed=25)
    Ad = np.broadcast_to(c["Ad"], (B, 4, 4)).copy() if per else c["Ad"]
    Bd = np.broadcast_to(c["Bd"], (B, 4, 1)).copy() if per else c["Bd"]
    K = MPC(Ad, Bd, Np=20, x0=X0, xref=Xref, uminus1=np.zeros(1), batch=B, **{k: c[k] for k in KEYS}); K.setup()
    U = K.output().copy()
    z4, z1 = np.zeros((4, 4)), np.zeros((1, 1))
    modes = ["host", "device"] if per else ["host"]
    for mode in modes:
        if mode == "host":
            with pytest.raises(BmpcError, match="not positive definite"):
                K.update_system(Qx=z4, QxN=z4, Qu=z1, QDu=z1)
        else:
            torch = pytest.importorskip("torch"); dev = torch.device("cuda", K.device)
            T = {k: torch.zeros((B,) + s, dtype=torch.float64, device=dev) for k, s in (("Qx", (4, 4)), ("QxN", (4, 4)), ("Qu", (1, 1)), ("QDu", (1, 1)))}
            torch.cuda.synchronize()
            with pytest.raises(BmpcError, match="not positive definite"):
                K.update_system_from_device(**T)
        with pytest.raises(BmpcError, match="update_system"):
            K.update(X0, U)
        # bounds leave definiteness as it was: still refused (a shared system is condensed again at once and fails its check)
        if per:
            K.update_system(umax=np.array([15.0]))
        else:
            with pytest.raises(BmpcError, match="not positive definite"):
                K.update_system(umax=np.array([15.0]))
        with pytest.raises(BmpcError, match="update_system"):
            K.update(X0, U)
        K.update_system(Qx=c["Qx"], QxN=c["QxN"], Qu=c["Qu"], QDu=c["QDu"], umax=c["umax"])
        K.update(X0, U)
        u = K.output()
        st = np.array(K.res.info.status_val); assert (st > 0).all() and (st == 1).mean() > 0.9
        for b in np.flatnonzero(st == 1)[:2]:
            ref, Q, z = _oracle(dict(c, x0=X0[b], xref=Xref[b], uminus1=U[b]))
            assert abs(u[b, 0] - ref[0]) < TOL
    K.close()


def test_mimo_qdu_that_stops_being_diagonal_leaves_the_multi_input_fast_path(MPC):
    c = mimo(); c.setdefault("eps_feas", 1e6); B = 128; rng = np.random.default_rng(8)
    X0 = 0.3 * rng.standard_normal((B, 8))
    kw = dict({k: c[k] for k in KEYS}, Np=40, batch=B, xref=c["xref"])
    K = MPC(c["Ad"], c["Bd"], x0=X0, uminus1=np.zeros(4), **kw); K.setup()
    X = X0.copy(); U = K.output()
    for t in range(2):
        X = X @ c["Ad"].T + U @ c["Bd"].T
        K.update(X, U); U = K.output()
    QDu2 = np.asarray(c["QDu"], float) + 0.02 * (np.ones((4, 4)) - np.eye(4))
    K.update_system(QDu=QDu2)
    K.update(X, U); _, info = K.output(return_u_seq=True); u1 = info["u_seq"].reshape(B, -1); s1 = np.array(K.res.info.status_val)
    F = MPC(c["Ad"], c["Bd"], x0=X, uminus1=U, **dict(kw, QDu=QDu2)); F.setup()
    _, info = F.output(return_u_seq=True); u2 = info["u_seq"].reshape(B, -1); s2 = np.array(F.res.info.status_val)
    both = (s1 == 1) & (s2 == 1)
    assert both.mean() > 0.9 and (s1 > 0).all()
    assert np.max(np.abs(u1[both] - u2[both])) < 1e-7
    for b in np.flatnonzero(both)[:3]:
        ref, Q, z = _oracle(dict(c, QDu=QDu2, x0=X[b], uminus1=U[b]))
        assert np.max(np.abs(u1[b] - ref)) < TOL, b
    K.close(); F.close()


@pytest.mark.parametrize("per", [False, True])
def test_update_with_the_current_arrays_is_a_no_op(MPC, per):
    c = pendulum(); B = 512
    X0, Xref = pendulum_random(B, seed=14)
    Ad = np.broadcast_to(c["Ad"], (B, 4, 4)).copy() if per else c["Ad"]
    Bd = np.broadcast_to(c["Bd"], (B, 4, 1)).copy() if per else c["Bd"]
    Ks = [MPC(Ad, Bd, Np=20, x0=X0, xref=Xref, uminus1=np.zeros(1), batch=B, **{k: c[k] for k in KEYS}) for _ in range(2)]
    for K in Ks:
        K.setup()
    X = X0.copy(); U = Ks[0].output().copy(); Ks[1].output()
    cur = {k: c[k] for k in PROBLEM if k != "uref"}; cur["uref"] = np.zeros(1)
    for t in range(4):
        X = _step(Ad, Bd, X, U)
        Ks[1].update_system(Ad, Bd, **cur)
        outs = []
        for K in Ks:
            K.update(X, U); outs.append(K.output().copy())
        assert np.array_equal(outs[0], outs[1]), t
        U = outs[0]
    for K in Ks:
        K.close()


def test_u_failure_follows_the_new_uref(MPC):
    """per-instance Dumin > Dumax on a few instances makes their QPs infeasible: they output the NEW uref"""
    c = pendulum(); B = 256; rng = np.random.default_rng(30)
    X0, Xref = pendulum_random(B, seed=31)
    Ad = np.broadcast_to(c["Ad"], (B, 4, 4)).copy(); Bd = np.broadcast_to(c["Bd"], (B, 4, 1)).copy()
    K = MPC(Ad, Bd, Np=20, x0=X0, xref=Xref, uminus1=np.zeros(1), batch=B, **{k: c[k] for k in KEYS}); K.setup()
    U = K.output().copy()
    bad = rng.choice(B, 5, replace=False)
    Dumin = np.tile(c["Dumin"], (B, 1)); Dumax = np.tile(c["Dumax"], (B, 1))
    Dumin[bad] = 1.0; Dumax[bad] = -1.0
    uref = rng.uniform(-0.5, 0.5, (B, 1))
    K.update_system(Dumin=Dumin, Dumax=Dumax, uref=uref)
    assert np.array_equal(K.u_failure, uref)
    X = _step(Ad, Bd, X0, U)
    with pytest.warns(UserWarning):
        K.update(X, U)
    u = K.output()
    st = np.array(K.res.info.status_val)
    assert (st[bad] < 0).all(), st[bad]
    assert np.array_equal(u[bad], uref[bad])
    good = np.setdiff1d(np.arange(B), bad)
    assert (st[good] > 0).all()
    K.close()


def test_attributes_and_objective_describe_the_new_problem(MPC):
    """after an update K.P, K.q, K.A, K.l, K.u equal the oracle assembly of the new problem (instance 0), and on a per-instance
    controller whose Qu and QDu differ per instance, output(return_obj_val=True) is the oracle objective plus each instance's own
    J_CNST (before, J_CNST used instance 0's weights and one shared uref for every instance)"""
    c = pendulum(); B = 512; rng = np.random.default_rng(41)
    X0, Xref = pendulum_random(B, seed=42)
    Ad = np.broadcast_to(c["Ad"], (B, 4, 4)).copy(); Bd = np.broadcast_to(c["Bd"], (B, 4, 1)).copy()
    Qu = rng.uniform(0.0, 0.05, (B, 1, 1)); QDu = rng.uniform(0.005, 0.05, (B, 1, 1))
    kw = {k: c[k] for k in KEYS}; kw.update(Qu=Qu, QDu=QDu)
    K = MPC(Ad, Bd, Np=20, x0=X0, xref=Xref, uminus1=np.zeros(1), batch=B, **kw); K.setup()
    U = K.output().copy()
    X = _step(Ad, Bd, X0, U)
    K.update(X, U)
    u, info = K.output(return_u_seq=True, return_obj_val=True)
    st = np.array(K.res.info.status_val)
    for b in [b for b in (1, 100, B - 1) if st[b] == 1]:
        ref, Q, z = _oracle(dict(c, Qu=Qu[b], QDu=QDu[b], x0=X[b], xref=Xref[b], uminus1=U[b]))
        obj = 0.5 * z @ (Q.P @ z) + Q.q @ z + 0.5 * U[b] @ QDu[b] @ U[b]
        assert abs(info["obj_val"][b] - obj) < 1e-6 * max(1.0, abs(obj)), (b, info["obj_val"][b], obj)
    # new weights, bounds and uref
    new = dict(Qx=np.diag([0.5, 0.01, 1.5, 0.01]), QxN=np.diag([0.6, 0.0, 1.2, 0.0]), Qu=rng.uniform(0.0, 0.05, (B, 1, 1)),
               QDu=rng.uniform(0.005, 0.05, (B, 1, 1)), umax=rng.uniform(10, 20, (B, 1)), xmin=np.array([-1.2, -100, -100, -100]),
               uref=rng.uniform(-0.1, 0.1, (B, 1)))
    K.update_system(**new)
    U = u.copy(); X = _step(Ad, Bd, X, U)
    K.update(X, U)
    inst0 = dict(c, **_inst(new, 0, True), x0=X[0], xref=Xref[0], uminus1=U[0])
    ref, Q, z = _oracle(inst0)
    # the reference-form QP of instance 0 at the last update() (before output() commits the new u as u_-1)
    for name in ("P", "q", "A", "l", "u"):
        got = getattr(K, name); want = getattr(Q, name)
        got = got.toarray() if hasattr(got, "toarray") else np.asarray(got)
        want = want.toarray() if hasattr(want, "toarray") else np.asarray(want)
        fin = np.isfinite(want)
        assert np.array_equal(np.isfinite(got), fin) and np.max(np.abs(got[fin] - want[fin]), initial=0.0) < 1e-9, name
    u, info = K.output(return_u_seq=True, return_obj_val=True)
    st = np.array(K.res.info.status_val)
    for b in [b for b in (0, 7, 300, B - 1) if st[b] == 1]:
        ref, Q, z = _oracle(dict(c, **_inst(new, b, True), x0=X[b], xref=Xref[b], uminus1=U[b]))
        ur = new["uref"][b]
        J = 0.5 * 20 * ur @ new["Qu"][b] @ ur + 0.5 * U[b] @ new["QDu"][b] @ U[b]
        obj = 0.5 * z @ (Q.P @ z) + Q.q @ z + J
        assert abs(info["obj_val"][b] - obj) < 1e-6 * max(1.0, abs(obj)), (b, info["obj_val"][b], obj)
    K.close()
