"""-m gpu: per-instance multi-input systems (n_sys = batch, 3-D Ad with nu > 1) on the multi-input fast path: k_tpm_pol reading each
instance's field-major parameter view.  Checked against the team kernels (fast_path=0), a shared-system handle, controllers set up
afresh and the CPU oracle on each sampled instance's own QP; after update_system (host arrays and device tensors) the warm steps that
k_tpm_pol finishes in one launch condense nothing and run no ADMM."""
import numpy as np
import pytest

from pympc_b200.workloads import mimo

pytestmark = pytest.mark.gpu
TOL = 1e-6
W = ("Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax")


@pytest.fixture(scope="module")
def MPC(bmpc_lib):
    assert bmpc_lib.bmpc_device_count() > 0, "GPU tests need a CUDA device; the product has no CPU fallback"
    from pympc_b200 import MPCController
    return MPCController


def _oracle_u(cfg):
    from oracle.qp_assembly import QPData
    from oracle.kkt import solve_exact
    Q = QPData(**cfg)
    z, y, r = solve_exact(Q.P, Q.q, Q.A, Q.l, Q.u)
    return z[Q.NX:Q.NX + Q.NU]


def _base(Np=40, Nc=None):
    c = dict(mimo(), Np=Np, Nc=Nc or Np)
    c["Qu"] = 0.01 * np.eye(4)                                  # (so that uref enters the cost)
    return c


def _fleet(c, B, rng):
    """governor systems perturbed inside their sparsity pattern (poles by 0.2 %, input gains by 10 %: the steady-state inputs stay
    inside every instance's umax), with per-instance Qx scale, umax, Dumax and uref"""
    Ad = c["Ad"][None] * (1.0 + 0.002 * rng.standard_normal((B, 8, 8)))   # (DC gain 1 - a1 - a2 = 0.046: +-8 %)
    Bd = c["Bd"][None] * (1.0 + 0.1 * rng.standard_normal((B, 8, 4)))
    s = rng.uniform(0.5, 2.0, B)[:, None, None]
    umax = rng.uniform(1.5, 3.0, (B, 4)); Dumax = rng.uniform(0.1, 0.3, (B, 4))
    P = dict(Qx=s * c["Qx"], QxN=s * c["QxN"], umin=-umax, umax=umax, Dumin=-Dumax, Dumax=Dumax, uref=0.05 * rng.standard_normal((B, 4)))
    return Ad, Bd, P


def _make(MPC, c, Ad, Bd, B, X0, fast_path, P=None, xref=None):
    K = MPC(Ad, Bd, Np=c["Np"], Nc=c["Nc"], x0=X0, xref=c["xref"] if xref is None else xref, uminus1=np.zeros(4), batch=B,
            fast_path=fast_path, **{k: c[k] for k in W})
    K.setup(solve=False)
    if P:
        K.update_system(**P)
    return K


def _inst(c, Ad, Bd, P, b):
    d = dict(c, Ad=Ad[b], Bd=Bd[b])
    for k, v in (P or {}).items():
        d[k] = v[b]
    return d


def _run(Ks, X, U, steps, c, Ad, Bd, P=None, xref=None, oracle=(1,), hook=None):
    """closed loop of the controllers Ks on the same states; per step: statuses, u*, stats; the loop follows Ks[-1]'s plan"""
    B = X.shape[0]; hist = []
    for t in range(steps):
        if hook:
            hook(t)
        outs, sts, stats = [], [], []
        for K in Ks:
            K.update(X, U, xref=xref) if xref is not None else K.update(X, U)
            Un, info = K.output(return_u_seq=True)
            outs.append(info["u_seq"].reshape(B, -1)); sts.append(np.array(K.res.info.status_val).copy())
            stats.append(dict(K.stats(), no_admm=int((np.array(K.res.info.iter) == 0).sum())))
            assert np.isin(sts[-1], (1, 2)).all(), (t, np.unique(sts[-1], return_counts=True))
        for b in oracle:
            if sts[0][b] == 1:
                ref = _oracle_u(dict(_inst(c, Ad, Bd, P, b), x0=X[b], uminus1=U[b], **({"xref": xref[b]} if xref is not None else {})))
                assert np.max(np.abs(outs[0][b] - ref)) < TOL, (t, b)
        hist.append((outs, sts, stats))
        U = outs[-1][:, :4].copy()
        X = np.einsum("bij,bj->bi", Ad, X) + np.einsum("bij,bj->bi", Bd, U)
    return hist, X, U


def _agree(hist, tol=TOL, share=0.97):
    for t, (outs, sts, _) in enumerate(hist):
        both = (sts[0] == 1) & (sts[1] == 1)
        assert both.mean() > share, (t, both.mean())
        assert np.max(np.abs(outs[0][both] - outs[1][both])) < tol, t


def _no_admm_share(hist, B):
    """share of the warm steps' instances each controller verified without any ADMM iteration (only k_tpm_pol does that)"""
    return [sum(h[2][i]["no_admm"] for h in hist[1:]) / (B * (len(hist) - 1)) for i in range(2)]


def test_heterogeneous_fleet_agrees_with_team_path(MPC):
    """512 perturbed governor systems with their own Qx scale, umax, Dumax and uref, 8 steps from a cold start: > 97 % verified by
    both paths and equal within 1e-6, samples equal the oracle, and k_tpm_pol verifies a large share of the warm steps' instances
    without ADMM (the team kernels never do).  (On this fleet the active per-instance input bounds leave 25-70 % of a warm step's
    instances to straggler rounds of 100 ADMM iterations, so the total ADMM count is NOT below the team path's: DESIGN §7.)"""
    c = _base(); B = 512; rng = np.random.default_rng(41)
    Ad, Bd, P = _fleet(c, B, rng)
    X0 = 0.3 * rng.standard_normal((B, 8))
    Ks = [_make(MPC, c, Ad, Bd, B, X0, f, P) for f in (1, 0)]
    hist, _, _ = _run(Ks, X0.copy(), np.zeros((B, 4)), 8, c, Ad, Bd, P, oracle=(1, B // 3, B - 5))
    _agree(hist)
    share = _no_admm_share(hist, B)
    assert share[0] > 0.3 and share[1] == 0.0, share
    for K in Ks:
        K.close()


def test_identical_instances_equal_a_shared_handle(MPC):
    """a per-instance handle whose 128 instances all hold the governor system gives the shared handle's u* (1e-9) at every step"""
    c = _base(); B = 128; rng = np.random.default_rng(3)
    X0 = 0.3 * rng.standard_normal((B, 8))
    Ad = np.broadcast_to(c["Ad"], (B, 8, 8)).copy(); Bd = np.broadcast_to(c["Bd"], (B, 8, 4)).copy()
    Kp = _make(MPC, c, Ad, Bd, B, X0, 1)
    Ks = _make(MPC, c, c["Ad"], c["Bd"], B, X0, 1)
    hist, _, _ = _run([Kp, Ks], X0.copy(), np.zeros((B, 4)), 8, c, Ad, Bd)
    for t, (outs, sts, stats) in enumerate(hist):
        assert np.array_equal(sts[0], sts[1]) and np.max(np.abs(outs[0] - outs[1])) < 1e-9, t
        assert stats[0]["admm_iters"] == stats[1]["admm_iters"] and stats[0]["rounds"] == stats[1]["rounds"], t   # the same kernels
    Kp.close(); Ks.close()


def test_pattern_outside_the_sparse_masks_and_a_held_input(MPC):
    """one instance with an entry outside the governor's sparsity pattern: the handle runs the dense entry, exactly.  So does
    (8,4,12,5) (Nc < Np) with per-instance systems and a time-varying xref"""
    c = _base(); B = 96; rng = np.random.default_rng(8)
    Ad, Bd, P = _fleet(c, B, rng)
    Ad[5, 0, 7] = 0.01; Bd[9, 3, 0] = 0.05
    X0 = 0.3 * rng.standard_normal((B, 8))
    Ks = [_make(MPC, c, Ad, Bd, B, X0, f, P) for f in (1, 0)]
    hist, _, _ = _run(Ks, X0.copy(), np.zeros((B, 4)), 6, c, Ad, Bd, P, oracle=(5, 9, 40))
    _agree(hist)
    share = _no_admm_share(hist, B)
    assert share[0] > 0.3 and share[1] == 0.0, share               # the dense entry of k_tpm_pol verifies warm instances alone
    for K in Ks:
        K.close()
    c = _base(12, 5); B = 256
    Ad, Bd, P = _fleet(c, B, rng)
    X0 = 0.3 * rng.standard_normal((B, 8))
    Xtv = c["xref"][None, None, :] * np.linspace(0.6, 1.0, 13)[None, :, None] * rng.uniform(0.8, 1.2, (B, 1, 1))
    Ks = [_make(MPC, c, Ad, Bd, B, X0, f, P) for f in (1, 0)]
    hist, _, _ = _run(Ks, X0.copy(), np.zeros((B, 4)), 6, c, Ad, Bd, P, xref=Xtv, oracle=(0, 77))
    _agree(hist, share=0.95)
    for K in Ks:
        K.close()


def _settle(K, c, Ad, Bd, B, steps=12):
    X = np.broadcast_to(c["xref"], (B, 8)).copy(); U = np.ones((B, 4))
    for _ in range(steps):
        K.update(X, U); U = K.output().copy()
        X = np.einsum("bij,bj->bi", Ad, X) + np.einsum("bij,bj->bi", Bd, U)
    return X, U


@pytest.mark.parametrize("from_device", [False, True])
def test_update_system_equals_a_fresh_setup_and_keeps_the_lazy_path(MPC, from_device):
    """update_system(Ad, Bd) (host arrays or device tensors): the next step equals a controller set up afresh with the new systems
    (1e-7 on instances both verified) and the oracle.  In a settled loop that updates (Ad, Bd) every step, every step that one
    launch finishes re-condenses nothing and runs no ADMM.  A device update that takes one instance outside the sparse masks is
    answered exactly"""
    torch = pytest.importorskip("torch") if from_device else None
    c = _base(); B = 128; rng = np.random.default_rng(23)
    Ad, Bd, P = _fleet(c, B, rng)
    K = _make(MPC, c, Ad, Bd, B, np.zeros((B, 8)), 1, P)
    X, U = _settle(K, c, Ad, Bd, B)

    def push(Ad_, Bd_):
        if from_device:
            dev = torch.device("cuda", K.device)
            Ta, Tb = (torch.tensor(np.ascontiguousarray(a), device=dev) for a in (Ad_, Bd_))
            torch.cuda.synchronize()
            K.update_system_from_device(Ta, Tb)
            return Ta, Tb
        K.update_system(Ad_, Bd_)
    one = 0
    for t in range(8):
        Ad = Ad * (1.0 + 1e-4 * rng.standard_normal(Ad.shape)); keep = push(Ad, Bd)
        K.update(X, U); Un = K.output().copy(); s = K.stats(); st = np.array(K.res.info.status_val)
        assert (st == 1).mean() > 0.99, (t, s)
        if s["rounds"] == 1:
            one += 1
            assert s["recondensed"] == 0 and s["admm_iters"] == 0, (t, s)
        U = Un; X = np.einsum("bij,bj->bi", Ad, X) + np.einsum("bij,bj->bi", Bd, U)
    assert one >= 4, one
    # a model change of a transient's size, compared with a fresh setup
    Ad2, Bd2, _ = _fleet(c, B, rng)
    X = X + 0.2 * rng.standard_normal(X.shape)
    if from_device:
        Ad2[7, 1, 6] = 0.02                                       # outside the sparse masks: the dense entry takes over
    keep = push(Ad2, Bd2)
    K.update(X, U); Un, info = K.output(return_u_seq=True); st = np.array(K.res.info.status_val)
    F = _make(MPC, c, Ad2, Bd2, B, X, 1, P); F.update(X, U); Fn, finfo = F.output(return_u_seq=True); fst = np.array(F.res.info.status_val)
    both = (st == 1) & (fst == 1)
    assert both.mean() > 0.97 and np.max(np.abs(info["u_seq"].reshape(B, -1)[both] - finfo["u_seq"].reshape(B, -1)[both])) < 1e-7
    for b in (0, 7, 100):
        if st[b] == 1:
            ref = _oracle_u(dict(_inst(c, Ad2, Bd2, P, b), x0=X[b], uminus1=U[b]))
            assert np.max(np.abs(info["u_seq"].reshape(B, -1)[b] - ref)) < TOL, b
    del keep
    K.close(); F.close()


def test_weight_bound_uref_updates_and_a_non_diagonal_qdu(MPC):
    """update_system(umax, Dumax, uref, Qx) equals a fresh setup; a non-diagonal QDu on one instance stays exact on the team
    kernels, and diagonal again returns a settled step to zero ADMM iterations"""
    c = _base(); B = 128; rng = np.random.default_rng(29)
    Ad, Bd, P = _fleet(c, B, rng)
    K = _make(MPC, c, Ad, Bd, B, np.zeros((B, 8)), 1, P)
    X, U = _settle(K, c, Ad, Bd, B)
    P2 = dict(P, umax=P["umax"] * 0.9, umin=-P["umax"] * 0.9, Dumax=P["Dumax"] * 1.1, Dumin=-P["Dumax"] * 1.1,
              uref=P["uref"] + 0.02, Qx=P["Qx"] * 1.5)
    K.update_system(umax=P2["umax"], umin=P2["umin"], Dumax=P2["Dumax"], Dumin=P2["Dumin"], uref=P2["uref"], Qx=P2["Qx"])
    K.update(X, U); Un, info = K.output(return_u_seq=True); st = np.array(K.res.info.status_val)
    F = _make(MPC, c, Ad, Bd, B, X, 1, P2); F.update(X, U); Fn, finfo = F.output(return_u_seq=True); fst = np.array(F.res.info.status_val)
    both = (st == 1) & (fst == 1)
    assert both.mean() > 0.97 and np.max(np.abs(info["u_seq"].reshape(B, -1)[both] - finfo["u_seq"].reshape(B, -1)[both])) < 1e-7
    F.close()
    U = Un.copy(); X = np.einsum("bij,bj->bi", Ad, X) + np.einsum("bij,bj->bi", Bd, U)
    QDu = np.broadcast_to(c["QDu"], (B, 4, 4)).copy(); QDu[3, 0, 1] = QDu[3, 1, 0] = 0.1
    K.update_system(QDu=QDu)
    P3 = dict(P2, QDu=QDu)
    for t in range(3):
        K.update(X, U); Un, info = K.output(return_u_seq=True); st = np.array(K.res.info.status_val); s = K.stats()
        assert s["admm_iters"] > 0, (t, s)                         # team kernels: every instance runs ADMM
        for b in (3, 50):
            assert st[b] == 1
            ref = _oracle_u(dict(_inst(c, Ad, Bd, P3, b), x0=X[b], uminus1=U[b]))
            assert np.max(np.abs(info["u_seq"].reshape(B, -1)[b] - ref)) < TOL, (t, b)
        U = Un.copy(); X = np.einsum("bij,bj->bi", Ad, X) + np.einsum("bij,bj->bi", Bd, U)
    K.update_system(QDu=np.broadcast_to(c["QDu"], (B, 4, 4)).copy())
    zero = 0
    for t in range(4):
        K.update(X, U); U = K.output().copy(); s = K.stats()
        zero += s["admm_iters"] == 0 and s["rounds"] == 1
        X = np.einsum("bij,bj->bi", Ad, X) + np.einsum("bij,bj->bi", Bd, U)
    assert zero >= 2, zero
    K.close()


def test_fast_path_2_builds_a_per_instance_shape_on_demand(MPC):
    """fast_path=2 at a per-instance shape outside the in-tree table, (3,2,10,6): the shape is built with the union of the
    instances' patterns and agrees with the team path and the oracle"""
    rng = np.random.default_rng(5); B = 256
    A = rng.standard_normal((3, 3)); A *= 0.95 / max(abs(np.linalg.eigvals(A))); A[2, 0] = 0.0
    Bm = rng.standard_normal((3, 2))
    Ad = A[None] * (1.0 + 0.05 * rng.standard_normal((B, 3, 3))); Bd = Bm[None] * (1.0 + 0.05 * rng.standard_normal((B, 3, 2)))
    c = dict(Np=10, Nc=6, Qx=np.diag([1.0, 0.5, 0.2]), QxN=np.diag([2.0, 0.5, 0.2]), Qu=np.array([[0.1, 0.02], [0.02, 0.3]]),
             QDu=np.diag([0.5, 0.2]), xmin=-1.5 * np.ones(3), xmax=1.5 * np.ones(3), umin=-np.array([0.8, 0.5]), umax=np.array([0.6, 0.9]),
             Dumin=-np.array([0.3, 0.4]), Dumax=np.array([0.4, 0.3]), eps_feas=1e3, uref=np.array([0.05, -0.05]))
    X0 = rng.uniform(-1.2, 1.2, (B, 3)); Xr = 0.3 * rng.standard_normal((B, 3))
    Ks = [MPC(Ad, Bd, **c, x0=X0, xref=Xr, uminus1=np.zeros(2), batch=B, fast_path=f) for f in (2, 0)]
    for K in Ks:
        K.setup()
    assert Ks[0]._L.bmpc_has_multi_input_fast_path(3, 2, 10, 6) == 1 and Ks[1]._L.bmpc_has_multi_input_fast_path(3, 2, 10, 6) == 0
    X = X0.copy(); U = np.zeros((B, 2)); its = [0, 0]
    for t in range(8):
        outs, sts = [], []
        for i, K in enumerate(Ks):
            K.update(X, U); Un, info = K.output(return_u_seq=True)
            outs.append(info["u_seq"].reshape(B, -1)); sts.append(np.array(K.res.info.status_val).copy()); its[i] += K.stats()["admm_iters"]
            assert np.isin(sts[-1], (1, 2)).all(), (t, i)
        both = (sts[0] == 1) & (sts[1] == 1)
        assert both.mean() > 0.95 and np.max(np.abs(outs[0][both] - outs[1][both])) < TOL, (t, both.mean())
        for b in (0, 101):
            if sts[0][b] == 1:
                ref = _oracle_u(dict(c, Ad=Ad[b], Bd=Bd[b], x0=X[b], xref=Xr[b], uminus1=U[b]))
                assert np.max(np.abs(outs[0][b] - ref)) < TOL, (t, b)
        U = outs[1][:, :2].copy(); X = np.einsum("bij,bj->bi", Ad, X) + np.einsum("bij,bj->bi", Bd, U)
    assert its[0] < 0.8 * its[1], its
    for K in Ks:
        K.close()
