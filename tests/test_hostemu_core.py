"""CPU checks of the DEVICE numerical core compiled for the host with a one-thread team
(tests/hostemu).  Catches index/algorithm errors without a GPU; parallel hazards are covered by the
-m gpu parity tests.  The emulation library is test infrastructure and is never loaded by pympc_b200."""
import numpy as np
import pytest

from conftest import golden
from emu import EmuSystem, launch_tiers
from oracle.qp_assembly import QPData
from pympc_b200.workloads import point_mass, pendulum, mimo

CASES = {"pm": point_mass, "pend": pendulum, "mimo": mimo}


def condensed_numpy(Q):
    """dense condensed operators from the oracle QP (eliminating X through the dynamics rows)"""
    NX, NU = Q.NX, Q.NU
    Ax = Q.A[:NX, :NX]; Bu = Q.A[:NX, NX:NX + NU]
    Bcal = -np.linalg.solve(Ax, Bu)
    H = Bcal.T @ Q.P[:NX, :NX] @ Bcal + Q.P[NX:NX + NU, NX:NX + NU]
    D = Q.A[2 * NX + NU:, NX:NX + NU]
    A = np.vstack([Bcal, np.eye(NU), D])
    return Bcal, H, A


@pytest.mark.parametrize("name", list(CASES))
def test_condense_matches_numpy(name):
    cfg = CASES[name](); Q = QPData(**cfg); E = EmuSystem(cfg)
    Bcal, H, A = condensed_numpy(Q)
    rel = lambda a, b: np.max(np.abs(a - b)) / max(1.0, np.max(np.abs(b)))
    assert rel(E.get("Bcal", Bcal.shape), Bcal) < 1e-12
    assert rel(E.get("H", H.shape), H) < 1e-12
    assert rel(E.get("Hinv", H.shape), np.linalg.inv(H)) < 1e-9
    rho = E.get("rho", (E.mc,))
    K = H + 1e-6 * np.eye(Q.NU) + A.T @ (rho[:, None] * A)
    assert rel(E.get("Kinv", H.shape), np.linalg.inv(K)) < 1e-9
    assert rel(E.get("M", (E.mc, E.mc)), A @ np.linalg.inv(H) @ A.T) < 1e-9


@pytest.mark.parametrize("name", list(CASES))
def test_first_solve_matches_golden(name):
    cfg = CASES[name](); g = golden(f"{name}_first.npz"); E = EmuSystem(cfg)
    U, st, it, ps, res = E.solve(cfg["x0"], cfg["uminus1"], cfg["xref"])
    assert st == 1
    assert np.max(np.abs(U - g["u_seq"])) < 1e-7


@pytest.mark.parametrize("name,steps", [("pm", 30), ("pend", 40), ("mimo", 6)])
def test_closed_loop_matches_golden(name, steps):
    cfg = CASES[name](); g = golden(f"{name}_loop.npz"); E = EmuSystem(cfg)
    x = np.array(cfg["x0"], float); um1 = np.array(cfg["uminus1"], float)
    for t in range(steps):
        U, st, it, ps, res = E.solve(x, um1, cfg["xref"])
        assert st == 1
        u0 = U[:E.nu]
        assert np.max(np.abs(u0 - g["u"][t])) < 1e-6, (t, u0, g["u"][t])
        x = cfg["Ad"] @ x + cfg["Bd"] @ u0; um1 = u0


def test_variants_match_golden():
    g = golden("variants.npz")
    c = point_mass(); c["Np"] = 25; c["Nc"] = 10; c["uref"] = np.array([0.1])
    c["xmin"] = np.array([-10.0, -10.0]); c["xmax"] = np.array([7.0, 10.0])
    E = EmuSystem(c); U, st, *_ = E.solve(c["x0"], c["uminus1"], g["a_xref"])
    assert st == 1 and np.max(np.abs(U - g["a_z"][26 * 2:26 * 2 + 10])) < 1e-7
    c = mimo(); c["Np"] = 12; c["Nc"] = 5; c["x0"] = np.array([0.3, -0.2, 0.1, 0.0, -0.4, 0.2, 0.0, 0.1])
    c["umin"] = -0.5 * np.ones(4); c["umax"] = 0.5 * np.ones(4); c["Qu"] = 0.1 * np.eye(4)
    E = EmuSystem(c); U, st, *_ = E.solve(c["x0"], c["uminus1"], c["xref"])
    assert st == 1 and np.max(np.abs(U - g["b_z"][13 * 8:13 * 8 + 20])) < 1e-7
    c = pendulum(); c["x0"] = np.array([0.45, 0.3, -0.05, 0.1])
    E = EmuSystem(c); U, st, *_ = E.solve(c["x0"], c["uminus1"], c["xref"])
    assert st == 1 and np.max(np.abs(U - g["c_z"][84:104])) < 1e-7


def test_random_batch_matches_golden():
    g = golden("pend_rand.npz"); cfg = pendulum()
    for b in range(g["X0"].shape[0]):
        E = EmuSystem(cfg)
        x = g["X0"][b].copy(); um1 = np.zeros(1)
        for t in range(g["U"].shape[0]):
            U, st, *_ = E.solve(x, um1, g["Xref"][b])
            assert st == 1 and abs(U[0] - g["U"][t, b, 0]) < 1e-6
            x = cfg["Ad"] @ x + cfg["Bd"] @ U[:1]; um1 = U[:1]


@pytest.mark.parametrize("name,steps", [("pm", 30), ("pend", 40)])
def test_tpi_fast_path_closed_loop(name, steps):
    """thread-per-instance ADMM + polish (bmpc_tpi.cuh), falling back to the team path like the library does"""
    cfg = CASES[name](); g = golden(f"{name}_loop.npz"); E = EmuSystem(cfg)
    x = np.array(cfg["x0"], float); um1 = np.array(cfg["uminus1"], float)
    used = 0
    for t in range(steps):
        U, ps = E.tpi_step(x, um1, cfg["xref"], pdas_steps=8)
        if ps <= 0:
            U, st, *_ = E.solve(x, um1, cfg["xref"]); assert st == 1
        else:
            used += 1
        assert np.max(np.abs(U[:E.nu] - g["u"][t])) < 1e-6, t
        x = cfg["Ad"] @ x + cfg["Bd"] @ U[:E.nu]; um1 = U[:E.nu]
    assert used >= steps - 2          # the fast path itself must carry the loop, not the fallback


def test_tpi_fast_path_random_batch():
    g = golden("pend_rand.npz"); cfg = pendulum()
    for b in range(g["X0"].shape[0]):
        E = EmuSystem(cfg)
        x = g["X0"][b].copy(); um1 = np.zeros(1)
        for t in range(g["U"].shape[0]):
            U, ps = E.tpi_step(x, um1, g["Xref"][b], pdas_steps=8)
            if ps <= 0:
                U, st, *_ = E.solve(x, um1, g["Xref"][b]); assert st == 1
            assert abs(U[0] - g["U"][t, b, 0]) < 1e-6
            x = cfg["Ad"] @ x + cfg["Bd"] @ U[:1]; um1 = U[:1]


@pytest.mark.parametrize("name,Nc,T", [("mimo", None, 4), ("pend", None, 4), ("pend", 7, 2), ("mimo", 12, 8), ("mimo", None, 2), ("pend", None, 8)])
def test_tile_admm_equals_team_admm(name, Nc, T):
    """The tile ADMM (T instances per CTA, Toeplitz prediction blocks) is the same iteration as the per-instance team
    ADMM: identical iterates (to rounding: the sums run in a different order), residuals and adaptive-rho moves."""
    cfg = CASES[name]()
    if Nc is not None:
        cfg = dict(cfg, Nc=Nc)
    E = EmuSystem(cfg); nx, nu = E.nx, E.nu
    rng = np.random.default_rng(5)
    X0 = np.asarray(cfg["x0"], float) + 0.3 * rng.standard_normal((T, nx))
    Um1 = 0.1 * rng.standard_normal((T, nu)); Xref = np.tile(np.asarray(cfg["xref"], float), (T, 1))
    ref, til = E.tile_compare(X0, Um1, Xref, niter=10, T=T)
    for k in ("x", "v", "xt"):
        assert np.abs(ref[k] - til[k]).max() <= 1e-9 * (1 + np.abs(ref[k]).max()), k
    assert np.allclose(ref["res"], til["res"], rtol=1e-7, atol=1e-12)
    assert (ref["lvl"] == til["lvl"]).all()
    # warm continuation on mixed ladder levels (instances of one tile may sit on different rho levels)
    lv = np.array([1, 2, 3, 2, 2, 4, 1, 2][:T], np.int32)
    ref2, til2 = E.tile_compare(X0, Um1, Xref, niter=7, lvl=lv, x_in=ref["x"], v_in=ref["v"], T=T)
    for k in ("x", "v", "xt"):
        assert np.abs(ref2[k] - til2[k]).max() <= 1e-9 * (1 + np.abs(ref2[k]).max()), k
    assert np.allclose(ref2["res"], til2["res"], rtol=1e-7, atol=1e-12)
    # time-varying reference (xref_mode 1)
    Xtv = np.tile(Xref[:, None, :], (1, E.Np + 1, 1)) * np.linspace(0.5, 1.0, E.Np + 1)[None, :, None]
    ref3, til3 = E.tile_compare(X0, Um1, Xtv, niter=5, T=T)
    assert np.abs(ref3["v"] - til3["v"]).max() <= 1e-9 * (1 + np.abs(ref3["v"]).max())


def test_primal_infeasibility_certificate():
    """OSQP's certificate as the straggler rounds evaluate it (bmpc_primal_infeasible): found for an initial state outside
    HARD state bounds (no feasible trajectory), not found for the same problem with a feasible start or with soft bounds."""
    cfg = point_mass(); cfg["xmax"] = np.array([3.0, 100.0])
    hard = EmuSystem(cfg, soft_on=0); soft = EmuSystem(cfg, soft_on=1)
    um1 = np.zeros(1)
    # the transient parts of y have to die out before the difference is a clean certificate (fixed rho here; the device
    # rounds also move rho, which speeds this up)
    assert hard.infeasible(np.array([3.5, 0.0]), um1, cfg["xref"], it0=400, it1=400)
    for it in (25, 400):
        assert not hard.infeasible(np.array([0.1, 0.2]), um1, cfg["xref"], it0=it, it1=it)
        assert not soft.infeasible(np.array([3.5, 0.0]), um1, cfg["xref"], it0=it, it1=it)


@pytest.mark.parametrize("name", ["pend", "pm"])
def test_tpi_fast_path_time_varying_reference(name):
    """SURVEY 8f-2 on the fast path: a (Np+1, nx) reference per instance (mpc.py:414-421) through the thread-per-instance
    ADMM (linear term by the adjoint recursion) and the Riccati polish (stage-wise linear terms): closed loop vs the exact
    solver on the oracle-assembled QP and vs the generic team code."""
    from oracle.kkt import solve_exact
    cfg = CASES[name](); Np = cfg.get("Np", 20); nx = len(cfg["x0"])
    rng = np.random.default_rng(8)
    E = EmuSystem(cfg); G = EmuSystem(cfg)
    x = np.asarray(cfg["x0"], float).copy(); um1 = np.asarray(cfg["uminus1"], float).reshape(-1).copy()
    fast = 0
    for t in range(6):
        # a reference that moves along the horizon (ramp + a wiggle on the first state)
        Xtv = np.tile(np.asarray(cfg["xref"], float), (Np + 1, 1)) * np.linspace(0.4, 1.0, Np + 1)[:, None]
        Xtv[:, 0] += 0.05 * np.sin(0.3 * (np.arange(Np + 1) + t)) + 0.02 * rng.standard_normal()
        U, ps = E.tpi_step(x, um1, Xtv, first_iters=10)
        fast += ps > 0
        if ps <= 0:                                             # stragglers take the generic route, like on the device
            U, st, *_ = E.solve(x, um1, Xtv); assert st == 1
        Ug, st, *_ = G.solve(x, um1, Xtv); assert st == 1
        Q = QPData(**dict(cfg, x0=x, uminus1=um1, xref=Xtv)); z, y, r = solve_exact(Q.P, Q.q, Q.A, Q.l, Q.u)
        ref = z[Q.NX:Q.NX + Q.NU]
        assert np.max(np.abs(Ug - ref)) < 1e-7
        assert np.max(np.abs(U - ref)) < 1e-7, (t, ps)
        um1 = U[:1].copy(); x = cfg["Ad"] @ x + cfg["Bd"] @ um1
    assert fast >= 4                                            # the fast path itself verified most steps


def test_tpi_fast_path_control_horizon_shorter_than_prediction():
    """Nc < Np on the fast path (mpc.py:513-517,540-543): the input is held after Nc moves.  ADMM sweeps collect the held
    stages into the last input; the Riccati polish treats stages k >= Nc as pinned to u_k = u_{k-1} without a row.
    Closed loop vs the exact solver on the oracle-assembled QP."""
    from oracle.kkt import solve_exact
    cfg = dict(pendulum(), Nc=10)
    E = EmuSystem(cfg); rng = np.random.default_rng(2)
    x = np.array([0.1, 0.2, 0.2, -0.1]); um1 = np.zeros(1); fast = 0
    for t in range(12):
        U, ps = E.tpi_step(x, um1, cfg["xref"], first_iters=10)
        assert ps != -100, "shape not compiled in the host emulation"
        fast += ps > 0
        if ps <= 0:
            U, st, *_ = E.solve(x, um1, cfg["xref"]); assert st == 1
        Q = QPData(**dict(cfg, x0=x, uminus1=um1)); z, y, r = solve_exact(Q.P, Q.q, Q.A, Q.l, Q.u)
        assert np.max(np.abs(U - z[Q.NX:Q.NX + Q.NU])) < 1e-7, (t, ps)
        um1 = U[:1].copy(); x = cfg["Ad"] @ x + cfg["Bd"] @ um1 + 0.01 * rng.standard_normal(4)
    assert fast >= 9


def test_tpi_fast_path_time_varying_reference_with_held_input():
    """Both f2 features at once on the fast path: (Np+1, nx) reference and Nc < Np (the adjoint recursion feeds the stages
    beyond Nc into the held last input)."""
    from oracle.kkt import solve_exact
    cfg = dict(pendulum(), Nc=10); Np = 20
    E = EmuSystem(cfg); x = np.array([0.1, 0.2, 0.2, -0.1]); um1 = np.zeros(1); fast = 0
    for t in range(6):
        Xtv = np.tile(np.asarray(cfg["xref"], float), (Np + 1, 1)) * np.linspace(0.4, 1.0, Np + 1)[:, None]
        Xtv[:, 0] += 0.05 * np.sin(0.3 * (np.arange(Np + 1) + t))
        U, ps = E.tpi_step(x, um1, Xtv, first_iters=10)
        assert ps != -100
        fast += ps > 0
        if ps <= 0:
            U, st, *_ = E.solve(x, um1, Xtv); assert st == 1
        Q = QPData(**dict(cfg, x0=x, uminus1=um1, xref=Xtv)); z, y, r = solve_exact(Q.P, Q.q, Q.A, Q.l, Q.u)
        assert np.max(np.abs(U - z[Q.NX:Q.NX + Q.NU])) < 1e-7, (t, ps)
        um1 = U[:1].copy(); x = cfg["Ad"] @ x + cfg["Bd"] @ um1
    assert fast >= 4


def test_random_systems_team_core_vs_oracle():
    """Property test of the generic (team) numerical core in host emulation: random small systems, weights and boxes
    (feasible by construction: soft state rows, input boxes around 0).  Whenever the polish verifies (status 1) the answer
    is the oracle's exact minimiser; a status-2 answer (degenerate vertex) is within OSQP's own accuracy."""
    from hypothesis import given, settings, strategies as st, HealthCheck
    from oracle.kkt import solve_exact

    @settings(max_examples=60, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
    @given(seed=st.integers(0, 10 ** 6), nx=st.integers(2, 4), nu=st.integers(1, 2), Np=st.integers(4, 9), short=st.booleans())
    def run(seed, nx, nu, Np, short):
        rng = np.random.default_rng(seed)
        A = rng.standard_normal((nx, nx)); A *= min(1.0, 1.05 / max(abs(np.linalg.eigvals(A))))
        Bm = rng.standard_normal((nx, nu))
        cfg = dict(Ad=A, Bd=Bm, Np=Np, Nc=(max(2, Np - 2) if short else Np), Qx=np.diag(rng.uniform(0.1, 2.0, nx)),
                   QxN=np.diag(rng.uniform(0.1, 2.0, nx)), Qu=np.diag(rng.uniform(0.0, 0.5, nu)), QDu=np.diag(rng.uniform(0.05, 1.0, nu)),
                   xmin=-rng.uniform(0.5, 3.0, nx), xmax=rng.uniform(0.5, 3.0, nx), umin=-rng.uniform(0.3, 2.0, nu),
                   umax=rng.uniform(0.3, 2.0, nu), Dumin=-rng.uniform(0.2, 1.0, nu), Dumax=rng.uniform(0.2, 1.0, nu),
                   eps_feas=10.0 ** rng.integers(2, 5), xref=0.5 * rng.standard_normal(nx), uminus1=np.zeros(nu), uref=np.zeros(nu))
        # start inside the state box (predictions may still leave it: the soft rows do get active).  Starts far outside the
        # box with eps_feas >= 1e5 AND a degenerate input vertex converge slower than OSQP's equilibrated iteration does
        # (no Ruiz scaling here) -- DESIGN.md section 7.
        cfg["x0"] = rng.uniform(0.9 * cfg["xmin"], 0.9 * cfg["xmax"])
        E = EmuSystem(cfg)
        U, status, it, ps, res = E.solve(cfg["x0"], cfg["uminus1"], cfg["xref"], rmax=E.mc)
        Q = QPData(**cfg); z, y, r = solve_exact(Q.P, Q.q, Q.A, Q.l, Q.u)
        ref = z[Q.NX:Q.NX + Q.NU]
        assert status in (1, 2)
        assert np.max(np.abs(U - ref)) < (1e-7 if status == 1 else 5e-2) * (1 + np.max(np.abs(ref)))
    run()


@pytest.mark.parametrize("eps_feas,scale,max_fail", [(1e5, 1.5, 0.01), (1e5, 2.5, 0.03), (1e3, 2.5, 0.0)])
def test_states_far_outside_the_soft_box_still_verify(eps_feas, scale, max_fail):
    """The regime round 1 documented as a behavioural gap (state far outside its soft box, large eps_feas; the reference's OSQP
    path reports 'solved', mpc.py:301-304): multipliers of order eps_feas * distance.  Three things closed it (bmpc_core.cuh):
    (1) the Schur-form polish used to reject the RIGHT working set — its hard-row regularisation delta shifts an active row off
    its bound by delta * mu (4e-8 at mu = 3e5, tolerance 1e-9), so 70 % of these instances never verified: one step of iterative
    refinement against the unregularised system; (2) the all-rows-at-once active-set update cycles when most hard rows are active:
    after BMPC_PDAS_FULL steps the hard rows change by single exchanges; (3) the rho ladder reaches 1e4 x (OSQP adapts up to 1e6).
    Host study (tools/soft_row_study.py, 400 systems): max-iter at eps_feas 1e5 / x0 up to 2.5x outside 17 % -> 0.5 %, at 1.5x
    11 % -> 0, ADMM iterations per solve 553 -> 72; every verified answer is the oracle's exact minimiser."""
    import sys, os
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "tools"))
    from soft_row_study import random_system
    from oracle.kkt import solve_exact
    rng = np.random.default_rng(2024); n = 120; tally = {1: 0, 2: 0, -2: 0}
    for i in range(n):
        nx, nu, Np = int(rng.integers(2, 5)), int(rng.integers(1, 3)), int(rng.integers(4, 10))
        c = random_system(rng, nx, nu, Np, None, eps_feas)
        c["x0"] = rng.uniform(scale * c["xmin"], scale * c["xmax"]); c["xref"] = 0.5 * rng.standard_normal(nx); c["uminus1"] = np.zeros(nu)
        E = EmuSystem(c)
        U, st, it, ps, res = E.solve(c["x0"], c["uminus1"], c["xref"], rmax=E.mc)
        tally[st if st in tally else -2] += 1
        if st == 1:
            Q = QPData(**c); z, y, r = solve_exact(Q.P, Q.q, Q.A, Q.l, Q.u); ref = z[Q.NX:Q.NX + Q.NU]
            assert np.max(np.abs(U - ref)) < 1e-6 * (1 + np.max(np.abs(ref))), (i, st)
            if i % 4 == 0:                              # ... and the algorithmically independent exact solver (least-distance form, NNLS)
                from oracle.ldp import solve_mpc
                ref2 = solve_mpc(Q)
                assert np.max(np.abs(U - ref2)) < 1e-6 * (1 + np.max(np.abs(ref2))), (i, "ldp")
    assert tally[-2] <= max_fail * n and tally[1] >= 0.9 * n, tally


def test_far_outside_failure_rate_is_the_osqp_restatements():
    """pendulum-size random systems (4 states, 1 input, Np = 20), eps_feas = 1e5, x0 up to 2.5x outside the soft box: the reference's own
    solver path (the oracle's OSQP restatement at the reference's settings, mpc.py:266: eps 1e-3; max_iter 4000) ends as max-iter on about
    one QP in twelve; the device core must not take the fallback u_failure (mpc.py:301-304) noticeably more often than that, and every
    answer it reports as solved-and-polished is exact (OSQP's 'solved' answers are 1e-3 .. 1e-1 off in relative terms)."""
    import sys, os
    import scipy.sparse as sp
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "tools"))
    from soft_row_study import random_system
    from oracle import osqp_port
    from oracle.ldp import solve_mpc
    from oracle.kkt import solve_exact
    rng = np.random.default_rng(2024); n = 48; ours = ref_fail = 0
    for i in range(n):
        c = random_system(rng, 4, 1, 20, None, 1e5)
        c["x0"] = rng.uniform(2.5 * c["xmin"], 2.5 * c["xmax"]); c["xref"] = 0.5 * rng.standard_normal(4); c["uminus1"] = np.zeros(1)
        E = EmuSystem(c)
        U, st, it, ps, res = E.solve(c["x0"], c["uminus1"], c["xref"], first_iters=50, tiers=launch_tiers(4, 1, 20, count=1))
        Q = QPData(**c)
        S = osqp_port.OSQP(); S.setup(sp.csc_matrix(Q.P), Q.q, sp.csc_matrix(Q.A), Q.l, Q.u, warm_start=True, verbose=False, eps_abs=1e-3, eps_rel=1e-3)
        ref_fail += S.solve().info.status_val != 1
        ours += st not in (1, 2)
        if st == 1:
            try:
                z, y, r = solve_exact(Q.P, Q.q, Q.A, Q.l, Q.u); exact = z[Q.NX:Q.NX + Q.NU]; tol = 1e-6
            except RuntimeError:                    # the stiffest QPs: only the least-distance solver answers, to NNLS accuracy
                exact = solve_mpc(Q); tol = 1e-4
            assert np.max(np.abs(U - exact)) < tol * (1 + np.max(np.abs(exact))), (i, tol)
    assert ours <= ref_fail + 3, (ours, ref_fail)


# ---- multi-input Riccati polish (bmpc_tpm.cuh): scalar sub-steps along the reference's scalar-shift delta-u chain ----

@pytest.mark.parametrize("name,steps", [("pm", 30), ("pend", 40), ("mimo", 6)])
def test_tpm_polish_closed_loop_matches_golden(name, steps):
    """the sweeps alone (no ADMM at all: working sets from zero, then shifted) reproduce the reference's closed loop; nu = 1
    shapes cross-check them against the single-input generation, the MIMO shape exercises chain rows, anchored runs and the
    interval test of degenerate vertices"""
    cfg = CASES[name](); g = golden(f"{name}_loop.npz"); E = EmuSystem(cfg)
    x = np.array(cfg["x0"], float); um1 = np.array(cfg["uminus1"], float)
    used = []
    for t in range(steps):
        U, ps = E.tpm_step(x, um1, cfg["xref"], mode=(0 if t == 0 else 1), max_ref=14)
        assert ps > 0, (t, ps)
        used.append(ps)
        assert np.max(np.abs(U[:E.nu] - g["u"][t])) < 1e-6, (t, ps)
        x = cfg["Ad"] @ x + cfg["Bd"] @ U[:E.nu]; um1 = U[:E.nu]
    assert np.mean(used[2:]) < (6.0 if name == "mimo" else 1.6)   # warm solves: about one refinement (MIMO: the early transient)


def test_tpm_polish_random_mimo_transients_vs_team_path():
    """random MIMO transients (the side bench's workload): every verified answer equals the team path's (ADMM + Schur-form
    polish, itself pinned to the oracle); the staged v* reproduces the verified working sets;
    most warm solves verify from the shifted working sets"""
    # (the multipliers of a degenerate vertex are not unique: v* is compared through what it is used for, not entry by entry)
    cfg = mimo(); rng = np.random.default_rng(11)
    ok = tot = 0
    for b in range(4):
        E = EmuSystem(cfg); x = 0.3 * rng.standard_normal(8); um1 = np.zeros(4)
        for t in range(9):
            Ut, st, *_ = E.solve(x, um1, cfg["xref"]); assert st == 1
            vteam = E.v.copy()
            if t == 0:
                U, ps = E.tpm_step(x, um1, cfg["xref"], mode=2, max_ref=2); assert ps > 0     # working sets from v*: verified at once
                E.Uplan = U.copy()
            else:
                E.mcodes, E.Uplan = codes, plan
                U, ps = E.tpm_step(x, um1, cfg["xref"], mode=1, max_ref=8)
                tot += 1; ok += ps > 0
                if ps <= 0:
                    E.v = vteam.copy()
                    U, ps = E.tpm_step(x, um1, cfg["xref"], mode=2, max_ref=2); assert ps > 0
            assert np.max(np.abs(U - Ut)) < 1e-7, (b, t, ps)
            # the staged fixed point v* round-trips: working sets derived from it are the stored ones and verify at once
            codes = E.mcodes.copy()
            U2, ps2 = E.tpm_step(x, um1, cfg["xref"], mode=2, max_ref=1)
            assert ps2 == 1 and np.max(np.abs(U2 - U)) < 1e-9 and np.array_equal(E.mcodes, codes), (b, t, ps2)
            E.mcodes = codes
            codes, plan = E.mcodes.copy(), U.copy()
            x = cfg["Ad"] @ x + cfg["Bd"] @ U[:4]; um1 = U[:4].copy()
    assert ok >= 0.7 * tot, (ok, tot)


def test_tpm_exchange_mode_finishes_the_stragglers():
    """the straggler rounds of the multi-input fast path (bmpc.cu::enqueue_round: ADMM chunk from the previous v*, then the polish from
    the iterate) in exchange mode (tpm_forward<S, true>: hard rows change by single exchanges): the warm MIMO solves whose first
    attempt (all-at-once updates from the shifted sets, 12 refinements) cycled all verify within 12 refinements of the first
    straggler round (all-at-once capped at 4, round 2's policy: about half), and a verified plan is the team path's exact answer"""
    cfg = mimo(); rng = np.random.default_rng(4)
    done = {"x": 0, "a": 0}; n = 0
    for b in range(16):
        E = EmuSystem(cfg); x = 0.3 * rng.standard_normal(8); um1 = np.zeros(4)
        for t in range(9):
            if t == 0:
                Ut, st, *_ = E.solve(x, um1, cfg["xref"]); assert st == 1
                U, ps = E.tpm_step(x, um1, cfg["xref"], mode=2, max_ref=2); assert ps > 0
            else:
                E.mcodes, E.Uplan = codes.copy(), plan.copy(); vprev = E.v.copy()
                U, ps = E.tpm_step(x, um1, cfg["xref"], mode=1, max_ref=12)
                if ps <= 0:
                    n += 1
                    E.v = vprev.copy(); E.x = plan.copy(); E.cold = 0
                    Ut, st, *_ = E.solve(x, um1, cfg["xref"]); assert st == 1
                    for key, cap, xf in (("a", 4, -1), ("x", 12, 0)):
                        E.v = vprev.copy(); E.x = plan.copy(); E.cold = 0; E.lvl = 2
                        E.admm_only(x, um1, cfg["xref"], 100)
                        U2, ps2 = E.tpm_step(x, um1, cfg["xref"], mode=2, max_ref=cap, exchange_from=xf)
                        if ps2 > 0:
                            done[key] += 1
                            assert np.max(np.abs(U2 - Ut)) < 1e-7, (b, t, key)
                    E.v = vprev.copy(); E.x = plan.copy(); E.cold = 0
                    Ut, st, *_ = E.solve(x, um1, cfg["xref"]); assert st == 1
                    U, ps = E.tpm_step(x, um1, cfg["xref"], mode=2, max_ref=4); assert ps > 0
            codes, plan = E.mcodes.copy(), U.copy()
            x = cfg["Ad"] @ x + cfg["Bd"] @ U[:4]; um1 = U[:4].copy()
    assert n >= 5, n                                    # the workload does produce stragglers
    assert done["x"] >= 0.95 * n and done["x"] > done["a"], (done, n)


def test_multi_input_round_loop_policy_in_emulation():
    """the multi-input fast path's round loop with the library's own round plans (tools/mimo_flow_study.py takes chunks, caps and
    modes from bmpc_rounds.cuh): cold solves finish within two rounds, warm transient solves within the first launch plus ONE straggler round, nothing
    falls through to the Schur-form polish (round 2's measured policy: five rounds for a cold solve, up to three straggler rounds)"""
    import sys, os
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "tools"))
    from mimo_flow_study import run
    r = run(40, 3)
    assert r["fallthrough"] == 0
    assert len(r["cold_rounds"]) <= 3 and r["cold_rounds"][1] >= 36, r           # [_, in one round, in two]
    assert len(r["warm_rounds"]) <= 3 and r["warm_rounds"][1] >= 0.8 * r["warm_rounds"].sum(), r


def test_tpm_polish_variants_vs_oracle():
    """input bounds, Nc < Np (held stages), soft state rows and a full Qu on a MIMO shape; time-varying reference on a small
    two-input system: verified answers equal the exact solver's on the oracle-assembled QP"""
    from oracle.kkt import solve_exact
    c = mimo(); c["Np"] = 12; c["Nc"] = 5; c["x0"] = np.array([0.3, -0.2, 0.1, 0.0, -0.4, 0.2, 0.0, 0.1])
    c["umin"] = -0.5 * np.ones(4); c["umax"] = 0.5 * np.ones(4); c["Qu"] = 0.1 * np.eye(4) + 0.02 * np.ones((4, 4))
    c["xmin"] = -0.6 * np.ones(8); c["xmax"] = 0.6 * np.ones(8); c["eps_feas"] = 1e3
    E = EmuSystem(c); x = c["x0"].copy(); um1 = np.zeros(4); fast = 0
    for t in range(8):
        U, ps = E.tpm_step(x, um1, c["xref"], mode=(0 if t == 0 else 1), max_ref=14)
        assert ps != -100 and ps != -101
        st = 1
        if ps <= 0:
            # (this heavily constrained short-horizon variant is beyond the plain active-set search from a shifted guess: the
            # sweeps then serve as the verifier of the team path's answer — working sets from its v* verify within 3 refinements)
            U, st, *_ = E.solve(x, um1, c["xref"]); assert st in (1, 2)
            U2, ps2 = E.tpm_step(x, um1, c["xref"], mode=2, max_ref=3); E.Uplan = U.copy()
            if st == 1:
                assert ps2 > 0 and np.max(np.abs(U2 - U)) < 1e-7, (t, ps2)
        else:
            fast += 1
        Q = QPData(**dict(c, x0=x, uminus1=um1)); z, y, r = solve_exact(Q.P, Q.q, Q.A, Q.l, Q.u)
        assert np.max(np.abs(U - z[Q.NX:Q.NX + Q.NU])) < (1e-7 if st == 1 else 1e-3), (t, ps)
        x = c["Ad"] @ x + c["Bd"] @ U[:4]; um1 = U[:4].copy()
    rng = np.random.default_rng(5)
    for Nc in (10, 6):
        A = rng.standard_normal((3, 3)); A *= 0.95 / max(abs(np.linalg.eigvals(A)))
        c = dict(Ad=A, Bd=rng.standard_normal((3, 2)), Np=10, Nc=Nc, Qx=np.diag([1.0, 0.5, 0.2]), QxN=np.diag([2.0, 0.5, 0.2]),
                 Qu=np.diag([0.1, 0.3]), QDu=np.diag([0.5, 0.2]), xmin=-1.5 * np.ones(3), xmax=1.5 * np.ones(3),
                 umin=-np.array([0.8, 0.5]), umax=np.array([0.6, 0.9]), Dumin=-np.array([0.3, 0.4]), Dumax=np.array([0.4, 0.3]),
                 eps_feas=1e3, uminus1=np.zeros(2), uref=np.array([0.05, -0.05]), x0=np.array([1.2, -0.8, 0.5]), xref=np.zeros(3))
        E = EmuSystem(c); x = c["x0"].copy(); um1 = np.zeros(2); fast = 0
        for t in range(8):
            Xtv = 0.3 * np.sin(0.4 * (np.arange(11)[:, None] + t) + np.arange(3)[None, :])
            U, ps = E.tpm_step(x, um1, Xtv, mode=(0 if t == 0 else 1), max_ref=14)
            assert ps != -100 and ps != -101
            st = 1
            if ps <= 0:
                U, st, *_ = E.solve(x, um1, Xtv); assert st in (1, 2)
                E.tpm_step(x, um1, Xtv, mode=2, max_ref=3); E.Uplan = U.copy()
            else:
                fast += 1
            Q = QPData(**dict(c, x0=x, uminus1=um1, xref=Xtv)); z, y, r = solve_exact(Q.P, Q.q, Q.A, Q.l, Q.u)
            assert np.max(np.abs(U - z[Q.NX:Q.NX + Q.NU])) < (1e-7 if st == 1 else 1e-3), (Nc, t, ps)
            x = c["Ad"] @ x + c["Bd"] @ U[:2]; um1 = U[:2].copy()
        assert fast >= 5, (Nc, fast)


def test_tpm_pattern_specialised_shape_equals_dense(monkeypatch):
    """the instantiation with the MIMO reference governor's (Ad, Bd) sparsity pattern fixed at compile time (what the device runs
    for that system) follows the dense instantiation refinement by refinement"""
    cfg = mimo(); x0 = 0.3 * np.random.default_rng(3).standard_normal(8)
    runs = []
    for sparse in (False, True):
        if sparse:
            monkeypatch.setenv("EMU_TPM_SPARSE", "1")
        E = EmuSystem(cfg); x = x0.copy(); um1 = np.zeros(4); out = []
        for t in range(8):
            if t == 0:
                Ut, st, *_ = E.solve(x, um1, cfg["xref"]); assert st == 1
                U, ps = E.tpm_step(x, um1, cfg["xref"], mode=2, max_ref=2); assert ps > 0
            else:
                U, ps = E.tpm_step(x, um1, cfg["xref"], mode=1, max_ref=16)
                if ps <= 0:
                    U, st, *_ = E.solve(x, um1, cfg["xref"]); assert st == 1
                    E.tpm_step(x, um1, cfg["xref"], mode=2, max_ref=2); E.Uplan = U.copy()
            out.append((ps, U.copy()))
            x = cfg["Ad"] @ x + cfg["Bd"] @ U[:4]; um1 = U[:4].copy()
        runs.append(out)
    assert sum(ps > 0 for ps, _ in runs[0]) >= 6
    for (pa, Ua), (pb, Ub) in zip(*runs):
        assert pa == pb and np.max(np.abs(Ua - Ub)) < 1e-10


@pytest.mark.parametrize("nx,Np,Nc,min_direct", [(1, 31, 31, 1.0), (8, 16, 16, 1.0), (13, 8, 8, 0.75)])
def test_tpi_polish_at_the_edges_of_the_shape_domain(nx, Np, Nc, min_direct):
    """The fast path's Riccati polish (tpi2_*, host build) at the edges of its shape domain — the longest horizon, Np * nx = 128 and
    a code word of exactly 32 bits — along the golden closed loops of tests/golden/shapes.npz (make_golden.py shapes).  Like on the
    device, a warm step starts from the stored working sets shifted one stage (8 refinements); a step it cannot verify that way takes
    the device's straggler route: ADMM + team polish, then the working sets read off that v*.  Every plan the polish verifies equals
    the golden to 1e-6 (1 + |u|); the team core answers the rest exactly.  At nx = 13 the active-set iteration verifies about 85 % of
    the warm steps alone (measured), the other shapes all of them."""
    g = golden("shapes.npz"); tag = f"{nx}_{Np}_{Nc}_"
    cfg = {k: g[tag + k] for k in ("Ad", "Bd", "Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax")}
    cfg.update(Np=Np, Nc=Nc, eps_feas=float(g[tag + "eps_feas"]))
    X, U, S, Xref = g[tag + "X"], g[tag + "U"], g[tag + "useq"], g[tag + "Xref"]
    T, N = U.shape
    direct = warm = 0
    for i in range(N):
        E = EmuSystem(cfg)
        for t in range(T):
            um1 = np.array([U[t - 1, i] if t > 0 else 0.0])
            scale = 1.0 + np.max(np.abs(S[t, i]))
            ps = 0
            if t > 0:
                u, ps = E.tpi2_step(X[t, i], um1, Xref[i], mode=1, max_ref=8)
                warm += 1; direct += ps > 0
            if ps <= 0:
                ut, st, it, pst, res = E.solve(X[t, i], um1, Xref[i])
                assert st == 1 and np.max(np.abs(ut - S[t, i])) < 1e-6 * scale, (i, t, st)
                u, ps = E.tpi2_step(X[t, i], um1, Xref[i], mode=2, max_ref=8)
                if ps <= 0:
                    continue
            assert np.max(np.abs(u - S[t, i])) < 1e-6 * scale, (i, t)
    assert direct >= min_direct * warm, (direct, warm)


# (shape, compiled pattern, least share of warm steps the polish verifies alone from the shifted sets: measured 100 % at
# (2,6,12,12), (4,1,40,40), (1,5,20,10), 95-98 % at the others, 55 % at (7,5,8,4))
MIMO_EDGE = [((2, 6, 12, 12), False, 0.9), ((7, 5, 8, 4), False, 0.5), ((8, 4, 25, 1), False, 0.9), ((8, 4, 25, 1), True, 0.9),
             ((3, 2, 60, 60), False, 0.9), ((4, 1, 40, 40), False, 0.9), ((1, 5, 20, 10), False, 0.9), ((13, 2, 6, 6), False, 0.9),
             ((13, 1, 10, 10), False, 0.9)]


@pytest.mark.parametrize("shape,pattern,min_direct", MIMO_EDGE,
                         ids=["-".join(map(str, s)) + ("-pattern" if p else "") for s, p, _ in MIMO_EDGE])
def test_tpm_polish_at_the_edges_of_the_shape_domain(monkeypatch, shape, pattern, min_direct):
    nx, nu, Np, Nc = shape
    if pattern:
        assert shape == tuple(int(v) for v in golden("mimo_shapes.npz")["pattern"])
        monkeypatch.setenv("EMU_TPM_PATTERN", "1")
    g = golden("mimo_shapes.npz"); tag = f"{nx}_{nu}_{Np}_{Nc}_"
    cfg = {k: g[tag + k] for k in ("Ad", "Bd", "Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "uref")}
    cfg.update(Np=Np, Nc=Nc, eps_feas=float(g[tag + "eps_feas"]))
    X, U, S, Xref = g[tag + "X"], g[tag + "U"], g[tag + "useq"], g[tag + "Xref"]
    T, N = U.shape[:2]
    direct = warm = verified = 0
    for i in range(N):
        E = EmuSystem(cfg)
        for t in range(T):
            um1 = U[t - 1, i] if t > 0 else np.zeros(nu)
            xr = Xref[i] if Xref.ndim == 2 else Xref[t, i]
            scale = 1.0 + np.max(np.abs(S[t, i]))
            ps = 0
            if t > 0:
                u, ps = E.tpm_step(X[t, i], um1, xr, mode=1, max_ref=12)
                assert ps != -100 and ps != -101
                warm += 1; direct += ps > 0
            if ps <= 0:
                ut, st, it, pst, res = E.solve(X[t, i], um1, xr)
                assert st == 1 and np.max(np.abs(ut - S[t, i])) < 1e-6 * scale, (i, t, st)
                u, ps = E.tpm_step(X[t, i], um1, xr, mode=2, max_ref=12, exchange_from=0)
                E.Uplan = ut.copy()
                if ps <= 0:
                    continue
            verified += 1
            assert np.max(np.abs(u - S[t, i])) < 1e-6 * scale, (i, t, ps)
    print(f"shape {shape}{' pattern' if pattern else ''}: polish alone on {direct} of {warm} warm steps, verified {verified} of {N * T}")
    assert direct >= min_direct * warm, (direct, warm)
