"""Generates the committed golden fixtures (run HERE, where /root/reference exists).

For every case the QP is assembled by the UNMODIFIED reference (pyMPC.mpc.MPCController with a
stub ``osqp`` module, tests/refharness.py), solved by ``oracle.kkt.solve_exact`` and certified by
the solver-independent KKT residuals (< 1e-9) on the reference-assembled (P, q, A, l, u).
Closed loops use the linear plant x+ = Ad x + Bd u (README.md:59-77 pattern).

    python tests/golden/make_golden.py              # every fixture
    python tests/golden/make_golden.py reference    # only ref_assembly.npz and ref_on_port.npz
    python tests/golden/make_golden.py shapes       # only shapes.npz (single-input shapes at the edges of the fast path)
    python tests/golden/make_golden.py mimo_shapes  # only mimo_shapes.npz (shapes at the edges of the multi-input fast path)
    python tests/golden/make_golden.py team_shapes  # only team_shapes.npz (team kernels: shape edges and polish capacity)
"""
import os
import sys

if sys.argv[1:] in (["shapes"], ["mimo_shapes"], ["team_shapes"]):
    # one process per shape: single-threaded BLAS keeps them from competing and the results reproducible
    for _v in ("OPENBLAS_NUM_THREADS", "OMP_NUM_THREADS", "MKL_NUM_THREADS"):
        os.environ.setdefault(_v, "1")

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from refharness import load_reference_controller  # noqa: E402
from oracle.kkt import solve_exact, kkt_residuals  # noqa: E402
from pympc_b200.workloads import point_mass, pendulum, mimo, pendulum_random  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
MPC = load_reference_controller()


def exact(K, warm=None):
    P, A = K.P.toarray(), K.A.toarray()
    z, y, r = solve_exact(P, K.q, A, K.l, K.u, warm=warm)
    assert max(r.values()) < 1e-9, r
    return z, y, r


def first_solve(name, cfg):
    K = MPC(**cfg); K.setup(solve=False)
    z, y, r = exact(K)
    NX = (K.Np + 1) * K.nx; NU = K.Nc * K.nu
    obj = 0.5 * z @ (K.P @ z) + K.q @ z
    np.savez_compressed(os.path.join(OUT, f"{name}_first.npz"), z=z, y=y, q=K.q, l=K.l, u=K.u,
                        P_data=K.P.toarray()[np.nonzero(K.P.toarray())], A_sum=np.array([K.A.toarray().sum(), np.abs(K.A.toarray()).sum()]),
                        u_seq=z[NX:NX + NU], x_seq=z[:NX], eps_seq=z[NX + NU:], obj=obj, J_CNST=K.J_CNST,
                        kkt=np.array([r['stat'], r['prim'], r['comp']]))
    print(name, "first u0", z[NX:NX + K.nu], r)


def closed_loop(name, cfg, nsteps, xref_fn=None):
    K = MPC(**cfg); K.setup(solve=False)
    Ad, Bd = np.asarray(cfg['Ad']), np.asarray(cfg['Bd'])
    NX = (K.Np + 1) * K.nx
    x = np.array(cfg['x0'], float); um1 = np.array(cfg['uminus1'], float)
    xs, us, warm = [], [], None
    for t in range(nsteps):
        K.update(x, um1, xref=(xref_fn(t) if xref_fn else None), solve=False)
        z, y, r = exact(K, warm)
        warm = (z, y)
        u0 = z[NX:NX + K.nu].copy()
        xs.append(x.copy()); us.append(u0)
        x = Ad @ x + Bd @ u0; um1 = u0
    np.savez_compressed(os.path.join(OUT, f"{name}_loop.npz"), x=np.array(xs), u=np.array(us))
    print(name, "loop u[:8]", np.array(us)[:8].ravel())


def random_batch(B=24, nsteps=4):
    cfg = pendulum()
    X0, Xref = pendulum_random(B, seed=0)
    Ad, Bd = cfg['Ad'], cfg['Bd']
    U = np.zeros((nsteps, B, 1)); X = np.zeros((nsteps, B, 4))
    for b in range(B):
        c = dict(cfg); c['x0'] = X0[b]; c['xref'] = Xref[b]
        K = MPC(**c); K.setup(solve=False)
        x = X0[b].copy(); um1 = np.zeros(1); warm = None
        for t in range(nsteps):
            K.update(x, um1, solve=False)
            z, y, r = exact(K, warm); warm = (z, y)
            u0 = z[84:85].copy(); U[t, b] = u0; X[t, b] = x
            x = Ad @ x + Bd @ u0; um1 = u0
    np.savez_compressed(os.path.join(OUT, "pend_rand.npz"), X0=X0, Xref=Xref, U=U, X=X)
    print("pend_rand", U[0, :4].ravel())


def variants():
    out = {}
    # (a) Nc < Np, time-varying xref, nonzero uref, Qu > 0  (mpc.py:618-692 demo shape)
    c = point_mass(); c['Np'] = 25; c['Nc'] = 10; c['uref'] = np.array([0.1])
    c['xmin'] = np.array([-10.0, -10.0]); c['xmax'] = np.array([7.0, 10.0])
    Xref = np.kron(np.ones((26, 1)), c['xref']); Xref[:, 0] = np.linspace(5.0, 7.0, 26)
    c['xref'] = Xref
    K = MPC(**c); K.setup(solve=False); z, y, r = exact(K)
    out['a_z'] = z; out['a_xref'] = Xref
    # (b) small MIMO with Nc < Np (channel-mixing delta-u quirk live)
    c = mimo(); c['Np'] = 12; c['Nc'] = 5; c['x0'] = np.array([0.3, -0.2, 0.1, 0.0, -0.4, 0.2, 0.0, 0.1])
    c['umin'] = -0.5 * np.ones(4); c['umax'] = 0.5 * np.ones(4); c['Qu'] = 0.1 * np.eye(4)
    K = MPC(**c); K.setup(solve=False); z, y, r = exact(K)
    out['b_z'] = z
    # (c) pendulum starting outside the soft position bound (slacks strongly active)
    c = pendulum(); c['x0'] = np.array([0.45, 0.3, -0.05, 0.1])
    K = MPC(**c); K.setup(solve=False); z, y, r = exact(K)
    out['c_z'] = z
    np.savez_compressed(os.path.join(OUT, "variants.npz"), **out)
    print("variants ok")


def _put_csc(out, key, M):
    M = M.tocsc()
    out[key + "_data"] = M.data; out[key + "_indices"] = M.indices; out[key + "_indptr"] = M.indptr
    out[key + "_shape"] = np.array(M.shape)


def reference_assembly():
    """What the reference's own assembly hands to the solver for every variant of tests/test_oracle.py: (P, A, q, l, u) after
    setup and (q, l, u, J_CNST) after each of three updates at the seeded inputs the test replays."""
    from test_oracle import ASSEMBLY_VARIANTS, assembly_variant
    out = {}
    for v in ASSEMBLY_VARIANTS:
        cfg = assembly_variant(v)
        K = MPC(**cfg); K.setup(solve=False)
        _put_csc(out, f"{v}_P", K.P); _put_csc(out, f"{v}_A", K.A)
        out[f"{v}_q"] = K.q.copy(); out[f"{v}_l"] = K.l.copy(); out[f"{v}_u"] = K.u.copy()
        rng = np.random.default_rng(3)
        for t in range(3):
            x = rng.normal(size=K.nx); um1 = rng.normal(size=K.nu)
            xr = cfg["xref"] if t == 0 else rng.normal(size=np.shape(cfg["xref"]))
            K.update(x, um1, xref=xr, solve=False)
            for k, a in (("x", x), ("um1", um1), ("xref", xr), ("q", K.q), ("l", K.l), ("u", K.u), ("J_CNST", K.J_CNST)):
                out[f"{v}_{t}_{k}"] = np.array(a, float)
    np.savez_compressed(os.path.join(OUT, "ref_assembly.npz"), **out)
    print("ref_assembly", len(ASSEMBLY_VARIANTS), "variants")


def reference_on_port(nsteps=5):
    """The unmodified reference controller (pendulum, eps 1e-9) run end to end with oracle/osqp_port as its ``osqp``: the solver
    calls it makes — setup(P, q, A, l, u), then update(q, l, u) before each step's solve — are stored, and so is the u it outputs."""
    from oracle import osqp_port
    cfg = pendulum()
    K = MPC(**cfg, eps_abs=1e-9, eps_rel=1e-9)
    K.setup(solve=False)
    out = {}
    _put_csc(out, "P", K.P); _put_csc(out, "A", K.A)
    out["q"] = K.q.copy(); out["l"] = K.l.copy(); out["u"] = K.u.copy()
    # the reference does not forward max_iter; tight tolerance needs more than OSQP's 4000 default
    K.prob = osqp_port.OSQP()
    K.prob.setup(K.P, K.q, K.A, K.l, K.u, warm_start=True, eps_abs=1e-9, eps_rel=1e-9, max_iter=200000)
    K.solve()
    x = np.array(cfg["x0"], float); um1 = np.array(cfg["uminus1"], float); us = []
    for t in range(nsteps):
        K.update(x, um1); u = np.array(K.output())
        out[f"{t}_q"] = K.q.copy(); out[f"{t}_l"] = K.l.copy(); out[f"{t}_u"] = K.u.copy()
        us.append(u)
        x = cfg["Ad"] @ x + cfg["Bd"] @ u; um1 = u
    out["u_out"] = np.array(us); out["u_slice"] = np.array([(K.Np + 1) * K.nx, (K.Np + 1) * K.nx + K.nu])
    np.savez_compressed(os.path.join(OUT, "ref_on_port.npz"), **out)
    print("ref_on_port u", np.array(us).ravel())


# Single-input shapes at the edges of the fast path's domain (tests/test_gpu_shapes.py, tests/test_hostemu_core.py):
# (nx, Np, Nc, instances).  nu = 1 throughout.
SHAPES = [(1, 31, 31, 32), (2, 29, 29, 32), (2, 31, 16, 32), (4, 25, 25, 16), (4, 31, 1, 16), (5, 17, 17, 16), (6, 21, 21, 16),
          (8, 16, 16, 16), (13, 8, 8, 32), (14, 7, 7, 32)]
SHAPE_STEPS = 4


def random_system(rng, nx, nu, Np, Nc=None, eps_feas=1e3):
    """Seeded random system: spectral radius <= 1.05, random Bd, diagonal weights, finite boxes on every row
    (the recipe of tests/test_gpu_parity.py::_random_system)."""
    A = rng.standard_normal((nx, nx)); A *= min(1.0, 1.05 / max(abs(np.linalg.eigvals(A))))
    return dict(Ad=A, Bd=rng.standard_normal((nx, nu)), Np=Np, Nc=Nc or Np, Qx=np.diag(rng.uniform(0.1, 2.0, nx)),
                QxN=np.diag(rng.uniform(0.1, 2.0, nx)), Qu=np.diag(rng.uniform(0.0, 0.5, nu)), QDu=np.diag(rng.uniform(0.05, 1.0, nu)),
                xmin=-rng.uniform(0.5, 3.0, nx), xmax=rng.uniform(0.5, 3.0, nx), umin=-rng.uniform(0.3, 2.0, nu),
                umax=rng.uniform(0.3, 2.0, nu), Dumin=-rng.uniform(0.2, 1.0, nu), Dumax=rng.uniform(0.2, 1.0, nu), eps_feas=eps_feas)


def certified(K, warm=None):
    """Exact minimiser of the QP the reference assembled, KKT residuals < 1e-9: the ADMM -> active-set oracle, or, when it cannot
    certify the QP, the least-distance solver (oracle/ldp.py) whose active set one primal-dual active-set solve then certifies."""
    from types import SimpleNamespace
    from oracle.kkt import _pdas
    from oracle.ldp import solve_mpc
    P, A = K.P.toarray(), K.A.toarray()
    try:
        return exact(K, warm)
    except (RuntimeError, AssertionError):
        pass
    NX, NU = (K.Np + 1) * K.nx, K.Nc * K.nu
    l = np.where(K.l < -1e20, -np.inf, K.l); u = np.where(K.u > 1e20, np.inf, K.u)
    U = solve_mpc(SimpleNamespace(NX=NX, NU=NU, A=A, P=P, q=K.q, l=l, u=u))
    X = np.linalg.solve(A[:NX, :NX], l[:NX] - A[:NX, NX:NX + NU] @ U)
    E = np.clip(X, l[NX:2 * NX], u[NX:2 * NX]) - X                 # slack of the soft rows xmin <= X + E <= xmax
    z = np.concatenate([X, U, E]); Az = A @ z
    out = _pdas(P, K.q, A, l, u, Az <= l + 1e-7 * (1 + np.abs(l)), Az >= u - 1e-7 * (1 + np.abs(u)), max_steps=20)
    assert out is not None, "least-distance fallback not certified"
    z, y = out
    r = kkt_residuals(P, K.q, A, l, u, z, y)
    assert max(r.values()) < 1e-9, r
    return z, y, r


def shape_case(spec):
    nx, Np, Nc, N = spec
    rng = np.random.default_rng([2026, nx, Np, Nc])
    c = random_system(rng, nx, 1, Np, Nc)
    X0 = rng.uniform(1.3 * c["xmin"], 1.3 * c["xmax"], (N, nx)); Xref = 0.5 * rng.standard_normal((N, nx))
    NX = (Np + 1) * nx
    X = np.zeros((SHAPE_STEPS, N, nx)); U = np.zeros((SHAPE_STEPS, N)); useq = np.zeros((SHAPE_STEPS, N, Nc))
    for b in range(N):
        K = MPC(**dict(c, x0=X0[b], xref=Xref[b], uminus1=np.zeros(1))); K.setup(solve=False)
        x = X0[b].copy(); um1 = np.zeros(1); warm = None
        for t in range(SHAPE_STEPS):
            K.update(x, um1, solve=False)
            z, y, r = certified(K, warm); warm = (z, y)
            X[t, b] = x; useq[t, b] = z[NX:NX + Nc]; U[t, b] = z[NX]
            um1 = z[NX:NX + 1].copy(); x = c["Ad"] @ x + c["Bd"] @ um1
    tag = f"{nx}_{Np}_{Nc}_"
    out = {tag + k: np.asarray(v, float) for k, v in c.items() if k not in ("Np", "Nc")}
    out.update({tag + "X": X, tag + "U": U, tag + "useq": useq, tag + "Xref": Xref})
    print("shapes", spec, "u0[:3]", U[0, :3], flush=True)
    return out


def shapes():
    from multiprocessing import Pool
    with Pool(min(len(SHAPES), os.cpu_count() or 1)) as pool:
        parts = pool.map(shape_case, sorted(SHAPES, key=lambda s: -s[0] * s[1] * s[3]))
    out = {}
    for p in parts:
        out.update(p)
    np.savez_compressed(os.path.join(OUT, "shapes.npz"), shapes=np.array(SHAPES), steps=SHAPE_STEPS, **out)


# Shapes at the edges of the multi-input fast path's domain (tests/test_gpu_mimo_shapes.py, tests/test_hostemu_core.py):
# (nx, nu, Np, Nc, instances, options).  Options: "qu" a full Qu, "uref" a non-zero uref, "tv" a time-varying (Np+1, nx)
# reference per instance and step, "pattern" the non-symmetric sparsity pattern below.
MIMO_SHAPES = [
    (2, 6, 12, 12, 32, ("qu", "uref")),    # 2 nx + 10 nu = 64: the code word is full, the last channel's hint bits are 62-63
    (7, 5, 8, 4, 16, ("tv", "zeros")),     # full code word; nx nu = 35 > 32: no pattern masks, a sparse system takes the dense entry
    (8, 4, 25, 1, 16, ("pattern",)),       # Nc = 1 with four inputs: first-block row and spurious last row on one stage
    (3, 2, 60, 60, 16, ("tv", "uref")),    # long horizon
    (4, 1, 40, 40, 16, ()),                # pendulum-size single-input system outside the single-input domain (Np >= 32)
    (1, 5, 20, 10, 32, ("qu",)),           # one state, five inputs, Nc < Np
    # the widest states of the domain (nx = 13, build.tpm_shape_supported).  They stand in for (22, 2, 6, 6) and (27, 1, 4, 4), the
    # widest states the code word holds, whose k_tpm_pol needs a stack frame of 44-68 KB per thread; those run on the team kernels
    (13, 2, 6, 6, 16, ()),
    (13, 1, 10, 10, 16, ()),               # (single-input, Np nx > 128: outside the single-input domain)
    # outside the domain: with fast_path=2 they run on the team kernels, with the same exact answers
    (22, 2, 6, 6, 16, ()),
    (27, 1, 4, 4, 16, ()),
    (14, 1, 7, 7, 32, ()),                 # single-input state too wide for either fast path
]
MIMO_STEPS = 5


def mimo_pattern(nx, nu):
    """Structural non-zeros of the pattern case: a lower-Hessenberg Ad (Ad[q][b] for b <= q + 1: NOT symmetric, so a transposed
    mask skips real terms) and a Bd with one block of two rows per channel plus one entry off that pattern"""
    am = np.array([[b <= q + 1 for b in range(nx)] for q in range(nx)])
    bm = np.array([[a // 2 == j for j in range(nu)] for a in range(nx)]); bm[0, nu - 1] = True
    return am, bm


def mimo_shape_case(spec):
    nx, nu, Np, Nc, N, opts = spec
    rng = np.random.default_rng([2027, nx, nu, Np, Nc])
    c = random_system(rng, nx, nu, Np, Nc)
    if "pattern" in opts:
        am, bm = mimo_pattern(nx, nu)
        A = rng.standard_normal((nx, nx)) * am; A *= min(1.0, 1.05 / max(abs(np.linalg.eigvals(A))))
        c["Ad"] = A; c["Bd"] = rng.uniform(0.5, 1.5, (nx, nu)) * rng.choice([-1.0, 1.0], (nx, nu)) * bm
    if "zeros" in opts:
        c["Ad"][0, nx - 1] = c["Ad"][nx - 1, 1] = 0.0; c["Bd"][1, 0] = 0.0        # structural zeros that no mask can hold
    if "qu" in opts:
        M = rng.standard_normal((nu, nu))
        c["Qu"] = 0.1 * M @ M.T / nu + np.diag(rng.uniform(0.0, 0.3, nu))
    c["uref"] = rng.uniform(-0.3, 0.3, nu) if "uref" in opts else np.zeros(nu)
    X0 = rng.uniform(1.3 * c["xmin"], 1.3 * c["xmax"], (N, nx)); Xr = 0.5 * rng.standard_normal((N, nx))
    if "tv" in opts:
        # per instance and step: the base reference on a ramp over the horizon plus a wave that moves with the step
        ramp = np.linspace(0.4, 1.0, Np + 1)[:, None]
        Xref = np.stack([Xr[:, None, :] * ramp[None] + 0.2 * np.sin(0.3 * (np.arange(Np + 1)[None, :, None] + t) + np.arange(nx)[None, None, :])
                         for t in range(MIMO_STEPS)])                     # (T, N, Np+1, nx)
    else:
        Xref = Xr
    NX, NU = (Np + 1) * nx, Nc * nu
    X = np.zeros((MIMO_STEPS, N, nx)); U = np.zeros((MIMO_STEPS, N, nu)); useq = np.zeros((MIMO_STEPS, N, NU))
    for b in range(N):
        K = MPC(**dict(c, x0=X0[b], xref=(Xref[0, b] if "tv" in opts else Xref[b]), uminus1=np.zeros(nu))); K.setup(solve=False)
        x = X0[b].copy(); um1 = np.zeros(nu); warm = None
        for t in range(MIMO_STEPS):
            K.update(x, um1, xref=(Xref[t, b] if "tv" in opts else None), solve=False)
            z, y, r = certified(K, warm); warm = (z, y)
            X[t, b] = x; useq[t, b] = z[NX:NX + NU]; U[t, b] = z[NX:NX + nu]
            um1 = z[NX:NX + nu].copy(); x = c["Ad"] @ x + c["Bd"] @ um1
    tag = f"{nx}_{nu}_{Np}_{Nc}_"
    out = {tag + k: np.asarray(v, float) for k, v in c.items() if k not in ("Np", "Nc")}
    out.update({tag + "X": X, tag + "U": U, tag + "useq": useq, tag + "Xref": Xref})
    print("mimo_shapes", spec[:4], "u0[:2]", U[0, :2].ravel(), flush=True)
    return out


def mimo_shapes():
    from multiprocessing import Pool
    with Pool(min(len(MIMO_SHAPES), os.cpu_count() or 1)) as pool:
        parts = pool.map(mimo_shape_case, sorted(MIMO_SHAPES, key=lambda s: -((s[2] + 1) * s[0] + s[3] * s[1]) ** 2 * s[4]))
    out = {}
    for p in parts:
        out.update(p)
    np.savez_compressed(os.path.join(OUT, "mimo_shapes.npz"), shapes=np.array([s[:5] for s in MIMO_SHAPES]), steps=MIMO_STEPS,
                        pattern=np.array([s[:4] for s in MIMO_SHAPES if "pattern" in s[5]][0]), **out)


# Team / tile kernels (k_admm, k_admm_tile, the Schur-form k_polish) at the edges of their shape domain and of the polish's
# working-set capacity (tests/test_gpu_team_shapes.py, tests/test_team_capacity_cpu.py): (name, nx, nu, Np, Nc, scales, options).
# Instance b starts at scales[b] times a random point of the state box: the further outside the soft box, the more soft rows are
# violated at the optimum and the larger the polish's working set.  Options: "hard" hard state rows (SOFT_ON = False; the states
# start inside the box), "ride" (hard) a reference beyond one state's bound, so that the state rides that bound over many stages.
TEAM_SHAPES = [
    ("warp_cap", 7, 1, 20, 20, (1.0, 1.4, 1.8, 2.2, 2.6, 3.0, 3.4, 4.0), ()),      # mc = 188: warp team, tiers 64 and 188
    ("cta_cap", 5, 2, 25, 25, (1.0, 2.0, 3.0, 4.5, 6.0, 8.0, 10.0, 5.0), ()),        # mc = 232: CTA team / tile, tiers 80 and 232
    ("mc192", 9, 1, 18, 10, (1.0, 1.5, 2.0, 3.0), ()),                             # mc = 192: the largest warp-team shape
    ("mc193", 8, 1, 19, 16, (1.0, 1.5, 2.0, 3.0), ()),                             # mc = 193: CTA team
    ("nu64", 1, 2, 32, 32, (1.0, 3.0, 6.0, 10.0), ()),                              # NU = 64: warp team
    ("nu65", 1, 5, 13, 13, (1.0, 3.0, 6.0, 10.0), ()),                              # NU = 65: CTA team
    ("tiny", 1, 1, 2, 2, (0.5, 1.5, 3.0, 6.0), ()),                                # Np = 2, nx = 1
    ("nc1", 2, 3, 5, 1, (0.5, 1.5, 3.0, 6.0), ()),                                 # Nc = 1 with nu = 3 > nx
    ("warp_hard", 7, 1, 20, 20, (0.05, 0.1, 0.2, 0.3), ("hard", "ride")),          # hard state rows on the warp team
    ("cta_hard", 5, 2, 25, 25, (0.05, 0.1, 0.2, 0.3), ("hard", "ride")),           # hard state rows on the CTA team / tile
]
TEAM_STEPS = 4


def working_set_size(K, z, y, tol=1e-7):
    """size of the polish's working set at the optimum (z, y) of the reference-assembled QP: soft rows outside their box (non-zero
    slack) plus inequality rows without slack at a bound with a non-zero multiplier"""
    A = K.A.toarray(); NX, NU = (K.Np + 1) * K.nx, K.Nc * K.nu
    nz = A.shape[1] - NX - NU                                    # slack columns (SOFT_ON)
    soft_rows = np.abs(A[:, NX + NU:]).sum(axis=1) > 0 if nz else np.zeros(A.shape[0], bool)
    ineq = (K.u - K.l) > 1e-12
    slack = np.abs(z[NX + NU:]) > tol * (1.0 + np.abs(z[:NX]).max()) if nz else np.zeros(0, bool)
    hard = ineq & ~soft_rows & (np.abs(y) > tol * (1.0 + np.abs(y).max()))
    return int(slack.sum() + hard.sum())


def team_shape_case(spec):
    name, nx, nu, Np, Nc, scales, opts = spec
    rng = np.random.default_rng([2028, nx, nu, Np, Nc, len(opts)])
    c = random_system(rng, nx, nu, Np, Nc)
    c["uref"] = np.zeros(nu)
    N = len(scales)
    P0 = rng.uniform(c["xmin"], c["xmax"], (N, nx))
    X0 = np.array(scales)[:, None] * np.where(rng.uniform(size=(N, nx)) < 0.5, c["xmin"], c["xmax"]) if "hard" not in opts else \
        np.array(scales)[:, None] * P0
    if "hard" not in opts:
        X0 = 0.5 * (X0 + np.array(scales)[:, None] * P0)
    Xref = 0.5 * rng.standard_normal((N, nx))
    if "ride" in opts:
        c["Qx"][0, 0] = c["QxN"][0, 0] = 20.0                      # a heavy weight on a reference beyond the hard bound: state 0
        Xref[:, 0] = 3.0 * c["xmax"][0]                            # rides its bound over the horizon
    NX, NU = (Np + 1) * nx, Nc * nu
    X = np.zeros((TEAM_STEPS, N, nx)); U = np.zeros((TEAM_STEPS, N, nu)); useq = np.zeros((TEAM_STEPS, N, NU))
    WS = np.zeros((TEAM_STEPS, N), np.int64)
    for b in range(N):
        K = MPC(**dict(c, x0=X0[b], xref=Xref[b], uminus1=np.zeros(nu)))
        if "hard" in opts:
            K.SOFT_ON = False
        K.setup(solve=False)
        x = X0[b].copy(); um1 = np.zeros(nu); warm = None
        for t in range(TEAM_STEPS):
            K.update(x, um1, solve=False)
            z, y, r = certified(K, warm); warm = (z, y)
            X[t, b] = x; useq[t, b] = z[NX:NX + NU]; U[t, b] = z[NX:NX + nu]; WS[t, b] = working_set_size(K, z, y)
            um1 = z[NX:NX + nu].copy(); x = c["Ad"] @ x + c["Bd"] @ um1
    tag = name + "_"
    out = {tag + k: np.asarray(v, float) for k, v in c.items() if k not in ("Np", "Nc")}
    out.update({tag + "X": X, tag + "U": U, tag + "useq": useq, tag + "Xref": Xref, tag + "ws": WS,
                tag + "shape": np.array([nx, nu, Np, Nc]), tag + "hard": np.array("hard" in opts)})
    print("team_shapes", name, (nx, nu, Np, Nc), "working sets", WS.tolist(), flush=True)
    return out


def team_shapes():
    from multiprocessing import Pool
    with Pool(min(len(TEAM_SHAPES), os.cpu_count() or 1)) as pool:
        parts = pool.map(team_shape_case, sorted(TEAM_SHAPES, key=lambda s: -((s[3] + 1) * s[1] + s[4] * s[2]) ** 2 * len(s[5])))
    out = {}
    for p in parts:
        out.update(p)
    np.savez_compressed(os.path.join(OUT, "team_shapes.npz"), names=np.array([s[0] for s in TEAM_SHAPES]), steps=TEAM_STEPS, **out)


if __name__ == "__main__":
    if sys.argv[1:] == ["shapes"]:
        shapes()
        sys.exit(0)
    if sys.argv[1:] == ["mimo_shapes"]:
        mimo_shapes()
        sys.exit(0)
    if sys.argv[1:] == ["team_shapes"]:
        team_shapes()
        sys.exit(0)
    if sys.argv[1:] == ["reference"]:        # only the records of the reference's solver inputs (tests/test_oracle.py)
        reference_assembly(); reference_on_port()
        sys.exit(0)
    first_solve("pm", point_mass()); first_solve("pend", pendulum()); first_solve("mimo", mimo())
    closed_loop("pm", point_mass(), 30)
    closed_loop("pend", pendulum(), 40)
    closed_loop("mimo", mimo(), 12)
    random_batch()
    variants()
    reference_assembly(); reference_on_port()
    shapes()
    mimo_shapes()
    team_shapes()
