"""-m gpu: the multi-input fast path (thread-per-instance Riccati polish over the scalar delta-u chain, k_tpm_pol) at the edges of
its shape domain.

Every shape of tests/golden/mimo_shapes.npz (make_golden.py mimo_shapes) is a seeded random system whose instances start up to
1.3x outside their soft state box; the golden is the exact minimiser of each step's reference-assembled QP along a 5-step closed
loop.  The controller (fast_path=2: the multi-input polish is built on demand for the shape and the system's sparsity pattern) is
fed the golden states and inputs step by step, so every step is compared with its own exact answer.  The batch (333) puts every
golden instance into many lanes and chunks and leaves the last chunk partial; replicas of one instance that the polish verified
alone must agree bit for bit.  The team kernels (fast_path=0) run the same inputs as a control.  Shapes outside the domain
(pympc_b200.build.tpm_shape_supported) must run on the team kernels instead, with the same answers."""
import numpy as np
import pytest

from conftest import golden
from pympc_b200 import _lib, build

pytestmark = pytest.mark.gpu
TOL = 1e-6
B = 333
SYS_KEYS = ("Ad", "Bd", "Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "uref")
SHAPES = [tuple(int(v) for v in s[:4]) for s in golden("mimo_shapes.npz")["shapes"]]
# Least share of the warm steps' instances that k_tpm_pol verifies alone, without any ADMM iteration (res.info.iter == 0), per
# shape, a little below what an H100 showed (the shares are printed; DESIGN.md §4 (i-b) lists them).  Each golden instance is
# about 6 % of the batch at N = 16.  Shapes not listed: outside the domain.
DIRECT_FLOOR = {
    (2, 6, 12, 12): 0.95, (7, 5, 8, 4): 0.3, (8, 4, 25, 1): 0.8, (3, 2, 60, 60): 0.85, (4, 1, 40, 40): 0.95, (1, 5, 20, 10): 0.95,
    (13, 2, 6, 6): 0.85, (13, 1, 10, 10): 0.8,
}


@pytest.fixture(scope="module")
def MPC(bmpc_lib):
    assert bmpc_lib.bmpc_device_count() > 0, "GPU tests need a CUDA device; the product has no CPU fallback"
    from pympc_b200 import MPCController
    return MPCController


def _golden_case(nx, nu, Np, Nc):
    g = golden("mimo_shapes.npz"); tag = f"{nx}_{nu}_{Np}_{Nc}_"
    cfg = {k: g[tag + k] for k in SYS_KEYS}
    cfg.update(Np=Np, Nc=Nc, eps_feas=float(g[tag + "eps_feas"]))
    return cfg, g[tag + "X"], g[tag + "U"], g[tag + "useq"], g[tag + "Xref"]


def _tiling(N):
    # chunk c (32 lanes) starts at golden instance c: every instance lands in a different lane of each chunk it sits in
    return (np.arange(B) + np.arange(B) // 32) % N


def _xref(GXref, t, idx):
    # constant (N, nx) or time-varying per step (T, N, Np+1, nx)
    return GXref[idx] if GXref.ndim == 2 else GXref[t][idx]


def _run(K, X, um1, xref, NU):
    K.update(X, um1, xref=xref)
    _, info = K.output(return_u_seq=True)
    return info["u_seq"].reshape(-1, NU), np.asarray(K.res.info.status_val).copy()


@pytest.mark.parametrize("nx,nu,Np,Nc", SHAPES, ids=[f"{nx}-{nu}-{Np}-{Nc}" for nx, nu, Np, Nc in SHAPES])
def test_multi_input_shape_vs_golden(MPC, nx, nu, Np, Nc):
    cfg, GX, GU, GS, GXref = _golden_case(nx, nu, Np, Nc)
    T, N, NU = GS.shape
    idx = _tiling(N)
    supported = build.tpm_shape_supported(nx, nu, Np, Nc)
    assert supported == ((nx, nu, Np, Nc) in DIRECT_FLOOR)
    Ks = [MPC(**cfg, x0=GX[0][idx], xref=_xref(GXref, 0, idx), uminus1=np.zeros(nu), batch=B, fast_path=f) for f in (2, 0)]
    for K in Ks:
        K.setup(solve=False)
    # the multi-input polish is there exactly for the shapes the predicate accepts; the control never has it
    assert Ks[0]._L.bmpc_has_multi_input_fast_path(nx, nu, Np, Nc) == int(supported)
    assert Ks[1]._L.bmpc_has_multi_input_fast_path(nx, nu, Np, Nc) == 0
    assert Ks[0]._L.bmpc_has_fast_path(nx, nu, Np, Nc) == 0
    scale = 1.0 + np.max(np.abs(GS), axis=2)                               # (T, N): 1 + |u_seq|_inf of each golden QP
    for t in range(T):
        um1 = (GU[t - 1] if t > 0 else np.zeros((N, nu)))[idx]
        for fast, K in zip((1, 0), Ks):
            useq, st = _run(K, GX[t][idx], um1, _xref(GXref, t, idx), NU)
            err = np.max(np.abs(useq - GS[t][idx]), axis=1) / scale[t][idx]
            if fast and supported:
                assert (st == 1).all(), (t, np.flatnonzero(st != 1)[:8], st[st != 1][:8])
                assert err.max() < TOL, (t, int(idx[np.argmax(err)]), err.max())
                if t > 0:
                    # warm steps: on these shapes only k_tpm_pol verifies an instance without ADMM; the others take ADMM rounds
                    direct = np.asarray(K.res.info.iter) == 0
                    s = K.stats()
                    print(f"shape ({nx},{nu},{Np},{Nc}) step {t}: polish alone {direct.mean():.3f}, admm_iters {s['admm_iters']}, "
                          f"rounds {s['rounds']}")
                    assert direct.mean() >= DIRECT_FLOOR[(nx, nu, Np, Nc)], (t, direct.mean(), s["admm_iters"])
                    # replicas of one instance the polish verified alone (other lanes, chunks): bit-identical plans
                    for i in range(N):
                        rows = useq[(idx == i) & direct]
                        assert (rows == rows[:1]).all(), (t, i)
            else:
                # team kernels (the control; the only path of a shape outside the domain): all solved, the polished ones exact
                assert (st > 0).all(), (fast, t)
                ok = st == 1
                assert ok.mean() > 0.95, (fast, t, ok.mean())
                assert err[ok].max() < TOL, (fast, t, err[ok].max())
    for K in Ks:
        K.close()


def _oracle_u(cfg):
    from oracle.qp_assembly import QPData
    from oracle.kkt import solve_exact
    Q = QPData(**cfg)
    try:
        z, y, r = solve_exact(Q.P, Q.q, Q.A, Q.l, Q.u)
        return z[Q.NX:Q.NX + Q.NU]
    except RuntimeError:
        from oracle.ldp import solve_mpc
        return solve_mpc(Q)


def _on_library(MPC, path, **kw):
    """a controller that runs on the library at `path` (the one _pick_library would choose for another pattern)"""
    K = MPC(**kw)
    K._pick_library = lambda: _lib.load(path)
    K.setup(solve=False)
    return K


def test_pattern_instantiation_equals_dense(MPC):
    """The non-symmetric sparsity pattern (lower-Hessenberg Ad, make_golden.mimo_pattern) compiled into k_tpm_pol against the dense
    instantiation of the same shape, on identical inputs: the terms the pattern skips are exact zeros (an fma with them changes
    nothing), so plans, statuses and the work done must be identical, step by step."""
    g = golden("mimo_shapes.npz")
    nx, nu, Np, Nc = (int(v) for v in g["pattern"])
    cfg, GX, GU, GS, GXref = _golden_case(nx, nu, Np, Nc)
    T, N, NU = GS.shape
    idx = _tiling(N)
    libs = [build.jit_multi_input_shape(nx, nu, Np, Nc, cfg["Ad"], cfg["Bd"]), build.jit_multi_input_shape(nx, nu, Np, Nc)]
    assert libs[0] != libs[1]                                          # the system's pattern is not dense: its own build
    Ks = [_on_library(MPC, lib, **cfg, x0=GX[0][idx], xref=GXref[idx], uminus1=np.zeros(nu), batch=B, fast_path=2) for lib in libs]
    for K in Ks:
        assert K._L.bmpc_has_multi_input_fast_path(nx, nu, Np, Nc) == 1
    for t in range(T):
        um1 = (GU[t - 1] if t > 0 else np.zeros((N, nu)))[idx]
        outs = [_run(K, GX[t][idx], um1, GXref[idx], NU) for K in Ks]
        work = [(K.stats()["polish_steps"], K.stats()["admm_iters"], K.stats()["rounds"]) for K in Ks]
        iters = [np.asarray(K.res.info.iter).copy() for K in Ks]
        assert np.array_equal(outs[0][1], outs[1][1]), t
        assert np.array_equal(outs[0][0], outs[1][0]), (t, np.max(np.abs(outs[0][0] - outs[1][0])))
        assert work[0] == work[1] and np.array_equal(iters[0], iters[1]), (t, work)
        assert (outs[0][1] == 1).all() and np.max(np.abs(outs[0][0] - GS[t][idx])) < TOL * (1.0 + np.abs(GS).max()), t
    for K in Ks:
        K.close()


@pytest.mark.parametrize("where", ["Ad", "Bd"])
def test_system_outside_the_compiled_pattern_takes_the_dense_entry(MPC, where):
    """One non-zero outside the compiled masks (Ad[0][nx-1], above the Hessenberg band, or Bd[nx-1][0], off the channel blocks) on
    the pattern library: bmpc_setup must pick the dense entry of the shape; the sparse one would silently drop that term (the
    sweeps and their verification would agree on the wrong model).  All instances against the team kernels, a sample against the
    oracle on its own QP."""
    g = golden("mimo_shapes.npz")
    nx, nu, Np, Nc = (int(v) for v in g["pattern"])
    cfg, GX, GU, GS, GXref = _golden_case(nx, nu, Np, Nc)
    lib = build.jit_multi_input_shape(nx, nu, Np, Nc, cfg["Ad"], cfg["Bd"])
    Ad, Bd = cfg["Ad"].copy(), cfg["Bd"].copy()
    if where == "Ad":
        assert Ad[0, nx - 1] == 0.0
        Ad[0, nx - 1] = 0.3
    else:
        assert Bd[nx - 1, 0] == 0.0
        Bd[nx - 1, 0] = 0.5
    cfg = dict(cfg, Ad=Ad, Bd=Bd)
    N = GX.shape[1]; idx = _tiling(N); X = GX[0][idx]; U = np.zeros((B, nu)); NU = Nc * nu
    Ks = [_on_library(MPC, lib, **cfg, x0=X, xref=GXref[idx], uminus1=U, batch=B, fast_path=2),
          MPC(**cfg, x0=X, xref=GXref[idx], uminus1=U, batch=B, fast_path=0)]
    Ks[1].setup(solve=False)
    rng = np.random.default_rng(17)
    for t in range(4):
        outs = [_run(K, X, U, GXref[idx], NU) for K in Ks]
        assert (outs[0][1] == 1).all(), t
        both = outs[1][1] == 1
        assert both.mean() > 0.95 and np.max(np.abs(outs[0][0][both] - outs[1][0][both])) < TOL, t
        for b in rng.choice(B, 4, replace=False):
            c = dict(cfg, x0=X[b], xref=GXref[idx][b], uminus1=U[b])
            assert np.max(np.abs(outs[0][0][b] - _oracle_u(c))) < TOL, (t, b)
        if t > 0:
            # the multi-input polish did run: on this shape only k_tpm_pol verifies an instance without ADMM
            direct = np.asarray(Ks[0].res.info.iter) == 0
            print(f"extra non-zero in {where}, step {t}: polish alone {direct.mean():.3f}")
            assert direct.any(), t
        U = outs[0][0][:, :nu].copy(); X = X @ Ad.T + U @ Bd.T
    for K in Ks:
        K.close()


def test_non_diagonal_rate_weight_runs_on_the_team_kernels(MPC):
    """A non-diagonal QDu: the multi-input polish keeps one previous value per channel, so tpm_fill declines the system and every
    instance runs on the team kernels (ADMM on every step) — with exact answers, although the controller's library has the shape."""
    nx, nu, Np, Nc = 1, 5, 20, 10
    cfg, GX, GU, GS, GXref = _golden_case(nx, nu, Np, Nc)
    rng = np.random.default_rng(23)
    M = rng.standard_normal((nu, nu))
    cfg = dict(cfg, QDu=cfg["QDu"] + 0.1 * M @ M.T / nu)
    N = GX.shape[1]; idx = _tiling(N); X = GX[0][idx]; U = np.zeros((B, nu)); NU = Nc * nu
    Ks = [MPC(**cfg, x0=X, xref=GXref[idx], uminus1=U, batch=B, fast_path=f) for f in (2, 0)]
    for K in Ks:
        K.setup(solve=False)
    assert Ks[0]._L.bmpc_has_multi_input_fast_path(nx, nu, Np, Nc) == 1
    for t in range(4):
        outs = [_run(K, X, U, GXref[idx], NU) for K in Ks]
        for useq, st in outs:
            assert (st > 0).all() and (st == 1).mean() > 0.95, t
        assert (np.asarray(Ks[0].res.info.iter) > 0).all(), t                  # no instance was verified without ADMM
        both = (outs[0][1] == 1) & (outs[1][1] == 1)
        assert np.max(np.abs(outs[0][0][both] - outs[1][0][both])) < TOL, t
        for b in rng.choice(np.flatnonzero(both), 4, replace=False):
            c = dict(cfg, x0=X[b], xref=GXref[idx][b], uminus1=U[b])
            assert np.max(np.abs(outs[0][0][b] - _oracle_u(c))) < TOL, (t, b)
        U = outs[0][0][:, :nu].copy(); X = X @ cfg["Ad"].T + U @ cfg["Bd"].T
    for K in Ks:
        K.close()
