"""-m gpu: the team / tile kernels (k_admm, k_admm_tile, the Schur-form k_polish) at the edges of their shape domain and of the
polish's working-set capacity.

Every case of tests/golden/team_shapes.npz (make_golden.py team_shapes) is a seeded random system along a 4-step closed loop whose
instances start further and further outside their soft state box; the golden is the exact minimiser of each step's
reference-assembled QP, and the golden also records the size of its working set (violated soft rows + active hard rows), so each
case states which capacity edge it reaches.  The controller runs on the team kernels (fast_path=0) and is fed the golden states
step by step.  The polish tiers each case meets are the library's own (bmpc_launch.cuh; tests/test_team_capacity_cpu.py pins
them): warp team 64 with its overflow to a CTA tier of mc rows, CTA team 80 then the largest capacity that fits."""
import numpy as np
import pytest

from conftest import golden

pytestmark = pytest.mark.gpu
TOL = 1e-6
B = 333
BIG = 5000           # more open instances than the CTA tier takes alone (BMPC_FB_MAX_LIST = 4096)
SYS_KEYS = ("Ad", "Bd", "Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "uref")
NAMES = [str(n) for n in golden("team_shapes.npz")["names"]]


@pytest.fixture(scope="module")
def MPC(bmpc_lib):
    assert bmpc_lib.bmpc_device_count() > 0, "GPU tests need a CUDA device; the product has no CPU fallback"
    from pympc_b200 import MPCController
    return MPCController


def _case(name):
    g = golden("team_shapes.npz"); tag = name + "_"
    nx, nu, Np, Nc = (int(v) for v in g[tag + "shape"])
    cfg = {k: g[tag + k] for k in SYS_KEYS}
    cfg.update(Np=Np, Nc=Nc, eps_feas=float(g[tag + "eps_feas"]))
    return cfg, bool(g[tag + "hard"]), g[tag + "X"], g[tag + "U"], g[tag + "useq"], g[tag + "Xref"], g[tag + "ws"]


def _controller(MPC, cfg, hard, X0, Xref, batch, per_instance=False, **opts):
    if per_instance:                                   # one system per instance (n_sys = batch): copies of the shared one
        cfg = dict(cfg, Ad=np.repeat(cfg["Ad"][None], batch, 0), Bd=np.repeat(cfg["Bd"][None], batch, 0))
    K = MPC(**cfg, x0=X0, xref=Xref, uminus1=np.zeros(cfg["Bd"].shape[-1]), batch=batch, fast_path=0, **opts)
    if hard:
        K.SOFT_ON = False
    K.setup(solve=False)
    return K


def _closed_loop(K, GX, GU, GXref, idx, NU):
    """the golden states step by step; returns per step (u_seq (batch, NU), status (batch,), u (batch, nu))"""
    out = []
    nu = GU.shape[2]
    for t in range(GX.shape[0]):
        um1 = (GU[t - 1] if t > 0 else np.zeros((GX.shape[1], nu)))[idx]
        K.update(GX[t][idx], um1, xref=GXref[idx])
        u, info = K.output(return_u_seq=True)
        out.append((info["u_seq"].reshape(-1, NU).copy(), np.asarray(K.res.info.status_val).copy(), np.asarray(u).reshape(-1, nu).copy()))
    return out


def _check_exact(name, out, GS, idx, bitwise=True):
    scale = 1.0 + np.max(np.abs(GS), axis=2)
    for t, (useq, st, u) in enumerate(out):
        ok = st == 1
        err = np.max(np.abs(useq - GS[t][idx]), axis=1) / scale[t][idx]
        assert (st > 0).all(), (name, t, np.flatnonzero(st <= 0)[:8])
        assert ok.mean() > 0.95, (name, t, ok.mean())
        assert err[ok].max() < TOL, (name, t, int(idx[ok][np.argmax(err[ok])]), err[ok].max())
        if bitwise:
            for i in range(GS.shape[1]):                 # replicas of one golden instance: bit for bit
                rows = useq[(idx == i) & ok]
                assert (rows == rows[:1]).all(), (name, t, i)


@pytest.mark.parametrize("name", NAMES)
def test_team_shape_vs_golden(MPC, name):
    cfg, hard, GX, GU, GS, GXref, WS = _case(name)
    T, N, NU = GS.shape
    idx = np.arange(B) % N
    K = _controller(MPC, cfg, hard, GX[0][idx], GXref[idx], B)
    _check_exact(name, _closed_loop(K, GX, GU, GXref, idx, NU), GS, idx)
    K.close()


@pytest.mark.parametrize("name", ["warp_cap", "cta_cap", "mc192"])
def test_capacity_does_not_depend_on_batch_size(MPC, name):
    """Working sets beyond the first tier (64 for a warp team, 80 for a CTA team) up to mc: every instance verifies, in a batch of
    333 and in a batch of 5 000 replicas of the instances beyond the first tier, whose straggler rounds hold more instances than
    the CTA tier takes alone.  The answers agree across batch sizes and with the golden."""
    cfg, hard, GX, GU, GS, GXref, WS = _case(name)
    T, N, NU = GS.shape
    first = 64 if name != "cta_cap" else 80
    assert WS.max() > first and (WS <= first).any()          # both sides of the first tier's capacity
    outs = []
    over = np.flatnonzero(WS[0] > first)              # the big batch: replicas of the instances the first tier cannot hold
    for batch, members in ((B, np.arange(N)), (BIG, over)):
        idx = members[np.arange(batch) % len(members)]
        K = _controller(MPC, cfg, hard, GX[0][idx], GXref[idx], batch)
        out = _closed_loop(K, GX, GU, GXref, idx, NU)
        K.close()
        scale = 1.0 + np.max(np.abs(GS), axis=2)
        for t, (useq, st, u) in enumerate(out):
            assert (st == 1).all(), (name, batch, t, sorted(set(idx[st != 1].tolist())), st[st != 1][:8])
            err = np.max(np.abs(useq - GS[t][idx]), axis=1) / scale[t][idx]
            assert err.max() < TOL, (name, batch, t, err.max())
        outs.append([useq[:len(members)] for useq, st, u in out])
    for t in range(T):
        assert np.max(np.abs(outs[0][t][over] - outs[1][t])) < TOL * (1.0 + np.abs(GS[t]).max()), (name, t)


def test_working_sets_beyond_capacity_end_with_the_admm_verdict(MPC):
    """A polish capacity of 40 rows (one CTA tier: team_threads=256, rmax=40) on instances whose optimal working sets reach 135:
    those beyond 40 cannot be verified.  They must never come back as verified (status 1) with a wrong answer: status 2 is within
    OSQP's accuracy class, status -2 returns u_failure."""
    cfg, hard, GX, GU, GS, GXref, WS = _case("warp_cap")
    T, N, NU = GS.shape
    cap = 40
    assert (WS > cap).any() and (WS <= cap).any()
    idx = np.arange(2 * N) % N
    K = _controller(MPC, cfg, hard, GX[0][idx], GXref[idx], 2 * N, team_threads=256, rmax=cap)
    out = _closed_loop(K, GX, GU, GXref, idx, NU)
    nu = GU.shape[2]
    for t, (useq, st, u) in enumerate(out):
        scale = 1.0 + np.max(np.abs(GS[t][idx]), axis=1)
        err = np.max(np.abs(u - GS[t][idx][:, :nu]), axis=1) / scale
        beyond = WS[t][idx] > cap
        assert (st[beyond] != 1).all(), (t, st[beyond])
        assert not (st == 1).any() or err[st == 1].max() < TOL, t
        two = st == 2
        assert not two.any() or err[two].max() < 2e-2, (t, err[two].max())
        bad = (st != 1) & (st != 2)
        assert (u[bad] == np.asarray(K.u_failure, float).ravel()[:nu]).all(), (t, st[bad])
        print(f"beyond capacity, step {t}: status {dict(zip(*np.unique(st[beyond], return_counts=True)))}")
    K.close()


@pytest.mark.parametrize("name", ["cta_cap", "cta_hard", "warp_hard"])
def test_per_instance_systems_vs_golden(MPC, name):
    """One system per instance (n_sys = batch): the CTA team runs k_admm<false> and the polish tiers without tiles, the warp team
    its per-instance blocks; same exact answers."""
    cfg, hard, GX, GU, GS, GXref, WS = _case(name)
    T, N, NU = GS.shape
    idx = np.arange(B) % N
    K = _controller(MPC, cfg, hard, GX[0][idx], GXref[idx], B, per_instance=True)
    _check_exact(name, _closed_loop(K, GX, GU, GXref, idx, NU), GS, idx)
    K.close()


def test_shape_beyond_shared_memory_is_refused(MPC):
    """(8, 4, 314): mc = 5 036 rows.  Not even an 8-row working set fits next to the polish's per-row vectors in the 227 KB a CTA
    can opt into (tests/test_team_capacity_cpu.py pins (8, 4, 313) as the last shape that fits).  setup() must refuse it with the
    library's message; a small controller still runs afterwards."""
    from pympc_b200 import BmpcError
    from pympc_b200.workloads import point_mass
    nx, nu, Np = 8, 4, 314
    rng = np.random.default_rng(5)
    A = 0.9 * np.eye(nx) + 0.01 * rng.standard_normal((nx, nx))
    K = MPC(A, rng.standard_normal((nx, nu)), Np=Np, x0=np.zeros(nx), xref=np.zeros(nx), uminus1=np.zeros(nu), batch=4,
            Qx=np.eye(nx), QxN=np.eye(nx), Qu=0.1 * np.eye(nu), QDu=0.1 * np.eye(nu), xmin=-np.ones(nx), xmax=np.ones(nx),
            umin=-np.ones(nu), umax=np.ones(nu), fast_path=0)
    with pytest.raises(BmpcError, match="problem too large for the shared-memory resident kernels"):
        K.setup(solve=False)
    c = point_mass()
    K2 = MPC(c["Ad"], c["Bd"], Np=20, x0=np.zeros(2), xref=np.zeros(2), uminus1=np.zeros(1), batch=4, fast_path=0,
             **{k: c[k] for k in ("Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax")})
    K2.setup(solve=False)
    K2.update(np.tile([1.0, 0.0], (4, 1)), np.zeros((4, 1)))
    K2.output()
    assert (np.asarray(K2.res.info.status_val) > 0).all()
    K2.close()
