"""-m gpu tests of bmpc_setup on a live handle: a set-up handle may be set up again (include/bmpc.h).  A re-setup whose condensed
Hessian is not positive definite returns BMPC_ERR_NOT_PD and leaves the handle refused, like a failed bmpc_update_problem:
bmpc_solve returns BMPC_ERR_STATE instead of solving on a failed factorisation with the previous problem's fast-path parameters.
Updates that leave the weights singular keep it refused: a uref-only update (on per-instance systems it defers the condense and
leaves definiteness as the setup left it) and an (Ad, Bd)-only one.  A valid bmpc_setup restores it, and its next solve equals a
fresh controller's, in every kernel family."""
import numpy as np
import pytest

from pympc_b200._lib import ptr
from pympc_b200.workloads import pendulum, pendulum_random, mimo

pytestmark = pytest.mark.gpu
KEYS = ("Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "eps_feas")
WEIGHTS = ("Qx", "QxN", "Qu", "QDu")
BMPC_OK, BMPC_ERR_STATE, BMPC_ERR_NOT_PD = 0, -3, -4


@pytest.fixture(scope="module")
def MPC(bmpc_lib):
    assert bmpc_lib.bmpc_device_count() > 0, "GPU tests need a CUDA device; the product has no CPU fallback"
    from pympc_b200 import MPCController
    return MPCController


def _family(name):
    """-> (Ad, Bd, constructor keywords, X0, fast-path check)"""
    if name == "mimo":
        c = mimo(); c.setdefault("eps_feas", 1e6); B = 256
        X0 = 0.3 * np.random.default_rng(4).standard_normal((B, 8))
        kw = dict({k: c[k] for k in KEYS}, Np=40, batch=B, xref=c["xref"], uminus1=np.zeros(4))
        return c["Ad"], c["Bd"], kw, X0, lambda L: L.bmpc_has_multi_input_fast_path(8, 4, 40, 40) == 1
    c = pendulum(); B = 512
    X0, Xref = pendulum_random(B, seed=6)
    kw = dict({k: c[k] for k in KEYS}, Np=20, batch=B, xref=Xref, uminus1=np.zeros(1), **({"fast_path": 0} if name == "team" else {}))
    Ad, Bd = c["Ad"], c["Bd"]
    if name == "per_instance":
        Ad = np.broadcast_to(Ad, (B, 4, 4)).copy(); Bd = np.broadcast_to(Bd, (B, 4, 1)).copy()
    return Ad, Bd, kw, X0, lambda L: name == "team" or L.bmpc_has_fast_path(4, 1, 20, 20) == 1


def _step(Ad, Bd, X, U):
    if np.ndim(Ad) == 3:
        return np.einsum("bij,bj->bi", Ad, X) + np.einsum("bij,bj->bi", Bd, U)
    return X @ Ad.T + U @ Bd.T


@pytest.mark.parametrize("name", ["tpi", "per_instance", "mimo", "team"])
def test_failed_resetup_is_refused_until_a_valid_one(MPC, name):
    Ad, Bd, kw, X0, on_fast_path = _family(name)
    K = MPC(Ad, Bd, x0=X0, **kw); K.setup()
    assert on_fast_path(K._L)
    U = K.output().copy()
    L, h = K._L, K._h
    sent = K._device_arrays(K._setup_arrays())
    bad = {n: np.zeros_like(a) if n in WEIGHTS else a for n, a in sent.items()}
    args = lambda arrays: [ptr(arrays[n]) for n, _, _ in K._PROBLEM]
    assert L.bmpc_setup(h, *args(bad)) == BMPC_ERR_NOT_PD
    assert b"not positive definite" in L.bmpc_last_error(h)
    assert L.bmpc_solve(h) == BMPC_ERR_STATE
    assert b"bmpc_setup" in L.bmpc_last_error(h)
    shared = np.ndim(Ad) == 2
    assert L.bmpc_update_problem(h, *[None] * 12, ptr(sent["uref"]), 0) == (BMPC_ERR_NOT_PD if shared else BMPC_OK)
    assert L.bmpc_solve(h) == BMPC_ERR_STATE
    assert L.bmpc_update_problem(h, ptr(sent["Ad"]), *[None] * 12, 0) == BMPC_ERR_NOT_PD
    assert L.bmpc_solve(h) == BMPC_ERR_STATE
    assert L.bmpc_setup(h, *args(sent)) == BMPC_OK
    X = _step(Ad, Bd, X0, U)
    K.update(X, U); u1 = K.output().copy(); s1 = np.array(K.res.info.status_val)
    F = MPC(Ad, Bd, x0=X0, **kw); F.setup(solve=False)
    F.update(X, U); u2 = F.output().copy(); s2 = np.array(F.res.info.status_val)
    assert (s1 > 0).all() and np.array_equal(s1, s2), (name, np.unique(s1, return_counts=True), np.unique(s2, return_counts=True))
    assert np.max(np.abs(u1 - u2)) < 1e-9, name
    K.close(); F.close()
