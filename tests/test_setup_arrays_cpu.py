"""CPU tests of the arrays MPCController.setup() hands bmpc_setup (MPCController._device_arrays over _setup_arrays, the conversion
update_system shares): float64, C-contiguous, in the argument order of bmpc_setup, the weights zeroed by JX_ON / JU_ON / JDU_ON, and on
per-instance controllers every array with a leading batch dimension (an array given once is broadcast).  The expected arrays are
built here independently from the constructor's arguments and compared exactly, bit for bit.  A weight whose flag is off is sent as
+0.0 zeros on every path; per-instance setup once sent 0 * Q instead, which is -0.0 where an entry of Q is negative (equal values)."""
import numpy as np
import pytest
import scipy.sparse as sp

NAMES = ("Ad", "Bd", "Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "uref")
WEIGHT_FLAG = {"Qx": "JX_ON", "QxN": "JX_ON", "Qu": "JU_ON", "QDu": "JDU_ON"}
B, NX, NU = 5, 3, 2


def _spd(rng, n):
    M = rng.standard_normal((n, n))
    return M @ M.T + n * np.eye(n)


def _problem(rng):
    """a shared problem with dense non-diagonal weights (signed off-diagonal entries), integer-valued Ad and (1, n) bounds"""
    return dict(Ad=np.array([[1, 1, 0], [0, 1, 1], [0, 0, 1]]), Bd=rng.standard_normal((NX, NU)), Np=6, Nc=4,
                Qx=_spd(rng, NX), QxN=_spd(rng, NX), Qu=_spd(rng, NU), QDu=_spd(rng, NU),
                xmin=-rng.uniform(1, 2, (1, NX)), xmax=rng.uniform(1, 2, NX), umin=-rng.uniform(1, 2, NU), umax=rng.uniform(1, 2, NU),
                Dumin=-np.full(NU, np.inf), Dumax=rng.uniform(0.1, 0.5, NU), uref=rng.standard_normal(NU))


def _expected(kw, flags, batched):
    """the 13 arrays by hand: shared arrays as given (dense, float64, bounds flattened); a weight whose flag is off: zeros;
    batched: every array (B, ...), from the argument where it has a batch dimension, else the shared one repeated"""
    shapes = dict(Ad=(NX, NX), Bd=(NX, NU), Qx=(NX, NX), QxN=(NX, NX), Qu=(NU, NU), QDu=(NU, NU), xmin=(NX,), xmax=(NX,))
    out = {}
    for name in NAMES:
        shape = shapes.get(name, (NU,))
        a = kw[name]
        a = a.toarray() if sp.issparse(a) else np.asarray(a, dtype=float)
        per = a.ndim == len(shape) + 1 and a.shape[0] == B and batched
        a = a if per else a.reshape(shape)
        if not flags.get(WEIGHT_FLAG.get(name), True):
            a = np.zeros(a.shape)
        if batched and not per:
            a = np.stack([a] * B)
        out[name] = a
    return out


def _assert_sent(K, exp, batched):
    sent = K._device_arrays(K._setup_arrays())
    assert list(sent) == list(NAMES)
    for name in NAMES:
        a, e = sent[name], exp[name]
        assert a.shape == e.shape and a.dtype == np.float64 and a.flags.c_contiguous, name
        assert a.tobytes() == e.tobytes(), name
    # the weights the controller records as sent: instance 0's for the reference-form QP, every instance's for J_CNST
    for name in WEIGHT_FLAG:
        d = getattr(K, "_" + name + "_d")
        assert np.array_equal(d, exp[name][0] if batched else exp[name]), name
        if batched:
            assert np.array_equal(K._w_full[name], exp[name]), name


@pytest.mark.parametrize("off", [None, "JX_ON", "JU_ON", "JDU_ON"])
def test_shared_controller_arrays(bmpc_lib, off):
    from pympc_b200 import MPCController
    kw = _problem(np.random.default_rng(1))
    kw["QxN"] = sp.csc_matrix(kw["QxN"])                      # a sparse weight is sent dense
    K = MPCController(batch=B, **kw)
    flags = {off: False} if off else {}
    for f, v in flags.items():
        setattr(K, f, v)
    _assert_sent(K, _expected(kw, flags, batched=False), batched=False)


@pytest.mark.parametrize("off", [None, "JX_ON", "JU_ON", "JDU_ON"])
def test_per_instance_controller_arrays(bmpc_lib, off):
    """Ad, Bd, Qx, Qu, xmin, umax, Dumin with a batch dimension, the other arrays shared"""
    from pympc_b200 import MPCController
    rng = np.random.default_rng(2)
    kw = _problem(rng)
    kw["Ad"] = np.stack([kw["Ad"] + 0.1 * i for i in range(B)])
    kw["Bd"] = kw["Bd"] * rng.uniform(0.5, 1.5, (B, 1, 1))
    kw["Qx"] = np.stack([_spd(rng, NX) for _ in range(B)])
    kw["Qu"] = np.stack([_spd(rng, NU) for _ in range(B)])
    kw["xmin"] = -rng.uniform(1, 2, (B, NX))
    kw["umax"] = rng.uniform(1, 2, (B, NU))
    kw["Dumin"] = -rng.uniform(0.1, 0.5, (B, NU))
    K = MPCController(batch=B, **kw)
    assert K._per_instance
    flags = {off: False} if off else {}
    for f, v in flags.items():
        setattr(K, f, v)
    _assert_sent(K, _expected(kw, flags, batched=True), batched=True)
