"""Batched drop-in for ``pyMPC.mpc.MPCController`` on H100 (host side, Python over ctypes).

Mirrors the reference class (/root/reference/pyMPC/mpc.py:27-615): same constructor arguments,
defaults, validation messages and method surface — ``setup()`` (mpc.py:254), ``output()`` (:271),
``update()`` (:338), ``solve()`` (:366), ``__controller_function__`` (:377) — but every numerical
step runs in hand-written CUDA kernels behind the C ABI of ``include/bmpc.h``:
``_compute_QP_matrices_`` + ``OSQP.setup`` -> ``bmpc_setup`` (condense on device),
``_update_QP_matrices_`` + ``OSQP.update`` -> ``bmpc_update``, ``OSQP.solve`` -> ``bmpc_solve``
(ADMM + verified active-set polish), result slicing -> ``bmpc_output``.

Batching (extension): ``batch=B`` runs B independent instances that share (Ad, Bd, weights,
bounds) and differ in (x0, uminus1, xref).  With ``batch=None`` (default) the class behaves like
the reference: 1-D inputs, 1-D ``output()``.

There is no CPU fallback: constructing a controller without the CUDA library or without a GPU
raises.  Unlike OSQP at its default tolerance the solver returns the exact QP minimiser (KKT
verified), which is what parity at 1e-6 needs (SURVEY.md §7.3); ``eps_abs``/``eps_rel`` keep
OSQP's meaning for instances the polish cannot verify, and in ``polish=False`` mode.
"""
import ctypes
import os
import warnings

import numpy as np

from . import _lib
from ._lib import BmpcConfig, BmpcError, BmpcStats, PinnedArray, ptr

_STATUS_STR = {1: "solved", 2: "solved", -2: "maximum iterations reached", -3: "primal infeasible", -10: "unsolved"}


class _ResInfo:
    """`res.info` of the last solve like OSQP's (the reference reads status / obj_val, mpc.py:301-327,372): status_val (int or
    int32 array), status (OSQP's strings), polished, and — fetched from the device on first access — obj_val (objective of the
    reference-form QP, without J_CNST) and iter (ADMM iterations; 0 when the polish verified the warm start directly)."""
    __slots__ = ("_st", "_scalar", "_B", "_K", "_cache", "_id")

    def __init__(self, st, scalar, B, K=None, solve_id=0):
        self._st, self._scalar, self._B, self._K, self._cache, self._id = st, scalar, B, K, {}, solve_id

    @property
    def status_val(self):
        return int(self._st[0]) if self._scalar else self._st

    @property
    def status(self):
        if self._scalar:
            return _STATUS_STR.get(int(self._st[0]), "unsolved")
        return np.array([_STATUS_STR.get(int(s), "unsolved") for s in self._st]) if self._B <= 4096 else None

    @property
    def polished(self):
        return bool(self._st[0] == 1) if self._scalar else self._st == 1

    def _fetch(self, what):
        if what not in self._cache:
            self._cache[what] = self._K._res_fetch(what, self._id)
        v = self._cache[what]
        return (v[0].item() if self._scalar else v)

    @property
    def obj_val(self):
        return self._fetch("obj_val")

    @property
    def iter(self):
        return self._fetch("iter")


class _Res:
    """Result object of the last solve with the attributes the reference reads from OSQP's (mpc.py:302-327): `x` — the primal
    solution in the reference's variable order [x_0..x_Np | u_0..u_{Nc-1} | eps_0..eps_Np] (fetched from the device on first
    access; shape (n,) unbatched, (B, n) batched) — and `info`."""
    __slots__ = ("info", "_K", "_x", "_id")

    def __init__(self, info, K, solve_id=0):
        self.info, self._K, self._x, self._id = info, K, None, solve_id

    @property
    def x(self):
        if self._x is None:
            self._x = self._K._res_fetch("x", self._id)
        return self._x[0] if self._K.batch is None else self._x


def __is_vector__(vec):
    # same acceptance rule as the reference helper (mpc.py:8-17)
    if vec.ndim == 1:
        return True
    if vec.ndim == 2:
        if vec.shape[0] == 1 or vec.shape[1] == 0:
            return True
    return False


def __is_matrix__(mat):
    return mat.ndim == 2


def _dense(M):
    return np.ascontiguousarray(M.toarray() if hasattr(M, "toarray") else M, dtype=float)


class MPCController:
    """Linear constrained MPC controller, batched on one H100.  Arguments as in the reference
    (mpc.py:30-74), plus:

    batch : int or None
        Number of independent instances.  ``None``: reference behaviour (one instance, 1-D I/O).
    device : int
        CUDA device ordinal.
    solver options (keyword only): ``rho`` (<=0: automatic), ``sigma``, ``alpha``, ``max_iter``,
        ``first_iters``, ``pdas_steps``, ``polish``, ``team_threads``, ``warps_per_block``, ``rmax``.
    """

    def __init__(self, Ad, Bd, Np=20, Nc=None,
                 x0=None, xref=None, uref=None, uminus1=None,
                 Qx=None, QxN=None, Qu=None, QDu=None,
                 xmin=None, xmax=None, umin=None, umax=None, Dumin=None, Dumax=None,
                 eps_feas=1e6, eps_rel=1e-3, eps_abs=1e-3, batch=None, device=0, **solver_options):
        Ad = np.asarray(Ad.toarray() if hasattr(Ad, "toarray") else Ad)
        Bd = np.asarray(Bd.toarray() if hasattr(Bd, "toarray") else Bd)
        # extension (SURVEY.md 8f-3): Ad of shape (B, nx, nx) selects one system per instance; Bd, the weights and the
        # bounds may then carry a leading batch dimension too (otherwise they are shared)
        self._per_instance = batch is not None and Ad.ndim == 3
        if self._per_instance:
            if Ad.shape[0] != int(batch) or Ad.shape[1] != Ad.shape[2]:
                raise ValueError(self._MSG["Ad"])
            self._sys_full = dict(Ad=Ad, Bd=Bd, Qx=Qx, QxN=QxN, Qu=Qu, QDu=QDu, xmin=xmin, xmax=xmax, umin=umin, umax=umax,
                                  Dumin=Dumin, Dumax=Dumax)
            pick = lambda a, nd: None if a is None else (np.asarray(a)[0] if np.ndim(a) == nd + 1 else a)
            Ad = Ad[0]; Bd = pick(Bd, 2)
            Qx, QxN, Qu, QDu = pick(Qx, 2), pick(QxN, 2), pick(Qu, 2), pick(QDu, 2)
            xmin, xmax, umin, umax, Dumin, Dumax = (pick(a, 1) for a in (xmin, xmax, umin, umax, Dumin, Dumax))
        if __is_matrix__(Ad) and (Ad.shape[0] == Ad.shape[1]):
            self.Ad = Ad
            self.nx = Ad.shape[0]
        else:
            raise ValueError(self._MSG["Ad"])
        if __is_matrix__(Bd) and Bd.shape[0] == self.nx:
            self.Bd = Bd
            self.nu = Bd.shape[1]
        else:
            raise ValueError(self._MSG["Bd"])
        if Np > 1:
            self.Np = Np
        else:
            raise ValueError("Np should be > 1!")
        if Nc is not None:
            if Nc <= Np:
                self.Nc = Nc
            else:
                raise ValueError("Nc should be <= Np!")
        else:
            self.Nc = self.Np
        self.batch = batch
        self._B = 1 if batch is None else int(batch)
        if self._B < 1:
            raise ValueError("batch should be >= 1!")
        nx, nu, B = self.nx, self.nu, self._B

        # per-instance quantities: accepted exactly like the reference when unbatched (mpc.py:108-142),
        # or with a leading batch dimension
        self.x0 = self._vec_or_batch(x0, nx, "x0 should be an array of dimension (nx,)!", np.zeros(nx))
        self.xref = self._xref_arg(xref)
        if uref is not None:
            uref = np.asarray(uref, dtype=float)
            if __is_vector__(uref) and uref.size == nu:
                self.uref = uref.ravel()
            else:
                raise ValueError(self._MSG["uref"])
        else:
            self.uref = np.zeros(nu)
        self.uminus1 = self._vec_or_batch(uminus1, nu, "uminus1 should be a vector of shape (nu,)!", self.uref)

        def weight(name, Q, n, default):
            if Q is None:
                return default
            Qd = Q if hasattr(Q, "toarray") else np.asarray(Q)
            if Qd.ndim == 2 and Qd.shape[0] == n and Qd.shape[1] == n:
                return Q
            raise ValueError(self._MSG[name])
        self.Qx = weight("Qx", Qx, nx, np.zeros((nx, nx)))   # zeros, not eye (mpc.py:150)
        self.QxN = weight("QxN", QxN, nx, self.Qx)
        self.Qu = weight("Qu", Qu, nu, np.zeros((nu, nu)))
        self.QDu = weight("QDu", QDu, nu, np.zeros((nu, nu)))

        def bound(name, v, n, default):
            if v is None:
                return default
            v = np.asarray(v, dtype=float)
            if __is_vector__(v) and v.size == n:
                return v.ravel()
            raise ValueError(self._MSG[name])
        inf = np.inf
        self.xmin = bound("xmin", xmin, nx, -np.ones(nx) * inf)
        self.xmax = bound("xmax", xmax, nx, np.ones(nx) * inf)
        self.umin = bound("umin", umin, nu, -np.ones(nu) * inf)
        self.umax = bound("umax", umax, nu, np.ones(nu) * inf)
        self.Dumin = bound("Dumin", Dumin, nu, -np.ones(nu) * inf)
        self.Dumax = bound("Dumax", Dumax, nu, np.ones(nu) * inf)

        self.eps_feas = eps_feas
        self.Qeps = eps_feas * np.eye(nx)
        self.eps_rel = eps_rel
        self.eps_abs = eps_abs
        self.u_failure = self.uref

        # hidden settings of the reference (mpc.py:233-238)
        self.raise_error = False
        self.JX_ON = True
        self.JU_ON = True
        self.JDU_ON = True
        self.SOFT_ON = True
        self.COMPUTE_J_CNST = False

        self.device = int(device)
        self.solver_options = dict(solver_options)
        # zero_copy (default on): the kernels read x0 / u_-1 from, and write u* to, pinned host memory in place (see _push / solve)
        self._zero_copy = bool(self.solver_options.pop("zero_copy", True))
        self._stats_buf = BmpcStats(); self._stats_ref = ctypes.byref(self._stats_buf)
        self._external_output = False        # set by whoever binds the solver's output buffer himself (bmpc_bind_output: bench.py's gather)
        self._bound_u = None
        self._out_pool = []
        self._out_pins = []; self._u0_pooled = False
        self._pin_ptr = getattr(self, "_pin_ptr", {})
        self._L = _lib.load()                      # raises if the CUDA extension is missing
        self._h = None
        self.res = None
        self.x0_rh = None
        self.uminus1_rh = None
        self._J_CNST = None
        self._w_full = {}
        self._J_dirty = True
        self._pin = {}
        self._pin_flip = {}
        self._status = None
        self._u0 = None

    # ------------------------------------------------------------------ argument helpers
    def _vec_or_batch(self, v, n, msg, default):
        if v is None:
            return np.array(default, dtype=float, copy=True)
        v = np.asarray(v, dtype=float)
        if self.batch is not None and v.ndim == 2 and v.shape == (self._B, n):
            return v
        if __is_vector__(v) and v.size == n:
            return v.ravel()
        raise ValueError(msg)

    def _xref_arg(self, xref):
        nx, Np, B = self.nx, self.Np, self._B
        if xref is None:
            return np.zeros(nx)
        xref = np.asarray(xref, dtype=float)
        if self.batch is not None:
            if xref.ndim == 3 and xref.shape[0] == B and xref.shape[2] == nx and (xref.shape[1] >= Np or xref.shape[1] == 1):
                return xref                                     # (B, Np+1, nx) per-instance trajectories, (B, 1, nx) per-instance constants
            if xref.ndim == 2 and xref.shape == (B, nx) and not (B >= Np and B == Np + 1):
                return xref
        if __is_vector__(xref) and xref.size == nx:
            return xref.ravel()
        if __is_matrix__(xref) and xref.shape[1] == nx and xref.shape[0] >= Np:
            return xref                                         # same acceptance as mpc.py:120 (quirk Q6)
        raise ValueError("xref should be either a vector of shape (nx,) or a matrix of shape (Np+1, nx)!")

    def _xref_device_layout(self, xref):
        """-> (array [B,nx] or [B,(Np+1)*nx], rows)"""
        nx, Np, B = self.nx, self.Np, self._B
        xref = np.asarray(xref, dtype=float)
        if xref.ndim == 1:
            return np.broadcast_to(xref, (B, nx)), 1
        if xref.ndim == 3 and xref.shape[1] == 1:
            return xref.reshape(B, nx), 1                       # explicit per-instance constant references (unambiguous for any batch size)
        if xref.ndim == 3:
            if xref.shape[1] != Np + 1:
                raise ValueError("time-varying xref needs exactly Np+1 rows")   # the reference crashes here too (Q6)
            return xref.reshape(B, (Np + 1) * nx), Np + 1
        if self.batch is not None and xref.shape == (B, nx) and not xref.shape[0] == Np + 1:
            return xref, 1
        if xref.shape[0] >= Np + 1:
            if xref.shape[0] != Np + 1:
                raise ValueError("time-varying xref needs exactly Np+1 rows")
            if self.batch is not None and B == Np + 1:
                warnings.warn("xref of shape (Np+1, nx) with batch == Np+1 is read as ONE time-varying reference shared by all instances "
                              "(the reference's meaning of a 2-D xref); pass shape (batch, 1, nx) for per-instance constant references")
            return np.broadcast_to(xref.reshape(1, -1), (B, (Np + 1) * nx)), Np + 1
        raise ValueError("time-varying xref needs exactly Np+1 rows")

    def _stage(self, name, arr, shape):
        """copy into a pinned staging buffer (two per name, used alternately: the asynchronous H2D copy of the previous call may
        still be reading the other one) and return it"""
        flip = self._pin_flip[name] = 1 - self._pin_flip.get(name, 1)
        key = name if flip == 0 else name + "#1"
        arr_in = np.asarray(arr)
        for k in (name, name + "#1"):                       # the caller's own pinned buffer (pinned_buffer()): no staging copy
            pk = self._pin.get(k)
            if pk is not None and arr_in.shape == pk.array.shape and arr_in.ctypes.data == pk.array.ctypes.data:
                return pk.array
        pin = self._pin.get(key)
        if pin is None or pin.array.shape != tuple(shape):
            pin = PinnedArray(shape); self._pin[key] = pin
        arr = np.asarray(arr)
        if not (arr.shape == pin.array.shape and arr.ctypes.data == pin.array.ctypes.data):
            np.copyto(pin.array, np.broadcast_to(arr, shape))
        return pin.array

    def pinned_buffer(self, name):
        """Pinned host arrays the caller may fill in place and pass to update()/output() to avoid a staging
        copy: 'x0' [B,nx], 'uminus1' [B,nu], 'xref' [B,nx], 'u' [B,nu] (output)."""
        shapes = {"x0": (self._B, self.nx), "uminus1": (self._B, self.nu), "xref": (self._B, self.nx), "u": (self._B, self.nu)}
        if name not in self._pin:
            self._pin[name] = PinnedArray(shapes[name])
        pin = self._pin[name]
        self._pin_ptr[id(pin.array)] = pin                   # update() recognises the caller's pinned buffers by identity (no per-call ctypes work)
        return pin.array

    def _check(self, rc):
        if rc < 0:
            msg = self._L.bmpc_last_error(self._h)
            raise BmpcError(f"libbmpc error {rc}: {msg.decode() if msg else ''}")
        return rc

    # ------------------------------------------------------------------ reference API
    def setup(self, solve=True):
        """Set up the QP (condense + factor on the GPU).  mpc.py:254-269."""
        self._L = self._pick_library()
        L = self._L
        B, nx, nu = self._B, self.nx, self.nu
        self.x0_rh = np.copy(self.x0)
        self.uminus1_rh = np.copy(self.uminus1)
        if self._h is not None:
            L.bmpc_destroy(self._h); self._h = None
        self._bound_u = None
        self._out_pool = []
        cfg = BmpcConfig(); L.bmpc_default_config(cfg)
        cfg.nx, cfg.nu, cfg.Np, cfg.Nc, cfg.batch, cfg.device = nx, nu, self.Np, self.Nc, B, self.device
        cfg.soft_on = 1 if self.SOFT_ON else 0
        cfg.eps_feas = float(self.eps_feas)
        # quirk Q1: the reference hands eps_rel to OSQP as eps_abs and vice versa (mpc.py:266)
        cfg.eps_abs, cfg.eps_rel = float(self.eps_rel), float(self.eps_abs)
        if self._per_instance:
            cfg.n_sys = B
        for k, v in self.solver_options.items():
            if not hasattr(cfg, k):
                raise TypeError(f"unknown solver option {k!r}")
            setattr(cfg, k, v)
        h = ctypes.c_void_p()
        rc = L.bmpc_create(cfg, ctypes.byref(h))
        if rc < 0:
            msg = L.bmpc_last_error(None)
            raise BmpcError(f"bmpc_create failed ({rc}): {msg.decode() if msg else ''}")
        self._h = h
        sent = self._device_arrays(self._setup_arrays())
        self._check(L.bmpc_setup(self._h, *[ptr(sent[name]) for name, _, _ in self._PROBLEM]))
        self._qp_static = None
        self._um1_for_J = self.uminus1_rh
        self._push(self.x0_rh, self.uminus1_rh, self.xref)
        self._J_dirty = True
        if solve:
            self.solve()

    def _pick_library(self):
        """The in-tree build, or — for a single-input shape its fast-path table does not hold — a per-shape build made on the spot
        (pympc_b200.build.jit_shape, cached): every (nx, 1, Np, Nc) runs on the thread-per-instance kernels, like the reference
        handles every shape uniformly (mpc.py:456-615).  Falls back to the generic team kernels with a warning if that build is
        not possible (no nvcc available).  With fast_path=2 a multi-input shape missing from the in-tree table is built the same
        way (build.jit_multi_input_shape), per-instance multi-input systems included (the union of the instances' patterns)."""
        from . import build
        L = _lib.load()
        opts = self.solver_options
        wants_fast = opts.get("fast_path", 1) and not opts.get("team_threads", 0) and opts.get("polish", 1) and self.SOFT_ON and not self._per_instance
        NX, NU = (self.Np + 1) * self.nx, self.Nc * self.nu
        small = (NX + NU + (self.Nc + 1) * self.nu) <= 192 and NU <= 64          # the library's own rule for the warp-team family
        tpi_fits = small and build.tpi_shape_supported(self.nx, self.nu, self.Np, self.Nc)    # the single-input kernels hold this shape
        # per-instance systems (3-D Ad) with several inputs take the multi-input fast path too (the union of the instances' patterns)
        wants_tpm = wants_fast or (self._per_instance and self.nu > 1 and opts.get("fast_path", 1) and not opts.get("team_threads", 0)
                                   and opts.get("polish", 1) and self.SOFT_ON)
        if wants_tpm and int(opts.get("fast_path", 1)) >= 2 and not tpi_fits and build.tpm_shape_supported(self.nx, self.nu, self.Np, self.Nc) \
                and not L.bmpc_has_multi_input_fast_path(self.nx, self.nu, self.Np, self.Nc) and not os.environ.get("BMPC_NO_JIT"):
            # fast_path=2: also build the multi-input Riccati polish for this shape (and this system's sparsity pattern) on the spot
            try:
                return _lib.load(build.jit_multi_input_shape(self.nx, self.nu, self.Np, self.Nc, self.Ad, self.Bd))
            except Exception as exc:
                warnings.warn(f"building a multi-input fast path for shape (nx={self.nx}, nu={self.nu}, Np={self.Np}, Nc={self.Nc}) failed ({exc}): "
                              "running on the generic team kernels")
                return L
        if not (wants_fast and tpi_fits) or L.bmpc_has_fast_path(self.nx, self.nu, self.Np, self.Nc):
            return L                            # (a shape outside the fast path's domain runs on the team kernels)
        if os.environ.get("BMPC_NO_JIT"):
            warnings.warn(f"no compiled fast path for shape (nx={self.nx}, nu=1, Np={self.Np}, Nc={self.Nc}): running on the generic team "
                          f"kernels (about 15x slower); add it with  python -m pympc_b200.build --add-shape {self.nx},1,{self.Np},{self.Nc}")
            return L
        try:
            return _lib.load(build.jit_shape(self.nx, 1, self.Np, self.Nc))
        except Exception as exc:
            warnings.warn(f"no compiled fast path for shape (nx={self.nx}, nu=1, Np={self.Np}, Nc={self.Nc}) and building one failed ({exc}): "
                          "running on the generic team kernels (about 15x slower)")
            return L

    def _push(self, x0, um1, xref, borrow=False):
        """hand (x0, u_-1, xref) to the device.  borrow=True: x0 / u_-1 sit in pinned, device-mapped staging buffers that the
        solver kernels read IN PLACE over PCIe while they compute (no H2D copy phase) — only valid when the solve is issued and
        retired before the buffers can change, i.e. from update(..., solve=True)"""
        B, nx, nu = self._B, self.nx, self.nu
        px = pu = pr = None; rows = 1
        if borrow and xref is None and x0 is not None:
            # the per-step call of a closed loop with the caller's own pinned buffers: two dictionary look-ups, one C call
            ex = self._pin_ptr.get(id(x0)); eu = self._pin_ptr.get(id(um1)) if um1 is not None else None
            if ex is not None and ex.array is x0 and (um1 is None or (eu is not None and eu.array is um1)):
                self._check(self._L.bmpc_update(self._h, ex.ptr, eu.ptr if eu is not None else None, None, 1, 2))
                return
        if x0 is not None:
            px = ptr(self._stage("x0", np.asarray(x0, dtype=float).reshape(-1, nx) if np.ndim(x0) > 1 else np.asarray(x0, dtype=float), (B, nx)))
        if um1 is not None:
            pu = ptr(self._stage("uminus1", np.asarray(um1, dtype=float).reshape(-1, nu) if np.ndim(um1) > 1 else np.asarray(um1, dtype=float), (B, nu)))
        if xref is not None:
            arr, rows = self._xref_device_layout(xref)
            pr = ptr(self._stage("xref" if rows == 1 else "xref_tv", arr, arr.shape))
        if borrow and pr is not None:
            self._check(self._L.bmpc_update(self._h, None, None, pr, rows, 0)); pr = None      # xref is always copied
        self._check(self._L.bmpc_update(self._h, px, pu, pr, rows, 2 if borrow else 0))

    def update(self, x, u=None, xref=None, solve=True):
        """New measurement (and optionally u_{-1}, xref); re-solve warm-started.  mpc.py:338-364."""
        if self._h is None:
            raise BmpcError("update() before setup()")
        self.x0_rh = x
        if u is not None:
            self.uminus1_rh = u
        if xref is not None:
            self.xref = xref
        # u=None: the device already holds the previously output control as uminus1 (committed by output(), Q9)
        self._um1_for_J = self.uminus1_rh
        self._push(x, u, xref, borrow=bool(solve) and self._zero_copy)
        self._J_dirty = True           # J_CNST is recomputed lazily (it is O(B) host work and rarely read)
        if solve:
            self.solve()

    def update_from_device(self, x_ptr, u_ptr=None, solve=True, borrow=False):
        """update() with x (and optionally u_-1) already resident on this device, e.g. the state of a
        ``pympc_b200.kalman.LinearStateEstimator`` — no host round trip between estimator and K3.  borrow=True: the kernels read
        the buffers in place (no device-to-device copy); keep them unchanged until output() has returned."""
        if self._h is None:
            raise BmpcError("update_from_device() before setup()")
        self._check(self._L.bmpc_update(self._h, x_ptr, u_ptr, None, 1, 2 if borrow else 1))
        self._J_dirty = True
        if solve:
            self.solve()

    # the arrays of bmpc_setup / bmpc_update_problem in argument order: (name, kind, hidden flag that zeroes it on the device)
    _PROBLEM = (("Ad", "system", None), ("Bd", "system", None), ("Qx", "weight", "JX_ON"), ("QxN", "weight", "JX_ON"),
                ("Qu", "weight", "JU_ON"), ("QDu", "weight", "JDU_ON"), ("xmin", "vector", None), ("xmax", "vector", None),
                ("umin", "vector", None), ("umax", "vector", None), ("Dumin", "vector", None), ("Dumax", "vector", None),
                ("uref", "vector", None))
    # the constructor's messages
    _MSG = {"Ad": "Ad should be a square matrix of dimension (nx,nx)!", "Bd": "Bd should be a matrix of dimension (nx, nu)!",
            "Qx": "Qx should be a matrix of shape (nx, nx)!", "QxN": "QxN should be a square matrix of shape (nx, nx)!",
            "Qu": "Qu should be a square matrix of shape (nu, nu)!", "QDu": "QDu should be a square matrix of shape (nu, nu)!",
            "xmin": "xmin should be a vector of shape (nx,)!", "xmax": "xmax should be a vector of shape (nx,)!",
            "umin": "umin should be a vector of shape (nu,)!", "umax": "umax should be a vector of shape (nu,)!",
            "Dumin": "Dumin should be a vector of shape (nu,)!", "Dumax": "Dumax should be a vector of shape (nu,)!",
            "uref": "uref should be a vector of shape (nu,)!"}

    def _problem_shape(self, name):
        nx, nu = self.nx, self.nu
        return {"Ad": (nx, nx), "Bd": (nx, nu), "Qx": (nx, nx), "QxN": (nx, nx), "Qu": (nu, nu), "QDu": (nu, nu)}.get(
            name, (nx,) if name in ("xmin", "xmax") else (nu,))

    def _setup_arrays(self):
        """the 13 arrays setup() hands the library, by name: the attributes; per-instance controllers take an array given with a
        leading batch dimension (at construction or by update_system) over the attribute, which then holds instance 0's"""
        arrays = {name: getattr(self, name) for name, _, _ in self._PROBLEM}
        if self._per_instance:
            for name, _, _ in self._PROBLEM:
                full = self._sys_full.get(name)
                if full is not None and np.ndim(full) == len(self._problem_shape(name)) + 1:
                    arrays[name] = full
        return arrays

    def _device_arrays(self, arrays):
        """{name: array} of bmpc_setup / bmpc_update_problem -> the arrays the library receives: float64 and C-contiguous, a weight
        whose JX_ON / JU_ON / JDU_ON is off as zeros, and on per-instance controllers with a leading batch dimension (an array given
        once is broadcast to every instance).  Records the weights sent: _Qx_d ... _QDu_d (instance 0's; the reference-form QP)
        and on per-instance controllers every instance's in _w_full (J_CNST)."""
        B, per = self._B, self._per_instance
        sent = {}
        for name, kind, flag in self._PROBLEM:
            if name not in arrays:
                continue
            M = _dense(arrays[name])
            if flag is not None and not getattr(self, flag):
                M = np.zeros(M.shape)
            sent[name] = np.ascontiguousarray(np.broadcast_to(M, (B,) + self._problem_shape(name))) if per else M
            if kind == "weight":
                setattr(self, "_" + name + "_d", sent[name][0] if per else sent[name])
                if per:
                    self._w_full[name] = sent[name]
        return sent

    def update_system(self, Ad=None, Bd=None, *, Qx=None, QxN=None, Qu=None, QDu=None, xmin=None, xmax=None, umin=None, umax=None,
                      Dumin=None, Dumax=None, uref=None):
        """Time-varying problem data (successive linearisation, gain scheduling, derated actuator limits, tightened constraints):
        replace any of the system matrices, weights, bounds and uref of the set-up controller without a new setup().  The next
        update() is a WARM solve of the QP the reference would assemble with the new arrays (working sets, ADMM state, the committed
        u_{-1} and the rho the setup chose are kept; eps_feas, SOFT_ON, the horizons and the solver options stay as set up).

        Shared controller: Ad (nx, nx), Bd (nx, nu), weights (n, n), bounds and uref vectors (n,) as the constructor takes them.
        Per-instance controller: the same, or with a leading batch dimension — (batch, n, n) matrices, (batch, n) vectors — for one
        set per instance.  Matrices dense or scipy.sparse.  None keeps an array.  JX_ON / JU_ON / JDU_ON zero the weights sent to
        the device as in setup().  The reference-form attributes (Ad, ..., uref, P, q, A, l, u, J_CNST) and u_failure follow;
        assigning ``K.xmin = ...`` directly keeps the reference's meaning: no effect until setup()."""
        per = self._per_instance
        vals = dict(Ad=Ad, Bd=Bd, Qx=Qx, QxN=QxN, Qu=Qu, QDu=QDu, xmin=xmin, xmax=xmax, umin=umin, umax=umax, Dumin=Dumin, Dumax=Dumax,
                    uref=uref)
        given = {name: self._problem_arg(vals[name], name) for name, _, _ in self._PROBLEM if vals[name] is not None}
        if self._h is None:
            raise BmpcError("update_system() before setup()")
        if not given:
            return
        sent = self._device_arrays(given)
        args = [ptr(sent[name]) if name in sent else None for name, _, _ in self._PROBLEM]
        if set(given) <= {"Ad", "Bd"}:
            rc = self._L.bmpc_update_system(self._h, args[0], args[1], 0)
        else:
            rc = self._L.bmpc_update_problem(self._h, *args, 0)
        # the handle holds the new arrays even when the check fails (then solve() raises until a valid update): so do the attributes
        for name, kind, flag in self._PROBLEM:
            if name not in given:
                continue
            M = given[name]
            full = M.ndim == len(self._problem_shape(name)) + 1
            if per:
                self._sys_full[name] = M
            if kind == "weight":
                setattr(self, name, M[0] if full else (vals[name] if hasattr(vals[name], "toarray") else M))   # (sparse stays sparse, Q16)
            else:
                setattr(self, name, M[0] if full else M)
            if name == "uref":
                self.u_failure = M                          # what an instance that fails outputs (per instance when given so)
        self._qp_static = None
        self._J_dirty = True
        self._check(rc)

    def _problem_arg(self, val, name):
        """validated copy (the caller may reuse its buffer) of one array of update_system: the constructor's acceptance rule and
        message, plus a leading batch dimension on per-instance controllers"""
        shape, B = self._problem_shape(name), self._B
        M = np.array(val.toarray() if hasattr(val, "toarray") else val, dtype=float)
        # a leading batch dimension: 3-D matrices; (batch, n) vectors (a (1, n) array is a vector in the reference's sense)
        batched = M.ndim == 3 if len(shape) == 2 else (M.ndim == 2 and M.shape == (B, shape[0]) and B > 1)
        if batched and not self._per_instance:
            raise ValueError(f"per-instance {name} of shape (batch, ...) needs a controller set up with per-instance systems "
                             "(Ad of shape (batch, nx, nx) at construction)")
        if len(shape) == 2:
            if M.shape not in (shape, (B,) + shape):
                raise ValueError(self._MSG[name])
            return M
        if batched and M.shape == (B,) + shape:
            return M
        if __is_vector__(M) and M.size == shape[0]:
            return M.ravel()
        raise ValueError(self._MSG[name])

    def update_system_from_device(self, Ad_ptr=None, Bd_ptr=None, *, Qx=None, QxN=None, Qu=None, QDu=None, xmin=None, xmax=None,
                                  umin=None, umax=None, Dumin=None, Dumax=None, uref=None):
        """update_system() with the arrays already on this controller's device (raw pointers, or contiguous float64 torch tensors),
        e.g. a batch of linearisations or of derated limits computed by torch: no host round trip.  Per-instance controllers take
        (batch, ...) arrays — (batch, nx, nx), (batch, nx, nu), (batch, n, n) weights, (batch, n) bounds and uref —, shared ones the
        unbatched shapes.  The library reads them in stream order on the controller's stream: whatever wrote them must be ordered
        before (same stream, or synchronised); keep them unchanged until the next solve has been retired.  New weights are condensed
        and checked at once (their definiteness is not known on the host).  With JX_ON / JU_ON / JDU_ON off the weights sent are
        zeros, as in setup().  The host-side attributes (Ad, ..., uref, P, q, A, l, u, J_CNST, u_failure) keep describing the last
        host-side arrays."""
        if self._h is None:
            raise BmpcError("update_system_from_device() before setup()")
        n = self._B if self._per_instance else 1
        vals = dict(Ad=Ad_ptr, Bd=Bd_ptr, Qx=Qx, QxN=QxN, Qu=Qu, QDu=QDu, xmin=xmin, xmax=xmax, umin=umin, umax=umax, Dumin=Dumin,
                    Dumax=Dumax, uref=uref)

        def dev_ptr(M, name, flag):
            if M is None or isinstance(M, int):
                return M
            shape = self._problem_shape(name)
            ok = ((n,) + shape,) if n > 1 else (shape, (1,) + shape)
            if tuple(M.shape) not in ok or not M.is_contiguous() or str(M.dtype) != "torch.float64" or not M.is_cuda \
                    or M.device.index != self.device:
                raise ValueError(f"{name} must be a contiguous float64 CUDA tensor of shape {ok[0]}")
            if flag is not None and not getattr(self, flag):
                # the weight is off: zeros go to the device (a buffer the controller keeps, so it outlives the stream-ordered read)
                zeros = self.__dict__.setdefault("_dev_zeros", {})
                if name not in zeros:
                    import torch
                    zeros[name] = torch.zeros(ok[0], dtype=torch.float64, device=M.device)
                return zeros[name].data_ptr()
            return M.data_ptr()
        args = [dev_ptr(vals[name], name, flag) for name, _, flag in self._PROBLEM]
        if all(a is None for a in args[2:]):
            self._check(self._L.bmpc_update_system(self._h, args[0], args[1], 1))
        else:
            self._check(self._L.bmpc_update_problem(self._h, *args, 1))

    def solve(self):
        """Solve the QP batch.  mpc.py:366-375."""
        B, nu = self._B, self.nu
        u = self._next_result_array() if (self._zero_copy and not self._external_output) else None
        self._u0_pooled = u is not None
        if u is None:
            u = self._pin.get("u") or self._pin.setdefault("u", PinnedArray((B, nu)))
        st = self._pin.get("status") or self._pin.setdefault("status", PinnedArray((B,), np.int32))
        if self._zero_copy and not self._external_output and self._bound_u != u.ptr.value:
            # the solver epilogue stores u* straight into a pinned (device-mapped) result array: no D2H copy after the solve — and, with a
            # small pool of such arrays, none on the host either: output() hands the array itself to the caller
            self._check(self._L.bmpc_bind_output(self._h, u.ptr)); self._bound_u = u.ptr.value
        self._check(self._L.bmpc_solve(self._h))
        self._check(self._L.bmpc_output(self._h, u.ptr, st.ptr, 0, 0))
        self._u0, self._status = u.array, st.array
        self._make_res()
        # only instances that were never KKT-verified or were certified infeasible can carry a negative status: skip the
        # scan of the status array when the solve reports none of either
        s = self._stats_buf
        self._check(self._L.bmpc_get_stats(self._h, self._stats_ref))
        if (s.unsolved != 0 or s.infeasible != 0) and np.any(self._status < 0):
            warnings.warn('OSQP did not solve the problem!')
            if self.raise_error:
                raise ValueError('OSQP did not solve the problem!')

    def _make_res(self):
        # the reference reads res.info.status / res.info.obj_val (mpc.py:301-327,372); built lazily: nothing is derived from
        # the status array until somebody looks
        self._solve_id = getattr(self, "_solve_id", 0) + 1
        self.res = _Res(_ResInfo(self._status, self.batch is None, self._B, self, self._solve_id), self, self._solve_id)

    def _res_fetch(self, what, solve_id):
        """lazy part of `res`: device -> host on first access (bmpc_get_sequences); only the latest solve is on the device"""
        if solve_id != self._solve_id:
            raise BmpcError("this `res` belongs to an earlier solve: its lazily fetched fields are no longer on the device")
        B, nx, nu, Np, Nc = self._B, self.nx, self.nu, self.Np, self.Nc
        if what == "iter":
            it = np.empty(B, np.int32)
            self._check(self._L.bmpc_get_sequences(self._h, None, None, None, None, ptr(it)))
            return it
        if what == "obj_val":
            obj = np.empty(B)
            self._check(self._L.bmpc_get_sequences(self._h, None, None, None, ptr(obj), None))
            return obj
        useq = np.empty((B, Nc * nu)); xseq = np.empty((B, (Np + 1) * nx)); eseq = np.empty((B, (Np + 1) * nx))
        self._check(self._L.bmpc_get_sequences(self._h, ptr(useq), ptr(xseq), ptr(eseq), None, None))
        return np.hstack([xseq, useq, eseq] if self.SOFT_ON else [xseq, useq])

    def output(self, return_x_seq=False, return_u_seq=False, return_eps_seq=False, return_status=False, return_obj_val=False):
        """First optimal input (and optional info); commits it as the next u_{-1}.  mpc.py:271-336."""
        if self._u0 is None:
            raise BmpcError("output() before a solve")
        B, nx, nu, Np, Nc = self._B, self.nx, self.nu, self.Np, self.Nc
        # failed instances already carry u_failure = uref (written by the device epilogue, mpc.py:303-304)
        uMPC = self._u0 if self._u0_pooled else self._fresh_output()
        info = {}
        if return_x_seq or return_u_seq or return_eps_seq or return_obj_val:
            useq = np.empty((B, Nc * nu)) if return_u_seq else None
            xseq = np.empty((B, (Np + 1) * nx)) if return_x_seq else None
            eseq = np.empty((B, (Np + 1) * nx)) if return_eps_seq else None
            obj = np.empty(B) if return_obj_val else None
            self._check(self._L.bmpc_get_sequences(self._h, ptr(useq), ptr(xseq), ptr(eseq), ptr(obj), None))
            if return_x_seq:
                info['x_seq'] = xseq.reshape(B, -1, nx) if self.batch is not None else xseq.reshape(-1, nx)
            if return_u_seq:
                info['u_seq'] = useq.reshape(B, -1, nu) if self.batch is not None else useq.reshape(-1, nu)
            if return_eps_seq:
                info['eps_seq'] = eseq.reshape(B, -1, nx) if self.batch is not None else eseq.reshape(-1, nx)
            if return_obj_val:
                val = obj + self.J_CNST
                info['obj_val'] = val if self.batch is not None else float(val[0])
        if return_status:
            if self.batch is None:
                info['status'] = self.res.info.status
            else:
                info['status'] = np.array([_STATUS_STR.get(int(s), "unsolved") for s in self._status])
        # side effect of the reference: uminus1_rh = uMPC (mpc.py:330) — committed on the device as well
        self._check(self._L.bmpc_output(self._h, None, None, 1, 0))
        if self.batch is None:
            uMPC = uMPC[0]
        self.uminus1_rh = uMPC
        if len(info) == 0:
            return uMPC
        return uMPC, info

    def _next_result_array(self):
        """a pinned result array nobody outside holds any more (the caller dropped what output() gave it two steps ago; the current
        result and uminus1_rh are references too), or a new one while the pool is small; None: fall back to one array + a copy"""
        import sys
        for pin in self._out_pins:
            if sys.getrefcount(pin.array) <= 2:                  # pin.array + getrefcount's argument
                return pin
        if len(self._out_pins) < 6:
            pin = PinnedArray((self._B, self.nu)); self._out_pins.append(pin)
            return pin
        return None

    def _fresh_output(self):
        """a copy of the result the caller owns, like the reference returns a new array every call — but without paying an
        mmap + page faults per call for a 0.5 MB batch: arrays handed out earlier are reused once NOBODY references them any
        more (the caller dropped them), which sys.getrefcount tells"""
        import sys
        pool = self._out_pool
        for i in range(len(pool)):
            a = pool[i]
            if a is not self.uminus1_rh and sys.getrefcount(a) <= 3 and a.shape == self._u0.shape:      # pool + local name + getrefcount's argument
                np.copyto(a, self._u0)
                return a
        a = self._u0.copy()
        if a.nbytes >= (64 << 10) and len(pool) < 8:
            pool.append(a)
        return a

    def __controller_function__(self, x, u, xref=None):
        """Debug helper of the reference (mpc.py:377-384)."""
        self.update(x, u, xref=xref, solve=True)
        return self.output()

    # ------------------------------------------------------------------ extras
    @property
    def J_CNST(self):
        """Constant term of the cost (mpc.py:412-442), evaluated on demand."""
        if self._J_dirty and self.uminus1_rh is not None:
            self._compute_J_CNST()
            self._J_dirty = False
        return self._J_CNST

    @J_CNST.setter
    def J_CNST(self, value):
        self._J_CNST = value
        self._J_dirty = False

    def _compute_J_CNST(self):
        """Constant of the cost exactly as the reference accumulates it (mpc.py:412-442; quirk Q7).  Per-instance controllers: each
        instance with its own weights and uref."""
        B, Np, nu = self._B, self.Np, self.nu
        J = np.zeros(B)
        um1 = np.broadcast_to(np.asarray(self._um1_for_J, dtype=float).reshape(-1, nu), (B, nu))
        if self._per_instance:
            W = self._w_full
            Qx, QxN, Qu, QDu = W["Qx"], W["QxN"], W["Qu"], W["QDu"]
            uref = self._sys_full.get("uref")
            uref = np.broadcast_to(np.asarray(self.uref if uref is None else uref, dtype=float).reshape(-1, nu), (B, nu))
            quad = lambda sub, a, Q, b: np.einsum(sub.replace("ij", "bij"), a, Q, b)
        else:
            Qx, QxN, Qu, QDu = self._Qx_d, self._QxN_d, self._Qu_d, self._QDu_d
            uref = self.uref
            quad = np.einsum
        if self.JX_ON and self.COMPUTE_J_CNST:
            arr, rows = self._xref_device_layout(self.xref)
            if rows == 1:
                xr = np.asarray(arr)
                J += 0.5 * Np * quad('bi,ij,bj->b', xr, QxN, xr) + 0.5 * quad('bi,ij,bj->b', xr, QxN, xr)
            else:
                xr = np.asarray(arr).reshape(B, Np + 1, self.nx)
                J += 0.5 * quad('bki,ij,bkj->b', xr[:, :Np], Qx, xr[:, :Np]) + 0.5 * quad('bi,ij,bj->b', xr[:, Np], QxN, xr[:, Np])
        if self.JU_ON:
            J += 0.5 * Np * (quad('bi,ij,bj->b', uref, Qu, uref) if self._per_instance else uref @ (Qu @ uref))
        if self.JDU_ON:
            J += 0.5 * quad('bi,ij,bj->b', um1, QDu, um1)
        self._J_CNST = J if self.batch is not None else float(J[0])

    # ---- reference-form QP attributes (mpc.py:597-606), built lazily on the host for instance 0 ----
    def _qp_view(self):
        from . import qp_view
        first = lambda a, nd: np.asarray(a, dtype=float)[0] if np.ndim(a) == nd + 1 else np.asarray(a, dtype=float)
        if getattr(self, "_qp_static", None) is None:
            z = np.zeros
            Qx = self._Qx_d; QxN = self._QxN_d; Qu = self._Qu_d; QDu = self._QDu_d
            self._qp_static = qp_view.assemble(np.asarray(self.Ad, float), np.asarray(self.Bd, float), self.Np, self.Nc, Qx, QxN, Qu, QDu,
                                               self.xmin, self.xmax, self.umin, self.umax, self.Dumin, self.Dumax,
                                               float(self.eps_feas), self.uref, bool(self.SOFT_ON))
        P, A, n, w = self._qp_static
        x0 = first(self.x0_rh, 1); um1 = first(self.uminus1_rh, 1)
        xr = np.asarray(self.xref, dtype=float)
        if self.batch is not None and (xr.ndim == 3 or (xr.ndim == 2 and xr.shape == (self._B, self.nx) and xr.shape[0] != self.Np + 1)):
            xr = xr[0]
        q, l, u = qp_view.vectors(self.Np, self.Nc, self.nx, self.nu, self._Qx_d, self._QxN_d, self._Qu_d, self._QDu_d, w, self.xmin,
                                  self.xmax, self.umin, self.umax, self.Dumin, self.Dumax, self.uref, x0, um1, xr, bool(self.SOFT_ON))
        return P, q, A, l, u

    P = property(lambda self: self._qp_view()[0])
    q = property(lambda self: self._qp_view()[1])
    A = property(lambda self: self._qp_view()[2])
    l = property(lambda self: self._qp_view()[3])
    u = property(lambda self: self._qp_view()[4])

    def stats(self):
        """Counters of the last solve (ADMM iterations, rounds, device time of the kernels)."""
        s = BmpcStats()
        self._check(self._L.bmpc_get_stats(self._h, ctypes.byref(s)))
        return {f: getattr(s, f) for f, _ in BmpcStats._fields_}

    def iterations(self):
        it = np.empty(self._B, np.int32)
        self._check(self._L.bmpc_get_sequences(self._h, None, None, None, None, ptr(it)))
        return it

    def condensed(self, name):
        """Export one array of the condensed system computed on the device (parity tests)."""
        dims = np.zeros(8, np.int32); self._L.bmpc_get_dims(self._h, ptr(dims))
        nx, nu, Np, Nc, NX, NU, mc, _ = [int(v) for v in dims]
        shapes = {"Bcal": (NX, NU), "Acal": (NX, nx), "H": (NU, NU), "Hinv": (NU, NU), "K": (NU, NU), "Kinv": (NU, NU),
                  "M": (mc, mc), "AHinv": (mc, NU), "Gx0": (NU, nx), "Gref": (NU, nx), "g0": (NU,), "lo0": (mc,),
                  "hi0": (mc,), "rho": (mc,), "scal": (8,)}
        out = np.empty(shapes[name])
        self._check(self._L.bmpc_get_sys(self._h, name.encode(), ptr(out), out.size))
        return out

    @property
    def handle(self):
        return self._h

    def close(self):
        if getattr(self, "_h", None) is not None:
            self._L.bmpc_destroy(self._h); self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
