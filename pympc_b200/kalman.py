"""Kalman design and the batched ``LinearStateEstimator`` on the GPU — the input side of the MPC path (SURVEY.md §8f-4).

Mirrors ``/root/reference/pyMPC/kalman.py``:

* ``dare`` replaces the ``control.dare`` calls of the reference (kalman.py:67, 96); ``kalman_design`` (kalman.py:24-70) and
  ``kalman_design_simple`` (kalman.py:73-106) follow the reference's formulas on top of it.  The Riccati equations are solved on
  the device (``bmpc_dare``: structured doubling, one warp per instance), a whole fleet of per-instance systems in one call.
* ``LinearStateEstimator`` (kalman.py:109-152) for a batch of B estimators that share (A, B, C, D, L) or carry one system per
  instance: ``predict(u)`` does ``x <- A x + B u; y <- C x`` (kalman.py:126-129) and ``update(y_meas)`` does
  ``x <- x + L (y_meas - y)`` (kalman.py:131-133, ``y`` is not refreshed — as in the reference).  The state stays on the device;
  ``device_state()`` feeds ``MPCController.update_from_device``.
* ``KalmanFilter``: the same estimator with the gain computed every step by the Kalman filter's covariance recursion
  (``predict``: ``P <- A P A' + Qn``; ``update``: ``K = P C' (C P C' + Rn)^-1``, Joseph-form ``P``), for models that change between
  steps.  With a constant model it settles on ``kalman_design_simple(..., type='filter')``'s gain.
* ``update_system`` / ``update_system_from_device`` replace the matrices of either estimator between steps, as assigning the
  reference's ``A``, ``B``, ``C`` attributes does (kalman.py:126-133).

Batching follows ``MPCController``: a 2-D array is shared by every instance, a 3-D array carries a leading batch dimension.
"""
import ctypes

import numpy as np

from . import _lib
from ._lib import BmpcError, ptr


_DARE_STATUS = {-1: "no stabilising solution", -2: "R not positive definite"}
_T = lambda a: np.swapaxes(a, -1, -2)


def _arrays(names, arrays):
    """float arrays of 2 or 3 dimensions and the common leading batch size of the 3-D ones (None when all are 2-D)"""
    out, sizes = [], set()
    for name, a in zip(names, arrays):
        a = np.asarray(a, float)
        if a.ndim not in (2, 3):
            raise ValueError(f"{name} should be a matrix (2-D) or a batch of matrices (3-D), got shape {a.shape}")
        if a.ndim == 3:
            sizes.add(a.shape[0])
        out.append(a)
    if len(sizes) > 1:
        raise ValueError(f"batched arrays disagree on the batch size: {sorted(sizes)}")
    return out, (sizes.pop() if sizes else None)


def dare(A, B, Q, R, S=None, E=None, return_status=False, device=0):
    """Stabilising solution of the discrete algebraic Riccati equation, python-control's ``dare(A, B, Q, R, S, E)`` with E = I:

        X = A'XA - (A'XB + S)(R + B'XB)^-1 (B'XA + S') + Q,      G = (R + B'XB)^-1 (B'XA + S')

    Returns ``(X, L, G)`` in python-control's order, L the closed-loop eigenvalues eig(A - B G).  Any argument may carry a
    leading batch dimension (one system per instance); all instances are solved in one call on the GPU (1 <= n, m <= 32).
    An instance without a stabilising solution, or with R not positive definite, raises ``numpy.linalg.LinAlgError``;
    with ``return_status=True`` the per-instance status (1 solved, -1 no stabilising solution, -2 R not positive definite)
    is returned as a fourth element instead, and the failed instances hold NaN in X, G and L."""
    names = ("A", "B", "Q", "R") + (() if S is None else ("S",))
    arrs, batch = _arrays(names, (A, B, Q, R) + (() if S is None else (S,)))
    A, B, Q, R = arrs[:4]; S = arrs[4] if S is not None else None
    n, m = A.shape[-1], B.shape[-1]
    want = {"A": (n, n), "B": (n, m), "Q": (n, n), "R": (m, m), "S": (n, m)}
    for name, a in zip(names, arrs):
        if a.shape[-2:] != want[name]:
            raise ValueError(f"{name} should have shape {want[name]} (n = {n} states, m = {m} inputs), got {a.shape[-2:]}")
    if not (1 <= n <= 32 and 1 <= m <= 32):
        raise ValueError(f"dare supports 1 <= n, m <= 32 (got n = {n}, m = {m})")
    if E is not None:
        E = np.asarray(E, float)
        if E.shape[-2:] != (n, n) or not np.array_equal(E, np.broadcast_to(np.eye(n), E.shape)):
            raise ValueError("dare: only E = I (or None) is supported")
    nb = 1 if batch is None else batch
    full = lambda a: np.ascontiguousarray(np.broadcast_to(a, (nb,) + a.shape[-2:]))
    A, B, Q, R = full(A), full(B), full(Q), full(R)
    S = None if S is None else full(S)
    L = _lib.load()
    X = np.empty((nb, n, n)); G = np.empty((nb, m, n)); st = np.empty(nb, np.int32); it = np.empty(nb, np.int32)
    rc = L.bmpc_dare(n, m, nb, int(device), ptr(A), ptr(B), ptr(Q), ptr(R), ptr(S), ptr(X), ptr(G), ptr(st), ptr(it))
    if rc < 0:
        raise BmpcError(f"bmpc_dare failed ({rc}): {L.bmpc_last_error(None).decode()}")
    ok = st == 1
    W = np.full((nb, n), np.nan, complex)
    if ok.any():
        W[ok] = np.linalg.eigvals(A[ok] - B[ok] @ G[ok])
    if not ok.all() and not return_status:
        bad = np.flatnonzero(~ok)[:8]
        raise np.linalg.LinAlgError("dare: " + ", ".join(f"instance {b}: {_DARE_STATUS.get(int(st[b]), st[b])} (status {st[b]})"
                                                         for b in bad) + (" ..." if (~ok).sum() > len(bad) else ""))
    out = (X, W, G) if batch is not None else (X[0], W[0], G[0])
    return out + ((st if batch is not None else st[:1]),) if return_status else out


def kalman_design(A, B, C, D, Qn, Rn, Nn=None, return_status=False, device=0):
    """General Kalman design (kalman.py:24-70) for x+ = A x + B [u; w], y = C x + D [u; w] + v with E[ww'] = Qn, E[vv'] = Rn,
    E[wv'] = Nn: the last nw = Qn.shape[0] columns of B and D carry the noise w.  Returns ``(L, P, W)``: gain, Riccati
    solution and closed-loop eigenvalues.  Batched like ``dare``."""
    (A, B, C, D, Qn, Rn), _ = _arrays(("A", "B", "C", "D", "Qn", "Rn"), (A, B, C, D, Qn, Rn))
    nw = Qn.shape[-1]; nu = B.shape[-1] - nw; ny = C.shape[-2]
    if nu < 0 or D.shape[-1] != B.shape[-1] or D.shape[-2] != ny or Rn.shape[-2:] != (ny, ny):
        raise ValueError("kalman_design: B [nx, nu + nw] and D [ny, nu + nw] must hold the nw = Qn.shape[0] noise inputs last, "
                         "and Rn must be [ny, ny]")
    Nn = np.zeros((nw, ny)) if Nn is None else _arrays(("Nn",), (Nn,))[0][0]
    Bw, Dw = B[..., nu:], D[..., nu:]
    Hn = Dw @ Nn                                                   # kalman.py:58
    Rb = Rn + Hn + _T(Hn) + Dw @ Qn @ _T(Dw)                       # kalman.py:59
    Qb = Bw @ Qn @ _T(Bw)                                          # kalman.py:60
    Nb = Bw @ (Qn @ _T(Dw) + Nn)                                   # kalman.py:61
    Qb = (Qb + _T(Qb)) / 2; Rb = (Rb + _T(Rb)) / 2                 # kalman.py:64-65
    res = dare(_T(A), _T(C), Qb, Rb, Nb, return_status=return_status, device=device)      # kalman.py:67
    P, W, K = res[:3]
    return (_T(K), P, W) + tuple(res[3:])                          # kalman.py:69-70


def kalman_design_simple(A, B, C, D, Qn, Rn, type='filter', return_status=False, device=0):
    """Simplified Kalman design (kalman.py:73-106) for x+ = A x + B u + w, y = C x + D u + v with E[ww'] = Qn, E[vv'] = Rn:
    ``type='filter'`` gives L = P C' (C P C' + Rn)^-1, ``'predictor'`` L = A P C' (C P C' + Rn)^-1.  Returns ``(L, P, W)``.
    B and D are not used (as in the reference).  Batched like ``dare``."""
    if type not in ('filter', 'predictor'):
        raise ValueError("Unknown Kalman design type. Specify either filter or predictor!")
    (A, C, Qn, Rn), _ = _arrays(("A", "C", "Qn", "Rn"), (A, C, Qn, Rn))
    res = dare(_T(A), _T(C), Qn, Rn, return_status=return_status, device=device)          # kalman.py:96
    P, W = res[0], res[1]
    with np.errstate(invalid="ignore"):
        PCt = P @ _T(C)
        Sinv = np.linalg.inv(C @ PCt + Rn)
        L = PCt @ Sinv if type == 'filter' else A @ PCt @ Sinv                           # kalman.py:99-102
    return (L, P, W) + tuple(res[3:])


class _DeviceEstimator:
    """What both estimators share: the state on the device (bmpc_est_*), predict / update, the on-device chain, model updates."""

    def _shape(self, a, n):
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(a, float).reshape(-1, n), (self._B, n)))
        return a

    def _out(self, a):
        return a if self.batch is not None else a[0]

    @property
    def x(self):
        x = np.empty((self._B, self.nx)); self._L.bmpc_est_get(self._h, ptr(x), None); return self._out(x)

    @property
    def y(self):
        y = np.empty((self._B, self.ny)); self._L.bmpc_est_get(self._h, None, ptr(y)); return self._out(y)

    def out_y(self, u):
        return self.y

    def predict(self, u):
        rc = self._L.bmpc_est_predict(self._h, ptr(self._shape(u, self.nu)), 0)
        if rc < 0:
            raise BmpcError("bmpc_est_predict failed")
        return self.x

    def update(self, y_meas):
        rc = self._L.bmpc_est_update(self._h, ptr(self._shape(y_meas, self.ny)), 0)
        if rc < 0:
            raise BmpcError("bmpc_est_update failed")
        return self.x

    def predict_device(self, u_ptr):
        """u already on the device (e.g. the MPC output buffer): no host traffic."""
        return self._L.bmpc_est_predict(self._h, u_ptr, 1)

    def update_device(self, y_ptr):
        return self._L.bmpc_est_update(self._h, y_ptr, 1)

    def attach(self, controller):
        """Chain this estimator with an MPCController on the device (estimate -> update_from_device -> u0 -> predict_device)
        without host reads in between: both run on the controller's stream, and the controller's deferred solve is retired before
        its output buffer is consumed.  `None` detaches."""
        rc = self._L.bmpc_est_attach(self._h, controller.handle if controller is not None else None)
        if rc < 0:
            raise BmpcError("bmpc_est_attach failed (controller on another device?)")

    def device_state(self):
        """Device pointer (int) of x [B, nx], usable as bmpc_update(x0=..., on_device=1)."""
        return self._L.bmpc_est_state_ptr(self._h)

    def _model_shape(self, name):
        nx, nu, ny = self.nx, self.nu, self.ny
        return {"A": (nx, nx), "B": (nx, nu), "C": (ny, nx), "L": (nx, ny), "Qn": (nx, nx), "Rn": (ny, ny)}[name]

    def _set_model(self, vals, on_device):
        args = [vals.get(name) for name in ("A", "B", "C", "L", "Qn", "Rn")]
        rc = self._L.bmpc_est_set_model(self._h, *args, on_device)
        if rc < 0:
            raise BmpcError(f"bmpc_est_set_model failed ({rc})")

    def _update_system(self, **vals):
        """update_system: host arrays, validated like the constructor; 2-D (every instance) or, for an estimator with one model
        per instance, 3-D (batch, ...).  Takes effect from the next predict (A, B, Qn) or update (C, L, Rn); y is not recomputed."""
        given = {}
        for name, a in vals.items():
            if a is None:
                continue
            shape = self._model_shape(name)
            M = np.array(a.toarray() if hasattr(a, "toarray") else a, dtype=float)
            if M.ndim == 3 and not self._per:
                raise ValueError(f"{name}: this estimator was created with one shared model and takes {shape} matrices only")
            if M.shape not in (shape, (self._B,) + shape):
                raise ValueError(f"{name} should have shape {shape}" + (f" or {(self._B,) + shape}" if self._per else "") +
                                 f", got {M.shape}")
            if name in ("Qn", "Rn"):
                M = (M + _T(M)) / 2
            given[name] = M
        if not given:
            return
        n = self._B if self._per else 1
        sent = {name: np.ascontiguousarray(np.broadcast_to(M, (n,) + M.shape[-2:])) for name, M in given.items()}
        self._set_model({name: ptr(M) for name, M in sent.items()}, 0)
        self._sent = sent                                   # host buffers of stream-ordered copies: kept until the next update
        for name, M in given.items():
            setattr(self, name, sent[name] if self._per else M)

    def _update_system_from_device(self, **vals):
        """update_system_from_device: raw device pointers (int) or contiguous float64 CUDA tensors on the estimator's device, of
        shape (batch, ...) for one model per instance, (...) or (1, ...) for a shared model.  Read in stream order on the
        estimator's stream (the controller's once attached): whatever wrote them must be ordered before.  The host-side attributes
        keep describing the last host arrays."""
        n = self._B if self._per else 1
        args = {}
        for name, M in vals.items():
            if M is None or isinstance(M, int):
                args[name] = M
                continue
            shape = self._model_shape(name)
            ok = ((n,) + shape,) if self._per else (shape, (1,) + shape)
            if tuple(M.shape) not in ok or not M.is_contiguous() or str(M.dtype) != "torch.float64" or not M.is_cuda \
                    or M.device.index != self.device:
                raise ValueError(f"{name} must be a contiguous float64 CUDA tensor of shape {ok[0]}")
            args[name] = M.data_ptr()
        if any(a is not None for a in args.values()):
            self._set_model(args, 1)

    def close(self):
        if getattr(self, "_h", None):
            self._L.bmpc_est_destroy(self._h); self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class LinearStateEstimator(_DeviceEstimator):
    def __init__(self, x0, A, B, C, D, L, batch=None, device=0):
        """Any of A, B, C, L may carry a leading batch dimension (one system per instance); `batch` then defaults to it."""
        self._L = _lib.load()
        self._per = any(np.ndim(a) == 3 for a in (A, B, C, L))
        if not self._per:
            A = np.ascontiguousarray(A, float); B = np.ascontiguousarray(B, float).reshape(A.shape[0], -1)
            C = np.ascontiguousarray(C, float).reshape(-1, A.shape[0]); Lg = np.ascontiguousarray(L, float).reshape(A.shape[0], -1)
        else:
            (A, B, C, Lg), nb = _arrays(("A", "B", "C", "L"), (A, B, C, L))
            if batch is None:
                batch = nb
            elif int(batch) != nb:
                raise ValueError(f"batch = {batch} but the per-instance matrices carry {nb} systems")
            full = lambda a: np.ascontiguousarray(np.broadcast_to(a, (nb,) + a.shape[-2:]))
            A, B, C, Lg = full(A), full(B), full(C), full(Lg)
        self.A, self.B, self.C, self.D, self.L = A, B, C, np.asarray(D, float), Lg
        self.nx, self.nu, self.ny = A.shape[-1], B.shape[-1], C.shape[-2]
        if B.shape[-2] != self.nx or C.shape[-1] != self.nx or Lg.shape[-2:] != (self.nx, self.ny):
            raise ValueError("LinearStateEstimator: A [nx, nx], B [nx, nu], C [ny, nx] and L [nx, ny] do not agree")
        self.batch = batch
        self._B = 1 if batch is None else int(batch)
        self.device = int(device)
        x0 = np.ascontiguousarray(np.broadcast_to(np.asarray(x0, float).reshape(-1, self.nx), (self._B, self.nx)))
        h = ctypes.c_void_p()
        if not self._per:
            rc = self._L.bmpc_est_create(self.nx, self.nu, self.ny, self._B, int(device), ptr(A), ptr(B), ptr(C), ptr(Lg), ptr(x0),
                                         ctypes.byref(h))
        else:
            rc = self._L.bmpc_est_create_ex(self.nx, self.nu, self.ny, self._B, self._B, int(device), ptr(A), ptr(B), ptr(C),
                                            ptr(Lg), ptr(x0), ctypes.byref(h))
        if rc < 0:
            raise BmpcError(f"bmpc_est_create failed ({rc}): {self._L.bmpc_last_error(None).decode()}")
        self._h = h

    def update_system(self, A=None, B=None, C=None, L=None):
        """Replace any of (A, B, C, L) between steps, as assigning the reference's attributes does: A and B act from the next
        predict, C and L from the next update; y is not recomputed.  2-D matrices, or (batch, ...) on an estimator created with one
        system per instance."""
        self._update_system(A=A, B=B, C=C, L=L)

    def update_system_from_device(self, A=None, B=None, C=None, L=None):
        """update_system with device arrays: raw pointers or contiguous float64 CUDA tensors (batch, ...) per instance, (...) shared;
        read in stream order on the estimator's stream, no host round trip."""
        self._update_system_from_device(A=A, B=B, C=C, L=L)

    def sim(self, u_seq, x=None):
        """Open-loop output prediction on the host, as the reference does (kalman.py:136-152); B = 1 only."""
        if self._per:
            raise ValueError("sim() predicts one instance of a shared system; this estimator has one system per instance")
        x = np.array(self.x if x is None else x, float).reshape(-1)
        u_seq = np.asarray(u_seq, float).reshape(len(u_seq), -1)
        assert u_seq.shape[1] == self.nu
        y = np.zeros((u_seq.shape[0], self.ny))
        for i in range(u_seq.shape[0]):
            y[i] = self.C @ x + self.D.reshape(self.ny, -1) @ u_seq[i]
            x = self.A @ x + self.B @ u_seq[i]
        return y


class KalmanFilter(_DeviceEstimator):
    _STATUS = {1: "ok", -2: "innovation covariance not positive definite"}

    def __init__(self, x0, A, B, C, D, Qn, Rn, P0=None, batch=None, device=0):
        """Batched Kalman filter for x+ = A x + B u + w, y = C x + v with E[ww'] = Qn, E[vv'] = Rn (the model of
        kalman_design_simple; no cross covariance: pass Bw Qw Bw' as Qn).  Holds the a-priori estimate x[k|k-1] and its covariance:
        predict(u) does x <- A x + B u, P <- A P A' + Qn, y <- C x; update(y_meas) computes the gain K = P C' (C P C' + Rn)^-1 and
        does x <- x + K (y_meas - y) with the Joseph-form covariance update.  D is accepted and not used, as in the reference.

        Any of A, B, C, Qn, Rn may carry a leading batch dimension (one model per instance); `batch` then defaults to it.  P0
        (nx, nx) or (batch, nx, nx) defaults to each instance's steady-state a-priori covariance dare(A', C', Qn, Rn): the filter
        then starts on the gain of kalman_design_simple(..., type='filter').  Qn, Rn and P0 are symmetrised.  An instance whose
        innovation covariance is not positive definite keeps its x and P at that update; ``status`` reports it (update() does not
        raise)."""
        self._L = _lib.load()
        (A, B, C, Qn, Rn), nb = _arrays(("A", "B", "C", "Qn", "Rn"), (A, B, C, Qn, Rn))
        self._per = nb is not None
        if self._per:
            if batch is None:
                batch = nb
            elif int(batch) != nb:
                raise ValueError(f"batch = {batch} but the per-instance matrices carry {nb} systems")
        self.nx, self.nu, self.ny = A.shape[-1], B.shape[-1], C.shape[-2]
        want = {"A": (self.nx, self.nx), "B": (self.nx, self.nu), "C": (self.ny, self.nx), "Qn": (self.nx, self.nx),
                "Rn": (self.ny, self.ny)}
        for name, a in zip(("A", "B", "C", "Qn", "Rn"), (A, B, C, Qn, Rn)):
            if a.shape[-2:] != want[name]:
                raise ValueError(f"KalmanFilter: {name} should have shape {want[name]} (nx = {self.nx}, nu = {self.nu}, "
                                 f"ny = {self.ny}), got {a.shape[-2:]}")
        if not (1 <= self.nx <= 32 and 1 <= self.ny <= 32):
            raise ValueError(f"KalmanFilter supports 1 <= nx, ny <= 32 (got nx = {self.nx}, ny = {self.ny})")
        self.batch = batch
        self._B = 1 if batch is None else int(batch)
        self.device = int(device)
        Qn, Rn = (Qn + _T(Qn)) / 2, (Rn + _T(Rn)) / 2
        x0 = np.ascontiguousarray(np.broadcast_to(np.asarray(x0, float).reshape(-1, self.nx), (self._B, self.nx)))
        if P0 is None:
            X, _, _, st = dare(_T(A), _T(C), Qn, Rn, return_status=True, device=device)
            if (np.asarray(st) != 1).any():
                bad = np.flatnonzero(np.asarray(st) != 1)[:8]
                raise ValueError("KalmanFilter: dare(A', C', Qn, Rn) has no stabilising solution for instance(s) "
                                 f"{bad.tolist()}: pass the initial covariance P0")
            P0 = X
        P0 = np.asarray(P0, float)
        if P0.shape not in ((self.nx, self.nx), (self._B, self.nx, self.nx)):
            raise ValueError(f"KalmanFilter: P0 should have shape {(self.nx, self.nx)} or {(self._B, self.nx, self.nx)}, got {P0.shape}")
        P0 = np.ascontiguousarray(np.broadcast_to((P0 + _T(P0)) / 2, (self._B, self.nx, self.nx)))
        n = self._B if self._per else 1
        full = lambda a: np.ascontiguousarray(np.broadcast_to(a, (n,) + a.shape[-2:]))
        A, B, C, Qn, Rn = full(A), full(B), full(C), full(Qn), full(Rn)
        one = lambda a: a if self._per else a[0]
        self.A, self.B, self.C, self.D, self.Qn, self.Rn = one(A), one(B), one(C), np.asarray(D, float), one(Qn), one(Rn)
        h = ctypes.c_void_p()
        rc = self._L.bmpc_est_create_kf(self.nx, self.nu, self.ny, self._B, n, self.device, ptr(A), ptr(B), ptr(C), ptr(Qn),
                                        ptr(Rn), ptr(x0), ptr(P0), ctypes.byref(h))
        if rc < 0:
            raise BmpcError(f"bmpc_est_create_kf failed ({rc}): {self._L.bmpc_last_error(None).decode()}")
        self._h = h

    @property
    def P(self):
        """covariance of the a-priori estimate (after predict) or of the a-posteriori one (after update): (nx, nx) per instance"""
        P = np.empty((self._B, self.nx, self.nx)); self._check(self._L.bmpc_est_get_cov(self._h, ptr(P), None)); return self._out(P)

    @property
    def status(self):
        """per instance: 1, or -2 when the last update found the innovation covariance C P C' + Rn not positive definite (that
        instance's x and P were left as they were)"""
        st = np.empty(self._B, np.int32); self._check(self._L.bmpc_est_get_cov(self._h, None, ptr(st))); return self._out(st)

    def _check(self, rc):
        if rc < 0:
            raise BmpcError(f"bmpc_est_get_cov failed ({rc})")

    def update_system(self, A=None, B=None, C=None, Qn=None, Rn=None):
        """Replace any of (A, B, C, Qn, Rn) between steps: A, B and Qn act from the next predict, C and Rn from the next update; y
        is not recomputed.  2-D matrices, or (batch, ...) on a filter created with one model per instance."""
        self._update_system(A=A, B=B, C=C, Qn=Qn, Rn=Rn)

    def update_system_from_device(self, A=None, B=None, C=None, Qn=None, Rn=None):
        """update_system with device arrays: raw pointers or contiguous float64 CUDA tensors (batch, ...) per instance, (...) shared;
        read in stream order on the filter's stream (the controller's once attached), no host round trip.  Qn and Rn are not
        symmetrised: their upper (Qn) and lower (Rn) triangles are read."""
        self._update_system_from_device(A=A, B=B, C=C, Qn=Qn, Rn=Rn)
