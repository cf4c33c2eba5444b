"""ctypes binding of libbmpc.so (include/bmpc.h).  There is no CPU fallback: if the CUDA
extension is missing or no device is visible, importing/creating fails loudly."""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# BMPC_LIB: load another build of the same library (kernel-variant sweeps of tools/gpu_sweep.py); default = the in-tree build
LIB_PATH = os.environ.get("BMPC_LIB") or os.path.join(_HERE, "libbmpc.so")
_lib = None

P = ctypes.c_void_p
DP = ctypes.c_void_p


class BmpcConfig(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in
                ("nx", "nu", "Np", "Nc", "batch", "device", "soft_on", "max_iter", "first_iters", "pdas_steps",
                 "rmax", "polish", "team_threads", "warps_per_block", "fast_path", "n_sys", "shift_warm", "candidate_warm", "cold_iters")] + \
               [(n, ctypes.c_double) for n in ("eps_feas", "rho", "sigma", "alpha", "eps_abs", "eps_rel")]


class BmpcStats(ctypes.Structure):
    _fields_ = [("admm_iters", ctypes.c_int64), ("rounds", ctypes.c_int32), ("unsolved", ctypes.c_int32),
                ("polish_steps", ctypes.c_int64), ("ms_admm", ctypes.c_float), ("ms_polish", ctypes.c_float),
                ("launches", ctypes.c_int32), ("infeasible", ctypes.c_int32), ("recondensed", ctypes.c_int32)]


EXPORTS = ["bmpc_default_config", "bmpc_create", "bmpc_destroy", "bmpc_last_error", "bmpc_setup", "bmpc_update", "bmpc_update_system", "bmpc_update_problem",
           "bmpc_solve", "bmpc_output", "bmpc_get_sequences", "bmpc_bind_output", "bmpc_bind_output_peers", "bmpc_bind_gather_flags",
           "bmpc_gather_arrive", "bmpc_set_stream",
           "bmpc_synchronize", "bmpc_get_stats", "bmpc_get_sys", "bmpc_get_dims", "bmpc_host_alloc",
           "bmpc_host_free", "bmpc_device_count", "bmpc_has_fast_path", "bmpc_has_multi_input_fast_path", "bmpc_est_create", "bmpc_est_create_ex", "bmpc_est_destroy", "bmpc_est_predict",
           "bmpc_est_update", "bmpc_est_get", "bmpc_est_state_ptr", "bmpc_est_set_stream", "bmpc_est_attach", "bmpc_est_create_kf",
           "bmpc_est_get_cov", "bmpc_est_set_model", "bmpc_dare"]


class BmpcError(RuntimeError):
    pass


_libs = {}


def load(path=None):
    """Load libbmpc.so (or, with `path`, a per-shape build of it made by pympc_b200.build.jit_shape); raises BmpcError if it has
    not been built (run ``python -m pympc_b200.build``)."""
    global _lib
    path = os.path.abspath(path or LIB_PATH)
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise BmpcError(f"{path} not found: build the CUDA extension first (python -m pympc_b200.build). "
                        "pympc_b200 has no CPU fallback.")
    L = ctypes.CDLL(path)
    L.bmpc_default_config.argtypes = [ctypes.POINTER(BmpcConfig)]; L.bmpc_default_config.restype = None
    L.bmpc_create.argtypes = [ctypes.POINTER(BmpcConfig), ctypes.POINTER(P)]; L.bmpc_create.restype = ctypes.c_int
    L.bmpc_destroy.argtypes = [P]; L.bmpc_destroy.restype = None
    L.bmpc_last_error.argtypes = [P]; L.bmpc_last_error.restype = ctypes.c_char_p
    L.bmpc_setup.argtypes = [P] + [DP] * 13; L.bmpc_setup.restype = ctypes.c_int
    L.bmpc_update.argtypes = [P, DP, DP, DP, ctypes.c_int, ctypes.c_int]; L.bmpc_update.restype = ctypes.c_int
    L.bmpc_update_system.argtypes = [P, DP, DP, ctypes.c_int]; L.bmpc_update_system.restype = ctypes.c_int
    L.bmpc_update_problem.argtypes = [P] + [DP] * 13 + [ctypes.c_int]; L.bmpc_update_problem.restype = ctypes.c_int
    L.bmpc_solve.argtypes = [P]; L.bmpc_solve.restype = ctypes.c_int
    L.bmpc_output.argtypes = [P, DP, DP, ctypes.c_int, ctypes.c_int]; L.bmpc_output.restype = ctypes.c_int
    L.bmpc_get_sequences.argtypes = [P, DP, DP, DP, DP, DP]; L.bmpc_get_sequences.restype = ctypes.c_int
    L.bmpc_bind_output.argtypes = [P, DP]; L.bmpc_bind_output.restype = ctypes.c_int
    L.bmpc_set_stream.argtypes = [P, P]; L.bmpc_set_stream.restype = ctypes.c_int
    L.bmpc_bind_output_peers.argtypes = [P, ctypes.POINTER(ctypes.c_void_p), ctypes.c_int]; L.bmpc_bind_output_peers.restype = ctypes.c_int
    L.bmpc_bind_gather_flags.argtypes = [P, P, ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int64]; L.bmpc_bind_gather_flags.restype = ctypes.c_int
    L.bmpc_gather_arrive.argtypes = [P, ctypes.c_int64]; L.bmpc_gather_arrive.restype = ctypes.c_int
    L.bmpc_synchronize.argtypes = [P]; L.bmpc_synchronize.restype = ctypes.c_int
    L.bmpc_get_stats.argtypes = [P, ctypes.POINTER(BmpcStats)]; L.bmpc_get_stats.restype = ctypes.c_int
    L.bmpc_get_sys.argtypes = [P, ctypes.c_char_p, DP, ctypes.c_int]; L.bmpc_get_sys.restype = ctypes.c_int
    L.bmpc_get_dims.argtypes = [P, DP]; L.bmpc_get_dims.restype = ctypes.c_int
    L.bmpc_host_alloc.argtypes = [ctypes.c_uint64]; L.bmpc_host_alloc.restype = P
    L.bmpc_host_free.argtypes = [P]; L.bmpc_host_free.restype = None
    L.bmpc_device_count.argtypes = []; L.bmpc_device_count.restype = ctypes.c_int
    L.bmpc_est_create.argtypes = [ctypes.c_int32] * 5 + [DP] * 5 + [ctypes.POINTER(P)]; L.bmpc_est_create.restype = ctypes.c_int
    L.bmpc_est_create_ex.argtypes = [ctypes.c_int32] * 6 + [DP] * 5 + [ctypes.POINTER(P)]; L.bmpc_est_create_ex.restype = ctypes.c_int
    L.bmpc_est_destroy.argtypes = [P]; L.bmpc_est_destroy.restype = None
    L.bmpc_est_predict.argtypes = [P, DP, ctypes.c_int]; L.bmpc_est_predict.restype = ctypes.c_int
    L.bmpc_est_update.argtypes = [P, DP, ctypes.c_int]; L.bmpc_est_update.restype = ctypes.c_int
    L.bmpc_est_get.argtypes = [P, DP, DP]; L.bmpc_est_get.restype = ctypes.c_int
    L.bmpc_est_state_ptr.argtypes = [P]; L.bmpc_est_state_ptr.restype = P
    L.bmpc_est_set_stream.argtypes = [P, P]; L.bmpc_est_set_stream.restype = ctypes.c_int
    L.bmpc_est_attach.argtypes = [P, P]; L.bmpc_est_attach.restype = ctypes.c_int
    L.bmpc_est_create_kf.argtypes = [ctypes.c_int32] * 6 + [DP] * 7 + [ctypes.POINTER(P)]; L.bmpc_est_create_kf.restype = ctypes.c_int
    L.bmpc_est_get_cov.argtypes = [P, DP, DP]; L.bmpc_est_get_cov.restype = ctypes.c_int
    L.bmpc_est_set_model.argtypes = [P] + [DP] * 6 + [ctypes.c_int]; L.bmpc_est_set_model.restype = ctypes.c_int
    L.bmpc_dare.argtypes = [ctypes.c_int32] * 4 + [DP] * 9; L.bmpc_dare.restype = ctypes.c_int
    L.bmpc_has_fast_path.argtypes = [ctypes.c_int] * 4; L.bmpc_has_fast_path.restype = ctypes.c_int
    L.bmpc_has_multi_input_fast_path.argtypes = [ctypes.c_int] * 4; L.bmpc_has_multi_input_fast_path.restype = ctypes.c_int
    _libs[path] = L
    if path == os.path.abspath(LIB_PATH):
        _lib = L
    return L


def ptr(a):
    """Raw pointer of a C-contiguous numpy array (or None)."""
    if a is None:
        return None
    return a.ctypes.data_as(ctypes.c_void_p)


class PinnedArray:
    """numpy view over cudaHostAlloc'ed memory (freed with the object)."""

    def __init__(self, shape, dtype=np.float64):
        L = load()
        self.nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        self._p = L.bmpc_host_alloc(max(self.nbytes, 8))
        if not self._p:
            raise BmpcError("cudaHostAlloc failed")
        buf = (ctypes.c_char * max(self.nbytes, 8)).from_address(self._p)
        buf._owner = self                     # views handed out (numpy -> memoryview -> buf) keep the allocation alive
        self.array = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
        self.array[...] = 0
        self.ptr = ctypes.c_void_p(self._p)   # (a.ctypes.data_as costs ~2.5 us per call: cached for the per-step calls)

    def __del__(self):
        try:
            if getattr(self, "_p", None):
                load().bmpc_host_free(self._p); self._p = None
        except Exception:
            pass
