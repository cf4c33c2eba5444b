"""ctypes front-end of the host emulation of the device core (tests only)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libhostemu.so")
_NAMES = ["Ad", "Bd", "Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "uref",
          "pw", "Acal", "Bcal", "BcalT", "PB", "H", "Hinv", "K", "Kinv", "AHinv", "M", "Gx0", "Gref", "GrefFull",
          "g0", "lo0", "hi0", "rho", "scal"]


def build():
    src = os.path.join(_HERE, "hostemu.cpp")
    csrc = os.path.join(_HERE, "..", "..", "pympc_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("bmpc_core.cuh", "bmpc_rounds.cuh", "bmpc_launch.cuh", "bmpc_tpi.cuh", "bmpc_tile.cuh", "bmpc_tpm.cuh")]
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    if (not os.path.exists(_SO)) or os.path.getmtime(_SO) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-x", "c++", src, "-o", _SO])
    return ctypes.CDLL(_SO)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class EmuSystem:
    def __init__(self, cfg, rho=0.0, sigma=1e-6, alpha=1.6, soft_on=1):
        self.L = build()
        Ad = np.asarray(cfg["Ad"], float); Bd = np.asarray(cfg["Bd"], float)
        self.nx, self.nu = Bd.shape
        self.Np = cfg.get("Np", 20); self.Nc = cfg.get("Nc") or self.Np
        nx, nu, Np, Nc = self.nx, self.nu, self.Np, self.Nc
        self.NX, self.NU = (Np + 1) * nx, Nc * nu
        self.mc = self.NX + self.NU + (Nc + 1) * nu
        self.off = {n: self.L.emu_offset(nx, nu, Np, Nc, i) for i, n in enumerate(_NAMES)}
        self.sys = np.zeros(self.L.emu_sys_total(nx, nu, Np, Nc))
        inf = np.inf

        def put(name, val):
            val = np.asarray(val.toarray() if hasattr(val, "toarray") else val, float).ravel()
            self.sys[self.off[name]:self.off[name] + val.size] = val
        put("Ad", Ad); put("Bd", Bd)
        Qx = cfg.get("Qx", np.zeros((nx, nx))); put("Qx", Qx); put("QxN", cfg.get("QxN", Qx))
        put("Qu", cfg.get("Qu", np.zeros((nu, nu)))); put("QDu", cfg.get("QDu", np.zeros((nu, nu))))
        put("xmin", cfg.get("xmin", -inf * np.ones(nx))); put("xmax", cfg.get("xmax", inf * np.ones(nx)))
        put("umin", cfg.get("umin", -inf * np.ones(nu))); put("umax", cfg.get("umax", inf * np.ones(nu)))
        put("Dumin", cfg.get("Dumin", -inf * np.ones(nu))); put("Dumax", cfg.get("Dumax", inf * np.ones(nu)))
        put("uref", cfg.get("uref", np.zeros(nu)))
        self.L.emu_condense.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p] + [ctypes.c_double] * 4 + [ctypes.c_int]
        self.L.emu_condense(nx, nu, Np, Nc, _p(self.sys), rho, sigma, alpha, float(cfg.get("eps_feas", 1e6)), int(soft_on))
        self.x = np.zeros(self.NU); self.v = np.zeros(self.mc); self.cold = 1

    def get(self, name, shape):
        n = int(np.prod(shape))
        return self.sys[self.off[name]:self.off[name] + n].reshape(shape).copy()

    def solve(self, x0, um1, xref, first_iters=10, max_iter=4000, pdas_steps=10, rmax=64, eps_abs=1e-3, eps_rel=1e-3, tiers=None):
        """rounds of ADMM + Schur polish.  The polish capacity is rmax, or tiers = (first round, straggler rounds): the capacities of
        the device's polish tiers in each (launch_tiers), smallest first."""
        x0 = np.ascontiguousarray(x0, float); um1 = np.ascontiguousarray(um1, float); xref = np.ascontiguousarray(xref, float)
        mode = 0 if xref.ndim == 1 else 1
        t0, t1 = (np.ascontiguousarray(t, np.int32) for t in (tiers or ((rmax,), (rmax,))))
        U = np.zeros(self.NU); it = ctypes.c_int(); ps = ctypes.c_int(); res = np.zeros(4)
        f = self.L.emu_solve
        f.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p] * 4 + [ctypes.c_int] * 2 + [ctypes.c_void_p] * 3 + \
                     [ctypes.c_int] * 3 + [ctypes.c_void_p, ctypes.c_int] * 2 + [ctypes.c_double] * 2 + [ctypes.c_void_p] * 3
        st = f(self.nx, self.nu, self.Np, self.Nc, _p(self.sys), _p(x0), _p(um1), _p(xref), mode, self.cold,
               _p(self.x), _p(self.v), _p(U), first_iters, max_iter, pdas_steps, _p(t0), len(t0), _p(t1), len(t1), eps_abs, eps_rel,
               ctypes.byref(it), ctypes.byref(ps), _p(res))
        self.cold = 0
        return U, st, it.value, ps.value, res

    def tpi_step(self, x0, um1, xref, first_iters=10, pdas_steps=8):
        """TPI fast path (ADMM + Riccati polish) on the same generic-layout state; xref (nx) or time-varying (Np+1, nx).
        Returns (U, polish_steps)."""
        x0 = np.ascontiguousarray(x0, float); um1 = np.ascontiguousarray(um1, float); xref = np.ascontiguousarray(xref, float)
        mode = 0 if xref.ndim == 1 else 1
        U = np.zeros(self.NU)
        f = self.L.emu_tpi_step
        f.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p] * 4 + [ctypes.c_int] * 2 + [ctypes.c_void_p] * 3 + [ctypes.c_int] * 2
        ps = f(self.nx, self.nu, self.Np, self.Nc, _p(self.sys), _p(x0), _p(um1), _p(xref), mode, self.cold, _p(self.x), _p(self.v), _p(U),
               first_iters, pdas_steps)
        self.cold = 0
        return U, ps

    def polish_only(self, x0, um1, xref, pdas_steps=10, rmax=None):
        """team (Schur) polish alone from self.v; returns (U, refinements) and replaces self.v by v* when verified"""
        x0 = np.ascontiguousarray(x0, float); um1 = np.ascontiguousarray(um1, float); xref = np.ascontiguousarray(xref, float)
        mode = 0 if xref.ndim == 1 else 1
        U = np.zeros(self.NU)
        f = self.L.emu_polish_only
        f.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        ps = f(self.nx, self.nu, self.Np, self.Nc, _p(self.sys), _p(x0), _p(um1), _p(xref), mode, _p(self.v), _p(U), pdas_steps, rmax or self.mc)
        return U, ps

    def tpi2_step(self, x0, um1, xref, mode=1, max_ref=8):
        """second-generation Riccati polish on the stored working-set codes (mode 0 as stored, 1 shifted one stage, 2 from v);
        returns (U, refinements used); state: self.codes, self.v, self.mumax."""
        x0 = np.ascontiguousarray(x0, float); um1 = np.ascontiguousarray(um1, float); xref = np.ascontiguousarray(xref, float)
        tv = 0 if xref.ndim == 1 else 1
        if not hasattr(self, "codes"):
            self.codes = np.zeros(self.Np, np.uint32)
        U = np.zeros(self.NU); mm = np.zeros(1)
        f = self.L.emu_tpi2_step
        f.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        ps = f(self.nx, self.nu, self.Np, self.Nc, _p(self.sys), _p(x0), _p(um1), _p(xref), tv, _p(self.codes), mode, _p(self.v), _p(U), max_ref, _p(mm))
        return U, ps

    def tpm_step(self, x0, um1, xref, mode=1, max_ref=8, exchange_from=-1):
        """multi-input Riccati polish (bmpc_tpm.cuh) on the stored working-set codes (mode 0 as stored, 1 shifted one stage, 2 from
        self.v); exchange_from >= 0: refinements from that index on update the hard rows by single exchanges (the device's straggler
        rounds: 0); returns (U, refinements used); state: self.mcodes, self.v, self.mumax."""
        x0 = np.ascontiguousarray(x0, float); um1 = np.ascontiguousarray(um1, float); xref = np.ascontiguousarray(xref, float)
        tv = 0 if xref.ndim == 1 else 1
        if not hasattr(self, "mcodes"):
            self.mcodes = np.zeros(self.Np, np.uint64)
        U = np.ascontiguousarray(getattr(self, "Uplan", np.zeros(self.NU)), float).copy(); mm = np.zeros(1)
        f = self.L.emu_tpm_step
        f.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        ps = f(self.nx, self.nu, self.Np, self.Nc, _p(self.sys), _p(x0), _p(um1), _p(xref), tv, _p(self.mcodes), mode, _p(self.v), _p(U), max_ref, _p(mm), exchange_from)
        if ps > 0:
            self.Uplan = U.copy()
        return U, ps

    def admm_only(self, x0, um1, xref, niter):
        """niter team-core ADMM iterations on (self.x, self.v) with the adaptive-rho move; returns the residual quadruple"""
        x0 = np.ascontiguousarray(x0, float); um1 = np.ascontiguousarray(um1, float); xref = np.ascontiguousarray(xref, float)
        tv = 0 if xref.ndim == 1 else 1
        lvl = ctypes.c_int(getattr(self, "lvl", 2)); res = np.zeros(4)
        f = self.L.emu_admm_only
        f.restype = None
        f.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p] * 4 + [ctypes.c_int] * 2 + [ctypes.c_void_p] * 2 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        f(self.nx, self.nu, self.Np, self.Nc, _p(self.sys), _p(x0), _p(um1), _p(xref), tv, self.cold, _p(self.x), _p(self.v), niter, ctypes.byref(lvl), _p(res))
        self.cold = 0; self.lvl = lvl.value
        return res

    def tile_compare(self, X0, Um1, Xref, niter, lvl=None, x_in=None, v_in=None, T=4):
        """Run the tile ADMM and the per-instance team ADMM on the same T (2, 4 or 8) instances; returns (ref, tile) dicts."""
        X0 = np.ascontiguousarray(X0, float); Um1 = np.ascontiguousarray(Um1, float); Xref = np.ascontiguousarray(Xref, float)
        mode = 0 if Xref.ndim == 2 else 1
        Xref = Xref.reshape(T, -1)
        lvl = np.ascontiguousarray(lvl if lvl is not None else [2] * T, np.int32)
        cold = 1 if x_in is None else 0
        xin = np.ascontiguousarray(x_in if x_in is not None else np.zeros((T, self.NU)), float)
        vin = np.ascontiguousarray(v_in if v_in is not None else np.zeros((T, self.mc)), float)
        out = {}
        for tag in ("ref", "tile"):
            out[tag] = {"x": np.zeros((T, self.NU)), "v": np.zeros((T, self.mc)), "xt": np.zeros((T, self.NU)),
                        "res": np.zeros((T, 4)), "lvl": np.zeros(T, np.int32)}
        f = self.L.emu_tile_compare
        f.restype = None
        f.argtypes = [ctypes.c_int] * 5 + [ctypes.c_void_p] * 4 + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 13
        f(T, self.nx, self.nu, self.Np, self.Nc, _p(self.sys), _p(X0), _p(Um1), _p(Xref), mode, cold, niter, _p(lvl), _p(xin), _p(vin),
          *[_p(out[tag][k]) for tag in ("ref", "tile") for k in ("x", "v", "xt", "res", "lvl")])
        return out["ref"], out["tile"]

    def infeasible(self, x0, um1, xref, it0=25, it1=25, eps=1e-4):
        """OSQP's primal-infeasibility certificate between the ADMM states after it0 and it0+it1 iterations (cold start)."""
        x0 = np.ascontiguousarray(x0, float); um1 = np.ascontiguousarray(um1, float); xref = np.ascontiguousarray(xref, float)
        f = self.L.emu_infeasible
        f.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p] * 4 + [ctypes.c_int] * 2 + [ctypes.c_double]
        return bool(f(self.nx, self.nu, self.Np, self.Nc, _p(self.sys), _p(x0), _p(um1), _p(xref), it0, it1, eps))


# opt-in shared memory per block of an H100 (cudaDevAttrMaxSharedMemoryPerBlockOptin), bytes
H100_OPTIN = 232448
H100_SMS = 132                  # streaming multiprocessors of an H100 SXM (cudaDevAttrMultiProcessorCount)
_ADMM_KINDS = ("warp", "lone_warp", "tile", "cta")     # BmpcTeamAdmm
_LAUNCH_FIELDS = ("ok", "team", "wpb", "rmax", "rmax_small", "fb_team", "fb_rmax", "overflow", "tile_T", "tile_threads",
                  "smem_admm", "smem_polish", "smem_polish_small", "fb_smem_polish")


def plan_launch(nx, nu, Np, Nc=None, max_optin=H100_OPTIN, team_threads=0, warps_per_block=0, rmax=0, n_sys=1):
    """the launch configuration bmpc_create chooses (bmpc_launch.cuh: bmpc_plan_launch), as a dict"""
    L = build(); out = np.zeros(14, np.int64)
    f = L.emu_plan_launch
    f.restype = None
    f.argtypes = [ctypes.c_int] * 9 + [ctypes.c_void_p]
    f(nx, nu, Np, Nc or Np, max_optin, team_threads, warps_per_block, rmax, n_sys, _p(out))
    return dict(zip(_LAUNCH_FIELDS, (int(v) for v in out)))


def round_launch(nx, nu, Np, Nc=None, count=1, list_given=False, sm_count=H100_SMS, max_optin=H100_OPTIN, team_threads=0,
                 warps_per_block=0, rmax=0, n_sys=1):
    """the team / tile launches of one round over `count` open instances (bmpc_launch.cuh: bmpc_round_launch; list_given: a
    straggler round) as a dict: admm kind, tile size, grid, threads and shared memory of the ADMM, and the polish tiers, smallest
    capacity first; None for a shape bmpc_create refuses"""
    L = build(); out = np.zeros(16, np.int64)
    f = L.emu_round_launch
    f.argtypes = [ctypes.c_int] * 12 + [ctypes.c_void_p]
    if not f(nx, nu, Np, Nc or Np, max_optin, team_threads, warps_per_block, rmax, n_sys, count, int(list_given), sm_count, _p(out)):
        return None
    v = [int(x) for x in out]
    tiers = [dict(zip(("warp", "grid", "threads", "rmax", "smem"), v[6 + 5 * k:11 + 5 * k])) for k in range(v[5])]
    return dict(admm=_ADMM_KINDS[v[0]], tile_T=v[1], admm_grid=v[2], admm_threads=v[3], admm_smem=v[4], tiers=tiers)


def launch_tiers(nx, nu, Np, Nc=None, count=1, max_optin=H100_OPTIN, team_threads=0, warps_per_block=0, rmax=0, n_sys=1):
    """(first round, straggler rounds): capacities of the polish tiers an instance passes in a batch of `count` whose straggler
    rounds keep all of them open (bmpc_polish_tiers), smallest first"""
    L = build(); caps = np.zeros(2, np.int32)
    f = L.emu_polish_tiers
    f.argtypes = [ctypes.c_int] * 11 + [ctypes.c_void_p]
    out = []
    for given in (0, 1):
        n = f(nx, nu, Np, Nc or Np, max_optin, team_threads, warps_per_block, rmax, n_sys, count, given, _p(caps))
        out.append(tuple(int(c) for c in caps[:n]))
    return tuple(out)
