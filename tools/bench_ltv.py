"""Time-varying system matrices on the device: what a successive-linearisation step costs with bmpc_update_system.

Workload: B = 65 536 per-instance inverted pendulums (pympc_b200.workloads.pendulum weights and bounds, pendulum_random starts and
references) driven by the nonlinear cart-pole (RK4 of workloads.cartpole_rhs, on the device) and re-linearised about each instance's
state at every step (workloads.cartpole_linearised, torch on the device).  bench.py's method (DESIGN.md §5): device-resident x0 and
u_-1 read in place, u* written into a device buffer, ONE explicit stream for the solver, the plant, the L2 flush (256 MiB written
between timed steps, outside the events) and the CUDA events around each step.  Modes, each from a fresh setup at the same start:
  fixed       the model stays the one linearised at the start: the warm step alone
  ltv_device  bmpc_update_system(on_device = 1) with the torch-built matrices + the warm step
  ltv_host    the same matrices copied to host memory first (outside the events), bmpc_update_system(on_device = 0) + the warm step
  resetup     today's alternative: a new controller, setup() with the new matrices and its cold solve, per step (host wall clock,
              synchronised; fewer steps)
Per step: event time (mean / median / max), host wall clock of the timed calls (synchronised after the stop event), refinements,
rounds, ADMM iterations and instances re-condensed.  Checks in the same run: u* of the last ltv_device step against a controller set
up from scratch with that step's matrices and inputs (instances both verified), and four instances against the oracle.  The card's
name and power limit are read in the same run.  Prints one JSON line; --out FILE also writes it there.

usage: python tools/bench_ltv.py [--batch 65536] [--steps 30] [--warmup 5] [--resetup-steps 3] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.bench_kalman_design import card  # noqa: E402

KEYS = ("Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "eps_feas")


def controller(MPC, Ad, Bd, X, Xref, U, B):
    from pympc_b200.workloads import pendulum
    c = pendulum()
    K = MPC(Ad, Bd, Np=20, x0=X, xref=Xref, uminus1=U, batch=B, **{k: c[k] for k in KEYS})
    K.setup(solve=False)
    return K


def run_mode(torch, MPC, mode, B, X0, Xref, steps, warmup, flush):
    from pympc_b200.workloads import cartpole_rhs, cartpole_linearised, CARTPOLE
    Ts = CARTPOLE[6]; dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    torch.cuda.synchronize(dev)
    torch.cuda.set_stream(stream)

    def rk4(x, u):
        k1 = cartpole_rhs(x, u); k2 = cartpole_rhs(x + 0.5 * Ts * k1, u)
        k3 = cartpole_rhs(x + 0.5 * Ts * k2, u); k4 = cartpole_rhs(x + Ts * k3, u)
        return x + Ts / 6.0 * (k1 + 2 * k2 + 2 * k3 + k4)
    Ad0, Bd0 = cartpole_linearised(X0, np.zeros((B, 1)))
    K = controller(MPC, Ad0, Bd0, X0, Xref, np.zeros((B, 1)), B)
    L, h = K._L, K.handle
    assert L.bmpc_set_stream(h, stream.cuda_stream) == 0
    Xd = torch.tensor(X0, device=dev)
    Ubuf = torch.zeros((2, B, 1), dtype=torch.float64, device=dev)
    ev_ms, wall_ms, st_acc, last = [], [], [], None
    for t in range(warmup + steps):
        Uprev = Ubuf[(t & 1) ^ 1]
        assert L.bmpc_bind_output(h, Ubuf[t & 1].data_ptr()) == 0
        if t > 0:
            Xd = rk4(Xd, Uprev)                                   # the nonlinear plant (not the hot path)
        Ad_t, Bd_t = cartpole_linearised(Xd, Uprev)
        Ah = Bh = None
        if mode == "ltv_host":
            Ah, Bh = Ad_t.cpu().numpy(), Bd_t.cpu().numpy()
        flush.zero_()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(dev)
        w0 = time.perf_counter()
        e0.record(stream)
        if mode == "ltv_device":
            assert L.bmpc_update_system(h, Ad_t.data_ptr(), Bd_t.data_ptr(), 1) == 0, L.bmpc_last_error(h)
        elif mode == "ltv_host":
            assert L.bmpc_update_system(h, Ah.ctypes.data, Bh.ctypes.data, 0) == 0, L.bmpc_last_error(h)
        assert L.bmpc_update(h, Xd.data_ptr(), Uprev.data_ptr(), None, 1, 2) == 0
        assert L.bmpc_solve(h) == 0, L.bmpc_last_error(h)
        assert L.bmpc_output(h, None, None, 1, 1) == 0
        e1.record(stream)
        e1.synchronize()
        w1 = time.perf_counter()
        st = K.stats()
        if t >= warmup:
            ev_ms.append(e0.elapsed_time(e1)); wall_ms.append(1e3 * (w1 - w0)); st_acc.append(st)
        if t == warmup + steps - 1:
            stat = np.empty(B, np.int32)
            assert L.bmpc_output(h, None, stat.ctypes.data, 0, 0) == 0
            last = (Xd.cpu().numpy(), Uprev.cpu().numpy(), Ad_t.cpu().numpy(), Bd_t.cpu().numpy(), Ubuf[t & 1].cpu().numpy().copy(), stat)
    torch.cuda.synchronize(dev)
    torch.cuda.set_stream(torch.cuda.default_stream(dev))
    K.close()
    return ev_ms, wall_ms, st_acc, last


def summary(ev_ms, wall_ms, st_acc):
    f = lambda k: [s[k] for s in st_acc]
    out = {"steps": len(st_acc)}
    if ev_ms:
        out.update(event_ms_mean=float(np.mean(ev_ms)), event_ms_median=float(np.median(ev_ms)), event_ms_max=float(np.max(ev_ms)))
    out.update(wall_ms_mean=float(np.mean(wall_ms)), wall_ms_median=float(np.median(wall_ms)), wall_ms_max=float(np.max(wall_ms)),
               refinements_mean=float(np.mean(f("polish_steps"))), rounds_mean=float(np.mean(f("rounds"))), rounds_max=int(max(f("rounds"))),
               admm_iters_mean=float(np.mean(f("admm_iters"))), recondensed_mean=float(np.mean(f("recondensed"))),
               recondensed_max=int(max(f("recondensed"))), unsolved_max=int(max(f("unsolved"))))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--resetup-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from pympc_b200 import MPCController as MPC
    from pympc_b200.workloads import pendulum, pendulum_random, cartpole_rhs, cartpole_linearised, CARTPOLE
    from oracle.qp_assembly import QPData
    from oracle.kkt import solve_exact
    B = args.batch; dev = torch.device("cuda", 0)
    torch.zeros(1, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    X0, Xref = pendulum_random(B, seed=2026)
    rec = {"tool": "bench_ltv", **card(), "batch": B, "Np": 20, "workload": "per-instance pendulums, nonlinear cart-pole plant (RK4), "
           "re-linearised about every instance's state each step", "l2": "flushed between timed steps (256 MiB write)", "modes": {}}
    for mode in ("fixed", "ltv_device", "ltv_host"):
        ev, wall, sts, last = run_mode(torch, MPC, mode, B, X0, Xref, args.steps, args.warmup, flush)
        rec["modes"][mode] = summary(ev, wall, sts)
        if mode == "ltv_device":
            X, U, A, Bm, u, stat = last
            F = controller(MPC, A, Bm, X, Xref, U, B); F.solve()
            uf = F.output().copy(); sf = np.array(F.res.info.status_val); F.close()
            d = np.abs(u[:, 0] - uf[:, 0])[(sf == 1) & (stat == 1)]
            c = pendulum(); err = 0.0
            for b in np.random.default_rng(5).choice(B, 4, replace=False):
                Q = QPData(**dict(c, Ad=A[b], Bd=Bm[b], x0=X[b], xref=Xref[b], uminus1=U[b]))
                z, y, r = solve_exact(Q.P, Q.q, Q.A, Q.l, Q.u)
                err = max(err, abs(u[b, 0] - z[Q.NX]))
            rec["check_ltv_device_last_step"] = {"max_abs_diff_u_vs_fresh_setup": float(d.max()), "compared": int(d.size),
                                                 "verified": int((stat == 1).sum()),
                                                 "max_abs_err_u_vs_oracle_4": float(err)}
    # today's route: setup() + cold solve with the new matrices, every step
    Ts = CARTPOLE[6]
    Xd = torch.tensor(X0, device=dev); U = np.zeros((B, 1)); wall, sts = [], []
    for t in range(1 + args.resetup_steps):
        Ut = torch.tensor(U, device=dev)
        if t > 0:
            k1 = cartpole_rhs(Xd, Ut); k2 = cartpole_rhs(Xd + 0.5 * Ts * k1, Ut)
            k3 = cartpole_rhs(Xd + 0.5 * Ts * k2, Ut); k4 = cartpole_rhs(Xd + Ts * k3, Ut)
            Xd = Xd + Ts / 6.0 * (k1 + 2 * k2 + 2 * k3 + k4)
        A, Bm = [a.cpu().numpy() for a in cartpole_linearised(Xd, Ut)]
        X = Xd.cpu().numpy()
        torch.cuda.synchronize(dev)
        w0 = time.perf_counter()
        K = MPC(A, Bm, Np=20, x0=X, xref=Xref, uminus1=U, batch=B, **{k: pendulum()[k] for k in KEYS})
        K.setup()
        Un = K.output().copy()
        w1 = time.perf_counter()
        if t > 0:
            wall.append(1e3 * (w1 - w0)); sts.append(K.stats())
        K.close(); U = Un
    rec["modes"]["resetup"] = summary([], wall, sts)
    rec["modes"]["resetup"]["timing"] = "host wall clock of construct + setup() + cold solve + output(), synchronised"
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
