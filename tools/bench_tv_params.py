"""Time-varying bounds and uref on the device: what a step costs when every instance's limits change every step (bmpc_update_problem).

Workload: B = 65 536 per-instance inverted pendulums (pympc_b200.workloads.pendulum model, weights and bounds; pendulum_random
starts and references), each with its own umax, Dumax and uref schedule changed at every step (derated actuator limit, speed-dependent
rate limit, moving feed-forward).  The plant is the linear model, stepped on the device.  bench.py's method as in tools/bench_ltv.py:
device-resident x0 and u_-1 read in place, u* written into a device buffer, ONE explicit stream for the solver, the plant, the
schedules, the L2 flush (256 MiB written between timed steps, outside the events) and the CUDA events.  Modes, each from a fresh
setup at the same start:
  fixed        the parameters stay the ones set up: the warm step alone
  host         bmpc_update_problem(on_device = 0) with the step's umax, Dumax, uref (host arrays) + the warm step
  device       the same schedules computed by torch on the device, bmpc_update_problem(on_device = 1) + the warm step
  device_ltv   device schedules together with a new per-instance (Ad, Bd) every step (Ad scaled by 1 +- 1e-3 per instance)
  resetup      the alternative without this feature: a new controller, setup() with the step's arrays and its cold solve (host wall
               clock, synchronised; fewer steps)
  shared_host  one SHARED pendulum system (batch 65 536), shared umax / Dumax / uref changed every step from host arrays: the eager
               path (re-condense, one host synchronisation, the block copied back for the constant-bank refill)
Per step: event time of the whole step (mean / median / max), event time of the update call alone, host wall clock, rounds, ADMM
iterations and instances re-condensed.  The card's name and power limit are read in the same run.  Prints one JSON line; --out FILE
also writes it there.

usage: python tools/bench_tv_params.py [--batch 65536] [--steps 30] [--warmup 5] [--resetup-steps 3] [--out FILE]
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


def schedules(B, seed=7):
    rng = np.random.default_rng(seed)
    return rng.uniform(10.0, 20.0, (B, 1)), rng.uniform(2.0, 5.0, (B, 1)), rng.uniform(-0.05, 0.05, (B, 1))


def at(t, lim, rate, off):
    """the step-t arrays (numpy or torch): umax, Dumax, uref"""
    return lim * (1.0 - 0.05 * np.sin(0.1 * t)), rate * (1.0 + 0.1 * np.sin(t)), off * np.cos(0.3 * t)


def run_mode(torch, MPC, mode, B, X0, Xref, steps, warmup, flush):
    from pympc_b200.workloads import pendulum
    c = pendulum(); dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    torch.cuda.synchronize(dev)
    torch.cuda.set_stream(stream)
    shared = mode == "shared_host"
    Ad = c["Ad"] if shared else np.broadcast_to(c["Ad"], (B, 4, 4)).copy()
    Bd = c["Bd"] if shared else np.broadcast_to(c["Bd"], (B, 4, 1)).copy()
    K = MPC(Ad, Bd, Np=20, x0=X0, xref=Xref, uminus1=np.zeros((B, 1)), batch=B, **{k: c[k] for k in KEYS})
    K.setup(solve=False)
    L, h = K._L, K.handle
    assert L.bmpc_set_stream(h, stream.cuda_stream) == 0
    lim, rate, off = schedules(B)
    if shared:
        lim, rate, off = lim[:1], rate[:1], off[:1]
    limd, rated, offd = (torch.tensor(a, device=dev) for a in (lim, rate, off))
    Adt = torch.tensor(c["Ad"], device=dev); Bdt = torch.tensor(c["Bd"], device=dev)
    scale = torch.tensor(np.random.default_rng(3).uniform(-1, 1, (B, 1, 1)), device=dev)
    Xd = torch.tensor(X0, device=dev)
    Ubuf = torch.zeros((2, B, 1), dtype=torch.float64, device=dev)
    ev_ms, upd_ms, wall_ms, st_acc = [], [], [], []
    for t in range(warmup + steps):
        Uprev = Ubuf[(t & 1) ^ 1]
        assert L.bmpc_bind_output(h, Ubuf[t & 1].data_ptr()) == 0
        if t > 0:
            Xd = Xd @ Adt.T + Uprev @ Bdt.T                        # the plant (not the hot path)
        umax, Dumax, uref = at(t, lim, rate, off)
        dm = None
        if mode in ("device", "device_ltv"):
            dm = [a.contiguous() for a in at(t, limd, rated, offd)]
            if mode == "device_ltv":
                f = 1.0 + 1e-3 * np.sin(0.2 * t) * scale
                dm += [(Adt * f).contiguous(), (Bdt * f).contiguous()]
        flush.zero_()
        e0, eu0, eu1, e1 = (torch.cuda.Event(enable_timing=True) for _ in range(4))
        torch.cuda.synchronize(dev)
        w0 = time.perf_counter()
        e0.record(stream)
        eu0.record(stream)
        if mode in ("host", "shared_host"):
            a = [np.ascontiguousarray(v) for v in (umax, Dumax, uref)]
            rc = L.bmpc_update_problem(h, None, None, None, None, None, None, None, None, None, a[0].ctypes.data, None, a[1].ctypes.data,
                                       a[2].ctypes.data, 0)
            assert rc == 0, L.bmpc_last_error(h)
        elif dm is not None:
            A_, B_ = (dm[3].data_ptr(), dm[4].data_ptr()) if mode == "device_ltv" else (None, None)
            rc = L.bmpc_update_problem(h, A_, B_, None, None, None, None, None, None, None, dm[0].data_ptr(), None, dm[1].data_ptr(),
                                       dm[2].data_ptr(), 1)
            assert rc == 0, L.bmpc_last_error(h)
        eu1.record(stream)
        assert L.bmpc_update(h, Xd.data_ptr(), Uprev.data_ptr(), None, 1, 2) == 0
        assert L.bmpc_solve(h) == 0, L.bmpc_last_error(h)
        assert L.bmpc_output(h, None, None, 1, 1) == 0
        e1.record(stream)
        e1.synchronize()
        w1 = time.perf_counter()
        st = K.stats()
        if t >= warmup:
            ev_ms.append(e0.elapsed_time(e1)); upd_ms.append(eu0.elapsed_time(eu1)); wall_ms.append(1e3 * (w1 - w0)); st_acc.append(st)
    torch.cuda.synchronize(dev)
    torch.cuda.set_stream(torch.cuda.default_stream(dev))
    stat = np.empty(B, np.int32)
    assert L.bmpc_output(h, None, stat.ctypes.data, 0, 0) == 0
    K.close()
    return ev_ms, upd_ms, wall_ms, st_acc, float((stat == 1).mean())


def summary(ev_ms, upd_ms, wall_ms, st_acc):
    f = lambda k: [s[k] for s in st_acc]
    out = {"steps": len(st_acc)}
    if ev_ms:
        out.update(event_ms_mean=float(np.mean(ev_ms)), event_ms_median=float(np.median(ev_ms)), event_ms_max=float(np.max(ev_ms)),
                   update_event_ms_mean=float(np.mean(upd_ms)), update_event_ms_median=float(np.median(upd_ms)))
    out.update(wall_ms_mean=float(np.mean(wall_ms)), wall_ms_median=float(np.median(wall_ms)),
               rounds_mean=float(np.mean(f("rounds"))), rounds_max=int(max(f("rounds"))), admm_iters_mean=float(np.mean(f("admm_iters"))),
               recondensed_mean=float(np.mean(f("recondensed"))), recondensed_max=int(max(f("recondensed"))),
               unsolved_max=int(max(f("unsolved"))))
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
    from pympc_b200.workloads import pendulum, pendulum_random
    B = args.batch; dev = torch.device("cuda", 0)
    torch.zeros(1, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    X0, Xref = pendulum_random(B, seed=2026)
    X0 = 0.5 * X0
    rec = {"tool": "bench_tv_params", **card(), "batch": B, "Np": 20,
           "workload": "per-instance pendulums (linear plant), per-instance umax / Dumax / uref schedules changed every step",
           "l2": "flushed between timed steps (256 MiB write)", "modes": {}}
    for mode in ("fixed", "host", "device", "device_ltv", "shared_host"):
        ev, upd, wall, sts, ver = run_mode(torch, MPC, mode, B, X0, Xref, args.steps, args.warmup, flush)
        rec["modes"][mode] = summary(ev, upd, wall, sts)
        rec["modes"][mode]["verified_last_step"] = ver
    # the route without this feature: a new controller with the step's arrays, setup() + cold solve, every step
    c = pendulum(); lim, rate, off = schedules(B)
    Ad = np.broadcast_to(c["Ad"], (B, 4, 4)).copy(); Bd = np.broadcast_to(c["Bd"], (B, 4, 1)).copy()
    X = X0.copy(); U = np.zeros((B, 1)); wall, sts = [], []
    for t in range(1 + args.resetup_steps):
        umax, Dumax, uref = at(t, lim, rate, off)
        kw = {k: c[k] for k in KEYS}; kw.update(umax=umax, Dumax=Dumax)
        w0 = time.perf_counter()
        K = MPC(Ad, Bd, Np=20, x0=X, xref=Xref, uminus1=U, batch=B, **kw)
        K.setup(solve=False); K.update_system(uref=uref); K.solve()
        Un = K.output().copy()
        w1 = time.perf_counter()
        if t > 0:
            wall.append(1e3 * (w1 - w0)); sts.append(K.stats())
        K.close(); U = Un; X = X @ c["Ad"].T + U @ c["Bd"].T
    rec["modes"]["resetup"] = summary([], [], wall, sts)
    rec["modes"]["resetup"]["timing"] = "host wall clock of construct + setup() + cold solve + output(), synchronised"
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
