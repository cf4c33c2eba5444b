"""The batched Kalman filter on the device (k_kf / k_kf_pi): what a filter step costs, and what it adds to a successive-
linearisation loop.

Workloads:
  cartpole   65 536 per-instance cart-pole filters (nx = 4, nu = 1, ny = 2), the model (A, B) replaced from device arrays
             (workloads.cartpole_linearised on torch) every step
  governor   16 384 MIMO governor filters (workloads.mimo, nx = 8, nu = 4, ny = 4 outputs), one shared model
  ltv_loop   tools/bench_ltv.py's workload (65 536 per-instance pendulum controllers, nonlinear cart-pole plant, re-linearised every
             step, update_system(on_device = 1)) without and with the filter, alternated: with it, the filter's model follows
             the controller's and it predicts with the last u* and updates with y = C x of the plant, on the controller's stream
             inside the timed step.  The controller reads the plant state in both modes, so both solve the same QPs and the
             difference is the filter's work (the linearised model has no affine term, so the filter's estimate of the
             nonlinear plant is not what this measures)
  redesign   today's alternative for the cart-pole fleet: kalman_design_simple on the new models + a new LinearStateEstimator,
             per step (host wall clock, synchronised)
Timing: CUDA events on one explicit stream shared by torch, the controller and the filter; warm-up steps first; `--reps`
repetitions of `--steps` steps, each repetition reduced to its median, reported as the median and the spread (min, max) of those.
The card's name, power limit and SM clock are read in the same run.  Prints one JSON line; --out FILE also writes it there.

usage: python tools/bench_kf.py [--steps 50] [--warmup 10] [--reps 5] [--loop-steps 20] [--redesign-steps 3] [--out FILE]
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
from tools.bench_ltv import controller  # noqa: E402

C2 = np.array([[1.0, 0, 0, 0], [0, 0, 1.0, 0]])


def spread(reps):
    m = [float(np.median(r)) for r in reps]
    return {"median_ms": float(np.median(m)), "min_ms": float(min(m)), "max_ms": float(max(m)), "reps": len(m),
            "steps_per_rep": len(reps[0])}


def timed(torch, stream, fn):
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(stream); fn(); e1.record(stream)
    return e0, e1


def filter_steps(torch, F, stream, U, Y, models, steps, warmup, reps):
    """per step: [set_model from device] + predict_device + update_device; events around predict + update, around the update
    (measurement) call alone and around the model replacement"""
    L, h = F._L, F._h
    assert L.bmpc_est_set_stream(h, stream.cuda_stream) == 0
    kern, meas, upd = [], [], []
    for r in range(reps):
        ks, ms, us = [], [], []
        for t in range(warmup + steps):
            ev_u = None
            if models is not None:
                A, B = models[t % len(models)]
                ev_u = timed(torch, stream, lambda: F.update_system_from_device(A=A, B=B))
            ev_p = timed(torch, stream, lambda: F.predict_device(U.data_ptr()))
            ev_m = timed(torch, stream, lambda: F.update_device(Y.data_ptr()))
            stream.synchronize()
            if t >= warmup:
                ks.append(ev_p[0].elapsed_time(ev_m[1])); ms.append(ev_m[0].elapsed_time(ev_m[1]))
                if ev_u:
                    us.append(ev_u[0].elapsed_time(ev_u[1]))
        kern.append(ks); meas.append(ms); upd.append(us)
    out = {"predict_update_kernels": spread(kern), "update_call": spread(meas)}
    if models is not None:
        out["update_system_from_device"] = spread(upd)
    st = F.status
    out["status_ok"] = int((st == 1).sum())
    return out


def ltv_loop(torch, B, steps, warmup, with_filter, flush):
    from pympc_b200 import MPCController as MPC
    from pympc_b200.kalman import KalmanFilter
    from pympc_b200.workloads import cartpole_rhs, cartpole_linearised, CARTPOLE, pendulum_random
    Ts = CARTPOLE[6]; dev = torch.device("cuda", 0)
    X0, Xref = pendulum_random(B, seed=2026)
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
    F = None
    if with_filter:
        F = KalmanFilter(X0, Ad0, Bd0, C2, None, 1e-6 * np.eye(4), 1e-6 * np.eye(2), P0=1e-4 * np.eye(4))
        F.attach(K)
    C2d = torch.tensor(C2, device=dev)
    Xd = torch.tensor(X0, device=dev)
    Ubuf = torch.zeros((2, B, 1), dtype=torch.float64, device=dev)
    ev = []
    for t in range(warmup + steps):
        Uprev = Ubuf[(t & 1) ^ 1]
        assert L.bmpc_bind_output(h, Ubuf[t & 1].data_ptr()) == 0
        if t > 0:
            Xd = rk4(Xd, Uprev)
        Ad_t, Bd_t = cartpole_linearised(Xd, Uprev)
        Ad_t, Bd_t = Ad_t.contiguous(), Bd_t.contiguous()
        Y = (Xd @ C2d.T).contiguous()
        flush.zero_()
        torch.cuda.synchronize(dev)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        assert L.bmpc_update_system(h, Ad_t.data_ptr(), Bd_t.data_ptr(), 1) == 0, L.bmpc_last_error(h)
        if F is not None:                     # x[t-1|t-1] -> x[t|t-1] with u_{t-1}, then the measurement of step t
            F.update_system_from_device(A=Ad_t, B=Bd_t)
            assert t == 0 or F.predict_device(Uprev.data_ptr()) == 0
            assert F.update_device(Y.data_ptr()) == 0
        assert L.bmpc_update(h, Xd.data_ptr(), Uprev.data_ptr(), None, 1, 2) == 0
        assert L.bmpc_solve(h) == 0, L.bmpc_last_error(h)
        assert L.bmpc_output(h, None, None, 1, 1) == 0
        e1.record(stream)
        e1.synchronize()
        if t >= warmup:
            ev.append(e0.elapsed_time(e1))
    torch.cuda.synchronize(dev)
    out = {"event_ms_median": float(np.median(ev)), "event_ms_mean": float(np.mean(ev)), "event_ms_min": float(np.min(ev)),
           "event_ms_max": float(np.max(ev)), "steps": len(ev)}
    if F is not None:
        F.close()
    torch.cuda.set_stream(torch.cuda.default_stream(dev))
    K.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--loop-steps", type=int, default=20)
    ap.add_argument("--redesign-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from pympc_b200.kalman import KalmanFilter, LinearStateEstimator, kalman_design_simple
    from pympc_b200.workloads import cartpole_linearised, mimo, pendulum_random
    dev = torch.device("cuda", 0)
    torch.zeros(1, device=dev)
    rec = {"tool": "bench_kf", **card(), "timing": "CUDA events on one explicit stream; per repetition the median step, reported "
           "as median / min / max over repetitions", "workloads": {}}
    stream = torch.cuda.Stream(dev)
    # --- cart-pole fleet, model from device arrays every step
    B = 65536
    X0, _ = pendulum_random(B, seed=7)
    rng = np.random.default_rng(1)
    with torch.cuda.stream(stream):
        Xs = [torch.tensor(X0 * s, device=dev) for s in np.linspace(1.0, 0.2, 8)]
        U = torch.tensor(0.1 * rng.standard_normal((B, 1)), device=dev)
        models = [tuple(m.contiguous() for m in cartpole_linearised(x, U)) for x in Xs]
        Y = torch.tensor(X0 @ C2.T + 0.01 * rng.standard_normal((B, 2)), device=dev)
    stream.synchronize()
    A0, B0 = [m.cpu().numpy() for m in models[0]]
    F = KalmanFilter(X0, A0, B0, C2, None, 1e-6 * np.eye(4), 1e-6 * np.eye(2), P0=1e-4 * np.eye(4))
    rec["workloads"]["cartpole"] = {"batch": B, "nx": 4, "nu": 1, "ny": 2, "model": "per instance, replaced from device arrays "
                                    "every step", **filter_steps(torch, F, stream, U, Y, models, args.steps, args.warmup, args.reps)}
    F.close()
    # --- governor fleet, shared model
    Bg = 16384; g = mimo(); Cg = np.zeros((4, 8))
    for i in range(4):
        Cg[i, 2 * i + 1] = 1.0
    Fg = KalmanFilter(np.zeros((Bg, 8)), g["Ad"], g["Bd"], Cg, None, 0.1 * np.eye(8), 0.5 * np.eye(4), batch=Bg)
    with torch.cuda.stream(stream):
        Ug = torch.tensor(rng.standard_normal((Bg, 4)), device=dev); Yg = torch.tensor(rng.standard_normal((Bg, 4)), device=dev)
    stream.synchronize()
    rec["workloads"]["governor"] = {"batch": Bg, "nx": 8, "nu": 4, "ny": 4, "model": "shared",
                                    **filter_steps(torch, Fg, stream, Ug, Yg, None, args.steps, args.warmup, args.reps)}
    Fg.close()
    # --- the LTV loop of bench_ltv without and with the filter, alternated
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    runs = {"without_filter": [], "with_filter": []}
    for r in range(2):
        for name, wf in (("without_filter", False), ("with_filter", True)):
            runs[name].append(ltv_loop(torch, B, args.loop_steps, 5, wf, flush))
    rec["workloads"]["ltv_loop"] = {"batch": B, "Np": 20, "l2": "flushed between timed steps (256 MiB write)", "runs": runs}
    # --- today's alternative: re-design + new estimator per step
    Qn, Rn = 1e-6 * np.eye(4), 1e-6 * np.eye(2)
    wall = []
    for t in range(1 + args.redesign_steps):
        A, Bm = [m.cpu().numpy() for m in models[t % len(models)]]
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        Lg, _, _ = kalman_design_simple(A, Bm, C2, None, Qn, Rn, type='filter')
        E = LinearStateEstimator(X0, A, Bm, C2, None, Lg)
        E.predict(np.zeros((B, 1))); E.update(np.zeros((B, 2)))
        w1 = time.perf_counter()
        E.close()
        if t > 0:
            wall.append(1e3 * (w1 - w0))
    rec["workloads"]["redesign"] = {"batch": B, "wall_ms_median": float(np.median(wall)), "wall_ms_min": float(min(wall)),
                                    "wall_ms_max": float(max(wall)), "steps": len(wall),
                                    "timing": "host wall clock of kalman_design_simple + LinearStateEstimator + predict + update, "
                                              "synchronised"}
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
