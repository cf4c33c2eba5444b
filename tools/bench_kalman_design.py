"""Batched Kalman design on the GPU (bmpc_dare / k_dare, csrc/bmpc_dare.cuh) against per-instance scipy on the host.

Two seeded workloads of per-instance plants:
  pend  65 536 inverted pendulums of the reference's Kalman example (Ts = 5 ms, C = [[1,0,0,0],[0,0,1,0]], Q = 10 I, R = I), each
        perturbed like test_per_instance_systems_vs_oracle (non-zeros of Ad by 1 %, Bd by 10 %)
  mimo  16 384 MIMO block systems (pympc_b200.workloads.mimo, nx = 8, ny = 4 outputs x[2i+1]), perturbed the same way
For each: k_dare's own device time (torch.profiler, CUDA activities, a run of its own after a warm-up), the host wall clock of one
bmpc_dare call (copies and synchronise included) and of kalman_design_simple end to end, mean / max doubling steps, the largest
relative difference to the scipy oracle on 256 instances, and scipy's time per instance on the same inputs (single process, the
baseline).  The card's name and power limit are read in the same run.  Prints one JSON line; --out FILE also writes it there.

usage: python tools/bench_kalman_design.py [--reps 20] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception as exc:                                   # the power limit is part of the number: say it is missing
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({exc})"}


def perturb(rng, b, Ad, Bd):
    A = np.stack([Ad + 0.01 * rng.standard_normal(Ad.shape) * (Ad != 0) for _ in range(b)])
    B = np.stack([Bd * (1 + 0.1 * rng.standard_normal()) for _ in range(b)])
    return A, B


def workloads():
    from pympc_b200.workloads import mimo
    M, m, b, ftheta, l, g, Ts = 0.5, 0.2, 0.1, 0.1, 0.3, 9.81, 5e-3
    Ac = np.array([[0, 1, 0, 0],
                   [0, -b / M, -(g * m) / M, (ftheta * m) / M],
                   [0, 0, 0, 1],
                   [0, b / (M * l), (M * g + g * m) / (M * l), -(M * ftheta + ftheta * m) / (M * l)]])
    Bc = np.array([[0.0], [1.0 / M], [0.0], [-1 / (M * l)]])
    A, B = perturb(np.random.default_rng(2026), 65536, np.eye(4) + Ac * Ts, Bc * Ts)
    yield "pend", A, B, np.array([[1.0, 0, 0, 0], [0, 0, 1.0, 0]]), 10 * np.eye(4), np.eye(2)
    c = mimo()
    A, B = perturb(np.random.default_rng(2027), 16384, c["Ad"], c["Bd"])
    C = np.zeros((4, 8)); C[np.arange(4), 2 * np.arange(4) + 1] = 1.0
    yield "mimo", A, B, C, 10 * np.eye(8), np.eye(4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from pympc_b200 import _lib
    from pympc_b200.kalman import kalman_design_simple
    from oracle.kalman_design import dare as odare, kalman_design_simple as okds
    L = _lib.load()
    assert L.bmpc_device_count() > 0, "needs a CUDA device"
    torch.zeros(1, device="cuda")
    rec = {"tool": "bench_kalman_design", **card(), "reps": args.reps, "workloads": {}}
    for name, A, B, C, Q, R in workloads():
        b, n = A.shape[0], A.shape[1]; m = C.shape[0]
        # the filter DARE of kalman_design_simple: dare(A', C', Q, R)
        At = np.ascontiguousarray(A.transpose(0, 2, 1)); Ct = np.ascontiguousarray(np.broadcast_to(C.T, (b, n, m)))
        Qb = np.ascontiguousarray(np.broadcast_to(Q, (b, n, n))); Rb = np.ascontiguousarray(np.broadcast_to(R, (b, m, m)))
        X = np.empty((b, n, n)); G = np.empty((b, m, n)); st = np.empty(b, np.int32); it = np.empty(b, np.int32)
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        call = lambda: L.bmpc_dare(n, m, b, 0, p(At), p(Ct), p(Qb), p(Rb), None, p(X), p(G), p(st), p(it))
        for _ in range(3):
            assert call() == 0
        wall = []
        for _ in range(args.reps):
            t0 = time.perf_counter(); assert call() == 0; wall.append(time.perf_counter() - t0)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                assert call() == 0
            torch.cuda.synchronize()
        kern = [e for e in prof.key_averages() if "k_dare" in e.key]
        k_us = sum(e.device_time_total for e in kern) / max(1, sum(e.count for e in kern))
        # end to end through the Python layer
        kalman_design_simple(A, None, C, None, Q, R)
        e2e = []
        for _ in range(max(3, args.reps // 4)):
            t0 = time.perf_counter(); Lg, P, W = kalman_design_simple(A, None, C, None, Q, R); e2e.append(time.perf_counter() - t0)
        # accuracy on 256 instances and the scipy baseline on the same inputs
        idx = np.random.default_rng(1).choice(b, 256, replace=False)
        err_L = err_P = 0.0
        t0 = time.perf_counter()
        for i in idx:
            Lr, Pr, _ = okds(A[i], None, C, None, Q, R)
            err_L = max(err_L, np.abs(Lg[i] - Lr).max() / np.abs(Lr).max()); err_P = max(err_P, np.abs(P[i] - Pr).max() / np.abs(Pr).max())
        t_oracle = (time.perf_counter() - t0) / len(idx)
        t0 = time.perf_counter()
        for i in idx:
            odare(At[i], Ct[i], Q, R)
        t_scipy = (time.perf_counter() - t0) / len(idx)
        rec["workloads"][name] = {
            "batch": b, "n": n, "m": m, "solved": int((st == 1).sum()),
            "steps_mean": float(it.mean()), "steps_max": int(it.max()),
            "k_dare_device_ms": k_us / 1e3, "k_dare_launches_profiled": int(sum(e.count for e in kern)),
            "bmpc_dare_call_ms_median": 1e3 * float(np.median(wall)),
            "kalman_design_simple_ms_median": 1e3 * float(np.median(e2e)),
            "max_rel_err_L_vs_oracle_256": err_L, "max_rel_err_P_vs_oracle_256": err_P,
            "scipy_dare_ms_per_instance": 1e3 * t_scipy, "scipy_kalman_design_simple_ms_per_instance": 1e3 * t_oracle,
            "scipy_dare_full_batch_s_extrapolated": t_scipy * b,
        }
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
