"""Per-instance multi-input fleets: what a step costs on the multi-input fast path (k_tpm_pol on per-instance parameter views,
fast_path=1) against the team kernels (fast_path=0).

Workloads (per-instance systems, n_sys = batch):
  W1  4 096 MIMO reference governors (8,4,40,40), each Ad / Bd perturbed inside the governor's sparsity pattern, with its own Qx scale,
      umax, Dumax and uref; the closed loop from x0 = 0.3 N(0, 1): the transient steps 4-13 and a settled window (steps 40-49)
  W2  16 384 such systems at (8,4,12,5)
  W3  W1 with update_system_from_device(Ad, Bd) every step (the model drifts by 1e-4 relative per step, torch on the device)
Method (bench.py's, DESIGN.md §5): device-resident x0 and u_-1 read in place, u* written into a device buffer, one explicit stream for
the solver and the CUDA events around each step, 256 MiB written between timed steps (outside the events) to flush L2.  The modes
alternate on the same seeds; the second mode of a pair is driven through the first one's states and inputs, so u* is compared on the
same problems (instances both verified, the whole batch, every timed step).  Per mode: event ms per step (mean, median), the update
call's own event time (W3), rounds, ADMM iterations, refinements, instances re-condensed and unverified, device memory in use.  The
card's name, power limit and SM clock are read in the same run.  Prints one JSON line; --out FILE also writes it there.

usage: python tools/bench_mimo_fleet.py [--w1 4096] [--w2 16384] [--pairs 2] [--out profiles/mimo_fleet_h100.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
W = ("Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax")
TRANSIENT = range(4, 14)
SETTLED = range(40, 50)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk, mx = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": pl, "sm_clock_at_start": clk, "max_sm_clock": mx}
    except Exception as exc:                                   # the power limit is part of the number: say it is missing
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({exc})"}


def fleet(B, Np, Nc, seed):
    from pympc_b200.workloads import mimo
    rng = np.random.default_rng(seed)
    c = dict(mimo(), Np=Np, Nc=Nc); c["Qu"] = 0.01 * np.eye(4)
    Ad = c["Ad"][None] * (1.0 + 0.002 * rng.standard_normal((B, 8, 8)))   # (DC gain 1 - a1 - a2 = 0.046: +-8 %)
    Bd = c["Bd"][None] * (1.0 + 0.1 * rng.standard_normal((B, 8, 4)))
    s = rng.uniform(0.5, 2.0, B)[:, None, None]
    umax = rng.uniform(1.5, 3.0, (B, 4)); Dumax = rng.uniform(0.1, 0.3, (B, 4))
    P = dict(Qx=s * c["Qx"], QxN=s * c["QxN"], umin=-umax, umax=umax, Dumin=-Dumax, Dumax=Dumax, uref=0.05 * rng.standard_normal((B, 4)))
    return c, Ad, Bd, P, 0.3 * rng.standard_normal((B, 8))


def run(torch, MPC, fast_path, work, steps, drift, flush, drive=None):
    """one mode of one workload; drive: the (x0, u_-1) of every step from the other mode (else the loop follows its own plan)"""
    c, Ad, Bd, P, X0 = work
    B = X0.shape[0]; dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    torch.cuda.synchronize(dev); torch.cuda.set_stream(stream)
    K = MPC(Ad, Bd, Np=c["Np"], Nc=c["Nc"], x0=X0, xref=c["xref"], uminus1=np.zeros(4), batch=B, fast_path=fast_path, **{k: c[k] for k in W})
    K.setup(solve=False); K.update_system(**P)
    L, h = K._L, K.handle
    assert L.bmpc_set_stream(h, stream.cuda_stream) == 0
    Ad_d = torch.tensor(Ad, device=dev); Bd_d = torch.tensor(Bd, device=dev)
    Xd = torch.tensor(X0, device=dev); Ubuf = torch.zeros((2, B, 4), dtype=torch.float64, device=dev)
    g = torch.Generator(device=dev); g.manual_seed(7)
    rec = {"ev": [], "upd": [], "st": [], "u": [], "drive": [], "mem": 0}
    for t in range(steps):
        Uprev = Ubuf[(t & 1) ^ 1]
        if drive is not None:
            Xd.copy_(drive[t][0]); Uprev.copy_(drive[t][1])
        elif t > 0:
            Xd = torch.einsum("bij,bj->bi", Ad_d, Xd) + torch.einsum("bij,bj->bi", Bd_d, Uprev)
        if drift and t > 0:
            Ad_d = Ad_d * (1.0 + 1e-4 * torch.randn(Ad_d.shape, generator=g, device=dev, dtype=torch.float64))
        assert L.bmpc_bind_output(h, Ubuf[t & 1].data_ptr()) == 0
        flush.zero_()
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        torch.cuda.synchronize(dev)
        e0.record(stream)
        if drift:
            K.update_system_from_device(Ad_d, Bd_d)
        e1.record(stream)
        assert L.bmpc_update(h, Xd.data_ptr(), Uprev.data_ptr(), None, 1, 2) == 0
        assert L.bmpc_solve(h) == 0, L.bmpc_last_error(h)
        assert L.bmpc_output(h, None, None, 1, 1) == 0
        e2.record(stream)
        e2.synchronize()
        rec["ev"].append(e0.elapsed_time(e2)); rec["upd"].append(e0.elapsed_time(e1)); rec["st"].append(K.stats())
        stat = np.empty(B, np.int32)
        assert L.bmpc_output(h, None, stat.ctypes.data, 0, 0) == 0
        rec["u"].append((Ubuf[t & 1].cpu().numpy().copy(), stat))
        rec["drive"].append((Xd.clone(), Uprev.clone()))
        if t == 0:
            rec["mem"] = torch.cuda.mem_get_info(dev)
    torch.cuda.synchronize(dev); torch.cuda.set_stream(torch.cuda.default_stream(dev))
    K.close()
    return rec


def summary(rec, window):
    st = [rec["st"][t] for t in window]; ev = [rec["ev"][t] for t in window]; up = [rec["upd"][t] for t in window]
    f = lambda k: [s[k] for s in st]
    free, total = rec["mem"]
    return {"steps": list(window)[0:1] + list(window)[-1:], "ms_mean": float(np.mean(ev)), "ms_median": float(np.median(ev)),
            "update_ms_mean": float(np.mean(up)), "update_ms_median": float(np.median(up)),
            "rounds_mean": float(np.mean(f("rounds"))), "admm_iters_mean": float(np.mean(f("admm_iters"))),
            "refinements_mean": float(np.mean(f("polish_steps"))), "recondensed_mean": float(np.mean(f("recondensed"))),
            "unsolved_mean": float(np.mean(f("unsolved"))), "device_mem_in_use_gb": round((total - free) / 2**30, 2)}


def agreement(a, b, window):
    d = 0.0; n = 0
    for t in window:
        (ua, sa), (ub, sb) = a["u"][t], b["u"][t]
        both = (sa == 1) & (sb == 1); n += int(both.sum())
        if both.any():
            d = max(d, float(np.max(np.abs(ua[both] - ub[both]))))
    return {"max_abs_diff_u": d, "instances_compared": n}


def workload(torch, MPC, name, work, steps, drift, flush, pairs, windows):
    out = {"modes": {}, "pairs": []}
    drive = None
    for p in range(pairs):
        pair = {}
        for fp in ((1, 0) if p % 2 == 0 else (0, 1)):
            rec = run(torch, MPC, fp, work, steps, drift, flush, drive)
            if drive is None:
                drive = rec["drive"]
            pair[fp] = rec
            out["modes"].setdefault(f"fast_path={fp}", []).append({w: summary(rec, r) for w, r in windows.items()})
        out["pairs"].append({w: agreement(pair[1], pair[0], r) for w, r in windows.items()})
        del pair
    print(name, json.dumps(out)[:400], file=sys.stderr)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--w1", type=int, default=4096)
    ap.add_argument("--w2", type=int, default=16384)
    ap.add_argument("--pairs", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from pympc_b200 import MPCController as MPC
    dev = torch.device("cuda", 0)
    torch.zeros(1, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    rec = {"tool": "bench_mimo_fleet", **card(), "l2": "flushed between timed steps (256 MiB write)",
           "timing": "CUDA events around update_system_from_device (W3) + update + solve + output, per step", "workloads": {}}
    win = {"transient": TRANSIENT, "settled": SETTLED}
    rec["workloads"]["W1"] = dict(batch=args.w1, shape=[8, 4, 40, 40], **workload(torch, MPC, "W1", fleet(args.w1, 40, 40, 1), 50, False, flush, args.pairs, win))
    rec["workloads"]["W2"] = dict(batch=args.w2, shape=[8, 4, 12, 5], **workload(torch, MPC, "W2", fleet(args.w2, 12, 5, 2), 50, False, flush, args.pairs, win))
    rec["workloads"]["W3"] = dict(batch=args.w1, shape=[8, 4, 40, 40], update="update_system_from_device(Ad, Bd) every step",
                                  **workload(torch, MPC, "W3", fleet(args.w1, 40, 40, 1), 50, True, flush, args.pairs, win))
    rec["card_after"] = card()
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
