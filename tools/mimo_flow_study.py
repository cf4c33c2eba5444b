"""Host emulation of the multi-input fast path's round loop on the MIMO side bench's workload, with the device code compiled for the
host and every round's chunk, cap and update mode as the library plans it (pympc_b200/csrc/bmpc_rounds.cuh, through
tools/round_plan.py): cold solve = [tile ADMM -> polish from the iterate] rounds; warm solve = [polish from the shifted
sets] then straggler rounds [ADMM -> polish from the iterate].  Prints the distribution of rounds per solve and how many instances
would fall through to the Schur-form polish.
Usage: python tools/mimo_flow_study.py [instances] [warm steps]"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests", "hostemu"))
from emu import EmuSystem                       # noqa: E402
from round_plan import plan_round               # noqa: E402
from pympc_b200.workloads import mimo           # noqa: E402


def _riccati_plan(r, total, cold):
    """the library's plan of round r, or None once the Schur-form polish takes over"""
    p = plan_round("tpm", r, total, cold)
    return p if p is not None and p["polish"] == "tpm" else None


def _polish(E, cfg, x, um1, p, mode):
    return E.tpm_step(x, um1, cfg["xref"], mode=mode, max_ref=p["cap"], exchange_from=0 if p["exchange"] else -1)


def cold_solve(E, cfg, x, um1):
    """returns (U or None when the instance would go on to the Schur-form polish, rounds, ADMM iterations)"""
    total = 0; r = 0
    while (p := _riccati_plan(r, total, cold=True)) is not None:
        E.admm_only(x, um1, cfg["xref"], p["chunk"]); total += p["chunk"]
        vs = E.v.copy()
        if hasattr(E, "mcodes"):
            del E.mcodes
        U, ps = _polish(E, cfg, x, um1, p, mode=2)
        r += 1
        if ps > 0:
            return U, r, total
        E.v = vs
    return None, r, total


def warm_solve(E, cfg, x, um1, codes, plan):
    p = _riccati_plan(0, 0, cold=False)
    assert p["admm"] == "none" and p["ws"] == "record"
    E.mcodes, E.Uplan = codes.copy(), plan.copy(); vprev = E.v.copy()
    U, ps = _polish(E, cfg, x, um1, p, mode=1)
    if ps > 0:
        return U, 1, 0
    E.v = vprev; E.x = plan.copy(); E.cold = 0; E.lvl = 2
    total = 0; r = 1
    while (p := _riccati_plan(r, total, cold=False)) is not None:
        E.admm_only(x, um1, cfg["xref"], p["chunk"]); total += p["chunk"]
        vs = E.v.copy()
        U, ps = _polish(E, cfg, x, um1, p, mode=2)
        r += 1
        if ps > 0:
            return U, r, total
        E.v = vs
    return None, r, total


def run(n, steps, seed=4):
    cfg = mimo(); rng = np.random.default_rng(seed); X0 = 0.3 * rng.standard_normal((16384, 8))
    rc, rw, itc, itw = [], [], [], []; fall = 0
    for b in range(n):
        E = EmuSystem(cfg); x = X0[b].copy(); um1 = np.zeros(4)
        U, r, it = cold_solve(E, cfg, x, um1); rc.append(r); itc.append(it)
        if U is None:
            fall += 1; continue
        for t in range(steps):
            codes, plan = E.mcodes.copy(), U.copy()
            um1 = U[:4].copy(); x = cfg["Ad"] @ x + cfg["Bd"] @ um1
            U, r, it = warm_solve(E, cfg, x, um1, codes, plan); rw.append(r); itw.append(it)
            if U is None:
                fall += 1; break
    return dict(fallthrough=fall, cold_rounds=np.bincount(rc), warm_rounds=np.bincount(rw), cold_iters=float(np.mean(itc)),
                warm_iters=float(np.mean(itw)) if itw else 0.0)


if __name__ == "__main__":
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 100
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    t0 = time.time(); r = run(n, steps)
    print(f"instances {n}: to the Schur-form fallback {r['fallthrough']} | cold solves by rounds {r['cold_rounds']}, {r['cold_iters']:.0f} ADMM iterations"
          f" | warm solves by rounds {r['warm_rounds']}, {r['warm_iters']:.1f} iterations  [{time.time() - t0:.0f} s]")
