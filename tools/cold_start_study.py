"""Host-emulation study of the COLD first solve on the multi-input fast path (bmpc_rounds.cuh: tile ADMM chunk -> k_tpm_pol from the
iterate -> straggler rounds): ADMM iterations, rounds and refinements until an instance verifies, by first chunk and refinement cap per
round; the library's own point (first chunk and cold cap of its policy) is marked.  Result (48 random MIMO starts): cap 4 never verifies
in the first round (333 iterations, 4.5 rounds per solve); cap 24 after 25 iterations verifies all of them at once -> the policy's
tpm_cold_cap = 24 and cold chunk 25.  Usage: python tools/cold_start_study.py [n]"""
import os, sys, numpy as np, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests", "hostemu"))
from emu import EmuSystem
from round_plan import plan_round
from pympc_b200.workloads import mimo
cfg=mimo(); rng=np.random.default_rng(7); B=int(sys.argv[1]) if len(sys.argv)>1 else 48
first=plan_round("tpm",0,0,cold=True); lib=(first["chunk"],(first["cap"],))
# emulate the device's cold flow: first chunk c0, then chunks doubling the total; polish cap per round
def flow(c0, caps, x0):
    E=EmuSystem(cfg); um1=np.zeros(4); total=0; chunk=c0; cost_ref=0; r=0
    while total<800:
        E.admm_only(x0,um1,cfg["xref"],chunk); total+=chunk
        cap=caps[min(r,len(caps)-1)]
        vs=E.v.copy()
        if hasattr(E,"mcodes"): del E.mcodes
        U,ps=E.tpm_step(x0,um1,cfg["xref"],mode=2,max_ref=cap)
        cost_ref+= ps if ps>0 else cap
        if ps>0: return total, r+1, cost_ref
        E.v=vs; r+=1; chunk=total
    return total, r, cost_ref
X=[0.3*rng.standard_normal(8) for _ in range(B)]
grid=[(c0,caps) for c0 in (25,50) for caps in ((4,),(8,),(12,),(16,),(24,),(12,4),(16,8))]
if lib not in grid: grid.insert(0,lib)
for c0,caps in grid:
    out=[flow(c0,caps,x) for x in X]
    it=np.array([o[0] for o in out]); rd=np.array([o[1] for o in out]); rf=np.array([o[2] for o in out])
    print(f"c0={c0} caps={caps}: mean iters {it.mean():.0f} max {it.max()}, rounds mean {rd.mean():.2f} max {rd.max()}, verified in round 1: {(rd==1).mean()*100:.0f} %, refinements mean {rf.mean():.1f}"
          + ("  <- library policy" if (c0,caps)==lib else ""))
