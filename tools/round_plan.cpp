// C entry point of the solver's round policy (pympc_b200/csrc/bmpc_rounds.cuh) for the Python studies and tests: g++ builds the
// header on its own (tools/round_plan.py), no CUDA library and no emulation of the kernels needed.
#include <string.h>
#include "../pympc_b200/csrc/bmpc_rounds.cuh"

// the plan of the next round for a handle of the given family and options: out[10] = admm, chunk, polish, ws, capA, capB, cap,
// exchange, reset, infeas.  Returns 0 when the solve's iteration budget is spent.
extern "C" int round_plan(int family, int polish, int first_iters, int cold_iters, int max_iter, int pdas_steps, int shift_warm,
                          int round, int total, int cold, int codes_valid, int* out) {
    const BmpcPolicy P = bmpc_make_policy(family, polish, first_iters, cold_iters, max_iter, pdas_steps, shift_warm);
    BmpcRoundPlan r;
    if (!bmpc_plan_round(P, BmpcSolveState{round, total, cold != 0, codes_valid != 0}, &r)) return 0;
    const int v[10] = {r.admm, r.chunk, r.polish, r.ws, r.capA, r.capB, r.cap, r.exchange, r.reset, r.infeas};
    memcpy(out, v, sizeof(v));
    return 1;
}
