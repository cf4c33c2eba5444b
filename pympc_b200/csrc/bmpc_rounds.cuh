// bmpc_rounds.cuh — the round policy of a solve: which kernels each round runs, with which chunk, caps and working sets.
// Host code only, plain C++ (no CUDA types): libbmpc.so decides every round with bmpc_plan_round and the host emulation
// (tests/hostemu) runs the same function, so a policy change is made here once and the emulation measures the library's own policy.
//
// A solve runs in rounds.  A round is an optional ADMM chunk followed by one polish attempt over the instances that are still
// open; the first round covers the whole batch, the later ("straggler") rounds only the listed instances.
#pragma once
#include <stdio.h>
#include <stdlib.h>

// kernel family of a handle, chosen by bmpc_setup from the shape and the options
enum BmpcFamily {
    BMPC_FAM_TPI,        // single-input fast path, one shared system: k_tpi_admm + k_tpi_pol, the stragglers on the team ADMM
    BMPC_FAM_TPI_VIEW,   // single-input fast path, per-instance systems: k_tpi_pol on parameter views, every ADMM chunk on the team kernels
    BMPC_FAM_TPM,        // multi-input fast path (one shared system): k_tpm_pol after the team / tile ADMM
    BMPC_FAM_TEAM        // team / tile kernels with the Schur-form polish
};

// refinements allowed per Schur-form polish attempt: the configured count in the first two rounds of a solve (every instance passes
// there), three times as many for the instances that come back from further ADMM rounds (few, and single exchanges need the room)
inline int bmpc_polish_steps(int pdas_steps, int round) { return round >= 2 ? 3 * pdas_steps : pdas_steps; }

// per-handle policy, fixed at bmpc_setup
struct BmpcPolicy {
    int family;                                                   // BmpcFamily
    int polish, first_iters, cold_iters, max_iter, pdas_steps, shift_warm;   // the bmpc_config options of the same names
    // first chunk when first_iters is 0: a warm team solve (a warm fast-path solve starts with the polish alone: measured 0 vs
    // 1..10 iterations, DESIGN.md); a cold team / tile solve (10 iterations from the free response leave working sets of hundreds of
    // rows for the Schur polish: 180 ms launches on the MIMO shape); a cold fast-path solve (no active-set guess to refresh: 25 at
    // once, so that the first polish usually verifies and the whole batch does not take the straggler route).  cold_iters replaces
    // the cold chunk of the team and multi-input families.
    int warm_chunk = 10, cold_chunk = 50, fast_cold_chunk = 25;
    int round_total = 25;       // straggler rounds: the first brings the total to 25 iterations, each later one doubles it
    int check_chunk = 25;       // pure ADMM (polish = 0): OSQP's check_termination interval
    int infeas_after = 25;      // infeasible instances never pass the polish: straggler rounds look for OSQP's certificate from here on
    int schur_after = 200;      // the fast-path families polish their stragglers with the Riccati polish while the total stays within this
    // k_tpi_pol refinements per attempt (phase A + phase B), twice as many in a cold solve, which reads its working sets off a rough
    // ADMM iterate (host study on 300 random pendulum starts, first polish after 25 iterations: 88 % verify within 8 refinements,
    // 99 % within 16, at most 3 rounds instead of 5)
    int tpi_steps = 8;
    // k_tpm_pol: refinements of the first launch of a warm solve / of a straggler round, ADMM iterations of the first straggler round.
    // (12, 12, 100) was chosen in host emulation with the straggler rounds in exchange mode, where 12 refinements finish every
    // straggler of the study in the first round (all-at-once, cap 4: 54 %, three rounds for the rest); before exchange mode,
    // (12, 4, 100) measured 11.4 ms/step on the MIMO side bench against 13.3 ms at (8, 6, 25) (tools/sweep_tpm_caps.sh).
    int tpm_first_cap = 12, tpm_round_cap = 12, tpm_chunk = 100;
    // every attempt of a cold solve: working sets read off a rough ADMM iterate need 8 - 14 refinements, not 4 (host study on 48
    // random MIMO starts, first polish after 25 iterations: cap 4 verifies none and the solve takes 333 iterations in 4.5 rounds,
    // cap 12 79 %, cap 16 92 %, cap 24 all of them in the first round; after 50 iterations the same picture)
    int tpm_cold_cap = 24;
};

inline BmpcPolicy bmpc_make_policy(int family, int polish, int first_iters, int cold_iters, int max_iter, int pdas_steps, int shift_warm) {
    BmpcPolicy p;
    p.family = family; p.polish = polish; p.first_iters = first_iters; p.cold_iters = cold_iters; p.max_iter = max_iter;
    p.pdas_steps = pdas_steps; p.shift_warm = shift_warm;
    if (family == BMPC_FAM_TPM)         // tuning knob (tools/sweep_tpm_caps.sh): first cap, round cap, first straggler chunk, cold cap
        if (const char* e = getenv("BMPC_TPM_CAPS")) sscanf(e, "%d,%d,%d,%d", &p.tpm_first_cap, &p.tpm_round_cap, &p.tpm_chunk, &p.tpm_cold_cap);
    return p;
}

// progress of the solve in flight
struct BmpcSolveState {
    int round;          // rounds run so far
    int total;          // ADMM iterations so far (every open instance has run all of them)
    bool cold;          // the solve started cold (no previous solution to start from)
    bool codes_valid;   // the stored working sets come from a fast-path polish of the whole batch
};

enum BmpcAdmmKind { BMPC_ADMM_NONE, BMPC_ADMM_TPI, BMPC_ADMM_TEAM };   // none, k_tpi_admm, team / tile kernels (launch_admm)
enum BmpcPolishKind { BMPC_POL_TPI, BMPC_POL_TPM, BMPC_POL_SCHUR, BMPC_POL_CHECK };   // k_tpi_pol, k_tpm_pol, k_polish, k_check_converged
// working sets of the Riccati polishes (their mode argument): stored, stored and shifted one stage (receding horizon), read off the
// iterate v; k_tpm_pol's first launch: per instance the stored record shifted, else read off the previous v*, shifted
enum { BMPC_WS_RECORD = -1, BMPC_WS_STORED = 0, BMPC_WS_SHIFTED = 1, BMPC_WS_FROM_V = 2 };

struct BmpcRoundPlan {
    int admm, chunk;    // BmpcAdmmKind, iterations (a team chunk of 0 still runs the per-step prep)
    int polish;         // BmpcPolishKind
    int ws;             // k_tpi_pol / k_tpm_pol: working-set source (BMPC_WS_*)
    int capA, capB;     // k_tpi_pol: refinements of phase A (all rows at once) and phase B
    int cap;            // k_tpm_pol: refinements; k_polish: refinement steps
    int exchange;       // k_tpm_pol: hard rows change by single exchanges instead of all at once
    int reset;          // the round's first kernel resets the per-instance state and snapshots u_-1 (the first round)
    int infeas;         // the ADMM chunk is bracketed by the check of OSQP's infeasibility certificate
};

// The next round of a solve, or false when its iteration budget is spent (the first round is always planned).  The caller
// stops as well when no instance is left open.
inline bool bmpc_plan_round(const BmpcPolicy& p, const BmpcSolveState& s, BmpcRoundPlan* r) {
    if (s.round > 0 && s.total >= p.max_iter) return false;
    const bool tpi = p.family == BMPC_FAM_TPI || p.family == BMPC_FAM_TPI_VIEW, tpm = p.family == BMPC_FAM_TPM;
    int chunk;
    if (!p.polish) chunk = p.check_chunk;
    else if (s.round == 0 && p.first_iters > 0) chunk = p.first_iters;
    else if (s.round == 0 && !s.cold) chunk = tpi || tpm ? 0 : p.warm_chunk;
    else if (s.round == 0) chunk = tpi ? p.fast_cold_chunk : p.cold_iters > 0 ? p.cold_iters : tpm ? p.fast_cold_chunk : p.cold_chunk;
    else if (tpm && s.total == 0) chunk = p.tpm_chunk;
    else chunk = s.total < p.round_total ? p.round_total - s.total : s.total;
    if (chunk > p.max_iter - s.total) chunk = p.max_iter - s.total;
    *r = BmpcRoundPlan();
    r->chunk = chunk;
    r->reset = s.round == 0;
    const int tpi_steps = s.cold ? 2 * p.tpi_steps : p.tpi_steps;
    // first round on the single-input fast path: k_tpi_pol alone on the stored working sets, or after k_tpi_admm (shared system only:
    // its matrices live in the constant bank) from the iterate
    if (s.round == 0 && p.polish && tpi && (p.family == BMPC_FAM_TPI || chunk == 0)) {
        r->admm = chunk > 0 ? BMPC_ADMM_TPI : BMPC_ADMM_NONE;
        r->polish = BMPC_POL_TPI;
        r->ws = chunk > 0 || !s.codes_valid ? BMPC_WS_FROM_V : p.shift_warm ? BMPC_WS_SHIFTED : BMPC_WS_STORED;
        r->capA = 1; r->capB = tpi_steps - 1;
        return true;
    }
    // warm first round on the multi-input fast path: k_tpm_pol alone (no prep, no ADMM)
    if (s.round == 0 && tpm && chunk == 0 && !s.cold) {
        r->admm = BMPC_ADMM_NONE;
        r->polish = BMPC_POL_TPM; r->ws = BMPC_WS_RECORD; r->cap = p.tpm_first_cap;
        return true;
    }
    r->admm = BMPC_ADMM_TEAM;
    r->infeas = s.round > 0 && s.total >= p.infeas_after;
    // the fast-path families polish from the iterate with their Riccati polish (about 3x lower latency than the Schur-form one; on
    // the multi-input shapes a refinement costs about one ADMM iteration); the Schur-form polish takes the instances still open after
    // schur_after iterations, whatever their working sets
    const bool riccati = s.total + chunk <= p.schur_after;
    if (!p.polish) {
        r->polish = BMPC_POL_CHECK;
    } else if (tpi && riccati) {
        r->polish = BMPC_POL_TPI; r->ws = BMPC_WS_FROM_V; r->capA = 2; r->capB = tpi_steps - 2;
    } else if (tpm && riccati) {
        // the first attempt of a cold solve updates all rows at once, every later one by single exchanges (host study on 45 cold
        // stragglers: the cold cap finishes all of them in their first straggler round, cap 12 needs two or three)
        r->polish = BMPC_POL_TPM; r->ws = BMPC_WS_FROM_V;
        r->cap = s.cold ? p.tpm_cold_cap : p.tpm_round_cap;
        r->exchange = !(s.cold && s.round == 0);
    } else {
        r->polish = BMPC_POL_SCHUR; r->cap = bmpc_polish_steps(p.pdas_steps, s.round);
    }
    return true;
}
