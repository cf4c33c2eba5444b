// bmpc_launch.cuh — launch configuration of the team / tile kernels: team size, instances per CTA, the working-set capacity of
// every Schur-form polish tier and the tile size of the ADMM.  Host code only, plain C++: libbmpc.so configures a handle with
// bmpc_plan_launch at bmpc_create and launches every team round as bmpc_round_launch describes it; the host emulation
// (tests/hostemu) runs the same functions, so the capacities an instance meets in the emulation are the device's.
//
// The polish holds its working set (violated soft rows + active hard rows) in shared memory: its Schur matrix is packed,
// r(r+1)/2 doubles.  A working set larger than a tier's capacity makes bmpc_polish return -1 and the instance moves to the next
// tier of the same launch pair.  Tiers:
//   * warp team (mc <= 192, NU <= 64): `rmax` (64) per warp, several warps per CTA.  Overflow goes, in the same round, to the CTA
//     tier `fb_rmax`: the largest capacity <= mc that fits the opt-in shared memory.  The same CTA tier takes straggler rounds of at
//     most fb_max_list instances directly (they are latency-bound); that choice is about speed only, never about capacity.
//   * CTA team: the small tier `rmax_small` (80, several CTAs per SM) when the full tier is above 96, its overflow to the full tier
//     `rmax`: the largest capacity <= mc that fits.
// A working set above the last tier's capacity cannot be verified: the instance ends with ADMM's verdict (status 2 or -2).
#pragma once
#include <stddef.h>
#include <initializer_list>
#include "bmpc_tile.cuh"

// shared memory (doubles) per instance of k_admm / k_polish (bmpc.cu) — keep in sync with the carve-up of those kernels
BMPC_HOSTDEV size_t bmpc_admm_smem_doubles(const BmpcDims& d) { return 4 * (size_t)d.NU + d.NX + 2 * (size_t)d.mc + d.nu + 4 + 4; }
BMPC_HOSTDEV size_t bmpc_polish_smem_doubles(const BmpcDims& d, int rmax) {
    return 3 * (size_t)d.NU + d.NX + 4 * (size_t)d.mc + (size_t)rmax * (rmax + 1) / 2 + rmax + d.nu + 2 + (d.mc + rmax + 3) / 2;
}

struct BmpcLaunch {
    int ok;                      // 0: not even a small working set fits in shared memory (bmpc_create refuses the shape)
    int team;                    // threads per instance: 32 = warp team (k_admm<true>, k_polish<true>), else one CTA per instance
    int wpb;                     // warp team: instances (warps) per CTA; CTA team: team / 32
    int rmax;                    // warp tier, or the CTA team's full tier
    int rmax_small;              // CTA team: the small first tier (0: none)
    int fb_team, fb_rmax;        // warp team: the CTA tier of stragglers and of the warp tier's overflow (0: none)
    int overflow;                // warp team: the warp tier hands working sets beyond rmax to the CTA tier in the same round
    int tile_T, tile_threads;    // > 0: the ADMM runs on tiles of tile_T instances per CTA (one shared system, automatic team)
    size_t smem_admm, smem_polish, smem_polish_small, fb_smem_polish;   // dynamic shared memory per CTA (bytes)
};

// straggler rounds of a warp-team handle with at most this many instances run on one warp per CTA (ADMM) and the CTA tier
// alone (polish): they are latency-bound
enum { BMPC_FB_MAX_LIST = 4096 };

// largest capacity <= want whose polish fits `budget` bytes (one instance); shrinks to 8 at the least
inline int bmpc_fit_rmax(const BmpcDims& d, int want, size_t budget) {
    int r = want < d.mc ? want : d.mc;
    while (r > 8 && bmpc_polish_smem_doubles(d, r) * 8 > budget) r--;
    return r;
}

// max_optin: the device's opt-in shared memory per block (bytes); team_threads, warps_per_block, rmax, n_sys: bmpc_config
inline BmpcLaunch bmpc_plan_launch(const BmpcDims& d, int max_optin, int team_threads, int warps_per_block, int rmax_cfg, int n_sys) {
    BmpcLaunch L = {};
    const size_t budget = (size_t)max_optin - 1024;
    auto fits = [&](int r) { return bmpc_polish_smem_doubles(d, r) * 8 <= budget; };
    int team = team_threads;
    if (team <= 0) team = (d.mc <= 192 && d.NU <= 64) ? 32 : 256;
    if (team != 32) { team = ((team + 31) / 32) * 32; if (team > 1024) team = 1024; }
    L.team = team;
    // main tier: rmax > 0 caps it; automatic: 64 per warp, the largest that fits for a CTA
    const int rmax = bmpc_fit_rmax(d, rmax_cfg > 0 ? rmax_cfg : (team == 32 ? 64 : d.mc), budget);
    if (!fits(rmax) || bmpc_admm_smem_doubles(d) * 8 > budget) return L;
    L.ok = 1;
    L.rmax = rmax;
    if (team == 32) {
        int wpb = warps_per_block > 0 ? warps_per_block : 8;
        while (wpb > 1 && (size_t)wpb * bmpc_polish_smem_doubles(d, rmax) * 8 > budget) wpb--;
        L.wpb = wpb;
        L.smem_admm = (size_t)wpb * bmpc_admm_smem_doubles(d) * 8;
        L.smem_polish = (size_t)wpb * bmpc_polish_smem_doubles(d, rmax) * 8;
        const int frmax = bmpc_fit_rmax(d, d.mc, budget);
        if (fits(frmax)) {
            L.fb_team = 128; L.fb_rmax = frmax;
            L.fb_smem_polish = bmpc_polish_smem_doubles(d, frmax) * 8;
            L.overflow = frmax > rmax;
        }
    } else {
        // large shapes with one shared system: the ADMM runs on tiles of T instances per CTA (bmpc_tile.cuh)
        if (team_threads == 0 && n_sys <= 1) {
            for (int T : {8, 4, 2}) if (!L.tile_T && bmpc_tile_smem_doubles(d, T) * 8 <= budget) L.tile_T = T;
            int th = d.NX > 2 * d.NU ? d.NX : 2 * d.NU;
            th = ((th + 31) / 32) * 32; if (th < 128) th = 128; if (th > 512) th = 512;
            if (warps_per_block > 0) th = warps_per_block * 32 > 512 ? 512 : warps_per_block * 32;     // tuning override
            L.tile_threads = th;
        }
        if (rmax_cfg == 0 && rmax > 96) { L.rmax_small = 80; L.smem_polish_small = bmpc_polish_smem_doubles(d, 80) * 8; }
        L.wpb = team / 32;
        L.smem_admm = bmpc_admm_smem_doubles(d) * 8;
        L.smem_polish = bmpc_polish_smem_doubles(d, rmax) * 8;
    }
    return L;
}

// ADMM kernel of a team round
enum BmpcTeamAdmm {
    BMPC_TADMM_WARP,       // k_admm<true>, wpb instances per CTA
    BMPC_TADMM_LONE_WARP,  // k_admm<true>, one warp per CTA (short straggler lists)
    BMPC_TADMM_TILE,       // k_admm_tile of tile_T instances per CTA
    BMPC_TADMM_CTA         // k_admm<false>, one CTA per instance
};

// one Schur-form polish launch: k_polish<warp>
struct BmpcPolishTier {
    int warp;                    // 1: k_polish<true> (a warp per instance), 0: k_polish<false> (a CTA per instance)
    int grid, threads, rmax;
    size_t smem;
};

// the team / tile launches of one round (bmpc_round_launch)
struct BmpcRoundLaunch {
    int admm;                    // BmpcTeamAdmm
    int tile_T;                  // BMPC_TADMM_TILE: instances per CTA (8, 4 or 2)
    int admm_grid, admm_threads;
    size_t admm_smem;
    int ntiers;                  // bmpc_round_polish
    BmpcPolishTier tier[2];
};

// a straggler round of a warp-team / fast-path handle short enough for one warp per CTA (ADMM) and the CTA tier alone (polish)
inline bool bmpc_lone_stragglers(const BmpcLaunch& L, int count, bool list_given) {
    return L.team == 32 && L.fb_team && list_given && count <= BMPC_FB_MAX_LIST;
}

// the polish tiers of a round over `count` open instances (list_given: a straggler round; the first round covers the whole batch)
// of a handle planned as L (L.ok), smallest capacity first; returns how many (1 or 2).  The first tier reads the round's list and
// count and fills the overflow list only when a second tier follows; the second reads the overflow list and takes its count from
// the device.
inline int bmpc_round_polish(const BmpcLaunch& L, int count, bool list_given, BmpcPolishTier* tier) {
    int n = 0;
    auto add = [&](int warp, int grid, int threads, int rmax, size_t smem) { tier[n++] = BmpcPolishTier{warp, grid, threads, rmax, smem}; };
    if (bmpc_lone_stragglers(L, count, list_given)) {
        add(0, count, L.fb_team, L.fb_rmax, L.fb_smem_polish);
    } else if (L.team == 32) {
        // working sets beyond the warp tier go to the CTA tier right after: whether an instance can be verified must not depend
        // on how many instances are open
        add(1, (count + L.wpb - 1) / L.wpb, L.wpb * 32, L.rmax, L.smem_polish);
        if (L.overflow) add(0, count, L.fb_team, L.fb_rmax, L.fb_smem_polish);
    } else {
        // two capacity tiers: the small one keeps several CTAs resident per SM (the polish is latency-bound); working sets that
        // outgrow it are redone by the full tier right after
        if (L.rmax_small) add(0, count, L.team, L.rmax_small, L.smem_polish_small);
        add(0, count, L.team, L.rmax, L.smem_polish);
    }
    return n;
}

// capacities of the polish tiers of such a round (bmpc_round_polish), smallest first; returns how many (<= 2)
inline int bmpc_polish_tiers(const BmpcLaunch& L, int count, bool list_given, int* caps) {
    BmpcPolishTier tier[2];
    const int n = bmpc_round_polish(L, count, list_given, tier);
    for (int k = 0; k < n; k++) caps[k] = tier[k].rmax;
    return n;
}

// the launches of a team round over `count` open instances (as bmpc_round_polish) on a GPU of sm_count SMs
inline BmpcRoundLaunch bmpc_round_launch(const BmpcLaunch& L, const BmpcDims& d, int count, bool list_given, int sm_count) {
    BmpcRoundLaunch R = {};
    if (bmpc_lone_stragglers(L, count, list_given)) {
        // the lanes-own-rows ADMM has the shortest dependent chain per iteration for these small shapes: measured 5 % on the
        // random-instance bench vs a 128-thread CTA
        R.admm = BMPC_TADMM_LONE_WARP;
        R.admm_grid = count; R.admm_threads = 32; R.admm_smem = bmpc_admm_smem_doubles(d) * 8;
    } else if (L.team == 32) {
        R.admm = BMPC_TADMM_WARP;
        R.admm_grid = (count + L.wpb - 1) / L.wpb; R.admm_threads = L.wpb * 32; R.admm_smem = L.smem_admm;
    } else if (L.tile_T > 0) {
        // throughput tiles (8 instances share every K^-1 entry) while the batch fills the GPU twice over; straggler rounds with
        // few instances left use small tiles: more CTAs, a shorter dependent chain per iteration
        int T = L.tile_T;
        if (T == 8 && count <= 2 * sm_count * 8) T = 4;
        if (T == 4 && count <= 2 * sm_count * 2) T = 2;
        R.admm = BMPC_TADMM_TILE; R.tile_T = T;
        R.admm_grid = (count + T - 1) / T; R.admm_threads = L.tile_threads; R.admm_smem = bmpc_tile_smem_doubles(d, T) * 8;
    } else {
        R.admm = BMPC_TADMM_CTA;
        R.admm_grid = count; R.admm_threads = L.team; R.admm_smem = L.smem_admm;
    }
    R.ntiers = bmpc_round_polish(L, count, list_given, R.tier);
    return R;
}
