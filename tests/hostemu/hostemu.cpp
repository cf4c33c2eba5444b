// Host emulation of the device numerical core (TEST INFRASTRUCTURE ONLY).
// Compiles pympc_b200/csrc/bmpc_core.cuh for the CPU with a one-thread "team" so that index
// arithmetic and algorithm logic can be checked against numpy without a GPU.  This is NOT a CPU
// fallback: pympc_b200 never loads this library; it lives under tests/ and is built by the tests.
#define BMPC_HOSTEMU 1
#include <stdlib.h>
#include <stdio.h>
#include <string.h>
#include "../../pympc_b200/csrc/bmpc_core.cuh"
#include "../../pympc_b200/csrc/bmpc_tpi.cuh"
#include "../../pympc_b200/csrc/bmpc_tile.cuh"
#include "../../pympc_b200/csrc/bmpc_launch.cuh"
#include <stdlib.h>
#include <stdio.h>
#include <string.h>

extern "C" {

int emu_sys_total(int nx, int nu, int Np, int Nc) { BmpcDims d = bmpc_make_dims(nx, nu, Np, Nc); return bmpc_make_off(d).total; }

// offsets of a few arrays for inspection: returns offset by name index
int emu_offset(int nx, int nu, int Np, int Nc, int which) {
    BmpcDims d = bmpc_make_dims(nx, nu, Np, Nc); BmpcSysOff o = bmpc_make_off(d);
    int tab[] = {o.Ad, o.Bd, o.Qx, o.QxN, o.Qu, o.QDu, o.xmin, o.xmax, o.umin, o.umax, o.Dumin, o.Dumax, o.uref,
                 o.pw, o.Acal, o.Bcal, o.BcalT, o.PB, o.H, o.Hinv, o.K, o.Kinv, o.AHinv, o.M, o.Gx0, o.Gref, o.GrefFull,
                 o.g0, o.lo0, o.hi0, o.rho, o.scal};
    return tab[which];
}

void emu_condense(int nx, int nu, int Np, int Nc, double* sys, double rho, double sigma, double alpha, double eps_feas, int soft_on) {
    BmpcDims d = bmpc_make_dims(nx, nu, Np, Nc); BmpcSysOff o = bmpc_make_off(d);
    SeqTeam t;
    bmpc_condense(t, d, o, sys, rho, sigma, alpha, eps_feas, soft_on);
}

// the launch configuration bmpc_create chooses (bmpc_plan_launch): out[14] = ok, team, wpb, rmax, rmax_small, fb_team, fb_rmax,
// overflow, tile_T, tile_threads, smem_admm, smem_polish, smem_polish_small, fb_smem_polish
void emu_plan_launch(int nx, int nu, int Np, int Nc, int max_optin, int team_threads, int warps_per_block, int rmax, int n_sys, long long* out) {
    const BmpcLaunch L = bmpc_plan_launch(bmpc_make_dims(nx, nu, Np, Nc), max_optin, team_threads, warps_per_block, rmax, n_sys);
    const long long v[14] = {L.ok, L.team, L.wpb, L.rmax, L.rmax_small, L.fb_team, L.fb_rmax, L.overflow, L.tile_T, L.tile_threads,
                             (long long)L.smem_admm, (long long)L.smem_polish, (long long)L.smem_polish_small, (long long)L.fb_smem_polish};
    for (int k = 0; k < 14; k++) out[k] = v[k];
}

// capacities of the polish tiers of one round over `count` open instances (bmpc_polish_tiers); returns how many
int emu_polish_tiers(int nx, int nu, int Np, int Nc, int max_optin, int team_threads, int warps_per_block, int rmax, int n_sys,
                     int count, int list_given, int* caps) {
    const BmpcLaunch L = bmpc_plan_launch(bmpc_make_dims(nx, nu, Np, Nc), max_optin, team_threads, warps_per_block, rmax, n_sys);
    return L.ok ? bmpc_polish_tiers(L, count, list_given != 0, caps) : 0;
}

// the team / tile launches of one round over `count` open instances (bmpc_round_launch): out[16] = admm, tile_T, admm_grid,
// admm_threads, admm_smem, ntiers, then per tier warp, grid, threads, rmax, smem; returns 0 (out untouched) for a refused shape
int emu_round_launch(int nx, int nu, int Np, int Nc, int max_optin, int team_threads, int warps_per_block, int rmax, int n_sys,
                     int count, int list_given, int sm_count, long long* out) {
    const BmpcDims d = bmpc_make_dims(nx, nu, Np, Nc);
    const BmpcLaunch L = bmpc_plan_launch(d, max_optin, team_threads, warps_per_block, rmax, n_sys);
    if (!L.ok) return 0;
    const BmpcRoundLaunch R = bmpc_round_launch(L, d, count, list_given != 0, sm_count);
    const long long v[6] = {R.admm, R.tile_T, R.admm_grid, R.admm_threads, (long long)R.admm_smem, R.ntiers};
    for (int k = 0; k < 6; k++) out[k] = v[k];
    for (int k = 0; k < 2; k++) {
        const BmpcPolishTier& t = R.tier[k];
        const long long w[5] = {t.warp, t.grid, t.threads, t.rmax, (long long)t.smem};
        for (int j = 0; j < 5; j++) out[6 + 5 * k + j] = w[j];
    }
    return 1;
}

// one full solve of one instance: rounds of ADMM + polish, like the host loop of the library.  The polish of each round runs
// its tiers like the device: tiers0 [n0] in the first round, tiers1 [n1] in the straggler rounds, smallest capacity first; a
// working set beyond one tier's capacity is redone by the next.
// x,v: warm start in/out (cold != 0 -> initialise).  Returns status (1 solved+polished, 2 solved by eps only, -2 max iter).
int emu_solve(int nx, int nu, int Np, int Nc, const double* sys, const double* x0, const double* um1, const double* xref,
              int xref_mode, int cold, double* x, double* v, double* Uout, int first_iters, int max_iter, int pdas_steps,
              const int* tiers0, int n0, const int* tiers1, int n1, double eps_abs, double eps_rel, int* iters_out,
              int* polish_steps_out, double* res_out) {
    BmpcDims d = bmpc_make_dims(nx, nu, Np, Nc); BmpcSysOff o = bmpc_make_off(d);
    SeqTeam t;
    int rmax = 1;
    for (int k = 0; k < n0; k++) rmax = tiers0[k] > rmax ? tiers0[k] : rmax;
    for (int k = 0; k < n1; k++) rmax = tiers1[k] > rmax ? tiers1[k] : rmax;
    double* buf = (double*)calloc(8 * d.mc + 8 * d.NU + d.NX + rmax * (rmax + 1) / 2 + rmax + 16, sizeof(double));
    double *g = buf, *cc = g + d.NU, *w = cc + d.NX, *xt = w + d.mc, *r = xt + d.NU, *W0 = r + d.NU, *zz = W0 + d.mc,
           *murow = zz + d.mc, *S = murow + d.mc, *tt = S + rmax * (rmax + 1) / 2, *U0 = tt + rmax, *U = U0 + d.NU, *res = U + d.NU;
    int* st = (int*)calloc(d.mc + rmax, sizeof(int)); int* R = st + d.mc;
    bmpc_prep(t, d, o, sys, x0, um1, xref, xref_mode, g, cc);
    if (cold) { for (int a = 0; a < d.NU; a++) x[a] = 0.0; for (int i = 0; i < d.mc; i++) v[i] = i < d.NX ? cc[i] : 0.0; }
    int total = 0, status = -2, psteps = 0, lvl = BMPC_LEV0;
    const double* rhov = sys + o.rho;
    // the rounds of the library's team kernels: chunk and polish steps from its policy (first_iters 0: the automatic first chunk)
    const BmpcPolicy P = bmpc_make_policy(BMPC_FAM_TEAM, 1, first_iters, 0, max_iter, pdas_steps, 1);
    BmpcRoundPlan pl;
    for (int round = 0; bmpc_plan_round(P, BmpcSolveState{round, total, cold != 0, false}, &pl); round++) {
        bmpc_admm(t, d, o, sys, um1, g, cc, x, v, w, xt, r, pl.chunk, res, lvl);
        lvl = bmpc_adapt_level(t, d, o, sys, um1, v, res, lvl);
        total += pl.chunk;
        const int* tiers = round == 0 ? tiers0 : tiers1; const int ntiers = round == 0 ? n0 : n1;
        int ps = -1;
        for (int k = 0; k < ntiers && ps == -1; k++) ps = bmpc_polish(t, d, o, sys, um1, g, cc, v, W0, zz, murow, st, S, tt, R, U0, U, tiers[k], pl.cap);
        if (getenv("EMU_TRACE")) printf("TRACE %d %.3e %.3e %d\n", total, res[0] / fmax(res[2], 1e-12), res[1] / fmax(res[3], 1e-12), ps);
        if (ps > 0) {
            psteps += ps; status = 1;
            for (int a = 0; a < d.NU; a++) { Uout[a] = U[a]; x[a] = U[a]; }
            for (int i = 0; i < d.mc; i++) v[i] = zz[i] + murow[i] / rhov[i];
            break;
        }
        // the device policy for unverified candidates (early exit; bmpc_warm_from_candidate only with EMU_WARM = the solver option
        // candidate_warm, off by default on the device too), mirrored here
        if (getenv("EMU_WARM") && ps == 0 && bmpc_admm_stalled(res, total) && (getenv("EMU_ALWAYS") || bmpc_candidate_usable(t, d, o, sys, um1, zz, murow))) bmpc_warm_from_candidate(t, d, o, sys, zz, murow, U, x, v, lvl);
        if (!getenv("EMU_NOTIGHT") && bmpc_residuals_tight(res, total)) { status = 2; for (int a = 0; a < d.NU; a++) Uout[a] = xt[a]; break; }
        psteps += pl.cap;
    }
    if (status != 1 && status != 2) {
        bool conv = res[0] <= eps_abs + eps_rel * res[2] && res[1] <= eps_abs + eps_rel * res[3];
        status = conv ? 2 : -2;
        for (int a = 0; a < d.NU; a++) Uout[a] = xt[a];
    }
    *iters_out = total; *polish_steps_out = psteps;
    for (int k = 0; k < 4; k++) res_out[k] = res[k];
    free(buf); free(st);
    return status;
}

}  // extern "C"

// TPI fast path for one instance (nu == 1, Nc == Np shapes): first_iters ADMM iterations + Riccati polish on the
// generic-layout state (x [NU], v [mc], in/out) exactly like the device kernels.  Returns polish steps (>0 verified,
// 0 not verified, -100 shape not compiled).
template <class S, bool TV>
static int emu_tpi_run(const double* sys, const double* x0, const double* um1, const double* xref, int cold, double* x,
                           double* v, double* Uout, int first_iters, int pdas_steps) {
    const TpiXref<S, TV> xr{xref};
    BmpcDims d = bmpc_make_dims(S::nx, S::nu, S::Np, S::Nc); BmpcSysOff o = bmpc_make_off(d);
    using CT = typename TpiCode<S>::type;
    TpiAdmmParams<S>* PA = new TpiAdmmParams<S>(); TpiPolParams<S>* PR = new TpiPolParams<S>();
    tpi_fill_admm<S>(sys, o, *PA); tpi_fill_pol<S>(sys, o, *PR);
    double* col = (double*)calloc(S::Np * (S::nx + 2) + S::MT + S::NU + 8, sizeof(double));
    for (int i = 0; i < S::MT; i++) col[i] = v[i + S::nx];
    TpiAcc V{col, 1};
    TpiAcc G{col + S::Np * (S::nx + 2) + S::MT, 1};
    tpi_admm<S>(*PA, V, G, x0, um1, xr, x, first_iters, cold != 0);
    for (int i = 0; i < S::MT; i++) v[i + S::nx] = col[i];
    for (int i = 0; i < S::nx; i++) v[i] = x0[i];
    CT cur[S::Np];
    auto C = [&](int k) -> CT& { return cur[k]; };
    tpi2_codes_from_v<S>(*PR, um1[0], V, col[S::MT - 1], C);
    // the polish emits on every forward sweep; the values of the accepted one are the solution
    double Ustar[S::NU], mumax = 0.0, vq = 0.0;
    int ps = 0;
    for (int r = 0; r < pdas_steps; r++) {
        tpi2_backward<S>(*PR, V, C, xr);
        if (tpi2_forward<S>(*PR, V, C, x0, um1[0], mumax, vq, [&](int j, double u) { Ustar[j] = u; })) { ps = r + 1; break; }
    }
    if (ps > 0) {
        double vstar[S::MT];
        for (int i = 0; i < S::MT - 1; i++) vstar[i] = col[tpi_vstar_slot<S>(i)];
        vstar[S::MT - 1] = vq;
        for (int i = 0; i < S::MT; i++) v[i + S::nx] = vstar[i];
        for (int j = 0; j < S::NU; j++) { Uout[j] = Ustar[j]; x[j] = Ustar[j]; }
    }
    free(col); delete PA; delete PR;
    return ps;
}

extern "C" int emu_tpi_step(int nx, int nu, int Np, int Nc, const double* sys, const double* x0, const double* um1, const double* xref,
                 int xref_mode, int cold, double* x, double* v, double* Uout, int first_iters, int pdas_steps) {
#define EMU_TPI_ARGS sys, x0, um1, xref, cold, x, v, Uout, first_iters, pdas_steps
    if (nx == 4 && nu == 1 && Np == 20 && Nc == 20)
        return xref_mode ? emu_tpi_run<TpiShape<4, 1, 20, 20>, true>(EMU_TPI_ARGS) : emu_tpi_run<TpiShape<4, 1, 20, 20>, false>(EMU_TPI_ARGS);
    if (nx == 2 && nu == 1 && Np == 20 && Nc == 20)
        return xref_mode ? emu_tpi_run<TpiShape<2, 1, 20, 20>, true>(EMU_TPI_ARGS) : emu_tpi_run<TpiShape<2, 1, 20, 20>, false>(EMU_TPI_ARGS);
    if (nx == 4 && nu == 1 && Np == 20 && Nc == 10)                                                                 // held input
        return xref_mode ? emu_tpi_run<TpiShape<4, 1, 20, 10>, true>(EMU_TPI_ARGS) : emu_tpi_run<TpiShape<4, 1, 20, 10>, false>(EMU_TPI_ARGS);
#undef EMU_TPI_ARGS
    return -100;
}


// Team (Schur-form) polish alone from a given ADMM state v (e.g. the previous solve's v*): returns refinements used (> 0 verified,
// 0 not verified, -1 working set beyond rmax); on success U and v (= v*) are written.
extern "C" int emu_polish_only(int nx, int nu, int Np, int Nc, const double* sys, const double* x0, const double* um1, const double* xref,
                               int xref_mode, double* v, double* Uout, int pdas_steps, int rmax) {
    BmpcDims d = bmpc_make_dims(nx, nu, Np, Nc); BmpcSysOff o = bmpc_make_off(d);
    SeqTeam t;
    double* buf = (double*)calloc(8 * d.mc + 8 * d.NU + d.NX + rmax * (rmax + 1) / 2 + rmax + 16, sizeof(double));
    double *g = buf, *cc = g + d.NU, *W0 = cc + d.NX, *zz = W0 + d.mc, *murow = zz + d.mc, *S = murow + d.mc,
           *tt = S + rmax * (rmax + 1) / 2, *U0 = tt + rmax, *U = U0 + d.NU;
    int* st = (int*)calloc(d.mc + rmax, sizeof(int)); int* R = st + d.mc;
    bmpc_prep(t, d, o, sys, x0, um1, xref, xref_mode, g, cc);
    int ps = bmpc_polish(t, d, o, sys, um1, g, cc, v, W0, zz, murow, st, S, tt, R, U0, U, rmax, pdas_steps);
    if (ps > 0) {
        const double* rhov = sys + o.rho;
        for (int a = 0; a < d.NU; a++) Uout[a] = U[a];
        for (int i = 0; i < d.mc; i++) v[i] = zz[i] + murow[i] / rhov[i];
    }
    free(buf); free(st);
    return ps;
}

// Second-generation Riccati polish (tpi2_*): up to max_ref refinements from the working-set codes (mode 0: as stored,
// 1: shifted by one stage, 2: derived from the TPI rows of v).  codes: Np words in/out; v [mc] in (mode 2) / out (v* when verified);
// mumax in/out.  Returns refinements used (> 0 verified, 0 not verified, -100 shape not compiled).
template <class S, bool TV>
static int emu_tpi2_run(const double* sys, const double* x0, const double* um1, const double* xref, unsigned* codes, int mode,
                        double* v, double* Uout, int max_ref, double* mumax_io) {
    using CT = typename TpiCode<S>::type;
    const TpiXref<S, TV> xr{xref};
    BmpcDims d = bmpc_make_dims(S::nx, S::nu, S::Np, S::Nc); BmpcSysOff o = bmpc_make_off(d);
    TpiPolParams<S>* P = new TpiPolParams<S>(); tpi_fill_pol<S>(sys, o, *P);
    double* col = (double*)calloc(S::Np * (S::nx + 2) + S::MT + 8, sizeof(double));
    CT stored[S::Np], cur[S::Np];
    for (int k = 0; k < S::Np; k++) stored[k] = (CT)codes[k];
    TpiAcc W{col, 1};
    auto C = [&](int k) -> CT& { return cur[k]; };
    if (mode == 2) {
        for (int i = 0; i < S::MT; i++) col[i] = v[i + S::nx];
        tpi2_codes_from_v<S>(*P, um1[0], W, col[S::MT - 1], C);
    } else {
        for (int k = 0; k < S::Np; k++) cur[k] = (CT)tpi2_shifted_code<S>(stored, k, mode == 1);
    }
    double mumax = *mumax_io, vq = 0.0, U[S::NU];
    int used = 0;
    for (int r = 0; r < max_ref; r++) {
        tpi2_backward<S>(*P, W, C, xr);
        const bool ok = tpi2_forward<S>(*P, W, C, x0, um1[0], mumax, vq, [&](int j, double u) { U[j] = u; });
        if (ok) { used = r + 1; break; }
    }
    if (used > 0) {
        for (int i = 0; i < S::MT - 1; i++) v[i + S::nx] = col[tpi_vstar_slot<S>(i)];
        v[S::nx + S::MT - 1] = vq;
        for (int q = 0; q < S::nx; q++) v[q] = x0[q];
        for (int j = 0; j < S::NU; j++) Uout[j] = U[j];
    }
    for (int k = 0; k < S::Np; k++) codes[k] = cur[k];
    *mumax_io = mumax;
    free(col); delete P;
    return used;
}

extern "C" int emu_tpi2_step(int nx, int nu, int Np, int Nc, const double* sys, const double* x0, const double* um1, const double* xref,
                             int xref_mode, unsigned* codes, int mode, double* v, double* Uout, int max_ref, double* mumax_io) {
#define EMU_TPI2_ARGS sys, x0, um1, xref, codes, mode, v, Uout, max_ref, mumax_io
    if (nx == 4 && nu == 1 && Np == 20 && Nc == 20)
        return xref_mode ? emu_tpi2_run<TpiShape<4, 1, 20, 20>, true>(EMU_TPI2_ARGS) : emu_tpi2_run<TpiShape<4, 1, 20, 20>, false>(EMU_TPI2_ARGS);
    if (nx == 2 && nu == 1 && Np == 20 && Nc == 20)
        return xref_mode ? emu_tpi2_run<TpiShape<2, 1, 20, 20>, true>(EMU_TPI2_ARGS) : emu_tpi2_run<TpiShape<2, 1, 20, 20>, false>(EMU_TPI2_ARGS);
    if (nx == 4 && nu == 1 && Np == 20 && Nc == 10)
        return xref_mode ? emu_tpi2_run<TpiShape<4, 1, 20, 10>, true>(EMU_TPI2_ARGS) : emu_tpi2_run<TpiShape<4, 1, 20, 10>, false>(EMU_TPI2_ARGS);
    // edges of the fast path's domain (tests/golden/shapes.npz): longest horizon, Np * nx = 128, a code word of exactly 32 bits
    if (nx == 1 && nu == 1 && Np == 31 && Nc == 31)
        return xref_mode ? emu_tpi2_run<TpiShape<1, 1, 31, 31>, true>(EMU_TPI2_ARGS) : emu_tpi2_run<TpiShape<1, 1, 31, 31>, false>(EMU_TPI2_ARGS);
    if (nx == 8 && nu == 1 && Np == 16 && Nc == 16)
        return xref_mode ? emu_tpi2_run<TpiShape<8, 1, 16, 16>, true>(EMU_TPI2_ARGS) : emu_tpi2_run<TpiShape<8, 1, 16, 16>, false>(EMU_TPI2_ARGS);
    if (nx == 13 && nu == 1 && Np == 8 && Nc == 8)
        return xref_mode ? emu_tpi2_run<TpiShape<13, 1, 8, 8>, true>(EMU_TPI2_ARGS) : emu_tpi2_run<TpiShape<13, 1, 8, 8>, false>(EMU_TPI2_ARGS);
#undef EMU_TPI2_ARGS
    return -100;
}


// Tile ADMM (bmpc_tile.cuh) against the per-instance team ADMM on the same T instances (T, NS = the device's three tile variants): prep + niter iterations +
// adaptive-rho move.  x, v: [T][NU], [T][mc] warm start in (ignored when cold), results out (ref_* per-instance code,
// tile_* tile code); res [T][4]; lvl [T] in/out.
template <int T, int NS>
static void emu_tile_compare_t(int nx, int nu, int Np, int Nc, const double* sys, const double* x0, const double* um1, const double* xref,
                                 int xref_mode, int cold, int niter, const int* lvl_in, const double* x_in, const double* v_in,
                                 double* ref_x, double* ref_v, double* ref_xt, double* ref_res, int* ref_lvl,
                                 double* tile_x, double* tile_v, double* tile_xt, double* tile_res, int* tile_lvl) {
    BmpcDims d = bmpc_make_dims(nx, nu, Np, Nc); BmpcSysOff o = bmpc_make_off(d);
    SeqTeam t;
    const int xl = xref_mode ? d.NX : d.nx;
    // reference: one instance at a time
    double* buf = (double*)calloc(4 * d.NU + d.NX + 2 * d.mc + 8, sizeof(double));
    double *g = buf, *cc = g + d.NU, *w = cc + d.NX, *xt = w + d.mc, *r = xt + d.NU, *res = r + d.NU;
    for (int e = 0; e < T; e++) {
        double* x = ref_x + e * d.NU; double* v = ref_v + e * d.mc;
        bmpc_prep(t, d, o, sys, x0 + e * nx, um1 + e * nu, xref + e * xl, xref_mode, g, cc);
        if (cold) { for (int a = 0; a < d.NU; a++) x[a] = 0.0; for (int i = 0; i < d.mc; i++) v[i] = i < d.NX ? cc[i] : 0.0; }
        else { memcpy(x, x_in + e * d.NU, sizeof(double) * d.NU); memcpy(v, v_in + e * d.mc, sizeof(double) * d.mc); }
        bmpc_admm(t, d, o, sys, um1 + e * nu, g, cc, x, v, w, xt, r, niter, res, lvl_in[e]);
        ref_lvl[e] = bmpc_adapt_level(t, d, o, sys, um1 + e * nu, v, res, lvl_in[e]);
        memcpy(ref_xt + e * d.NU, xt, sizeof(double) * d.NU); memcpy(ref_res + e * 4, res, sizeof(double) * 4);
    }
    free(buf);
    // tile
    double* sm = (double*)calloc(bmpc_tile_smem_doubles(d, T) + 8, sizeof(double));
    BmpcTile<T> S; S.carve(sm, d);
    for (int e = 0; e < T; e++) { S.inst[e] = e; S.lvl[e] = lvl_in[e]; for (int q = 0; q < nu; q++) S.um1[e * nu + q] = um1[e * nu + q]; }
    bmpc_tile_load_phi(t, d, sys + o.Bcal, S.phi1, S.phi2);
    bmpc_tile_load_rows(t, d, o, sys, S.lo, S.hi, S.rho);
    bmpc_tile_prep(t, d, o, sys, S, x0, xref, xref_mode);
    for (int e = 0; e < T; e++) {
        for (int a = 0; a < d.NU; a++) S.x[a * T + e] = cold ? 0.0 : x_in[e * d.NU + a];
        for (int i = 0; i < d.mc; i++) S.v[i * T + e] = cold ? (i < d.NX ? S.cc[i * T + e] : 0.0) : v_in[e * d.mc + i];
    }
    if (nx == 8 && nu == 4) bmpc_admm_tile<T, NS, 8, 4>(t, d, o, sys, S, niter);      // the unrolled instantiation the device uses for this shape
    else bmpc_admm_tile<T, NS, 0, 0>(t, d, o, sys, S, niter);
    bmpc_tile_adapt(t, d, o, sys, S);
    for (int e = 0; e < T; e++) {
        for (int a = 0; a < d.NU; a++) { tile_x[e * d.NU + a] = S.x[a * T + e]; tile_xt[e * d.NU + a] = S.xt[a * T + e]; }
        for (int i = 0; i < d.mc; i++) tile_v[e * d.mc + i] = S.v[i * T + e];
        for (int k = 0; k < 4; k++) tile_res[e * 4 + k] = S.res[e * 4 + k];
        tile_lvl[e] = S.nlvl[e];
    }
    free(sm);
}

extern "C" void emu_tile_compare(int T, int nx, int nu, int Np, int Nc, const double* sys, const double* x0, const double* um1, const double* xref,
                                 int xref_mode, int cold, int niter, const int* lvl_in, const double* x_in, const double* v_in,
                                 double* ref_x, double* ref_v, double* ref_xt, double* ref_res, int* ref_lvl,
                                 double* tile_x, double* tile_v, double* tile_xt, double* tile_res, int* tile_lvl) {
#define EMU_TILE_ARGS nx, nu, Np, Nc, sys, x0, um1, xref, xref_mode, cold, niter, lvl_in, x_in, v_in, ref_x, ref_v, ref_xt, ref_res, ref_lvl, tile_x, tile_v, tile_xt, tile_res, tile_lvl
    if (T == 8) emu_tile_compare_t<8, 2>(EMU_TILE_ARGS);
    else if (T == 4) emu_tile_compare_t<4, 2>(EMU_TILE_ARGS);
    else emu_tile_compare_t<2, 1>(EMU_TILE_ARGS);
#undef EMU_TILE_ARGS
}


// OSQP's primal-infeasibility certificate as the straggler rounds evaluate it: ADMM state after it0 iterations vs after
// it0 + it1 iterations (cold start, base rho level).  Returns 1 when certified.
extern "C" int emu_infeasible(int nx, int nu, int Np, int Nc, const double* sys, const double* x0, const double* um1, const double* xref,
                              int it0, int it1, double eps) {
    BmpcDims d = bmpc_make_dims(nx, nu, Np, Nc); BmpcSysOff o = bmpc_make_off(d);
    SeqTeam t;
    double* buf = (double*)calloc(5 * d.NU + d.NX + 5 * d.mc + 8, sizeof(double));
    double *g = buf, *cc = g + d.NU, *x = cc + d.NX, *v = x + d.NU, *w = v + d.mc, *xt = w + d.mc, *r = xt + d.NU, *res = r + d.NU,
           *v0 = res + 8, *dy = v0 + d.mc;
    bmpc_prep(t, d, o, sys, x0, um1, xref, 0, g, cc);
    for (int i = 0; i < d.mc; i++) v[i] = i < d.NX ? cc[i] : 0.0;
    bmpc_admm(t, d, o, sys, um1, g, cc, x, v, w, xt, r, it0, res, BMPC_LEV0);
    memcpy(v0, v, sizeof(double) * d.mc);
    bmpc_admm(t, d, o, sys, um1, g, cc, x, v, w, xt, r, it1, res, BMPC_LEV0);
    int flag = bmpc_primal_infeasible(t, d, o, sys, um1, cc, v0, BMPC_LEV0, v, BMPC_LEV0, dy, eps) ? 1 : 0;
    free(buf);
    return flag;
}


// Multi-input Riccati polish (bmpc_tpm.cuh): up to max_ref refinements from the working-set codes (mode 0: as stored, 1: shifted
// by one stage — Uout then holds the previous plan on entry —, 2: derived from v in the standard row order, 3: from v of the
// previous problem, shifted).  codes: Np 64-bit words in/out; v [mc] in (modes 2, 3) / out (v* when verified); mumax in/out.
// Returns refinements used (> 0 verified, 0 not verified, -100 shape not compiled, -101 QDu not diagonal).
#include "../../pympc_b200/csrc/bmpc_tpm.cuh"
template <class S, bool TV>
static int emu_tpm_run(const double* sys, const double* x0, const double* um1, const double* xref, uint64_t* codes, int mode,
                       double* v, double* Uout, int max_ref, double* mumax_io, int exchange_from) {
    using L = TpmLayout<S>;
    const TpiXref<S, TV> xr{xref};
    BmpcDims d = bmpc_make_dims(S::nx, S::nu, S::Np, S::Nc); BmpcSysOff o = bmpc_make_off(d);
    TpmParams<S>* P = new TpmParams<S>();
    if (!tpm_fill<S>(sys, o, *P)) { delete P; return -101; }
    double* col = (double*)calloc(L::slots + 8, sizeof(double));
    uint64_t cur[S::Np], atb[S::Np], keep[S::Np];
    TpiAcc W{col, 1};
    auto C = [&](int k) -> uint64_t& { return cur[k]; };
    auto CB = [&](int k) -> uint64_t& { return atb[k]; };
    auto CK = [&](int k) -> uint64_t& { return keep[k]; };
    if (mode >= 2) { TpiAcc V{v, 1}; tpm_codes_from_v<S>(*P, um1, V, C, mode == 3); }
    else {
        unsigned first[S::nu];
        for (int j = 0; j < S::nu; j++) first[j] = (mode == 1 && S::Nc > 1) ? tpm_first_label<S>(*P, j, Uout[j], Uout[S::nu + j]) : 0u;
        const int tail = tpm_tail_start<S>(codes);
        for (int k = 0; k < S::Np; k++) cur[k] = tpm_shifted_code<S>(codes, k, mode == 1, first, tail);
    }
    double mumax = *mumax_io, vfirst[S::nu], vq = 0.0, U[S::NU];
    int used = 0;
    for (int r = 0; r < max_ref; r++) {
        tpm_backward<S>(*P, W, C, xr, um1);
        auto outu = [&](int k, int j, double u) { U[k * S::nu + j] = u; };
        const bool ex = exchange_from >= 0 && r >= exchange_from;
        const int fl = ex ? tpm_forward<S, true>(*P, W, C, CB, CK, x0, um1, mumax, vfirst, vq, outu)
                          : tpm_forward<S, false>(*P, W, C, CB, CK, x0, um1, mumax, vfirst, vq, outu);
        if (fl == 0) { used = r + 1; break; }
    }
    if (used > 0) {
        for (int k = 0; k < S::Np; k++)
            for (int p = 0; p < 2 * S::nu + S::nx; p++) { const int row = tpm_vstar_row<S>(k, p); if (row >= 0) v[row] = col[k * L::per_stage + p]; }
        for (int j = 0; j < S::nu; j++) v[S::NX + S::NU + j] = vfirst[j];
        v[S::mc - 1] = vq;
        for (int q = 0; q < S::nx; q++) v[q] = x0[q];
        for (int j = 0; j < S::NU; j++) Uout[j] = U[j];
    }
    for (int k = 0; k < S::Np; k++) codes[k] = (used > 0) ? atb[k] : cur[k];       // a verified vertex is described by the rows at their bounds
    *mumax_io = mumax;
    free(col); delete P;
    return used;
}

extern "C" int emu_tpm_step(int nx, int nu, int Np, int Nc, const double* sys, const double* x0, const double* um1, const double* xref,
                            int xref_mode, uint64_t* codes, int mode, double* v, double* Uout, int max_ref, double* mumax_io, int exchange_from) {
#define EMU_TPM_ARGS sys, x0, um1, xref, codes, mode, v, Uout, max_ref, mumax_io, exchange_from
#define EMU_TPM_SHAPE(a, b, c, e) \
    if (nx == a && nu == b && Np == c && Nc == e) \
        return xref_mode ? emu_tpm_run<TpiShape<a, b, c, e>, true>(EMU_TPM_ARGS) : emu_tpm_run<TpiShape<a, b, c, e>, false>(EMU_TPM_ARGS);
    if (nx == 8 && nu == 4 && Np == 40 && Nc == 40 && getenv("EMU_TPM_SPARSE")) {      // the device's pattern-specialised instantiation (MIMO reference governor)
        using SP = TpmSparseShape<8, 4, 40, 40, 0x40c01030040c0103ull, 0x8040201u>;
        return xref_mode ? emu_tpm_run<SP, true>(EMU_TPM_ARGS) : emu_tpm_run<SP, false>(EMU_TPM_ARGS);
    }
    EMU_TPM_SHAPE(8, 4, 40, 40)
    EMU_TPM_SHAPE(8, 4, 12, 5)
    EMU_TPM_SHAPE(8, 4, 12, 12)
    EMU_TPM_SHAPE(4, 1, 20, 20)
    EMU_TPM_SHAPE(2, 1, 20, 20)
    EMU_TPM_SHAPE(4, 1, 20, 10)
    EMU_TPM_SHAPE(3, 2, 10, 10)
    EMU_TPM_SHAPE(3, 2, 10, 6)
    // edges of the shape domain (tests/golden/mimo_shapes.npz): full code word, Nc = 1, long horizon, nu = 1, nx = 13;
    // EMU_TPM_PATTERN: the non-symmetric pattern of the (8, 4, 25, 1) case (lower-Hessenberg Ad), as the device compiles it
    if (nx == 8 && nu == 4 && Np == 25 && Nc == 1 && getenv("EMU_TPM_PATTERN")) {
        using SP = TpmSparseShape<8, 4, 25, 1, 0xffff7f3f1f0f0703ull, 0x88442219u>;
        return xref_mode ? emu_tpm_run<SP, true>(EMU_TPM_ARGS) : emu_tpm_run<SP, false>(EMU_TPM_ARGS);
    }
    EMU_TPM_SHAPE(2, 6, 12, 12)
    EMU_TPM_SHAPE(7, 5, 8, 4)
    EMU_TPM_SHAPE(8, 4, 25, 1)
    EMU_TPM_SHAPE(3, 2, 60, 60)
    EMU_TPM_SHAPE(4, 1, 40, 40)
    EMU_TPM_SHAPE(1, 5, 20, 10)
    EMU_TPM_SHAPE(13, 2, 6, 6)
    EMU_TPM_SHAPE(13, 1, 10, 10)
#undef EMU_TPM_SHAPE
#undef EMU_TPM_ARGS
    return -100;
}

// niter ADMM iterations of the team core on the generic-layout state (x [NU], v [mc], in/out; cold != 0 -> initialise), with the
// adaptive-rho move afterwards (lvl in/out); res_out [4].  Used by the policy studies of the polish kernels.
extern "C" void emu_admm_only(int nx, int nu, int Np, int Nc, const double* sys, const double* x0, const double* um1, const double* xref,
                              int xref_mode, int cold, double* x, double* v, int niter, int* lvl_io, double* res_out) {
    BmpcDims d = bmpc_make_dims(nx, nu, Np, Nc); BmpcSysOff o = bmpc_make_off(d);
    SeqTeam t;
    double* buf = (double*)calloc(4 * d.NU + d.NX + 2 * d.mc + 16, sizeof(double));
    double *g = buf, *cc = g + d.NU, *w = cc + d.NX, *xt = w + d.mc, *r = xt + d.NU, *res = r + d.NU;
    bmpc_prep(t, d, o, sys, x0, um1, xref, xref_mode, g, cc);
    if (cold) { for (int a = 0; a < d.NU; a++) x[a] = 0.0; for (int i = 0; i < d.mc; i++) v[i] = i < d.NX ? cc[i] : 0.0; }
    bmpc_admm(t, d, o, sys, um1, g, cc, x, v, w, xt, r, niter, res, *lvl_io);
    *lvl_io = bmpc_adapt_level(t, d, o, sys, um1, v, res, *lvl_io);
    for (int k = 0; k < 4; k++) res_out[k] = res[k];
    free(buf);
}
