// bmpc.cu — CUDA kernels (sm_90a) and the C ABI of libbmpc.so (see include/bmpc.h).
//
// Kernel map (SURVEY.md §2a K1-K6):
//   k_condense   K1/K2  one CTA per system: prediction matrices, H, K, inverses, dual operators
//   k_admm       K3+K4  one team (warp or CTA) per instance: per-step prep + ADMM iterations, state in smem
//   k_polish     K5+K6  one team per instance: active-set polish, KKT verification, output epilogue
//   k_finalize          status / fallback output for instances the polish never verified
//   k_sequences         optional x/u/eps sequences and objective value (output() info, mpc.py:307-328)
// Host side: handle management and the round loop  ADMM(first_iters) -> polish -> [ADMM(chunk) -> polish]*, each round as
// bmpc_rounds.cuh plans it.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <array>
#include <string>
#include <vector>

#include "../../include/bmpc.h"
#include "bmpc_core.cuh"
#include "bmpc_rounds.cuh"
#include "bmpc_tpi.cuh"
#include "bmpc_tile.cuh"
#include "bmpc_launch.cuh"
#include "bmpc_tpm.cuh"
#include "bmpc_dare.cuh"
#include "bmpc_kf.cuh"

// One block of round counters = BMPC_CNT ints (the handle keeps two, used alternately): [0] instances still unfinished (-> next list),
// [1] active-set refinements, [2] overflow of the small polish tier, [3] certified infeasible, [4..7] queue control of k_tpi_pol
// (cursor, head, and one 64-bit word: low = reserved queue tail, high = finished chunks), [8] instances that left as "solved,
// unpolished" on tight ADMM residuals.
// [10..11] / [12..13]: ~(earliest start) and latest end of k_tpi_pol in ns of the GPU's global timer (64-bit each): the kernel's
// own duration, for the roofline of bench.py (CUDA events around a launch also count launch gaps).
// [9]: instances re-condensed by k_condense_list in this round (rounds that report through a D2H copy; in the mapped-memory report of
// k_tpi_pol slot 9 carries the K6 arrival flag instead — those rounds never condense).
// [14]: warps of k_tpi_pol that have left; the last one copies the block into the handle's MAPPED pinned host buffer and raises
// [15] = launch epoch there: the host spins on that word instead of paying a D2H copy + stream synchronisation per solve.
enum { TPI_Q_CURSOR = 4, TPI_Q_HEAD = 5, TPI_Q_TAIL = 6, BMPC_CNT_TIGHT = 8, BMPC_CNT_COND = 9, BMPC_CNT_T0 = 10, BMPC_CNT_T1 = 12, BMPC_CNT_EXIT = 14, BMPC_CNT_EPOCH = 15, BMPC_CNT = 16 };
__device__ __forceinline__ unsigned long long bmpc_globaltimer() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }

// ------------------------------------------------------------------------------------------------
// teams
struct WarpTeam {
    int tid;
    static constexpr int n = 32;
    __device__ __forceinline__ WarpTeam() : tid(threadIdx.x & 31) {}
    __device__ __forceinline__ void sync() { __syncwarp(); }
    __device__ __forceinline__ bool all(bool p) { return __all_sync(0xffffffffu, p); }
    __device__ __forceinline__ double max(double v) {
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, s));
        return v;
    }
    __device__ __forceinline__ double sum(double v) {
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
        return v;
    }
    __device__ __forceinline__ int excl_scan(int f, int& total) {
        unsigned b = __ballot_sync(0xffffffffu, f);
        total = __popc(b);
        return __popc(b & ((1u << tid) - 1u));
    }
    __device__ __forceinline__ int warp() const { return 0; }
    __device__ __forceinline__ int nwarps() const { return 1; }
    __device__ __forceinline__ int lane() const { return tid; }
    __device__ __forceinline__ int lanes() const { return 32; }
    __device__ __forceinline__ void wsync() { __syncwarp(); }
    __device__ __forceinline__ double wsum(double v) { return sum(v); }
};

struct BlockTeam {
    int tid, n;
    double* sd;   // 32 doubles of scratch
    int* si;      // 32 ints of scratch
    __device__ __forceinline__ BlockTeam(double* sd_, int* si_) : tid(threadIdx.x), n(blockDim.x), sd(sd_), si(si_) {}
    __device__ __forceinline__ void sync() { __syncthreads(); }
    __device__ __forceinline__ bool all(bool p) { return __syncthreads_and(p) != 0; }
    __device__ __forceinline__ double max(double v) {
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, s));
        if ((tid & 31) == 0) sd[tid >> 5] = v;
        __syncthreads();
        double r = sd[0];
        for (int w = 1; w < (n + 31) / 32; w++) r = fmax(r, sd[w]);
        __syncthreads();
        return r;
    }
    __device__ __forceinline__ double sum(double v) {
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
        if ((tid & 31) == 0) sd[tid >> 5] = v;
        __syncthreads();
        double r = 0.0;
        for (int w = 0; w < (n + 31) / 32; w++) r += sd[w];
        __syncthreads();
        return r;
    }
    __device__ __forceinline__ int excl_scan(int f, int& total) {
        unsigned b = __ballot_sync(0xffffffffu, f);
        if ((tid & 31) == 0) si[tid >> 5] = __popc(b);
        __syncthreads();
        int off = 0, tot = 0;
        for (int w = 0; w < (n + 31) / 32; w++) { int c = si[w]; if (w < (tid >> 5)) off += c; tot += c; }
        __syncthreads();
        total = tot;
        return off + __popc(b & ((1u << (tid & 31)) - 1u));
    }
    __device__ __forceinline__ int warp() const { return tid >> 5; }
    __device__ __forceinline__ int nwarps() const { return n >> 5; }
    __device__ __forceinline__ int lane() const { return tid & 31; }
    __device__ __forceinline__ int lanes() const { return 32; }
    __device__ __forceinline__ void wsync() { __syncwarp(); }
    __device__ __forceinline__ double wsum(double v) {
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
        return v;
    }
};

// ------------------------------------------------------------------------------------------------
// per-instance device arrays
struct BmpcInst {
    const double* x0;     // [B,nx]
    const double* um1;    // [B,nu]
    const double* xref;   // [B,nx] or [B,NX]
    const double* um1_solved;  // [B,nu] copy of um1 as seen by the last solve (output() may overwrite um1)
    double* g;            // [B,NU]   scratch (per-step linear term)
    double* cc;           // [B,NX]   scratch (free response Acal x0)
    double* xw;           // [B,NU]   ADMM x (warm start)
    double* vw;           // [B,mc]   ADMM v (warm start)
    double* Ua;           // [B,NU]   last ADMM xt (fallback solution)
    double* Us;           // [B,NU]   solution
    double* res;          // [B,4]    residuals of the last ADMM iteration
    double* u0;           // [B,nu]   output
    int32_t* status;      // [B]
    int32_t* iters;       // [B]
    int32_t* psteps;      // [B]
    int32_t* lvl;         // [B] adaptive-rho ladder level (reset to the base level at every solve)
    double* u0_shadow;    // second copy of the output = the NEXT solve's u_-1 if output() commits it (a pointer swap instead of a copy)
    double* u0_peer[8];   // extra copies of the output slice in peer GPUs' buffers (NVLink peer stores), see bmpc_bind_output_peers
    int n_peer;
    size_t sys_stride;    // 0: all instances share one system block; o.total: instance i uses block i (per-instance Ad, Bd, ...)
};

// K6: the solver epilogue stores u* into this rank's output slice and, when peers are bound, straight into every peer
// GPU's copy of the gathered buffer over NVLink (the all-gather is fused into the kernel: no collective launch)
__device__ __forceinline__ void bmpc_publish_u0(const BmpcInst& I, double* u0_out, size_t idx, double val) {
    u0_out[idx] = val;
    I.u0_shadow[idx] = val;
    for (int p = 0; p < I.n_peer; p++) I.u0_peer[p][idx] = val;
}

// K6, arrival: after the epilogue's peer stores, every rank raises its flag (= the step counter) in every peer's flag array
// and waits until all peers have raised theirs here: when the kernel ends, the gathered buffer of this step is complete on
// this rank.  One tiny launch instead of a collective; the flag stores are ordered behind the data stores of the solver
// kernels by the stream and a system-scope fence.
struct BmpcPeerFlags { long long* p[8]; };
__global__ void k_gather_arrive(long long* mine, BmpcPeerFlags P, int n_peer, int rank, int world, long long epoch) {
    const int t = threadIdx.x;
    if (t < n_peer) { __threadfence_system(); *(volatile long long*)(P.p[t] + rank) = epoch; }
    if (t < world && t != rank) {
        const long long t0 = clock64();
        while (*(volatile long long*)(mine + t) < epoch) {
            if (clock64() - t0 > 20000000000ll) __trap();            // ~10 s: a peer died; fail loudly instead of hanging the GPU
            __nanosleep(100);
        }
    }
    __threadfence_system();
}

// smem (doubles) per instance of the two kernels: bmpc_admm_smem_doubles, bmpc_polish_smem_doubles (bmpc_launch.cuh)

__global__ void k_condense(BmpcDims d, BmpcSysOff o, double* sys, double rho, double sigma, double alpha, double eps_feas,
                           int soft_on) {
    __shared__ double sd[32];
    __shared__ int si[32];
    BlockTeam t(sd, si);
    bmpc_condense(t, d, o, sys + (size_t)blockIdx.x * o.total, rho, sigma, alpha, eps_feas, soft_on);
}

// ---- time-varying problem data without a new setup (bmpc_update_problem, bmpc_update_system)
// One input array of bmpc_setup that an update replaces: cnt doubles per system at block offset off, read from src (batch-major:
// system i's at src[i * cnt]); view >= 0: the field number where the fast path's parameter view holds the same numbers (Ad, Bd)
struct BmpcRefreshSeg { const double* src; int off, cnt, view; };
struct BmpcRefreshTab { BmpcRefreshSeg seg[13]; int n; };
// k_sys_refresh: one thread per (double of a replaced array, instance), field-major so that the stores into the fast path's
// field-major parameter view (TpiPolView: field f of instance i at view[f * B + i]) are coalesced.  Writes the table's arrays into
// every instance's system block and the view-held ones into the view as well.  The condensed part of the block is NOT touched here:
// the handle's generation counter has moved past every instance's stamp, and k_condense_list re-condenses an instance before the
// first launch that reads its condensed block.  (The view's fields derived from bounds, weights or uref are rebuilt from the raw
// fields by k_fill_view.)
__global__ void k_sys_refresh(double* __restrict__ sys, size_t sys_stride, int B, const __grid_constant__ BmpcRefreshTab T,
                              double* __restrict__ view) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    int f = (int)(idx / B), s = 0;
    const int inst = (int)(idx % B);
    while (s < T.n && f >= T.seg[s].cnt) { f -= T.seg[s].cnt; s++; }
    if (s >= T.n) return;
    const BmpcRefreshSeg& g = T.seg[s];
    const double v = g.src[(size_t)inst * g.cnt + f];
    sys[(size_t)inst * sys_stride + g.off + f] = v;
    if (view && g.view >= 0) view[(size_t)(g.view + f) * B + inst] = v;
}

// k_condense_list: K1 over the listed instances (list == nullptr: 0..count-1), one CTA each, with the rho the setup chose (read from
// the instance's own block: the ladder, the per-instance level and the staged v* = z* + y*/rho stay consistent).  gen != nullptr:
// instances whose stamp already equals `cur` are fresh and leave at once; the others are condensed and stamped.  ncount: number of
// instances condensed (per-solve statistics), may be null.
__global__ void k_condense_list(BmpcDims d, BmpcSysOff o, double* sys, size_t sys_stride, const int32_t* __restrict__ list, int count,
                                int32_t* gen, int32_t cur, double sigma, double alpha, double eps_feas, int soft_on, int32_t* ncount) {
    __shared__ double sd[32];
    __shared__ int si[32];
    const int idx = blockIdx.x;
    if (idx >= count) return;
    const int inst = list ? list[idx] : idx;
    if (gen && gen[inst] == cur) return;
    double* blk = sys + (size_t)inst * sys_stride;
    const double rho = blk[o.scal + BMPC_S_RHO];           // read before the condense rewrites scal (behind its first barrier)
    BlockTeam t(sd, si);
    bmpc_condense(t, d, o, blk, rho, sigma, alpha, eps_feas, soft_on);
    if (t.tid == 0) {
        if (gen) gen[inst] = cur;
        if (ncount) atomicAdd(ncount, 1);
    }
}

template <bool WARP>
__global__ void k_admm(BmpcDims d, BmpcSysOff o, const double* __restrict__ sys, BmpcInst I, const int32_t* __restrict__ list,
                       int count, int niter, int do_prep, int cold, int xref_mode, int adapt) {
    extern __shared__ double smem[];
    __shared__ double sd[32];
    __shared__ int si[32];
    int slot, idx;
    if (WARP) { slot = threadIdx.x >> 5; idx = blockIdx.x * (blockDim.x >> 5) + slot; }
    else { slot = 0; idx = blockIdx.x; }
    if (idx >= count) return;
    const int inst = list ? list[idx] : idx;
    sys += (size_t)inst * I.sys_stride;
    double* base = smem + (size_t)slot * bmpc_admm_smem_doubles(d);
    double *g = base, *cc = g + d.NU, *x = cc + d.NX, *v = x + d.NU, *w = v + d.mc, *xt = w + d.mc, *r = xt + d.NU,
           *um1 = r + d.NU, *res = um1 + d.nu + (d.nu & 1);
    auto run = [&](auto& t) {
        for (int q = t.tid; q < d.nu; q += t.n) um1[q] = I.um1[(size_t)inst * d.nu + q];
        t.sync();
        if (do_prep) {
            const int xl = xref_mode ? d.NX : d.nx;
            bmpc_prep(t, d, o, sys, I.x0 + (size_t)inst * d.nx, um1, I.xref + (size_t)inst * xl, xref_mode, g, cc);
            for (int a = t.tid; a < d.NU; a += t.n) I.g[(size_t)inst * d.NU + a] = g[a];
            for (int i = t.tid; i < d.NX; i += t.n) I.cc[(size_t)inst * d.NX + i] = cc[i];
        } else {
            for (int a = t.tid; a < d.NU; a += t.n) g[a] = I.g[(size_t)inst * d.NU + a];
            for (int i = t.tid; i < d.NX; i += t.n) cc[i] = I.cc[(size_t)inst * d.NX + i];
        }
        if (cold) {
            for (int a = t.tid; a < d.NU; a += t.n) x[a] = 0.0;
            t.sync();
            for (int i = t.tid; i < d.mc; i += t.n) v[i] = (i < d.NX) ? cc[i] : 0.0;
        } else {
            for (int a = t.tid; a < d.NU; a += t.n) x[a] = I.xw[(size_t)inst * d.NU + a];
            for (int i = t.tid; i < d.mc; i += t.n) v[i] = I.vw[(size_t)inst * d.mc + i];
        }
        t.sync();
        int lvl = I.lvl[inst];
        bmpc_admm(t, d, o, sys, um1, g, cc, x, v, w, xt, r, niter, res, lvl);
        if (adapt) {
            const int nl = bmpc_adapt_level(t, d, o, sys, um1, v, res, lvl);
            if (t.tid == 0 && nl != lvl) I.lvl[inst] = nl;
        }
        for (int a = t.tid; a < d.NU; a += t.n) { I.xw[(size_t)inst * d.NU + a] = x[a]; I.Ua[(size_t)inst * d.NU + a] = xt[a]; }
        for (int i = t.tid; i < d.mc; i += t.n) I.vw[(size_t)inst * d.mc + i] = v[i];
        if (t.tid < 4) I.res[(size_t)inst * 4 + t.tid] = res[t.tid];
        if (t.tid == 0) I.iters[inst] += niter;
    };
    if (WARP) { WarpTeam t; run(t); }
    else { BlockTeam t(sd, si); run(t); }
}


// K3+K4 for large shapes: one CTA per TILE of T instances (bmpc_tile.cuh).  Same contract as k_admm.
template <int T, int NS, int NXC, int NUC>
__global__ void __launch_bounds__(NS >= 4 ? 768 : 512) k_admm_tile(BmpcDims d, BmpcSysOff o, const double* __restrict__ sys, BmpcInst I, const int32_t* __restrict__ list,
                            int count, int niter, int do_prep, int cold, int xref_mode, int adapt) {
    extern __shared__ double smem[];
    __shared__ double sd[32];
    __shared__ int si[32];
    BlockTeam t(sd, si);
    BmpcTile<T> S; S.carve(smem, d);
    const int first = blockIdx.x * T;
    const int nact = (count - first) < T ? (count - first) : T;       // a partial tile repeats its last instance (no write-back)
    if (t.tid < T) {
        const int e = t.tid < nact ? t.tid : nact - 1;
        const int inst = list ? list[first + e] : first + e;
        S.inst[t.tid] = inst; S.lvl[t.tid] = I.lvl[inst];
    }
    t.sync();
    bmpc_tile_load_phi(t, d, sys + o.Bcal, S.phi1, S.phi2);
    bmpc_tile_load_rows(t, d, o, sys, S.lo, S.hi, S.rho);
    for (int idx = t.tid; idx < d.nu * T; idx += t.n) { const int e = idx / d.nu, q = idx % d.nu; S.um1[idx] = I.um1[(size_t)S.inst[e] * d.nu + q]; }
    if (do_prep) {
        // staging: v (mc T >= nx T doubles) is free until it is loaded below.  (r, NU T doubles, was too small when Nc nu < nx and
        // overwrote u_-1 and the other per-instance values carved behind it: g then held the wrong u_-1 term.)
        double* x0 = S.v;
        for (int idx = t.tid; idx < d.nx * T; idx += t.n) { const int e = idx / d.nx, c = idx % d.nx; x0[idx] = I.x0[(size_t)S.inst[e] * d.nx + c]; }
        t.sync();
        bmpc_tile_prep(t, d, o, sys, S, x0, I.xref, xref_mode);
        for (int idx = t.tid; idx < d.NU * nact; idx += t.n) { const int e = idx / d.NU, a = idx % d.NU; I.g[(size_t)S.inst[e] * d.NU + a] = S.g[(size_t)a * T + e]; }
        for (int idx = t.tid; idx < d.NX * nact; idx += t.n) { const int e = idx / d.NX, i = idx % d.NX; I.cc[(size_t)S.inst[e] * d.NX + i] = S.cc[(size_t)i * T + e]; }
    } else {
        for (int idx = t.tid; idx < d.NU * T; idx += t.n) { const int e = idx / d.NU, a = idx % d.NU; S.g[(size_t)a * T + e] = I.g[(size_t)S.inst[e] * d.NU + a]; }
        for (int idx = t.tid; idx < d.NX * T; idx += t.n) { const int e = idx / d.NX, i = idx % d.NX; S.cc[(size_t)i * T + e] = I.cc[(size_t)S.inst[e] * d.NX + i]; }
    }
    t.sync();
    if (cold) {
        for (int idx = t.tid; idx < d.NU * T; idx += t.n) S.x[idx] = 0.0;
        for (int idx = t.tid; idx < d.mc * T; idx += t.n) S.v[idx] = (idx / T < d.NX) ? S.cc[idx] : 0.0;
    } else {
        for (int idx = t.tid; idx < d.NU * T; idx += t.n) { const int e = idx / d.NU, a = idx % d.NU; S.x[(size_t)a * T + e] = I.xw[(size_t)S.inst[e] * d.NU + a]; }
        for (int idx = t.tid; idx < d.mc * T; idx += t.n) { const int e = idx / d.mc, i = idx % d.mc; S.v[(size_t)i * T + e] = I.vw[(size_t)S.inst[e] * d.mc + i]; }
    }
    t.sync();
    bmpc_admm_tile<T, NS, NXC, NUC>(t, d, o, sys, S, niter);
    if (adapt) {
        bmpc_tile_adapt(t, d, o, sys, S);
        if (t.tid < nact && S.nlvl[t.tid] != S.lvl[t.tid]) I.lvl[S.inst[t.tid]] = S.nlvl[t.tid];
    }
    for (int idx = t.tid; idx < d.NU * nact; idx += t.n) {
        const int e = idx / d.NU, a = idx % d.NU; const size_t gidx = (size_t)S.inst[e] * d.NU + a;
        I.xw[gidx] = S.x[(size_t)a * T + e]; I.Ua[gidx] = S.xt[(size_t)a * T + e];
    }
    for (int idx = t.tid; idx < d.mc * nact; idx += t.n) { const int e = idx / d.mc, i = idx % d.mc; I.vw[(size_t)S.inst[e] * d.mc + i] = S.v[(size_t)i * T + e]; }
    for (int idx = t.tid; idx < 4 * nact; idx += t.n) I.res[(size_t)S.inst[idx / 4] * 4 + idx % 4] = S.res[idx];
    if (t.tid < nact) I.iters[S.inst[t.tid]] += niter;
}

template <bool WARP>
__global__ void k_polish(BmpcDims d, BmpcSysOff o, const double* __restrict__ sys, BmpcInst I, const int32_t* __restrict__ list,
                         int count, int rmax, int max_steps, int32_t* next_list, int32_t* next_count, double* u0_out,
                         const int32_t* dev_count, int32_t* ovf_list, int cand_warm) {
    extern __shared__ double smem[];
    __shared__ double sd[32];
    __shared__ int si[32];
    int slot, idx;
    if (WARP) { slot = threadIdx.x >> 5; idx = blockIdx.x * (blockDim.x >> 5) + slot; }
    else { slot = 0; idx = blockIdx.x; }
    if (dev_count) count = *dev_count;                 // second tier: the list was filled by the launch before this one
    if (idx >= count) return;
    const int inst = list ? list[idx] : idx;
    sys += (size_t)inst * I.sys_stride;
    double* base = smem + (size_t)slot * bmpc_polish_smem_doubles(d, rmax);
    double *g = base, *cc = g + d.NU, *v = cc + d.NX, *W0 = v + d.mc, *zz = W0 + d.mc, *murow = zz + d.mc,
           *S = murow + d.mc, *tt = S + (size_t)rmax * (rmax + 1) / 2, *U0 = tt + rmax, *U = U0 + d.NU, *um1 = U + d.NU;
    int* st = (int*)(um1 + d.nu + (d.nu & 1));
    int* R = st + d.mc;
    auto run = [&](auto& t) {
        for (int q = t.tid; q < d.nu; q += t.n) um1[q] = I.um1[(size_t)inst * d.nu + q];
        for (int a = t.tid; a < d.NU; a += t.n) g[a] = I.g[(size_t)inst * d.NU + a];
        for (int i = t.tid; i < d.NX; i += t.n) cc[i] = I.cc[(size_t)inst * d.NX + i];
        for (int i = t.tid; i < d.mc; i += t.n) v[i] = I.vw[(size_t)inst * d.mc + i];
        t.sync();
        int ps = bmpc_polish(t, d, o, sys, um1, g, cc, v, W0, zz, murow, st, S, tt, R, U0, U, rmax, max_steps);
        if (ps > 0) {
            const double* rhov = sys + o.rho;
            for (int a = t.tid; a < d.NU; a += t.n) {
                double ua = U[a];
                I.Us[(size_t)inst * d.NU + a] = ua; I.xw[(size_t)inst * d.NU + a] = ua;
                if (a < d.nu) bmpc_publish_u0(I, u0_out, (size_t)inst * d.nu + a, ua);
            }
            // exact ADMM fixed point of this problem = warm start of the next one: v* = z* + y*/rho
            for (int i = t.tid; i < d.mc; i += t.n) I.vw[(size_t)inst * d.mc + i] = zz[i] + murow[i] / rhov[i];
            if (t.tid == 0) { I.status[inst] = BMPC_SOLVED; I.psteps[inst] += ps; atomicAdd(next_count + 1, ps); }
        } else if (ps == -1 && ovf_list) {
            // working set larger than this tier's capacity: hand the instance to the large-capacity launch that follows
            if (t.tid == 0) { int pos = atomicAdd(next_count + 2, 1); ovf_list[pos] = inst; }
        } else {
            // not verified.  (a) ADMM residuals far below any tolerance: the iterate is the answer to ~1e-8 although the active-set
            // iteration cannot certify it (degenerate vertex): "solved" like OSQP would say, no more rounds.  (b) otherwise, if the
            // last candidate is sane (hard rows feasible to 1e-2), its rows and multipliers become the ADMM state of the next
            // round: a strongly violated soft row carries the multiplier eps_feas * d, which ADMM alone builds in eps_feas d / rho steps
            const double* resg = I.res + (size_t)inst * 4;
            const int itsg = I.iters[inst];
            const bool tight = bmpc_residuals_tight(resg, itsg);
            if (tight) {
                for (int a = t.tid; a < d.NU; a += t.n) {
                    const double ua = I.Ua[(size_t)inst * d.NU + a];
                    I.Us[(size_t)inst * d.NU + a] = ua;
                    if (a < d.nu) bmpc_publish_u0(I, u0_out, (size_t)inst * d.nu + a, ua);
                }
            } else if (ps == 0 && cand_warm && bmpc_admm_stalled(resg, itsg) && bmpc_candidate_usable(t, d, o, sys, um1, zz, murow)) {
                const int lvl = I.lvl[inst];
                bmpc_warm_from_candidate(t, d, o, sys, zz, murow, U, I.xw + (size_t)inst * d.NU, I.vw + (size_t)inst * d.mc, lvl);
            }
            if (t.tid == 0) {
                int used = (ps < 0 ? 1 : max_steps);
                I.psteps[inst] += used; atomicAdd(next_count + 1, used);
                if (tight) { I.status[inst] = BMPC_SOLVED_UNPOLISHED; atomicAdd(next_count + BMPC_CNT_TIGHT, 1); }
                else if (I.status[inst] != BMPC_PRIMAL_INFEASIBLE) { int pos = atomicAdd(next_count, 1); next_list[pos] = inst; }   // a certified instance is finished
            }
        }
    };
    if (WARP) { WarpTeam t; run(t); }
    else { BlockTeam t(sd, si); run(t); }
}

// instances still unverified after the last round: OSQP's criterion decides between "solved" and "max iter";
// the output falls back to u_failure = uref when not solved (mpc.py:230,303-304).  pure_admm: no polish was run.
__global__ void k_finalize(BmpcDims d, BmpcSysOff o, const double* __restrict__ sys, BmpcInst I, const int32_t* __restrict__ list,
                           int count, double eps_abs, double eps_rel, double* u0_out) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    const int inst = list ? list[idx] : idx;
    sys += (size_t)inst * I.sys_stride;
    const double* res = I.res + (size_t)inst * 4;
    bool conv = res[0] <= eps_abs + eps_rel * res[2] && res[1] <= eps_abs + eps_rel * res[3];
    if (I.status[inst] == BMPC_PRIMAL_INFEASIBLE) return;               // certified: status and u_failure already written
    I.status[inst] = conv ? BMPC_SOLVED_UNPOLISHED : BMPC_MAX_ITER;
    for (int a = 0; a < d.NU; a++) I.Us[(size_t)inst * d.NU + a] = I.Ua[(size_t)inst * d.NU + a];
    for (int q = 0; q < d.nu; q++) bmpc_publish_u0(I, u0_out, (size_t)inst * d.nu + q, conv ? I.Ua[(size_t)inst * d.NU + q] : sys[o.uref + q]);
}


// ---- primal infeasibility (OSQP paper 3.4), checked on straggler rounds only: the change of the multipliers y over one
// ADMM round, projected like OSQP does, is a certificate when A' dy ~ 0 and the support function of the row box is negative.
// Soft rows are penalties, not constraints: they stay out.  k_snapshot keeps (v, level) of the listed instances before the
// round; k_infeas compares with the state after it.
__global__ void k_snapshot(BmpcDims d, BmpcInst I, const int32_t* __restrict__ list, int count, double* vprev, int32_t* lprev) {
    const int idx = blockIdx.x;
    if (idx >= count) return;
    const int inst = list ? list[idx] : idx;
    for (int i = threadIdx.x; i < d.mc; i += blockDim.x) vprev[(size_t)inst * d.mc + i] = I.vw[(size_t)inst * d.mc + i];
    if (threadIdx.x == 0) lprev[inst] = I.lvl[inst];
}

__global__ void k_infeas(BmpcDims d, BmpcSysOff o, const double* __restrict__ sys, BmpcInst I, const int32_t* __restrict__ list, int count,
                         const double* __restrict__ vprev, const int32_t* __restrict__ lprev, double eps_pinf, double* u0_out, int32_t* counts) {
    extern __shared__ double smem[];
    __shared__ double sd[32];
    __shared__ int si[32];
    const int idx = blockIdx.x;
    if (idx >= count) return;
    const int inst = list ? list[idx] : idx;
    sys += (size_t)inst * I.sys_stride;
    BlockTeam t(sd, si);
    double* dy = smem; double* um1 = dy + d.mc;
    for (int q = t.tid; q < d.nu; q += t.n) um1[q] = I.um1[(size_t)inst * d.nu + q];
    t.sync();
    if (bmpc_primal_infeasible(t, d, o, sys, um1, I.cc + (size_t)inst * d.NX, vprev + (size_t)inst * d.mc, lprev[inst],
                               I.vw + (size_t)inst * d.mc, I.lvl[inst], dy, eps_pinf)) {
        if (t.tid == 0) { I.status[inst] = BMPC_PRIMAL_INFEASIBLE; atomicAdd(counts + 3, 1); }
        for (int q = t.tid; q < d.nu; q += t.n) bmpc_publish_u0(I, u0_out, (size_t)inst * d.nu + q, sys[o.uref + q]);
    }
}

// pure-ADMM mode: list of instances not yet converged by OSQP's criterion
__global__ void k_check_converged(BmpcInst I, const int32_t* __restrict__ list, int count, double eps_abs, double eps_rel,
                                  int32_t* next_list, int32_t* next_count) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    const int inst = list ? list[idx] : idx;
    const double* res = I.res + (size_t)inst * 4;
    bool conv = res[0] <= eps_abs + eps_rel * res[2] && res[1] <= eps_abs + eps_rel * res[3];
    if (!conv && I.status[inst] != BMPC_PRIMAL_INFEASIBLE) { int pos = atomicAdd(next_count, 1); next_list[pos] = inst; }
}

__global__ void k_reset(BmpcInst I, int B) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B) { I.status[i] = BMPC_UNSOLVED; I.iters[i] = 0; I.psteps[i] = 0; I.lvl[i] = BMPC_LEV0; }
}

// x_seq = Acal x0 + Bcal U, eps_seq = distance back to the box, objective of the reference QP (without J_CNST).
// Recomputes g and cc from (x0, u_-1, xref) so it does not depend on which solve path ran.
__global__ void k_sequences(BmpcDims d, BmpcSysOff o, const double* __restrict__ sys, BmpcInst I, int B, int xref_mode,
                            double* xseq, double* epsseq, double* obj) {
    extern __shared__ double smem[];
    WarpTeam t;
    const int slot = threadIdx.x >> 5;
    int inst = blockIdx.x * (blockDim.x >> 5) + slot;
    if (inst >= B) return;
    sys += (size_t)inst * I.sys_stride;
    double* g = smem + (size_t)slot * (d.NU + d.NX + d.nu + 1);
    double* cc = g + d.NU;
    double* um1 = cc + d.NX;
    const double *BcalT = sys + o.BcalT, *H = sys + o.H, *lo0 = sys + o.lo0, *hi0 = sys + o.hi0;
    const double *Qx = sys + o.Qx, *QxN = sys + o.QxN;
    const double rho_e = sys[o.scal + BMPC_S_RHOE];
    const double* U = I.Us + (size_t)inst * d.NU;
    const double* xr = I.xref + (size_t)inst * (xref_mode ? d.NX : d.nx);
    for (int q = t.tid; q < d.nu; q += 32) um1[q] = I.um1_solved[(size_t)inst * d.nu + q];
    t.sync();
    bmpc_prep(t, d, o, sys, I.x0 + (size_t)inst * d.nx, um1, xr, xref_mode, g, cc);
    double part = 0.0;
    for (int i = t.tid; i < d.NX; i += 32) {
        double xi = bmpc_Arow_dot(d, BcalT, U, i) + cc[i];
        double e = xi > hi0[i] ? hi0[i] - xi : (xi < lo0[i] ? lo0[i] - xi : 0.0);
        if (!(rho_e > 0.0)) e = 0.0;
        xseq[(size_t)inst * d.NX + i] = xi; epsseq[(size_t)inst * d.NX + i] = e;
        part += 0.5 * rho_e * e * e;
        // 0.5 cc' P_X cc + q_X' cc  with q_X = -P_X xref
        int k = i / d.nx, a = i % d.nx; const double* Q = k < d.Np ? Qx : QxN; double pc = 0.0, pr = 0.0;
        for (int q = 0; q < d.nx; q++) {
            pc += Q[a * d.nx + q] * cc[k * d.nx + q];
            pr += Q[a * d.nx + q] * (xref_mode ? xr[k * d.nx + q] : xr[q]);
        }
        part += cc[i] * (0.5 * pc - pr);
    }
    for (int a = t.tid; a < d.NU; a += 32) {
        double hu = 0.0;
        for (int b = 0; b < d.NU; b++) hu += H[a * d.NU + b] * U[b];
        part += U[a] * (0.5 * hu + g[a]);
    }
    part = t.sum(part);
    if (t.tid == 0) obj[inst] = part;
}

// ------------------------------------------------------------------------------------------------
// TPI fast path (bmpc_tpi.cuh): one thread per instance, one warp (32 instances) per CTA.
// The iterate travels between global [inst][mc] and shared [row][lane] through a coalesced transpose.
constexpr int TPI_STR = 33;   // padded lane stride of the shared-memory columns

template <class S>
__device__ __forceinline__ void tpi_load_v(const BmpcInst& I, int inst0, int nvalid, double* smem, int row_off, int nrows = S::MT) {
    // coalesced global read -> transposed shared write, issued as asynchronous 8-byte copies (LDGSTS) so that the 125
    // copies of a lane are all in flight at once instead of one load->store round trip per element
    const double* src = I.vw + (size_t)inst0 * S::mc;
    for (int idx = threadIdx.x; idx < nvalid * S::mc; idx += 32) {
        int t = idx / S::mc, i = idx - t * S::mc;
        if (i >= S::nx && i - S::nx < nrows) {
            const unsigned dst = (unsigned)__cvta_generic_to_shared(smem + (row_off + i - S::nx) * TPI_STR + t);
            asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src + idx) : "memory");
        }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

template <class S, bool TV>
__global__ void __launch_bounds__(32) k_tpi_admm(const __grid_constant__ TpiAdmmParams<S> P, BmpcInst I, const int32_t* __restrict__ list, int B, int niter, int cold,
                                                 int reset, int32_t* counts, double* um1_solved) {
    // list == nullptr: instances blockIdx*32 .. +31 (coalesced transpose of the iterate through shared memory);
    // list != nullptr: B arbitrary instances (straggler rounds): each thread moves its own rows directly.
    extern __shared__ double smem[];
    const int lane = threadIdx.x, idx0 = blockIdx.x * 32;
    const int nvalid = (B - idx0) < 32 ? (B - idx0) : 32;
    const bool valid = lane < nvalid;
    const int inst = list ? (valid ? list[idx0 + lane] : 0) : idx0 + lane;
    TpiAcc V{smem + lane, TPI_STR};
    if (!cold) {
        if (list) {
            if (valid) { const double* src = I.vw + (size_t)inst * S::mc + S::nx; for (int i = 0; i < S::MT; i++) V(i) = src[i]; }
        } else { tpi_load_v<S>(I, idx0, nvalid, smem, 0); }
        __syncwarp();
    }
    double x0[S::nx], um1[S::nu], xref[S::nx], x[S::NU];
#pragma unroll
    for (int q = 0; q < S::nx; q++) { x0[q] = valid ? I.x0[(size_t)inst * S::nx + q] : 0.0; xref[q] = (valid && !TV) ? I.xref[(size_t)inst * S::nx + q] : 0.0; }
    // constant reference: in registers; time-varying: this instance's (Np+1) x nx block in global memory
    const TpiXref<S, TV> xr{TV ? I.xref + (size_t)inst * S::NX : xref};
#pragma unroll
    for (int q = 0; q < S::nu; q++) um1[q] = valid ? I.um1[(size_t)inst * S::nu + q] : 0.0;
#pragma unroll
    for (int a = 0; a < S::NU; a++) x[a] = (valid && !cold) ? I.xw[(size_t)inst * S::NU + a] : 0.0;
    if (reset) {
        // first round of a solve: the per-solve bookkeeping that k_reset / two memsets would do rides here (3 launches saved)
        if (valid) {
            I.status[inst] = BMPC_UNSOLVED; I.iters[inst] = 0; I.psteps[inst] = 0; I.lvl[inst] = BMPC_LEV0;
#pragma unroll
            for (int q = 0; q < S::nu; q++) um1_solved[(size_t)inst * S::nu + q] = um1[q];
        }
        if (blockIdx.x == 0 && lane < BMPC_CNT) counts[lane] = 0;        // (the polish launch behind this one zeroes the other half)
    }
    // g' (read once per iteration) lives in the instance's global scratch row I.g, not in shared memory: the column is
    // MT rows instead of MT + NU, which lets one more warp reside per SM (measured: ADMM kernel 12 % faster)
    const TpiAcc G{I.g + (size_t)inst * S::NU, 1};
    if (valid) tpi_admm<S>(P, V, G, x0, um1, xr, x, niter, cold != 0);
    __syncwarp();
    if (list) {
        if (valid) {
            double* dst = I.vw + (size_t)inst * S::mc;
            for (int i = 0; i < S::MT; i++) dst[S::nx + i] = V(i);
#pragma unroll
            for (int q = 0; q < S::nx; q++) dst[q] = x0[q];
        }
    } else {
        double* dst = I.vw + (size_t)idx0 * S::mc;
#pragma unroll 5
        for (int idx = lane; idx < nvalid * S::mc; idx += 32) {
            int t = idx / S::mc, i = idx - t * S::mc;
            dst[idx] = (i >= S::nx) ? smem[(i - S::nx) * TPI_STR + t] : I.x0[(size_t)(idx0 + t) * S::nx + i];
        }
    }
    if (valid) {
#pragma unroll
        for (int a = 0; a < S::NU; a++) { I.xw[(size_t)inst * S::NU + a] = x[a]; I.Ua[(size_t)inst * S::NU + a] = x[a]; }
        I.iters[inst] += niter;
    }
}

// ------------------------------------------------------------------------------------------------
// K5 + K6 of the fast path: persistent, work-stealing Riccati polish (bmpc_tpi.cuh, second generation).
// One CTA per SM, TpiPolLayout<S>::warps warps per CTA (as many as the gain workspaces let reside, at most TPI_POL_WARPS), every
// warp on its own: it
//   phase A  steals chunks of 32 instances off a cursor and runs capA active-set refinements on them (a warm solve: ONE, from
//            the stored working sets shifted by one stage); lanes that verified publish u*, U, status, v*; the others store
//            their updated working sets and enter a device-side queue;
//   phase B  when the cursor is exhausted the warp serves the queue: whatever instances are waiting (1..32) get up to capB more
//            refinements in-warp.  Stragglers therefore never make 31 verified lanes wait (the first-generation kernel lost
//            2/3 of its time to that on transient steps) and a warm solve is ONE launch whatever the refinement counts are.
// Instances still unverified after that go to next_list for the ADMM rounds of the host loop.
struct TpiPolArgs {
    const int32_t* list; int count;      // instances of phase A: list[0..count) or, list == nullptr, 0..count-1
    int mode;                            // 0 stored working sets, 1 stored and shifted one stage (receding horizon), 2 from the iterate v
    int capA, capB;                      // refinements per instance in phase A / in phase B (0: no phase B, failures go to next_list)
    int reset;                           // first round of a solve: per-solve bookkeeping rides here
    int32_t* counts_next;                // the 8 counters of the NEXT round: zeroed here (saves a memset launch per solve)
    int32_t* host_counts; int epoch;     // mapped pinned copy of the counters + the value the last warp stores into its epoch slot (0: off)
    long long* gflags; BmpcPeerFlags gpeers; int g_npeer, g_rank, g_world; long long g_epoch;   // K6 arrival folded into this launch (g_epoch 0: off)
    int32_t* next_list; int32_t* counts; // counts[0] unfinished (-> next_list), [1] refinements; counts[4..7] queue control, see below
    int32_t* queue; int qcap;            // phase-B queue (capacity qcap), all -1 between launches (consumers clear what they take)
    double* u0_out; double* um1_solved;
    const double* pview; int pstride;    // per-instance parameter blocks (PERINST instantiation): base and field stride (= batch)
    int cand_warm;                       // 1: an unverified instance hands its last candidate to the ADMM rounds when that candidate is sane
    unsigned char* codes; int code_stride;   // per instance: Np working-set codes + the multiplier scale (double) of the last refinement
};
constexpr int TPI_POL_WARPS = 7;                 // warps per CTA of k_tpi_pol when their workspaces fit (the pendulum: 230 720 B)
constexpr size_t TPI_POL_SMEM_MAX = 232448;      // dynamic shared memory a CTA can opt into on sm_90 (227 KB)

// bytes of one instance's working-set record in global memory: Np code words (2 bytes up to nx = 5, else 4) rounded up to 8,
// then the multiplier scale (double) of the last refinement.  Host-side twin of TpiPolLayout<S>::code_stride (bmpc_create
// sizes the records of a handle from its dims before a fast-path entry is chosen)
static constexpr int tpi_code_stride(int nx, int Np) { return ((Np * (2 * nx + 6 <= 16 ? 2 : 4) + 7) & ~7) + 8; }

template <class S>
struct TpiPolLayout {
    using CT = typename TpiCode<S>::type;
    static constexpr int GROWS = S::Np * (S::nx + 2);                      // gain rows = TPI rows of v minus the spurious last one
    static constexpr size_t gain_bytes = (size_t)GROWS * TPI_STR * 8;
    static constexpr size_t code_bytes = (((size_t)S::Np * 32 * sizeof(CT)) + 15) & ~(size_t)15;
    static constexpr size_t per_warp = gain_bytes + code_bytes;
    // as many warps per CTA as their workspaces fit in shared memory, at most TPI_POL_WARPS (one CTA per SM)
    static constexpr int warps = (int)(TPI_POL_SMEM_MAX / per_warp < (size_t)TPI_POL_WARPS ? TPI_POL_SMEM_MAX / per_warp : (size_t)TPI_POL_WARPS);
    static_assert(warps >= 1, "fast-path polish: one warp's workspace exceeds the shared memory of a CTA");
    static constexpr size_t smem = per_warp * warps;                         // dynamic shared memory of one CTA
    static constexpr int code_stride = (int)(((S::Np * sizeof(CT) + 7) & ~(size_t)7) + 8);   // bytes per instance in global memory
    static_assert(code_stride == tpi_code_stride(S::nx, S::Np), "record size");
    static constexpr int VROWS = S::MT - 1;                                 // TPI rows of v without the spurious last row
    static_assert(VROWS <= GROWS, "slot layout");
};

// one batch of up to 32 instances (one per lane) through up to cap refinements; returns the mask of verified lanes
template <class S, bool TV, class PP>
__device__ __forceinline__ void tpi_pol_batch(const PP& P, const BmpcInst& I, const TpiPolArgs& A, double* wsm, typename TpiCode<S>::type* csm,
                                              int inst, bool valid_in, int inst0_contig, int nvalid, int mode, int cap, bool to_queue, int reset) {
    bool valid = valid_in;
    using L = TpiPolLayout<S>; using CT = typename TpiCode<S>::type;
    constexpr int nx = S::nx;
    const int lane = threadIdx.x & 31;
    TpiAcc W{wsm + lane, TPI_STR};
    auto C = [&](int k) -> CT& { return csm[k * 32 + lane]; };
    double x0[nx], xref[nx], um1 = 0.0, mumax = 0.0, vq = 0.0;
#pragma unroll
    for (int q = 0; q < nx; q++) { x0[q] = valid ? I.x0[(size_t)inst * nx + q] : 0.0; xref[q] = (valid && !TV) ? I.xref[(size_t)inst * nx + q] : 0.0; }
    if (valid) um1 = I.um1[(size_t)inst];
    const TpiXref<S, TV> xr{TV ? I.xref + (size_t)inst * S::NX : xref};
    unsigned char* rec = A.codes + (size_t)inst * A.code_stride;
    if (mode == 2) {
        // working sets from the ADMM iterate: TPI rows of v into the (still unused) gain rows
        if (inst0_contig >= 0) tpi_load_v<S>(I, inst0_contig, nvalid, wsm, 0, L::VROWS);
        else if (valid) { const double* src = I.vw + (size_t)inst * S::mc + nx; for (int i = 0; i < L::VROWS; i++) W(i) = src[i]; }
        __syncwarp();
        if (valid) tpi2_codes_from_v<S>(P, um1, W, I.vw[(size_t)inst * S::mc + nx + S::MT - 1], C);
    } else if (valid) {
        // stored working sets (written by another SM when this batch comes from the queue: bypass L1)
        CT st[S::Np];
        const unsigned long long* src = (const unsigned long long*)rec;
        constexpr int NW = (int)((S::Np * sizeof(CT) + 7) / 8);
        unsigned long long wbuf[NW];
#pragma unroll
        for (int i = 0; i < NW; i++) wbuf[i] = __ldcg(src + i);
#pragma unroll
        for (int k = 0; k < S::Np; k++) st[k] = (CT)(wbuf[(k * sizeof(CT)) / 8] >> (8 * ((k * sizeof(CT)) % 8)));
#pragma unroll
        for (int k = 0; k < S::Np; k++) C(k) = (CT)tpi2_shifted_code<S>(st, k, mode == 1);
        if (!reset) mumax = __ldcg((const double*)(rec + A.code_stride - 8));
    }
    double* udst = I.Us + (size_t)inst * S::NU;
    double u_first = 0.0;
    bool done = !valid, ok = false;
    if (mode == 2 && A.list != nullptr && !reset && valid) {
        // straggler round (an ADMM chunk of the team kernels ran just before): residuals far below any tolerance end the instance
        // as "solved, unpolished" — its iterate is the answer although the active-set iteration cannot certify it (bmpc_residuals_tight)
        if (bmpc_residuals_tight(I.res + (size_t)inst * 4, I.iters[inst])) {
            const double* ua = I.Ua + (size_t)inst * S::NU;
            for (int j = 0; j < S::NU; j++) udst[j] = ua[j];
            bmpc_publish_u0(I, A.u0_out, (size_t)inst, ua[0]);
            I.status[inst] = BMPC_SOLVED_UNPOLISHED; atomicAdd(A.counts + BMPC_CNT_TIGHT, 1);
            done = true; valid = false;
        }
    }
    int used = 0;
    for (int r = 0; r < cap; r++) {
        if (!done) {
            tpi2_backward<S>(P, W, C, xr);
            ok = tpi2_forward<S>(P, W, C, x0, um1, mumax, vq, [&](int j, double u) { udst[j] = u; if (j == 0) u_first = u; });
            used++;
            done = ok;
        }
        if (__all_sync(0xffffffffu, done)) break;
    }
    ok = ok && valid;
    if (valid) {
        if (reset) {
            I.iters[inst] = 0; A.um1_solved[inst] = um1;
            if (!ok) { I.status[inst] = BMPC_UNSOLVED; I.lvl[inst] = BMPC_LEV0; }
        }
        if (ok) { bmpc_publish_u0(I, A.u0_out, (size_t)inst, u_first); I.status[inst] = BMPC_SOLVED; }
        // working sets of the accepted (or last) candidate: the next solve starts from them, phase B continues from them
        unsigned long long* dst = (unsigned long long*)rec;
        constexpr int NW = (int)((S::Np * sizeof(CT) + 7) / 8);
        unsigned long long wbuf[NW];
#pragma unroll
        for (int i = 0; i < NW; i++) wbuf[i] = 0ull;
#pragma unroll
        for (int k = 0; k < S::Np; k++) wbuf[(k * sizeof(CT)) / 8] |= (unsigned long long)C(k) << (8 * ((k * sizeof(CT)) % 8));
#pragma unroll
        for (int i = 0; i < NW; i++) dst[i] = wbuf[i];
        *(double*)(rec + A.code_stride - 8) = mumax;
    }
    // refinement count: one atomic per warp
    int tot = used;
#pragma unroll
    for (int sft = 16; sft > 0; sft >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, sft);
    if (lane == 0 && tot) atomicAdd(A.counts + 1, tot);
    // unfinished lanes: to the queue of phase B (their working sets must be visible first) or to the host's list
    const bool fail = valid && !ok && (reset || I.status[inst] != BMPC_PRIMAL_INFEASIBLE);
    const unsigned fmask = __ballot_sync(0xffffffffu, fail);
    const int nf = __popc(fmask), pos = __popc(fmask & ((1u << lane) - 1u));
    if (to_queue) {
        // one 64-bit atomic publishes "nf more entries reserved" and "one more chunk of phase A finished" together, so a
        // consumer that reads the word sees a tail that is final once the chunk count is complete
        if (fmask) {
            __threadfence();
            unsigned long long old = 0ull;
            if (lane == 0) old = atomicAdd((unsigned long long*)(A.counts + TPI_Q_TAIL), (1ull << 32) | (unsigned long long)nf);
            const int basep = (int)(unsigned)__shfl_sync(0xffffffffu, old, 0);
            if (fail) ((volatile int32_t*)A.queue)[basep + pos] = inst;
        } else if (lane == 0) atomicAdd((unsigned long long*)(A.counts + TPI_Q_TAIL), 1ull << 32);     // no return value: fire and forget
    } else if (fmask) {
        int basep = 0;
        if (lane == 0) basep = atomicAdd(A.counts, nf);
        basep = __shfl_sync(0xffffffffu, basep, 0);
        if (fail) {
            A.next_list[basep + pos] = inst;
            // its ADMM rounds start from the exact fixed point v* of its last verified solve, unless the last candidate is sane (hard
            // rows feasible to 1e-2): then from the candidate's rows and multipliers v = z + mu / rho (bmpc_candidate_usable's policy)
            bool usable = A.cand_warm != 0 && mode == 2 && A.list != nullptr && bmpc_admm_stalled(I.res + (size_t)inst * 4, I.iters[inst]);   // straggler rounds only
            double up = um1;
            for (int j = 0; j < S::NU && usable; j++) {
                const double u = udst[j], dz = u - up;
                const double uh = P.uhi, ul = P.ulo, dh = P.dhi, dl = P.dlo;
                usable = u <= uh + 1e-2 * (1.0 + fabs(uh)) && u >= ul - 1e-2 * (1.0 + fabs(ul)) &&
                         dz <= dh + 1e-2 * (1.0 + fabs(dh)) && dz >= dl - 1e-2 * (1.0 + fabs(dl));
                up = u;
            }
            if (usable) {
                double* dst = I.vw + (size_t)inst * S::mc;
                for (int i = 0; i < L::VROWS; i++) dst[nx + i] = W(tpi_vstar_slot<S>(i));
                dst[S::mc - 1] = vq;
#pragma unroll
                for (int q = 0; q < nx; q++) dst[q] = x0[q];
            }
        }
    }
    // v* = z* + y*/rho, the exact ADMM fixed point of this problem, staged in the consumed gain slots by the forward sweep: the
    // warm start of the ADMM rounds a later solve may need for this instance (measured: starting those rounds from the failed
    // candidate instead costs 10x the rounds).  Verified lanes only.
    const unsigned okmask = __ballot_sync(0xffffffffu, ok);
    if (okmask) {
        __syncwarp();
        if (ok) {
            double* dst = I.vw + (size_t)inst * S::mc;
#pragma unroll
            for (int q = 0; q < nx; q++) dst[q] = x0[q];
            dst[S::mc - 1] = vq;
        }
        if (inst0_contig >= 0) {
            // coalesced: for every verified instance t of the chunk the warp writes its rows 32 at a time (lane = row)
            constexpr int NG = (L::VROWS + 31) / 32;
            int soff[NG];
#pragma unroll
            for (int c = 0; c < NG; c++) { const int i = c * 32 + lane; soff[c] = (i < L::VROWS) ? tpi_vstar_slot<S>(i) * TPI_STR : -1; }
            double* dst = I.vw + (size_t)inst0_contig * S::mc + nx + lane;
            if (okmask == 0xffffffffu) {
                // every instance of the chunk verified (the steady state): 4 instances per trip, all loads ahead of the stores
#pragma unroll 1
                for (int t = 0; t < 32; t += 4) {
                    double val[4][NG];
#pragma unroll
                    for (int j = 0; j < 4; j++)
#pragma unroll
                        for (int c = 0; c < NG; c++) val[j][c] = (soff[c] >= 0) ? wsm[soff[c] + t + j] : 0.0;
#pragma unroll
                    for (int j = 0; j < 4; j++)
#pragma unroll
                        for (int c = 0; c < NG; c++) if (soff[c] >= 0) dst[(size_t)(t + j) * S::mc + c * 32] = val[j][c];
                }
            } else {
#pragma unroll 2
                for (int t = 0; t < nvalid; t++) {
                    if (!((okmask >> t) & 1u)) continue;
#pragma unroll
                    for (int c = 0; c < NG; c++) if (soff[c] >= 0) dst[(size_t)t * S::mc + c * 32] = wsm[soff[c] + t];
                }
            }
        } else if (ok) {
            double* dst = I.vw + (size_t)inst * S::mc;
            for (int i = 0; i < L::VROWS; i++) dst[nx + i] = W(tpi_vstar_slot<S>(i));
        }
    }
    __syncwarp();
}

// the parameters of one system that a fast path's per-instance view holds; false: QDu is not diagonal (the multi-input sweeps need
// it diagonal).  Both fills read only the raw inputs and scal: valid on a block whose condensed part is stale (after bmpc_update_problem)
template <class S>
__device__ __forceinline__ bool fill_view_params(const double* sys, const BmpcSysOff& o, TpiPolParams<S>& P) { tpi_fill_pol<S>(sys, o, P); return true; }
template <class S>
__device__ __forceinline__ bool fill_view_params(const double* sys, const BmpcSysOff& o, TpmParams<S>& P) { return tpm_fill<S>(sys, o, P); }

// per-instance parameter blocks (n_sys = batch) of either fast path, field-major in global memory (TpiPolView, TpmPolView): field f
// of instance i at pg[f * B + i].  nondiag: raised when some instance's QDu is not diagonal (never by the single-input fill)
template <class PS>
__global__ void k_fill_view(BmpcSysOff o, const double* __restrict__ sys, size_t sys_stride, int B, double* __restrict__ pg,
                            unsigned long long* nondiag) {
    const int inst = blockIdx.x * blockDim.x + threadIdx.x;
    if (inst >= B) return;
    PS P;
    const bool diag = fill_view_params(sys + (size_t)inst * sys_stride, o, P);
    const double* src = (const double*)&P;
    for (int f = 0; f < (int)(sizeof(PS) / sizeof(double)); f++) pg[(size_t)f * B + inst] = src[f];
    if (!diag) *nondiag = 1ull;
}

template <class S, bool TV, bool PERINST>
__global__ void __launch_bounds__(TpiPolLayout<S>::warps * 32, 1) k_tpi_pol(const __grid_constant__ TpiPolParams<S> P, BmpcInst I, TpiPolArgs A) {
    using L = TpiPolLayout<S>; using CT = typename TpiCode<S>::type;
    extern __shared__ double smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double* wsm = (double*)((char*)smem + (size_t)warp * L::per_warp);
    CT* csm = (CT*)((char*)wsm + L::gain_bytes);
    const int nchunks = (A.count + 31) / 32;
    if (blockIdx.x == 0 && threadIdx.x < BMPC_CNT) A.counts_next[threadIdx.x] = 0;
    if (threadIdx.x == 0) atomicMax((unsigned long long*)(A.counts + BMPC_CNT_T0), ~bmpc_globaltimer());
    // ---- phase A
    for (;;) {
        int chunk = 0;
        if (lane == 0) chunk = atomicAdd(A.counts + TPI_Q_CURSOR, 1);
        chunk = __shfl_sync(0xffffffffu, chunk, 0);
        if (chunk >= nchunks) break;
        const int idx0 = chunk * 32, nvalid = (A.count - idx0) < 32 ? (A.count - idx0) : 32;
        const bool valid = lane < nvalid;
        const int inst = A.list ? (valid ? A.list[idx0 + lane] : 0) : idx0 + lane;
        if constexpr (PERINST) { const TpiPolView<S> Pv(A.pview + inst, (size_t)A.pstride); tpi_pol_batch<S, TV>(Pv, I, A, wsm, csm, inst, valid, A.list ? -1 : idx0, nvalid, A.mode, A.capA, A.capB > 0, A.reset); }
        else tpi_pol_batch<S, TV>(P, I, A, wsm, csm, inst, valid, A.list ? -1 : idx0, nvalid, A.mode, A.capA, A.capB > 0, A.reset);
    }
    auto leave = [&]() {
        if (lane != 0) return;
        atomicMax((unsigned long long*)(A.counts + BMPC_CNT_T1), bmpc_globaltimer());
        if (A.epoch == 0) return;
        __threadfence_system();                 // this warp's u* stores (to peers / to mapped host memory too) before its exit count
        if (atomicAdd(A.counts + BMPC_CNT_EXIT, 1) == (int)(gridDim.x * L::warps) - 1) {          // (launch_tpi_pol: L::warps per CTA)
            // last warp out: every counter of the launch is final.
            __threadfence();
            volatile int32_t* src = (volatile int32_t*)A.counts; volatile int32_t* dst = (volatile int32_t*)A.host_counts;
            int gathered = 0;
            if (A.g_epoch > 0 && src[0] == 0) {
                // K6 arrival without a launch of its own: every instance of this rank is final and stored in every peer's gathered
                // buffer -> raise this rank's flag at the peers, then wait for theirs: when this kernel ends the gathered buffer of
                // the step is complete here.  (Instances left for straggler rounds: the host calls bmpc_gather_arrive afterwards.)
                __threadfence_system();
                for (int pr = 0; pr < A.g_npeer; pr++) *(volatile long long*)(A.gpeers.p[pr] + A.g_rank) = A.g_epoch;
                const long long t0 = clock64();
                for (int r = 0; r < A.g_world; r++) {
                    if (r == A.g_rank) continue;
                    while (*(volatile long long*)(A.gflags + r) < A.g_epoch) {
                        if (clock64() - t0 > 20000000000ll) __trap();        // ~10 s: a peer died; fail loudly instead of hanging the GPU
                        __nanosleep(100);
                    }
                }
                __threadfence_system();
                gathered = 1;
            }
            // ... and hand the counters to the host through mapped memory
            for (int i = 0; i < BMPC_CNT_EXIT; i++) dst[i] = src[i];
            dst[BMPC_CNT_TIGHT + 1] = gathered;
            __threadfence_system();
            dst[BMPC_CNT_EPOCH] = A.epoch;
        }
    };
    if (A.capB <= 0) { leave(); return; }
    // ---- phase B: serve the queue until every chunk of phase A is finished and the queue is empty.  Tickets: a warp takes the
    // next 32 queue slots with one fetch-and-add (no compare-and-swap races between a thousand warps) and waits until they are
    // filled or phase A has ended short of them, so batches are full while phase A still produces.
    volatile unsigned long long* ctl = (volatile unsigned long long*)(A.counts + TPI_Q_TAIL);
    for (;;) {
        int h = 0;
        if (lane == 0) h = atomicAdd(A.counts + TPI_Q_HEAD, 32);
        h = __shfl_sync(0xffffffffu, h, 0);
        const int idx = h + lane;
        int inst = -1;
        for (;;) {
            unsigned wlo = 0u, whi = 0u;
            if (lane == 0) { const unsigned long long w = *ctl; wlo = (unsigned)w; whi = (unsigned)(w >> 32); }   // tail | finished chunks
            wlo = __shfl_sync(0xffffffffu, wlo, 0); whi = __shfl_sync(0xffffffffu, whi, 0);
            const bool all_done = (int)whi >= nchunks;
            if (inst < 0 && idx < A.qcap && (idx < (int)wlo)) inst = ((volatile int32_t*)A.queue)[idx];
            const bool ready = inst >= 0 || (all_done && idx >= (int)wlo);
            if (__all_sync(0xffffffffu, ready)) break;
            __nanosleep(200);
        }
        const bool valid = inst >= 0;
        const unsigned vmask = __ballot_sync(0xffffffffu, valid);
        if (!vmask) break;                                            // ticket beyond the end of the queue: nothing left
        if (valid) ((volatile int32_t*)A.queue)[idx] = -1;            // the queue is all -1 again when the launch ends
        __threadfence();
        if constexpr (PERINST) { const TpiPolView<S> Pv(A.pview + (valid ? inst : 0), (size_t)A.pstride); tpi_pol_batch<S, TV>(Pv, I, A, wsm, csm, valid ? inst : 0, valid, -1, __popc(vmask), 0, A.capB, false, 0); }
        else tpi_pol_batch<S, TV>(P, I, A, wsm, csm, valid ? inst : 0, valid, -1, __popc(vmask), 0, A.capB, false, 0);
    }
    leave();
}


// ------------------------------------------------------------------------------------------------
// Multi-input fast path (bmpc_tpm.cuh): K5 of shapes with nu > 1, one shared system or per-instance systems (PERINST: parameters
// from each instance's view, TpmPolView) — the constrained Riccati polish with one
// THREAD per instance and one warp (32 instances) per CTA.  Gain rows in global memory (per resident warp: slots x 32 lanes,
// lane-interleaved), working sets in local memory, the system in the constant bank (kernel parameter).
//  mode -1: warm first round of a solve: per instance, the stored working sets shifted one stage (record flag set: its last
//           solve was verified here) or, failing that, the working sets read off its ADMM fixed point v* of the previous
//           problem (left by whichever kernel finished it), shifted;
//  mode  2: straggler rounds: an ADMM chunk of the team / tile kernels ran just before; working sets from the iterate v.
// Verified: plan, u0 (published like every epilogue: output slice, shadow, peers), status, v* (standard row order: the warm
// start of any later ADMM round), x (ADMM warm start), working-set record.  Not verified: listed for the next round.
struct TpmArgs {
    const int32_t* list; int count, mode, cap, reset;
    int32_t* counts; int32_t* next_list; double* u0_out; double* um1_solved;
    double* W; unsigned long long* rec; int rec_stride;               // record of instance i: Np code words, mumax, flag (rec_stride 64-bit words)
    const double* pview; int pstride;                                  // per-instance parameter blocks (PERINST instantiation): base and field stride (= batch)
};
struct TpmDiscard { unsigned long long sink; };

// the parameters k_tpm_pol's sweeps read: the kernel parameter (one shared system) or instance inst's view (per-instance systems)
template <bool PERINST, class S>
__device__ __forceinline__ decltype(auto) tpm_params_of(const TpmParams<S>& P, const TpmArgs& A, int inst) {
    if constexpr (PERINST) return TpmPolView<S>(A.pview + inst, (size_t)A.pstride);
    else return (P);
}

// sparsity pattern of n new per-instance matrices of cnt <= 64 entries (batch-major, instance i's at src[i * cnt]): bit f of *word is
// raised when entry f is non-zero in some instance (*word zeroed by the caller)
__global__ void k_tpm_pattern(const double* __restrict__ src, int cnt, int n, unsigned long long* word) {
    const int inst = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long m = 0ull;
    if (inst < n)
        for (int f = 0; f < cnt; f++) if (src[(size_t)inst * cnt + f] != 0.0) m |= 1ull << f;
    for (int s = 16; s > 0; s >>= 1) m |= __shfl_xor_sync(0xffffffffu, m, s);
    if ((threadIdx.x & 31) == 0 && m) atomicOr(word, m);
}

template <class S, bool TV, bool EX, bool PERINST>
__global__ void __launch_bounds__(32) k_tpm_pol(const __grid_constant__ TpmParams<S> Pk, BmpcInst I, TpmArgs A) {
    using L = TpmLayout<S>; using CD = TpmCode<S>;
    constexpr int nx = S::nx, nu = S::nu, Np = S::Np, NU = S::NU, mc = S::mc, NX = S::NX;
    const int lane = threadIdx.x, idx = blockIdx.x * 32 + lane;
    const bool valid = idx < A.count;
    const int inst = valid ? (A.list ? A.list[idx] : idx) : 0;
    auto&& P = tpm_params_of<PERINST>(Pk, A, inst);
    TpiStreamAcc W{A.W + (size_t)blockIdx.x * L::slots * 32 + lane, 32};
    uint64_t cur[Np], atb[Np];
    uint64_t dump = 0ull; uint64_t* const dp = &dump;
    auto C = [&](int k) -> uint64_t& { return cur[k]; };
    auto CB = [&](int k) -> uint64_t& { return atb[k]; };
    auto CK = [dp](int) -> uint64_t& { return *dp; };
    double x0[nx], um1[nu], xref[nx];
#pragma unroll
    for (int q = 0; q < nx; q++) { x0[q] = valid ? I.x0[(size_t)inst * nx + q] : 0.0; xref[q] = (valid && !TV) ? I.xref[(size_t)inst * nx + q] : 0.0; }
#pragma unroll
    for (int j = 0; j < nu; j++) um1[j] = valid ? I.um1[(size_t)inst * nu + j] : 0.0;
    const TpiXref<S, TV> xr{TV ? I.xref + (size_t)inst * NX : xref};
    unsigned long long* rec = A.rec + (size_t)inst * A.rec_stride;
    double mumax = 0.0;
    bool done = !valid, ok = false;
    if (valid) {
        const bool stored = A.mode < 0 && rec[Np + 1] == 1ull;
        if (stored) {
            uint64_t st[Np];
            for (int k = 0; k < Np; k++) st[k] = rec[k];
            unsigned first[nu];
#pragma unroll
            for (int j = 0; j < nu; j++) first[j] = (S::Nc > 1) ? tpm_first_label<S>(P, j, I.Us[(size_t)inst * NU + j], I.Us[(size_t)inst * NU + nu + j]) : 0u;
            const int tail = tpm_tail_start<S>(st);
            for (int k = 0; k < Np; k++) cur[k] = tpm_shifted_code<S>(st, k, true, first, tail);
            mumax = __longlong_as_double((long long)rec[Np]);
        } else {
            const double* v = I.vw + (size_t)inst * mc;
            tpm_codes_from_v<S>(P, um1, [&](int i) { return v[i]; }, C, A.mode < 0 ? 1 : 0);
        }
        if (A.mode == 2 && !A.reset && bmpc_residuals_tight(I.res + (size_t)inst * 4, I.iters[inst])) {
            // residuals far below any tolerance: the iterate is the answer although the active-set iteration cannot certify it
            const double* ua = I.Ua + (size_t)inst * NU;
            for (int a = 0; a < NU; a++) { I.Us[(size_t)inst * NU + a] = ua[a]; if (a < nu) bmpc_publish_u0(I, A.u0_out, (size_t)inst * nu + a, ua[a]); }
            I.status[inst] = BMPC_SOLVED_UNPOLISHED; atomicAdd(A.counts + BMPC_CNT_TIGHT, 1);
            done = true;
        }
    }
    const bool live = valid && !done;
    double vfirst[nu], vq = 0.0;
    double* udst = I.Us + (size_t)inst * NU;
    int used = 0;
    for (int r = 0; r < A.cap; r++) {
        if (!done) {
            tpm_backward<S>(P, W, C, xr, um1);
            const int fl = tpm_forward<S, EX>(P, W, C, CB, CK, x0, um1, mumax, vfirst, vq, [&](int k, int j, double u) { udst[k * nu + j] = u; });
            used++;
            ok = fl == 0; done = ok;
        }
        if (__all_sync(0xffffffffu, done)) break;
    }
    ok = ok && live;
    if (valid && A.reset) {
        I.iters[inst] = 0; I.psteps[inst] = 0; I.lvl[inst] = BMPC_LEV0;
#pragma unroll
        for (int j = 0; j < nu; j++) A.um1_solved[(size_t)inst * nu + j] = um1[j];
        if (!ok) I.status[inst] = BMPC_UNSOLVED;
    }
    if (live) {
        I.psteps[inst] += used;
        if (ok) {
#pragma unroll
            for (int j = 0; j < nu; j++) bmpc_publish_u0(I, A.u0_out, (size_t)inst * nu + j, udst[j]);
            I.status[inst] = BMPC_SOLVED;
            double* xw = I.xw + (size_t)inst * NU;
            for (int a = 0; a < NU; a++) xw[a] = udst[a];
            // v* in the standard row order
            double* v = I.vw + (size_t)inst * mc;
#pragma unroll
            for (int q = 0; q < nx; q++) v[q] = x0[q];
            for (int k = 0; k < Np; k++)
                for (int p = 0; p < 2 * nu + nx; p++) { const int row = tpm_vstar_row<S>(k, p); if (row >= 0) v[row] = W.ld(k * L::per_stage + p); }
#pragma unroll
            for (int j = 0; j < nu; j++) v[NX + NU + j] = vfirst[j];
            v[mc - 1] = vq;
            for (int k = 0; k < Np; k++) rec[k] = atb[k];
            rec[Np] = (unsigned long long)__double_as_longlong(mumax); rec[Np + 1] = 1ull;
        } else {
            rec[Np + 1] = 0ull;                                         // whoever finishes this instance leaves v*: the next solve starts from that
        }
    }
    int tot = live ? used : 0;
#pragma unroll
    for (int sft = 16; sft > 0; sft >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, sft);
    if (lane == 0 && tot) atomicAdd(A.counts + 1, tot);
    const bool fail = live && !ok && (A.reset || I.status[inst] != BMPC_PRIMAL_INFEASIBLE);
    const unsigned fmask = __ballot_sync(0xffffffffu, fail);
    if (fmask) {
        int basep = 0;
        if (lane == 0) basep = atomicAdd(A.counts, __popc(fmask));
        basep = __shfl_sync(0xffffffffu, basep, 0);
        if (fail) A.next_list[basep + __popc(fmask & ((1u << lane) - 1u))] = inst;
    }
}

// One compiled fast-path entry: a shape of the single-input fast path (one line of csrc/tpi_shapes.inc; `python -m pympc_b200.build
// --add-shape nx,1,Np` appends one and rebuilds) or a shape and (Ad, Bd) pattern of the multi-input one (csrc/tpm_shapes.inc)
struct BmpcFastEntry {
    int family;                        // BMPC_FAM_TPI or BMPC_FAM_TPM
    int nx, nu, Np, Nc;
    unsigned long long amask; unsigned bmask;   // (Ad, Bd) entries the kernels may find non-zero (all ones: any system)
    size_t par_bytes;                  // host copy of the parameters (single-input: k_tpi_admm's block, then k_tpi_pol's)
    int slots;                         // multi-input: gain slots per lane of the workspace
    bool (*fill)(const double* hs, const BmpcSysOff& o, void* par);   // from system 0's block; false: declines (QDu not diagonal)
    int view_fields, view_ad, view_bd; // per-instance parameter view: doubles per instance, field numbers of Ad and Bd (k_sys_refresh)
    void (*fill_view)(struct bmpc_handle* h);
    int (*configure)();                // single-input: shared-memory opt-in of its kernels (nullptr: none)
    void (*launch)(struct bmpc_handle* h, const int32_t* list, int count, const BmpcRoundPlan& p, int32_t* next_list);
};

// ------------------------------------------------------------------------------------------------
// host side
struct bmpc_handle {
    bmpc_config cfg;
    BmpcDims d;
    BmpcSysOff o;
    BmpcLaunch launch = {};            // team size, polish tiers and tile size (bmpc_plan_launch); each team round: bmpc_round_launch
    int sm_count = 132;
    cudaStream_t stream, own_stream;
    double* sys = nullptr;
    BmpcInst I;
    double *x0 = nullptr, *um1 = nullptr, *um1_alt = nullptr, *um1_solved = nullptr, *xref = nullptr, *u0_own = nullptr, *u0_bound = nullptr;
    const double *x0_cur = nullptr, *um1_cur = nullptr;    // what the next solve reads: the handle's copies or buffers borrowed from the caller (bmpc_update on_device = 2)
    int cpar = 0;                                          // which half of counts[16] the round in flight uses (the fast-path kernel zeroes the other half for the next one)
    double *seq_x = nullptr, *seq_e = nullptr, *seq_obj = nullptr;
    int32_t *listA = nullptr, *listB = nullptr, *counts = nullptr;  // counts[8]: [0..3] round counters, [4..7] queue control of k_tpi_pol
    long long* gflags = nullptr; BmpcPeerFlags gpeers = {}; int g_npeer = 0, g_rank = 0, g_world = 1;   // K6 arrival flags
    long long g_epoch = 0, g_done_epoch = 0;       // one epoch per solve while flags are bound; the last epoch whose arrival is complete
    int32_t* queue = nullptr; unsigned char* codes = nullptr;        // phase-B queue and stored working sets of the fast-path polish
    int code_stride = 0;                                             // bytes per instance of codes
    int32_t* h_count = nullptr;                                      // pinned, mapped
    int epoch = 0, spin_epoch = 0;                                   // launch epochs of the fast-path kernel's host notification
    cudaEvent_t ev[4];
    int xref_mode = 0;
    const int32_t* status_filled = nullptr;   // host status array last filled with BMPC_SOLVED everywhere (skip refilling it)
    bool sync_after_round = false;     // bmpc_output queued a result copy behind the round: wait for the stream, not only for the kernel
    bool is_setup = false, cold = true, solved = false, committed = true;   // committed: this solve's u0 already is the next u_-1
    bmpc_stats stats;
    std::string err;
    int32_t* ovf = nullptr;            // overflow list of the first polish tier, read by the second
    double* vprev = nullptr; int32_t* lprev = nullptr;   // snapshot of (v, level) for the infeasibility check of straggler rounds
    void (*tile_fn[3])(BmpcDims, BmpcSysOff, const double*, BmpcInst, const int32_t*, int, int, int, int, int, int) = {nullptr, nullptr, nullptr};   // tiles of 8, 4, 2
    struct { const int32_t* list; int count; int32_t *cur, *nxt; int total, chunk, round; bool need_prep; int tight; bool cold; } st = {};
    bool pending = false;              // a round is in flight and has not been retired by the host yet
    const BmpcFastEntry* fast = nullptr;   // the fast-path entry the handle runs on (select_fast); nullptr: the team kernels
    void* fast_par = nullptr;          // host copy of its parameters
    // the fast path's per-instance parameter blocks (n_sys = batch; TpiPolView or TpmPolView): field f of instance i at p[f * B + i],
    // in the layout of entry e.  Recorded once at setup; bmpc_update_problem writes Ad / Bd into fields e->view_ad / view_bd
    // (k_sys_refresh) and rebuilds the rest with e->fill_view
    struct { double* p; const BmpcFastEntry* e; } view = {};
    bool codes_valid = false;         // the stored working sets come from a fast-path polish of the whole batch
    double* tpm_W = nullptr; unsigned long long* tpm_rec = nullptr;   // gain rows of the resident warps, working-set records
    int tpm_W_slots = 0;               // gain slots per lane tpm_W was allocated for
    // per-instance systems on a multi-input view: the union of the instances' (Ad, Bd) patterns and whether some instance's QDu is not
    // diagonal decide the entry (select_fast).  tpm_word (device) / tpm_hword (pinned host): the pattern words of a device update
    // [0] Ad, [1] Bd, and [2] the "QDu not diagonal" flag of k_fill_view
    unsigned long long tpm_am = 0ull; unsigned tpm_bm = 0u; bool tpm_nondiag = false;
    unsigned long long *tpm_word = nullptr, *tpm_hword = nullptr;
    BmpcPolicy policy = {};            // round policy of the chosen kernel family (bmpc_rounds.cuh)
    // time-varying (Ad, Bd), bmpc_update_system.  Per-instance systems: every instance's condensed block carries the generation it
    // was condensed for (sys_gen[i]); bmpc_update_system moves the handle's counter ahead of all of them and k_condense_list brings
    // an instance up to date right before the first launch that reads its condensed block.
    int32_t* sys_gen = nullptr; int32_t sys_gen_cur = 0;
    bool sys_stale = false;            // some instance's condensed block may predate its (Ad, Bd)
    bool sys_lazy = false;             // H is positive definite whatever (Ad, Bd) are (decided at setup and whenever the weights
                                       // change): the condense may be deferred
    bool sys_bad = false;              // the last update failed the positive-definiteness check: bmpc_solve refuses
    double* sys_stage = nullptr;       // device copy of host arrays for k_sys_refresh: array f of all systems at sys_stage[B * o.f]
};

static std::string g_create_err;

#define BMPC_CUDA(call)                                                                            \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            h->err = std::string(#call) + ": " + cudaGetErrorString(e_);                           \
            return BMPC_ERR_CUDA;                                                                  \
        }                                                                                          \
    } while (0)

// host copy of a single-input entry's parameters: the constant-bank blocks of k_tpi_admm and k_tpi_pol
template <class S>
struct TpiHostParams { TpiAdmmParams<S> admm; TpiPolParams<S> pol; };

template <class S>
static void launch_tpi_pol(bmpc_handle* h, const int32_t* list, int count, int mode, int capA, int capB, int reset, int32_t* next_list) {
    using L = TpiPolLayout<S>;
    const TpiPolParams<S>& PP = ((const TpiHostParams<S>*)h->fast_par)->pol;
    TpiPolArgs A;
    A.list = list; A.count = count; A.mode = mode; A.capA = capA; A.capB = capB; A.reset = reset;
    A.next_list = next_list; A.counts = h->counts + BMPC_CNT * h->cpar; A.counts_next = h->counts + BMPC_CNT * (1 - h->cpar); A.queue = h->queue; A.qcap = h->cfg.batch; A.u0_out = h->I.u0; A.um1_solved = h->um1_solved;
    A.codes = h->codes; A.code_stride = L::code_stride; A.cand_warm = h->cfg.candidate_warm;
    const int nchunks = (count + 31) / 32;
    int grid = (nchunks + L::warps - 1) / L::warps;
    if (grid > h->sm_count) grid = h->sm_count;
    if (grid < 1) grid = 1;
    const size_t sm = L::smem;
    constexpr int threads = L::warps * 32;          // the kernel's last-warp exit count assumes exactly this block size
    A.pview = h->view.p; A.pstride = h->cfg.batch;
    A.host_counts = h->h_count; A.epoch = h->spin_epoch;
    A.gflags = h->gflags; A.gpeers = h->gpeers; A.g_npeer = h->g_npeer; A.g_rank = h->g_rank; A.g_world = h->g_world;
    A.g_epoch = (h->gflags && h->spin_epoch && h->g_world > 1) ? h->g_epoch : 0;
    if (h->view.p) {
        if (h->xref_mode) k_tpi_pol<S, true, true><<<grid, threads, sm, h->stream>>>(PP, h->I, A);
        else k_tpi_pol<S, false, true><<<grid, threads, sm, h->stream>>>(PP, h->I, A);
    } else {
        if (h->xref_mode) k_tpi_pol<S, true, false><<<grid, threads, sm, h->stream>>>(PP, h->I, A);
        else k_tpi_pol<S, false, false><<<grid, threads, sm, h->stream>>>(PP, h->I, A);
    }
    h->stats.launches++;
}

// k_tpi_pol of a round, after k_tpi_admm when the plan has it (first round of a cold or first_iters solve on a shared system: the
// polish then reads its working sets off the iterate).  Without ADMM in the round the first launch resets the instances itself.
template <class S>
static void launch_tpi(bmpc_handle* h, const int32_t* list, int count, const BmpcRoundPlan& p, int32_t* next_list) {
    if (p.admm == BMPC_ADMM_TPI) {
        const int grid = (count + 31) / 32;
        const TpiAdmmParams<S>& PA = ((const TpiHostParams<S>*)h->fast_par)->admm;
        const int cold = h->cold ? 1 : 0;
        const size_t sa = S::MT * TPI_STR * 8;
        if (h->xref_mode)   // one (Np+1) x nx reference per instance
            k_tpi_admm<S, true><<<grid, 32, sa, h->stream>>>(PA, h->I, list, count, p.chunk, cold, p.reset, h->counts + BMPC_CNT * h->cpar, h->um1_solved);
        else
            k_tpi_admm<S, false><<<grid, 32, sa, h->stream>>>(PA, h->I, list, count, p.chunk, cold, p.reset, h->counts + BMPC_CNT * h->cpar, h->um1_solved);
        h->stats.launches++;
        cudaEventRecord(h->ev[1], h->stream);
    }
    launch_tpi_pol<S>(h, list, count, p.ws, p.capA, p.capB, p.admm == BMPC_ADMM_NONE ? p.reset : 0, next_list);
}

template <class S>
static bool tpi_fill_entry(const double* hs, const BmpcSysOff& o, void* par) {
    TpiHostParams<S>& P = *(TpiHostParams<S>*)par;
    tpi_fill_admm<S>(hs, o, P.admm); tpi_fill_pol<S>(hs, o, P.pol);
    return true;
}
template <class S>
static int tpi_configure_entry() {
    if (cudaFuncSetAttribute(k_tpi_admm<S, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(S::MT * TPI_STR * 8)) != cudaSuccess) return 1;
    if (cudaFuncSetAttribute(k_tpi_admm<S, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(S::MT * TPI_STR * 8)) != cudaSuccess) return 1;
    const int sm = (int)TpiPolLayout<S>::smem;
    if (cudaFuncSetAttribute(k_tpi_pol<S, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm) != cudaSuccess) return 1;
    if (cudaFuncSetAttribute(k_tpi_pol<S, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm) != cudaSuccess) return 1;
    if (cudaFuncSetAttribute(k_tpi_pol<S, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm) != cudaSuccess) return 1;
    if (cudaFuncSetAttribute(k_tpi_pol<S, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm) != cudaSuccess) return 1;
    return 0;
}

// k_tpm_pol of a round.  Its first launch resets the instances itself when no ADMM ran before it in the round
template <class S>
static void launch_tpm(bmpc_handle* h, const int32_t* list, int count, const BmpcRoundPlan& p, int32_t* next_list) {
    TpmArgs A;
    A.list = list; A.count = count; A.mode = p.ws; A.cap = p.cap; A.reset = p.admm == BMPC_ADMM_NONE ? p.reset : 0;
    A.counts = h->counts + BMPC_CNT * h->cpar; A.next_list = next_list; A.u0_out = h->I.u0; A.um1_solved = h->um1_solved;
    A.W = h->tpm_W; A.rec = h->tpm_rec; A.rec_stride = S::Np + 2;
    A.pview = h->view.p; A.pstride = h->cfg.batch;
    const TpmParams<S>& P = *(const TpmParams<S>*)h->fast_par;
    const int grid = (count + 31) / 32;
    // exchange: the straggler rounds' instantiation (hard rows change by single exchanges, tpm_forward<S, true>); per-instance
    // systems (a view): the instantiation that reads each instance's view
    if (h->view.p) {
        if (p.exchange) {
            if (h->xref_mode) k_tpm_pol<S, true, true, true><<<grid, 32, 0, h->stream>>>(P, h->I, A);
            else k_tpm_pol<S, false, true, true><<<grid, 32, 0, h->stream>>>(P, h->I, A);
        } else {
            if (h->xref_mode) k_tpm_pol<S, true, false, true><<<grid, 32, 0, h->stream>>>(P, h->I, A);
            else k_tpm_pol<S, false, false, true><<<grid, 32, 0, h->stream>>>(P, h->I, A);
        }
    } else if (p.exchange) {
        if (h->xref_mode) k_tpm_pol<S, true, true, false><<<grid, 32, 0, h->stream>>>(P, h->I, A);
        else k_tpm_pol<S, false, true, false><<<grid, 32, 0, h->stream>>>(P, h->I, A);
    } else {
        if (h->xref_mode) k_tpm_pol<S, true, false, false><<<grid, 32, 0, h->stream>>>(P, h->I, A);
        else k_tpm_pol<S, false, false, false><<<grid, 32, 0, h->stream>>>(P, h->I, A);
    }
    h->stats.launches++;
}
template <class S>
static bool tpm_fill_entry(const double* hs, const BmpcSysOff& o, void* par) { return tpm_fill<S>(hs, o, *(TpmParams<S>*)par); }

// rebuilds the handle's view from every instance's block (PS: the parameter block of its entry); a multi-input view also gets the
// "QDu not diagonal" word tpm_word[2] (allocated with such a view only)
template <class PS>
static void fill_view_entry(bmpc_handle* h) {
    const int B = h->cfg.batch;
    unsigned long long* nondiag = h->tpm_word ? h->tpm_word + 2 : nullptr;
    if (nondiag) cudaMemsetAsync(nondiag, 0, sizeof(unsigned long long), h->stream);
    k_fill_view<PS><<<(B + 63) / 64, 64, 0, h->stream>>>(h->o, h->sys, (size_t)h->o.total, B, h->view.p, nondiag);
}
template <class PS>
static constexpr int view_field_ad() { return (int)(offsetof(PS, Ad) / sizeof(double)); }
template <class PS>
static constexpr int view_field_bd() { return (int)(offsetof(PS, Bd) / sizeof(double)); }

template <class S>
static constexpr BmpcFastEntry tpi_entry() {
    using PS = TpiPolParams<S>;
    return {BMPC_FAM_TPI, S::nx, S::nu, S::Np, S::Nc, S::amask, S::bmask, sizeof(TpiHostParams<S>), 0, tpi_fill_entry<S>,
            (int)(sizeof(PS) / sizeof(double)), view_field_ad<PS>(), view_field_bd<PS>(), fill_view_entry<PS>, tpi_configure_entry<S>, launch_tpi<S>};
}
template <class S>
static constexpr BmpcFastEntry tpm_entry() {
    using PS = TpmParams<S>;
    return {BMPC_FAM_TPM, S::nx, S::nu, S::Np, S::Nc, S::amask, S::bmask, sizeof(PS), TpmLayout<S>::slots, tpm_fill_entry<S>,
            (int)(sizeof(PS) / sizeof(double)), view_field_ad<PS>(), view_field_bd<PS>(), fill_view_entry<PS>, nullptr, launch_tpm<S>};
}
// BMPC_TPI_SHAPES_FILE / BMPC_TPM_SHAPES_FILE: pympc_b200.build.jit_shape() / jit_multi_input_shape() compile a copy of the library
// whose table holds the one shape a controller asked for when the in-tree table does not have it.  Entries are tried in order:
// single-input shapes first; of a multi-input shape the sparse patterns first, its dense instantiation last
#define BMPC_TPI_SHAPE(NX_, NU_, NP_, NC_) tpi_entry<TpiShape<NX_, NU_, NP_, NC_>>(),
#define BMPC_TPM_SHAPE(NX_, NU_, NP_, NC_) tpm_entry<TpiShape<NX_, NU_, NP_, NC_>>(),
#define BMPC_TPM_SPARSE_SHAPE(NX_, NU_, NP_, NC_, AM_, BM_) tpm_entry<TpmSparseShape<NX_, NU_, NP_, NC_, AM_, BM_>>(),
#ifndef BMPC_TPI_SHAPES_FILE
#define BMPC_TPI_SHAPES_FILE "tpi_shapes.inc"
#endif
#ifndef BMPC_TPM_SHAPES_FILE
#define BMPC_TPM_SHAPES_FILE "tpm_shapes.inc"
#endif
static const BmpcFastEntry g_fast[] = {
#include BMPC_TPI_SHAPES_FILE
#include BMPC_TPM_SHAPES_FILE
};
#undef BMPC_TPI_SHAPE
#undef BMPC_TPM_SHAPE
#undef BMPC_TPM_SPARSE_SHAPE

static bool same_shape(const BmpcFastEntry& e, const BmpcDims& d) { return e.nx == d.nx && e.nu == d.nu && e.Np == d.Np && e.Nc == d.Nc; }
static bool has_entry(int family, const BmpcDims& d) {
    for (const BmpcFastEntry& e : g_fast) if (e.family == family && same_shape(e, d)) return true;
    return false;
}

extern "C" {

static int finish_solve(bmpc_handle* h);

void bmpc_default_config(bmpc_config* c) {
    memset(c, 0, sizeof(*c));
    c->Np = 20; c->Nc = 0; c->batch = 1; c->device = 0; c->soft_on = 1;
    c->max_iter = 4000; c->first_iters = 0; c->pdas_steps = 10; c->rmax = 0; c->polish = 1;
    c->team_threads = 0; c->warps_per_block = 0; c->fast_path = 1; c->n_sys = 1; c->shift_warm = 1; c->candidate_warm = 0; c->cold_iters = 0;
    c->eps_feas = 1e6; c->rho = 0.0; c->sigma = 1e-6; c->alpha = 1.6; c->eps_abs = 1e-3; c->eps_rel = 1e-3;
}

int bmpc_has_fast_path(int nx, int nu, int Np, int Nc) {
    return has_entry(BMPC_FAM_TPI, bmpc_make_dims(nx, nu, Np, Nc <= 0 ? Np : Nc));
}

int bmpc_has_multi_input_fast_path(int nx, int nu, int Np, int Nc) {
    return has_entry(BMPC_FAM_TPM, bmpc_make_dims(nx, nu, Np, Nc <= 0 ? Np : Nc));
}

int bmpc_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

const char* bmpc_last_error(const bmpc_handle* h) { return h ? h->err.c_str() : g_create_err.c_str(); }

void* bmpc_host_alloc(uint64_t bytes) {
    void* p = nullptr;
    // mapped + portable: the device can read / write the buffer in place (bmpc_update on_device = 2, bmpc_bind_output): with unified
    // addressing the host pointer is the device pointer
    if (cudaHostAlloc(&p, bytes, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void bmpc_host_free(void* p) { if (p) cudaFreeHost(p); }

static int configure_launch(bmpc_handle* h) {
    const BmpcDims& d = h->d;
    int dev = h->cfg.device, max_optin = 0;
    cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    cudaDeviceGetAttribute(&h->sm_count, cudaDevAttrMultiProcessorCount, dev);
    // team size, tiers and tile size: one decision the host emulation shares (bmpc_launch.cuh)
    const BmpcLaunch& L = h->launch = bmpc_plan_launch(d, max_optin, h->cfg.team_threads, h->cfg.warps_per_block, h->cfg.rmax, h->cfg.n_sys);
    if (!L.ok) { h->err = "problem too large for the shared-memory resident kernels"; return BMPC_ERR_ARG; }
    if (L.tile_T) {
        // kernels per tile size {8, 4, 2}; shapes with a compiled (nx, nu) get the unrolled instantiation
        if (d.nx == 8 && d.nu == 4) { h->tile_fn[0] = k_admm_tile<8, 2, 8, 4>; h->tile_fn[1] = k_admm_tile<4, 2, 8, 4>; h->tile_fn[2] = k_admm_tile<2, 1, 8, 4>; }
        else { h->tile_fn[0] = k_admm_tile<8, 2, 0, 0>; h->tile_fn[1] = k_admm_tile<4, 2, 0, 0>; h->tile_fn[2] = k_admm_tile<2, 1, 0, 0>; }
        for (int k = 0; k < 3; k++) {
            const int T = 8 >> k;
            if (L.tile_T >= T) BMPC_CUDA(cudaFuncSetAttribute((const void*)h->tile_fn[k], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bmpc_tile_smem_doubles(d, T) * 8)));
        }
    }
    if (L.team == 32) {
        BMPC_CUDA(cudaFuncSetAttribute(k_admm<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem_admm));
        BMPC_CUDA(cudaFuncSetAttribute(k_polish<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem_polish));
        if (L.fb_team) BMPC_CUDA(cudaFuncSetAttribute(k_polish<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.fb_smem_polish));
    } else {
        BMPC_CUDA(cudaFuncSetAttribute(k_admm<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem_admm));
        BMPC_CUDA(cudaFuncSetAttribute(k_polish<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem_polish));
    }
    return BMPC_OK;
}

int bmpc_create(const bmpc_config* cfg, bmpc_handle** out) {
    if (!cfg || !out) { g_create_err = "null argument"; return BMPC_ERR_ARG; }
    *out = nullptr;
    if (cfg->nx < 1 || cfg->nu < 1 || cfg->Np < 2 || cfg->batch < 1 || (cfg->Nc > cfg->Np)) {
        g_create_err = "invalid dimensions (need nx,nu >= 1, Np > 1, Nc <= Np, batch >= 1)"; return BMPC_ERR_ARG;
    }
    int ndev = bmpc_device_count();
    if (ndev <= 0) { g_create_err = "no CUDA device visible: libbmpc has no CPU fallback"; return BMPC_ERR_NO_DEVICE; }
    if (cfg->device < 0 || cfg->device >= ndev) { g_create_err = "device ordinal out of range"; return BMPC_ERR_ARG; }
    if (cfg->n_sys != 0 && cfg->n_sys != 1 && cfg->n_sys != cfg->batch) { g_create_err = "n_sys must be 1 (shared system) or batch (one system per instance)"; return BMPC_ERR_ARG; }
    bmpc_handle* h = new bmpc_handle();
    h->cfg = *cfg;
    if (h->cfg.n_sys <= 0) h->cfg.n_sys = 1;
    if (h->cfg.Nc <= 0) h->cfg.Nc = h->cfg.Np;
    if (h->cfg.max_iter <= 0) h->cfg.max_iter = 4000;
    if (h->cfg.pdas_steps <= 0) h->cfg.pdas_steps = 10;
    h->d = bmpc_make_dims(cfg->nx, cfg->nu, h->cfg.Np, h->cfg.Nc);
    h->o = bmpc_make_off(h->d);
    memset(&h->I, 0, sizeof(h->I)); memset(&h->stats, 0, sizeof(h->stats));
    auto fail = [&](int code) { g_create_err = h->err; bmpc_destroy(h); return code; };
    cudaError_t e = cudaSetDevice(cfg->device);
    if (e != cudaSuccess) { h->err = cudaGetErrorString(e); return fail(BMPC_ERR_CUDA); }
    if (cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking) != cudaSuccess) { h->err = "stream create failed"; return fail(BMPC_ERR_CUDA); }
    h->stream = h->own_stream;
    for (int i = 0; i < 4; i++) cudaEventCreate(&h->ev[i]);
    int rc = configure_launch(h);
    if (rc) return fail(rc);
    const BmpcDims& d = h->d; size_t B = cfg->batch;
    auto dalloc = [&](void** p, size_t bytes) { return cudaMalloc(p, bytes ? bytes : 8) == cudaSuccess; };
    bool ok = true;
    ok &= dalloc((void**)&h->sys, sizeof(double) * (size_t)h->o.total * h->cfg.n_sys);
    ok &= dalloc((void**)&h->x0, sizeof(double) * B * d.nx);
    ok &= dalloc((void**)&h->um1, sizeof(double) * B * d.nu);
    ok &= dalloc((void**)&h->um1_alt, sizeof(double) * B * d.nu);
    ok &= dalloc((void**)&h->um1_solved, sizeof(double) * B * d.nu);
    ok &= dalloc((void**)&h->xref, sizeof(double) * B * d.NX);
    ok &= dalloc((void**)&h->u0_own, sizeof(double) * B * d.nu);
    ok &= dalloc((void**)&h->I.g, sizeof(double) * B * d.NU);
    ok &= dalloc((void**)&h->I.cc, sizeof(double) * B * d.NX);
    ok &= dalloc((void**)&h->I.xw, sizeof(double) * B * d.NU);
    ok &= dalloc((void**)&h->I.vw, sizeof(double) * B * d.mc);
    ok &= dalloc((void**)&h->I.Ua, sizeof(double) * B * d.NU);
    ok &= dalloc((void**)&h->I.Us, sizeof(double) * B * d.NU);
    ok &= dalloc((void**)&h->I.res, sizeof(double) * B * 4);
    ok &= dalloc((void**)&h->I.status, sizeof(int32_t) * B);
    ok &= dalloc((void**)&h->I.iters, sizeof(int32_t) * B);
    ok &= dalloc((void**)&h->I.psteps, sizeof(int32_t) * B);
    ok &= dalloc((void**)&h->I.lvl, sizeof(int32_t) * B);
    ok &= dalloc((void**)&h->listA, sizeof(int32_t) * B);
    ok &= dalloc((void**)&h->listB, sizeof(int32_t) * B);
    ok &= dalloc((void**)&h->counts, sizeof(int32_t) * 2 * BMPC_CNT);
    ok &= dalloc((void**)&h->queue, sizeof(int32_t) * B);
    h->code_stride = tpi_code_stride(d.nx, d.Np);          // the record of this shape's single-input entry (TpiPolLayout asserts it)
    ok &= dalloc((void**)&h->codes, (size_t)B * h->code_stride);
    ok &= dalloc((void**)&h->ovf, sizeof(int32_t) * (size_t)B);
    ok &= dalloc((void**)&h->vprev, sizeof(double) * (size_t)B * d.mc);
    ok &= dalloc((void**)&h->lprev, sizeof(int32_t) * (size_t)B);
    if (!ok) { h->err = "cudaMalloc failed"; cudaGetLastError(); return fail(BMPC_ERR_CUDA); }
    if (cudaHostAlloc((void**)&h->h_count, sizeof(int32_t) * BMPC_CNT, cudaHostAllocMapped) != cudaSuccess) { h->err = "cudaHostAlloc failed"; return fail(BMPC_ERR_CUDA); }
    cudaMemset(h->sys, 0, sizeof(double) * (size_t)h->o.total * h->cfg.n_sys);
    cudaMemset(h->x0, 0, sizeof(double) * B * d.nx);
    cudaMemset(h->um1, 0, sizeof(double) * B * d.nu);
    cudaMemset(h->xref, 0, sizeof(double) * B * d.NX);
    cudaMemset(h->u0_own, 0, sizeof(double) * B * d.nu);
    cudaMemset(h->I.Us, 0, sizeof(double) * B * d.NU);
    cudaMemset(h->I.Ua, 0, sizeof(double) * B * d.NU);
    cudaMemset(h->queue, 0xff, sizeof(int32_t) * B);
    cudaMemset(h->codes, 0, (size_t)B * h->code_stride);
    cudaMemset(h->counts, 0, sizeof(int32_t) * 2 * BMPC_CNT);
    cudaMemset(h->um1_alt, 0, sizeof(double) * B * d.nu);
    h->I.sys_stride = h->cfg.n_sys > 1 ? (size_t)h->o.total : 0;
    h->I.x0 = h->x0; h->I.um1 = h->um1; h->I.um1_solved = h->um1_solved; h->I.xref = h->xref; h->I.u0 = h->u0_own; h->I.u0_shadow = h->um1_alt;
    h->x0_cur = h->x0; h->um1_cur = h->um1;
    k_reset<<<(int)((B + 255) / 256), 256, 0, h->stream>>>(h->I, (int)B);
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { h->err = "device initialisation failed"; return fail(BMPC_ERR_CUDA); }
    *out = h;
    return BMPC_OK;
}

void bmpc_destroy(bmpc_handle* h) {
    if (!h) return;
    cudaSetDevice(h->cfg.device);
    if (h->pending) cudaStreamSynchronize(h->stream);
    void* ptrs[] = {h->sys, h->x0, h->um1, h->um1_alt, h->um1_solved, h->xref, h->u0_own, h->I.g, h->I.cc, h->I.xw, h->I.vw, h->I.Ua, h->I.Us, h->I.res,
                    h->I.status, h->I.iters, h->I.psteps, h->I.lvl, h->listA, h->listB, h->counts, h->queue, h->codes, h->ovf, h->vprev, h->lprev, h->seq_x, h->seq_e, h->seq_obj};
    for (void* p : ptrs) if (p) cudaFree(p);
    if (h->h_count) cudaFreeHost(h->h_count);
    free(h->fast_par);
    if (h->view.p) cudaFree(h->view.p);
    if (h->tpm_word) cudaFree(h->tpm_word);
    if (h->tpm_hword) cudaFreeHost(h->tpm_hword);
    if (h->tpm_W) cudaFree(h->tpm_W);
    if (h->tpm_rec) cudaFree(h->tpm_rec);
    if (h->sys_gen) cudaFree(h->sys_gen);
    if (h->sys_stage) cudaFree(h->sys_stage);
    for (int i = 0; i < 4; i++) if (h->ev[i]) cudaEventDestroy(h->ev[i]);
    if (h->own_stream) cudaStreamDestroy(h->own_stream);
    delete h;
}

int bmpc_set_stream(bmpc_handle* h, void* s) {
    if (!h) return BMPC_ERR_ARG;
    if (h->pending) { cudaSetDevice(h->cfg.device); int rc = finish_solve(h); if (rc) return rc; }
    h->stream = s ? (cudaStream_t)s : h->own_stream;
    return BMPC_OK;
}

int bmpc_synchronize(bmpc_handle* h) {
    if (!h) return BMPC_ERR_ARG;
    BMPC_CUDA(cudaSetDevice(h->cfg.device));
    if (h->pending) { int rc = finish_solve(h); if (rc) return rc; }
    BMPC_CUDA(cudaStreamSynchronize(h->stream));
    return BMPC_OK;
}

int bmpc_bind_output(bmpc_handle* h, double* dev_u0) {
    if (!h) return BMPC_ERR_ARG;
    // kernels in flight captured the old pointer: retire them first (the committed u_-1 of that solve stays what it was)
    if (h->pending) { cudaSetDevice(h->cfg.device); int rc = finish_solve(h); if (rc) return rc; }
    h->u0_bound = dev_u0;
    h->I.u0 = dev_u0 ? dev_u0 : h->u0_own;
    return BMPC_OK;
}

int bmpc_bind_output_peers(bmpc_handle* h, double* const* peer_u0, int n) {
    if (!h || n < 0 || n > 8 || (n > 0 && !peer_u0)) return BMPC_ERR_ARG;
    if (h->pending) { cudaSetDevice(h->cfg.device); int rc = finish_solve(h); if (rc) return rc; }
    h->I.n_peer = n;
    for (int p = 0; p < n; p++) h->I.u0_peer[p] = peer_u0[p];
    return BMPC_OK;
}

int bmpc_bind_gather_flags(bmpc_handle* h, int64_t* my_flags, int64_t* const* peer_flags, int n_peers, int rank, int world, int64_t base_epoch) {
    if (!h || n_peers < 0 || n_peers > 8 || world < 1 || world > 9 || rank < 0 || rank >= world || (n_peers > 0 && (!my_flags || !peer_flags))) return BMPC_ERR_ARG;
    h->gflags = (long long*)my_flags; h->g_npeer = n_peers; h->g_rank = rank; h->g_world = world;
    h->g_epoch = h->g_done_epoch = base_epoch;
    for (int p = 0; p < n_peers; p++) h->gpeers.p[p] = (long long*)peer_flags[p];
    return BMPC_OK;
}

int bmpc_gather_arrive(bmpc_handle* h, int64_t epoch) {
    if (!h) return BMPC_ERR_ARG;
    if (!h->gflags) { h->err = "bmpc_gather_arrive before bmpc_bind_gather_flags"; return BMPC_ERR_STATE; }
    BMPC_CUDA(cudaSetDevice(h->cfg.device));
    if (h->pending) { int rc = finish_solve(h); if (rc) return rc; }
    (void)epoch;                                       // the library counts the epochs itself (one per solve on every rank)
    if (h->g_done_epoch == h->g_epoch) return BMPC_OK;  // the solver kernel's last warp already signalled and waited
    k_gather_arrive<<<1, 32, 0, h->stream>>>(h->gflags, h->gpeers, h->g_npeer, h->g_rank, h->g_world, h->g_epoch);
    h->g_done_epoch = h->g_epoch;
    BMPC_CUDA(cudaGetLastError());
    return BMPC_OK;
}

int bmpc_get_dims(const bmpc_handle* h, int32_t* dims) {
    if (!h || !dims) return BMPC_ERR_ARG;
    dims[0] = h->d.nx; dims[1] = h->d.nu; dims[2] = h->d.Np; dims[3] = h->d.Nc; dims[4] = h->d.NX; dims[5] = h->d.NU;
    dims[6] = h->d.mc; dims[7] = h->launch.team;
    return BMPC_OK;
}

// ---- helpers of bmpc_setup and bmpc_update_problem
// the 13 input arrays of bmpc_setup / bmpc_update_problem in argument order: block offset and doubles per system
struct BmpcInput { int off, cnt; };
static std::array<BmpcInput, 13> problem_inputs(const BmpcDims& d, const BmpcSysOff& o) {
    const int xx = d.nx * d.nx, uu = d.nu * d.nu;
    return {{{o.Ad, xx}, {o.Bd, d.nx * d.nu}, {o.Qx, xx}, {o.QxN, xx}, {o.Qu, uu}, {o.QDu, uu}, {o.xmin, d.nx}, {o.xmax, d.nx},
             {o.umin, d.nu}, {o.umax, d.nu}, {o.Dumin, d.nu}, {o.Dumax, d.nu}, {o.uref, d.nu}}};
}

// x'Qx > 0 for every x != 0: Cholesky factorisation of the symmetric part
static bool host_pd(const double* Q, int n) {
    std::vector<double> L((size_t)n * n);
    for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) L[i * n + j] = 0.5 * (Q[i * n + j] + Q[j * n + i]);
    for (int j = 0; j < n; j++) {
        double s = L[j * n + j];
        for (int k = 0; k < j; k++) s -= L[j * n + k] * L[j * n + k];
        if (!(s > 0.0)) return false;
        L[j * n + j] = sqrt(s);
        for (int i = j + 1; i < n; i++) {
            double t = L[i * n + j];
            for (int k = 0; k < j; k++) t -= L[i * n + k] * L[j * n + k];
            L[i * n + j] = t / L[j * n + j];
        }
    }
    return true;
}
// x'Qx >= 0 for every x: a diagonal with non-negative entries, or positive definite (a singular non-diagonal Q counts as "no")
static bool host_psd(const double* Q, int n) {
    bool diag = true, nonneg = true;
    for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) {
        if (i != j && Q[i * n + j] != 0.0) diag = false;
        if (i == j && !(Q[i * n + j] >= 0.0)) nonneg = false;
    }
    return diag ? nonneg : host_pd(Q, n);
}
// H = B'P_X B + P_U is positive definite for ANY (Ad, Bd) when P_X >= 0 and P_U > 0 (Qx, QxN, Qu, QDu >= 0 and Qu or QDu > 0: the
// difference matrix T is positive definite).  Per-instance systems whose weights all do so may defer the condense (sys_lazy).
// w: the weights Qx, QxN, Qu, QDu of n systems, each system's contiguous as in its block, system i's at w + i * stride
static bool weights_keep_h_definite(const BmpcDims& d, const double* w, int n, size_t stride) {
    for (int i = 0; i < n; i++, w += stride) {
        const double *Qx = w, *QxN = Qx + d.nx * d.nx, *Qu = QxN + d.nx * d.nx, *QDu = Qu + d.nu * d.nu;
        if (!(host_psd(Qx, d.nx) && host_psd(QxN, d.nx) && host_psd(Qu, d.nu) && host_psd(QDu, d.nu) && (host_pd(Qu, d.nu) || host_pd(QDu, d.nu))))
            return false;
    }
    return true;
}

// condensed Hessians of all n_sys systems positive definite; otherwise bmpc_solve refuses until the next successful
// bmpc_update_problem / bmpc_setup.  who: the entry point named in the message
static int check_condensed(bmpc_handle* h, const char* who) {
    const int ns = h->cfg.n_sys; const BmpcSysOff& o = h->o;
    std::vector<double> errs(ns);
    BMPC_CUDA(cudaMemcpy2DAsync(errs.data(), sizeof(double), h->sys + o.scal + BMPC_S_ERR, sizeof(double) * o.total, sizeof(double), ns,
                                cudaMemcpyDeviceToHost, h->stream));
    BMPC_CUDA(cudaStreamSynchronize(h->stream));
    for (int si = 0; si < ns; si++) if (errs[si] != 0.0) {
        h->sys_bad = true;
        h->err = std::string(who) + ": condensed Hessian is not positive definite (the weights or (Ad, Bd) make the QP non-strictly convex in U)";
        return BMPC_ERR_NOT_PD;
    }
    return BMPC_OK;
}

// the (Ad, Bd) sparsity pattern of n systems (system i's Ad at Ad[i * stride], Bd at Bd[i * stride]), as the union over them: bit
// q nx + b of *am: Ad[q][b] non-zero in some system, bit a nu + j of *bm: Bd[a][j].  Shapes beyond the masks: all bits
static void tpm_pattern(const BmpcDims& d, const double* Ad, const double* Bd, int n, size_t stride, unsigned long long* am, unsigned* bm) {
    *am = 0ull; *bm = 0u;
    if (d.nx * d.nx > 64 || d.nx * d.nu > 32) { *am = ~0ull; *bm = ~0u; return; }
    for (int s = 0; s < n; s++) {
        if (Ad) for (int i = 0; i < d.nx * d.nx; i++) if (Ad[s * stride + i] != 0.0) *am |= 1ull << i;
        if (Bd) for (int i = 0; i < d.nx * d.nu; i++) if (Bd[s * stride + i] != 0.0) *bm |= 1u << i;
    }
}
// gain rows and working-set records of multi-input entry e.  fresh: the stored records start empty (the next warm solve reads its
// working sets off v*)
static int tpm_alloc(bmpc_handle* h, const BmpcFastEntry& e, bool fresh) {
    const size_t B = h->cfg.batch, nwarp = (B + 31) / 32;
    if (h->tpm_W && h->tpm_W_slots < e.slots) { cudaFree(h->tpm_W); h->tpm_W = nullptr; }
    if (!h->tpm_W) { BMPC_CUDA(cudaMalloc((void**)&h->tpm_W, sizeof(double) * nwarp * 32 * (size_t)e.slots)); h->tpm_W_slots = e.slots; }
    if (!h->tpm_rec) { BMPC_CUDA(cudaMalloc((void**)&h->tpm_rec, sizeof(unsigned long long) * B * (size_t)(h->d.Np + 2))); fresh = true; }
    if (fresh) BMPC_CUDA(cudaMemsetAsync(h->tpm_rec, 0, sizeof(unsigned long long) * B * (size_t)(h->d.Np + 2), h->stream));
    return BMPC_OK;
}

static int policy_family(const bmpc_handle* h) {
    if (!h->fast) return BMPC_FAM_TEAM;
    return h->fast->family == BMPC_FAM_TPI && h->view.p ? BMPC_FAM_TPI_VIEW : h->fast->family;
}

// the options let entry e take the handle's system, whatever its pattern: the handle's shape, fast_path, soft state rows (the Riccati
// polishes treat state rows as the soft penalty they are by default), and one-warp teams (single-input) or polish on (multi-input)
static bool fast_allowed(const bmpc_handle* h, const BmpcFastEntry& e) {
    const bmpc_config& c = h->cfg;
    return same_shape(e, h->d) && c.fast_path && c.soft_on && (e.family == BMPC_FAM_TPI ? h->launch.team == 32 : c.polish != 0);
}

// The fast-path entry of the handle (h->fast, nullptr: the team kernels), its parameters and the kernel family: the first entry of
// the table the options allow (fast_allowed) and that takes the system.  A single-input entry takes any system; a multi-input entry
// one whose (Ad, Bd) pattern its masks contain and whose QDu is diagonal.  Shared system: pattern and diagonality of system 0's block,
// read back only when the options allow some entry (the fill reports QDu).  Per-instance systems: the union the handle keeps over the
// instances (tpm_am, tpm_bm, tpm_nondiag); a multi-input entry reads only the view, and the block comes back only for a single-input
// entry's constant-bank fill.  The multi-input records restart empty when the entry changes or the caller asks for fresh ones.
static int select_fast(bmpc_handle* h, bool fresh) {
    const bool shared = h->cfg.n_sys <= 1;
    std::vector<double> hs;
    for (const BmpcFastEntry& e : g_fast)
        if (fast_allowed(h, e) && (shared || e.family == BMPC_FAM_TPI)) {
            hs.resize(h->o.total);
            BMPC_CUDA(cudaMemcpyAsync(hs.data(), h->sys, sizeof(double) * h->o.total, cudaMemcpyDeviceToHost, h->stream));
            BMPC_CUDA(cudaStreamSynchronize(h->stream));
            break;
        }
    unsigned long long am = h->tpm_am; unsigned bm = h->tpm_bm;
    if (shared && !hs.empty()) tpm_pattern(h->d, hs.data() + h->o.Ad, hs.data() + h->o.Bd, 1, 0, &am, &bm);
    if (!h->fast_par) {                                   // one host copy for whichever entry the handle takes: the largest
        size_t bytes = 0;
        for (const BmpcFastEntry& e : g_fast) bytes = e.par_bytes > bytes ? e.par_bytes : bytes;
        h->fast_par = calloc(1, bytes);
    }
    const BmpcFastEntry* old = h->fast;
    h->fast = nullptr;
    for (const BmpcFastEntry& e : g_fast) {
        if (!fast_allowed(h, e)) continue;
        if (e.family == BMPC_FAM_TPM && (h->tpm_nondiag || (am & ~e.amask) || (bm & ~e.bmask))) continue;
        if (!hs.empty() && !e.fill(hs.data(), h->o, h->fast_par)) continue;
        h->fast = &e;
        break;
    }
    if (h->fast && h->fast->family == BMPC_FAM_TPM) { int rc = tpm_alloc(h, *h->fast, fresh || h->fast != old); if (rc) return rc; }
    h->policy.family = policy_family(h);
    return BMPC_OK;
}

// per-instance systems after bmpc_update_system: bring the condensed blocks of the listed instances (nullptr: 0..count-1) up to date
// before a launch that reads them; instances already fresh cost one CTA that leaves at once.  Returns 1 if it launched.
static int condense_stale(bmpc_handle* h, const int32_t* list, int count, int32_t* ncount) {
    if (!h->sys_stale || count <= 0) return 0;
    k_condense_list<<<count, 256, 0, h->stream>>>(h->d, h->o, h->sys, h->I.sys_stride, list, count, h->sys_gen, h->sys_gen_cur,
                                                  h->cfg.sigma, h->cfg.alpha, h->cfg.eps_feas, h->cfg.soft_on, ncount);
    if (list == nullptr && count >= h->cfg.batch) h->sys_stale = false;
    return 1;
}

int bmpc_setup(bmpc_handle* h, const double* Ad, const double* Bd, const double* Qx, const double* QxN, const double* Qu,
               const double* QDu, const double* xmin, const double* xmax, const double* umin, const double* umax,
               const double* Dumin, const double* Dumax, const double* uref) {
    if (!h) return BMPC_ERR_ARG;
    const double* src[13] = {Ad, Bd, Qx, QxN, Qu, QDu, xmin, xmax, umin, umax, Dumin, Dumax, uref};
    for (const double* s : src) if (!s) { h->err = "bmpc_setup: null pointer"; return BMPC_ERR_ARG; }
    BMPC_CUDA(cudaSetDevice(h->cfg.device));
    const BmpcDims& d = h->d; const BmpcSysOff& o = h->o;
    const int ns = h->cfg.n_sys;
    const auto P = problem_inputs(d, o);
    std::vector<double> in((size_t)o.pw * ns, 0.0);
    for (int si = 0; si < ns; si++)
        for (int f = 0; f < 13; f++) memcpy(in.data() + (size_t)si * o.pw + P[f].off, src[f] + (size_t)si * P[f].cnt, sizeof(double) * P[f].cnt);
    BMPC_CUDA(cudaMemcpy2DAsync(h->sys, sizeof(double) * o.total, in.data(), sizeof(double) * o.pw, sizeof(double) * o.pw, ns,
                                cudaMemcpyHostToDevice, h->stream));
    k_condense<<<ns, 256, 0, h->stream>>>(d, o, h->sys, h->cfg.rho, h->cfg.sigma, h->cfg.alpha, h->cfg.eps_feas, h->cfg.soft_on);
    BMPC_CUDA(cudaGetLastError());
    // everything derived from the new arrays comes before the check: a handle refused after a failed setup still describes what its
    // blocks hold, so a later update decides and refreshes from the same state as after a failed update
    // per-instance systems: one parameter block per instance, built on the device from each instance's block, in the layout of the
    // first entry the options allow (a single-input shape: its entry; a multi-input shape: its first entry).  It is kept current
    // whichever family runs (a later update may bring the handle onto a multi-input entry)
    const BmpcFastEntry* ve = nullptr;
    if (ns > 1) for (const BmpcFastEntry& e : g_fast) if (fast_allowed(h, e)) { ve = &e; break; }
    if (ve && ve->family == BMPC_FAM_TPM) {
        if (!h->tpm_word) BMPC_CUDA(cudaMalloc((void**)&h->tpm_word, 3 * sizeof(unsigned long long)));
        if (!h->tpm_hword) BMPC_CUDA(cudaMallocHost((void**)&h->tpm_hword, 3 * sizeof(unsigned long long)));
        tpm_pattern(d, in.data() + P[0].off, in.data() + P[1].off, ns, o.pw, &h->tpm_am, &h->tpm_bm);
        h->tpm_nondiag = false;
        for (int si = 0; si < ns; si++) {
            const double* q = in.data() + (size_t)si * o.pw + P[5].off;
            for (int i = 0; i < d.nu * d.nu; i++) if (i / d.nu != i % d.nu && q[i] != 0.0) h->tpm_nondiag = true;
        }
    }
    if (ve) {
        if (!h->view.p) BMPC_CUDA(cudaMalloc((void**)&h->view.p, sizeof(double) * (size_t)ve->view_fields * h->cfg.batch));
        h->view.e = ve;
        ve->fill_view(h);
        BMPC_CUDA(cudaGetLastError());
    }
    int rc = select_fast(h, true);
    if (rc) return rc;
    if (h->fast && h->fast->configure && h->fast->configure()) { h->err = "fast path: shared-memory configuration failed"; return BMPC_ERR_CUDA; }
    const bmpc_config& c = h->cfg;
    h->policy = bmpc_make_policy(h->policy.family, c.polish, c.first_iters, c.cold_iters, c.max_iter, c.pdas_steps, c.shift_warm);
    // time-varying problem data on per-instance systems: when the weights keep H positive definite for ANY (Ad, Bd),
    // bmpc_update_problem may defer the condense to the launches that need it
    h->sys_lazy = ns > 1 && weights_keep_h_definite(d, in.data() + P[2].off, ns, o.pw);     // Qx .. QDu (inputs 2..5) are contiguous
    if (ns > 1) {
        if (!h->sys_gen) BMPC_CUDA(cudaMalloc((void**)&h->sys_gen, sizeof(int32_t) * (size_t)ns));
        BMPC_CUDA(cudaMemsetAsync(h->sys_gen, 0, sizeof(int32_t) * (size_t)ns, h->stream));
    }
    h->sys_gen_cur = 0; h->sys_stale = false;
    rc = check_condensed(h, "bmpc_setup");
    if (rc) return rc;
    h->sys_bad = false;
    // uminus1 default = uref for every instance (mpc.py:141); caller overrides through bmpc_update
    h->is_setup = true; h->cold = true; h->solved = false; h->pending = false; h->codes_valid = false;
    return BMPC_OK;
}



int bmpc_update(bmpc_handle* h, const double* x0, const double* uminus1, const double* xref, int xref_rows, int on_device) {
    if (!h) return BMPC_ERR_ARG;
    if (!h->is_setup) { h->err = "bmpc_update before bmpc_setup"; return BMPC_ERR_STATE; }
    BMPC_CUDA(cudaSetDevice(h->cfg.device));
    if (h->pending) { int rc = finish_solve(h); if (rc) return rc; }
    const BmpcDims& d = h->d; size_t B = h->cfg.batch;
    cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    if (on_device == 2) {
        // borrowed device buffers: the solver kernels read them in place (no copy); the caller keeps them unchanged until the
        // results of the next solve have been retired (bmpc_output / bmpc_synchronize)
        if (x0) h->x0_cur = x0;
        if (uminus1) h->um1_cur = uminus1;
    } else {
        if (x0) { BMPC_CUDA(cudaMemcpyAsync(h->x0, x0, sizeof(double) * B * d.nx, kind, h->stream)); h->x0_cur = h->x0; }
        if (uminus1) { BMPC_CUDA(cudaMemcpyAsync(h->um1, uminus1, sizeof(double) * B * d.nu, kind, h->stream)); h->um1_cur = h->um1; }
    }
    h->I.x0 = h->x0_cur; h->I.um1 = h->um1_cur;
    if (xref) {
        if (xref_rows != 1 && xref_rows != d.Np + 1) { h->err = "xref_rows must be 1 or Np+1"; return BMPC_ERR_ARG; }
        h->xref_mode = xref_rows == 1 ? 0 : 1;
        BMPC_CUDA(cudaMemcpyAsync(h->xref, xref, sizeof(double) * B * (h->xref_mode ? d.NX : d.nx), kind, h->stream));
    }
    return BMPC_OK;
}

int bmpc_update_problem(bmpc_handle* h, const double* Ad, const double* Bd, const double* Qx, const double* QxN, const double* Qu,
                        const double* QDu, const double* xmin, const double* xmax, const double* umin, const double* umax,
                        const double* Dumin, const double* Dumax, const double* uref, int on_device) {
    if (!h) return BMPC_ERR_ARG;
    if (!h->is_setup) { h->err = "bmpc_update_problem before bmpc_setup"; return BMPC_ERR_STATE; }
    if (on_device != 0 && on_device != 1) { h->err = "bmpc_update_problem: on_device must be 0 (host) or 1 (device)"; return BMPC_ERR_ARG; }
    BMPC_CUDA(cudaSetDevice(h->cfg.device));
    if (h->pending) { int rc = finish_solve(h); if (rc) return rc; }
    const BmpcDims& d = h->d; const BmpcSysOff& o = h->o;
    const double* src[13] = {Ad, Bd, Qx, QxN, Qu, QDu, xmin, xmax, umin, umax, Dumin, Dumax, uref};
    const auto P = problem_inputs(d, o);
    bool any = false;
    for (const double* s : src) any = any || s;
    if (!any) return BMPC_OK;
    const bool model = Ad || Bd, weights = Qx || QxN || Qu || QDu;
    if (h->cfg.n_sys <= 1) {
        // shared system: eager.  New inputs into the block, K1 with the kept rho, the check of bmpc_setup, then everything that was
        // derived from the condensed block on the host
        const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
        for (int f = 0; f < 13; f++)
            if (src[f]) BMPC_CUDA(cudaMemcpyAsync(h->sys + P[f].off, src[f], sizeof(double) * P[f].cnt, kind, h->stream));
        k_condense_list<<<1, 256, 0, h->stream>>>(d, o, h->sys, 0, nullptr, 1, nullptr, 0, h->cfg.sigma, h->cfg.alpha, h->cfg.eps_feas,
                                                  h->cfg.soft_on, nullptr);
        BMPC_CUDA(cudaGetLastError());
        int rc = check_condensed(h, "bmpc_update_problem");
        if (rc) return rc;
        rc = select_fast(h, false);
        if (rc) return rc;
        h->sys_bad = false;
        return BMPC_OK;
    }
    // per-instance systems: the new arrays go into every block and into the fast path's parameter view; the condense is deferred
    // to the launches that read a condensed block (condense_stale) — unless H may lose definiteness, then all of it now + the check
    const int B = h->cfg.batch;
    const bool hv = h->view.p != nullptr;                // the handle's parameter view (either fast path)
    const bool tpm_view = hv && h->view.e->family == BMPC_FAM_TPM;
    if (!on_device && !h->sys_stage) BMPC_CUDA(cudaMalloc((void**)&h->sys_stage, sizeof(double) * (size_t)B * o.pw));
    BmpcRefreshTab T = {}; size_t per = 0;
    bool view_fill = false;                              // an array the view holds only through derived fields (fill_view)
    for (int f = 0; f < 13; f++) {
        if (!src[f]) continue;
        const double* s = src[f];
        if (!on_device) {
            BMPC_CUDA(cudaMemcpyAsync(h->sys_stage + (size_t)B * P[f].off, s, sizeof(double) * B * P[f].cnt, cudaMemcpyHostToDevice, h->stream));
            s = h->sys_stage + (size_t)B * P[f].off;
        }
        const int view = !hv ? -1 : f == 0 ? h->view.e->view_ad : f == 1 ? h->view.e->view_bd : -1;
        view_fill = view_fill || (hv && f >= 2);
        T.seg[T.n++] = BmpcRefreshSeg{s, P[f].off, P[f].cnt, view};
        per += (size_t)P[f].cnt;
    }
    const size_t n = (size_t)B * per;
    k_sys_refresh<<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>(h->sys, h->I.sys_stride, B, T, h->view.p);
    BMPC_CUDA(cudaGetLastError());
    if (view_fill) { h->view.e->fill_view(h); BMPC_CUDA(cudaGetLastError()); }
    h->sys_gen_cur++; h->sys_stale = true;
    // multi-input fast path on per-instance systems: the union pattern of the new (Ad, Bd) and "QDu not diagonal" decide the entry
    // below.  Host arrays: decided here.  Device (Ad, Bd) on a sparse entry: k_tpm_pattern + one synchronising read of the pattern
    // words; on the dense entry or the team kernels the pattern is taken as dense (nothing is read back).  Device QDu: the flag
    // k_fill_view raised, read in the synchronisation of the definiteness check below
    const bool qdu_dev = tpm_view && QDu && on_device;
    if (tpm_view && model) {
        if (!on_device) {
            unsigned long long am; unsigned bm;
            if (Ad) { tpm_pattern(d, Ad, nullptr, B, (size_t)P[0].cnt, &am, &bm); h->tpm_am = am; }
            if (Bd) { tpm_pattern(d, nullptr, Bd, B, (size_t)P[1].cnt, &am, &bm); h->tpm_bm = bm; }
        } else if (h->fast && (~h->fast->amask || ~h->fast->bmask)) {        // a sparse entry
            BMPC_CUDA(cudaMemsetAsync(h->tpm_word, 0, 2 * sizeof(unsigned long long), h->stream));
            if (Ad) k_tpm_pattern<<<(B + 127) / 128, 128, 0, h->stream>>>(Ad, P[0].cnt, B, h->tpm_word);
            if (Bd) k_tpm_pattern<<<(B + 127) / 128, 128, 0, h->stream>>>(Bd, P[1].cnt, B, h->tpm_word + 1);
            BMPC_CUDA(cudaGetLastError());
            BMPC_CUDA(cudaMemcpyAsync(h->tpm_hword, h->tpm_word, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
            BMPC_CUDA(cudaStreamSynchronize(h->stream));
            if (Ad) h->tpm_am = h->tpm_hword[0];
            if (Bd) h->tpm_bm = (unsigned)h->tpm_hword[1];
        } else {
            if (Ad) h->tpm_am = ~0ull;
            if (Bd) h->tpm_bm = ~0u;
        }
    }
    if (tpm_view && QDu && !on_device) {
        h->tpm_nondiag = false;
        for (int si = 0; si < B; si++)
            for (int i = 0; i < d.nu * d.nu; i++) if (i / d.nu != i % d.nu && QDu[(size_t)si * d.nu * d.nu + i] != 0.0) h->tpm_nondiag = true;
    }
    if (qdu_dev) BMPC_CUDA(cudaMemcpyAsync(h->tpm_hword + 2, h->tpm_word + 2, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
    // definiteness depends on the weights alone: new host weights decide the deferral again (every instance, with the arrays this
    // call kept: read back from the blocks); device weights are condensed and checked at once
    bool check = model && !h->sys_lazy;
    if (weights && on_device) { h->sys_lazy = false; check = true; }
    else if (weights) {
        const int w0 = P[2].off, nw = P[5].off + P[5].cnt - w0;     // Qx, QxN, Qu, QDu (inputs 2..5) are contiguous in the block
        std::vector<double> w((size_t)B * nw);
        BMPC_CUDA(cudaMemcpy2DAsync(w.data(), sizeof(double) * nw, h->sys + w0, sizeof(double) * h->I.sys_stride, sizeof(double) * nw, B,
                                    cudaMemcpyDeviceToHost, h->stream));
        BMPC_CUDA(cudaStreamSynchronize(h->stream));
        h->sys_lazy = weights_keep_h_definite(d, w.data(), B, nw);
        check = !h->sys_lazy;
    }
    if (check) {
        condense_stale(h, nullptr, B, nullptr);
        BMPC_CUDA(cudaGetLastError());
        int rc = check_condensed(h, "bmpc_update_problem");
        if (qdu_dev) h->tpm_nondiag = h->tpm_hword[2] != 0ull;        // (check_condensed synchronised the stream)
        if (rc) { if (tpm_view) select_fast(h, false); return rc; }   // refused; the entry still follows the arrays the blocks hold
    }
    if (tpm_view) { int rc = select_fast(h, false); if (rc) return rc; }
    // (bounds and uref alone leave definiteness as it was: a handle refused after a failed update stays refused)
    if (check || h->sys_lazy) h->sys_bad = false;
    return BMPC_OK;
}

int bmpc_update_system(bmpc_handle* h, const double* Ad, const double* Bd, int on_device) {
    return bmpc_update_problem(h, Ad, Bd, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, on_device);
}

static void launch_admm(bmpc_handle* h, const BmpcRoundLaunch& R, const int32_t* list, int count, int niter, int do_prep) {
    const int cold = h->cold ? 1 : 0, polish = h->cfg.polish ? 1 : 0;
    switch (R.admm) {
    case BMPC_TADMM_WARP: case BMPC_TADMM_LONE_WARP:
        k_admm<true><<<R.admm_grid, R.admm_threads, R.admm_smem, h->stream>>>(h->d, h->o, h->sys, h->I, list, count, niter, do_prep, cold, h->xref_mode, polish);
        break;
    case BMPC_TADMM_TILE:
        h->tile_fn[R.tile_T == 8 ? 0 : R.tile_T == 4 ? 1 : 2]<<<R.admm_grid, R.admm_threads, R.admm_smem, h->stream>>>(h->d, h->o, h->sys, h->I, list, count, niter, do_prep, cold, h->xref_mode, polish);
        break;
    case BMPC_TADMM_CTA:
        k_admm<false><<<R.admm_grid, R.admm_threads, R.admm_smem, h->stream>>>(h->d, h->o, h->sys, h->I, list, count, niter, do_prep, cold, h->xref_mode, polish);
        break;
    }
    h->stats.launches++;
}

static void launch_polish(bmpc_handle* h, const BmpcRoundLaunch& R, const int32_t* list, int count, int steps, int32_t* next_list, int32_t* next_count) {
    for (int k = 0; k < R.ntiers; k++) {
        const BmpcPolishTier& t = R.tier[k];
        const int32_t* tlist = k == 0 ? list : h->ovf;
        const int32_t* dev_count = k == 0 ? nullptr : next_count + 2;     // filled by the tier before
        int32_t* ovf = k + 1 < R.ntiers ? h->ovf : nullptr;
        if (t.warp) k_polish<true><<<t.grid, t.threads, t.smem, h->stream>>>(h->d, h->o, h->sys, h->I, tlist, count, t.rmax, steps, next_list, next_count, h->I.u0, dev_count, ovf, h->cfg.candidate_warm);
        else k_polish<false><<<t.grid, t.threads, t.smem, h->stream>>>(h->d, h->o, h->sys, h->I, tlist, count, t.rmax, steps, next_list, next_count, h->I.u0, dev_count, ovf, h->cfg.candidate_warm);
        h->stats.launches++;
    }
}

// ---- solve = rounds of [ADMM chunk -> polish]; the host only needs the count of unfinished instances after each
// round.  bmpc_solve enqueues the first round and returns; whoever needs results next (bmpc_output, ...) waits once,
// and only if stragglers remain runs further rounds.  In the warm closed loop this is ONE host sync per step.
static bool plan_round(const bmpc_handle* h, BmpcRoundPlan* p) {
    const auto& st = h->st;
    return bmpc_plan_round(h->policy, BmpcSolveState{st.round, st.total, st.cold, h->codes_valid}, p);
}

// launches the round plan p: a first round without team ADMM is one fast-path launch pair over the batch (thread-per-instance
// kernels, throughput-optimised); the team rounds run the CTA-per-instance kernels, latency-bound on the few stragglers
static int enqueue_round(bmpc_handle* h, const BmpcRoundPlan& p) {
    auto& st = h->st;
    st.chunk = p.chunk;
    const bool team = p.admm == BMPC_ADMM_TEAM;
    const bool tpi_first = !team && p.polish == BMPC_POL_TPI;     // k_tpi_pol over the batch: it zeroes the next round's counters itself
    // straggler rounds read u_-1 from the snapshot the first round took: bmpc_output may already have queued the commit of
    // this solve's u0 into um1 (speculating that the first round finishes everything)
    h->cpar ^= 1;                                        // counters of this round: the half the previous round left zeroed
    int32_t* cnt = h->counts + BMPC_CNT * h->cpar;
    h->I.um1 = st.round > 0 ? h->um1_solved : h->um1_cur;
    h->I.x0 = h->x0_cur; h->I.u0_shadow = h->um1_alt;
    if (!tpi_first) {
        if (team && p.reset) {
            const int B = h->cfg.batch;
            k_reset<<<(B + 255) / 256, 256, 0, h->stream>>>(h->I, B);
            h->stats.launches++;
            BMPC_CUDA(cudaMemcpyAsync(h->um1_solved, h->um1_cur, sizeof(double) * (size_t)B * h->d.nu, cudaMemcpyDefault, h->stream));   // (um1_cur may be mapped host memory)
        }
        BMPC_CUDA(cudaMemsetAsync(h->counts, 0, sizeof(int32_t) * 2 * BMPC_CNT, h->stream));     // this round's half and the next one's
        // every team launch below reads the condensed blocks of exactly this round's instances (per-instance systems after
        // bmpc_update_system: bring them up to date first).  The fast-path rounds without team ADMM (k_tpi_pol, k_tpm_pol alone)
        // read only the parameters or the view, so a warm step they finish condenses nothing
        if (team) h->stats.launches += condense_stale(h, st.list, st.count, cnt + BMPC_CNT_COND);
    }
    h->spin_epoch = 0;
    if (p.admm == BMPC_ADMM_NONE && p.polish == BMPC_POL_TPI) { h->epoch = (h->epoch % 1000000000) + 1; h->spin_epoch = h->epoch; ((volatile int32_t*)h->h_count)[BMPC_CNT_EPOCH] = 0; }
    // (a warm fast-path round times itself with the global timer and reports through mapped memory: no event records in the stream)
    if (!h->spin_epoch) BMPC_CUDA(cudaEventRecord(h->ev[0], h->stream));
    if (team) {
        const BmpcRoundLaunch R = bmpc_round_launch(h->launch, h->d, st.count, st.list != nullptr, h->sm_count);
        if (p.infeas) { k_snapshot<<<st.count, 128, 0, h->stream>>>(h->d, h->I, st.list, st.count, h->vprev, h->lprev); h->stats.launches++; }
        launch_admm(h, R, st.list, st.count, p.chunk, st.need_prep ? 1 : 0);
        st.need_prep = false;
        if (p.infeas) {
            k_infeas<<<st.count, 128, sizeof(double) * (h->d.mc + h->d.nu + 2), h->stream>>>(h->d, h->o, h->sys, h->I, st.list, st.count, h->vprev, h->lprev, 1e-4, h->I.u0, cnt);
            h->stats.launches++;
        }
        BMPC_CUDA(cudaEventRecord(h->ev[1], h->stream));
        if (p.polish == BMPC_POL_SCHUR) launch_polish(h, R, st.list, st.count, p.cap, st.nxt, cnt);
        else if (p.polish == BMPC_POL_CHECK) { k_check_converged<<<(st.count + 255) / 256, 256, 0, h->stream>>>(h->I, st.list, st.count, h->cfg.eps_abs, h->cfg.eps_rel, st.nxt, cnt); h->stats.launches++; }
    } else if (!tpi_first) {
        BMPC_CUDA(cudaEventRecord(h->ev[1], h->stream));      // (k_tpi_admm, when a first round has it, records ev[1] behind itself)
    }
    if (p.polish == BMPC_POL_TPI || p.polish == BMPC_POL_TPM) h->fast->launch(h, st.list, st.count, p, st.nxt);
    if (tpi_first) h->codes_valid = true;
    h->I.um1 = h->um1_cur;
    if (!h->spin_epoch) BMPC_CUDA(cudaEventRecord(h->ev[2], h->stream));
    if (!h->spin_epoch) BMPC_CUDA(cudaMemcpyAsync(h->h_count, cnt, sizeof(int32_t) * BMPC_CNT, cudaMemcpyDeviceToHost, h->stream));
    BMPC_CUDA(cudaGetLastError());
    return BMPC_OK;
}

// waits for the round in flight; returns 1 in *more if another round was enqueued (stragglers), 0 if the solve is complete
static int retire_round(bmpc_handle* h, int* more) {
    auto& st = h->st;
    float a = 0.f, p = 0.f;
    bool spun = false;
    if (h->spin_epoch && !h->sync_after_round) {
        // the kernel's last warp raises the epoch word in mapped host memory when every counter is final: a few microseconds
        // after the kernel ends, instead of a D2H copy + cudaStreamSynchronize (the round trip sits in every step of a control loop)
        volatile int32_t* flag = (volatile int32_t*)h->h_count + BMPC_CNT_EPOCH;
        for (long spins = 0; *flag != h->spin_epoch; spins++)
            if (spins > 200000000L) break;                              // ~ seconds: fall back to the stream
        spun = *flag == h->spin_epoch;
    }
    if (!spun) {
        BMPC_CUDA(cudaStreamSynchronize(h->stream));
        if (h->spin_epoch && ((volatile int32_t*)h->h_count)[BMPC_CNT_EPOCH] != h->spin_epoch) { h->err = "fast-path kernel did not report"; return BMPC_ERR_CUDA; }
        if (!h->spin_epoch) { cudaEventElapsedTime(&a, h->ev[0], h->ev[1]); cudaEventElapsedTime(&p, h->ev[1], h->ev[2]); }
    }
    {   // a fast-path polish launch timed itself (global timer): more faithful than events, which also see launch gaps
        unsigned long long t0n, t1; memcpy(&t0n, h->h_count + BMPC_CNT_T0, 8); memcpy(&t1, h->h_count + BMPC_CNT_T1, 8);
        if (t1 != 0ull && t0n != 0ull && t1 > ~t0n) p = (float)((double)(t1 - ~t0n) * 1e-6);
    }
    h->stats.ms_admm += a; h->stats.ms_polish += p;
    h->stats.admm_iters += (int64_t)st.count * st.chunk;
    st.total += st.chunk; st.round++;
    h->cold = false;
    st.count = h->h_count[0];
    h->stats.polish_steps += h->h_count[1];
    h->stats.infeasible += h->h_count[3];
    if (!h->spin_epoch) h->stats.recondensed += h->h_count[BMPC_CNT_COND];
    st.tight += h->h_count[BMPC_CNT_TIGHT];
    if (spun && h->h_count[BMPC_CNT_TIGHT + 1] == 1) h->g_done_epoch = h->g_epoch;
    st.list = st.nxt; int32_t* tmp = st.cur; st.cur = st.nxt; st.nxt = tmp;
    BmpcRoundPlan next;
    if (st.count > 0 && plan_round(h, &next)) { *more = 1; return enqueue_round(h, next); }
    *more = 0;
    const int B = h->cfg.batch;
    if (!h->cfg.polish) {
        // pure-ADMM mode: every instance gets its status from OSQP's criterion on its last residuals
        k_finalize<<<(B + 127) / 128, 128, 0, h->stream>>>(h->d, h->o, h->sys, h->I, nullptr, B, h->cfg.eps_abs, h->cfg.eps_rel, h->I.u0);
        h->stats.launches++;
    } else if (st.count > 0) {
        k_finalize<<<(st.count + 127) / 128, 128, 0, h->stream>>>(h->d, h->o, h->sys, h->I, st.list, st.count, h->cfg.eps_abs, h->cfg.eps_rel, h->I.u0);
        h->stats.launches++;
    }
    BMPC_CUDA(cudaGetLastError());
    h->stats.rounds = st.round; h->stats.unsolved = h->cfg.polish ? st.count + st.tight : -1;   // not KKT-verified: status 2 or -2
    h->pending = false;
    return BMPC_OK;
}

static int finish_solve(bmpc_handle* h) {
    while (h->pending) { int more = 0; int rc = retire_round(h, &more); if (rc) return rc; }
    return BMPC_OK;
}

int bmpc_solve(bmpc_handle* h) {
    if (!h) return BMPC_ERR_ARG;
    if (!h->is_setup) { h->err = "bmpc_solve before bmpc_setup"; return BMPC_ERR_STATE; }
    if (h->sys_bad) { h->err = "bmpc_solve after a failed bmpc_setup / bmpc_update_problem / bmpc_update_system (condensed Hessian not positive definite): update again or set up anew"; return BMPC_ERR_STATE; }
    BMPC_CUDA(cudaSetDevice(h->cfg.device));
    if (h->pending) { int rc = finish_solve(h); if (rc) return rc; }
    const int B = h->cfg.batch;
    memset(&h->stats, 0, sizeof(h->stats));
    auto& st = h->st;
    st.list = nullptr; st.count = B; st.cur = h->listA; st.nxt = h->listB;
    st.total = 0; st.round = 0; st.need_prep = true; st.tight = 0; st.cold = h->cold;
    if (h->gflags) h->g_epoch++;                     // every rank solves in lockstep: the arrival epoch of this step
    BmpcRoundPlan first;
    plan_round(h, &first);                           // (the first round is always planned)
    int rc = enqueue_round(h, first);
    if (rc) return rc;
    h->pending = true; h->solved = true; h->committed = false;
    return BMPC_OK;
}

int bmpc_output(bmpc_handle* h, double* u0, int32_t* status, int commit_uminus1, int on_device) {
    if (!h) return BMPC_ERR_ARG;
    if (!h->solved) { h->err = "bmpc_output before bmpc_solve"; return BMPC_ERR_STATE; }
    BMPC_CUDA(cudaSetDevice(h->cfg.device));
    const BmpcDims& d = h->d; size_t B = h->cfg.batch;
    cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    const bool want_u = u0 && u0 != h->I.u0;
    auto copy_u = [&]() -> int {
        if (want_u) BMPC_CUDA(cudaMemcpyAsync(u0, h->I.u0, sizeof(double) * B * d.nu, kind, h->stream));
        return BMPC_OK;
    };
    bool u_copied = false;
    if (h->pending) {
        // speculate that the round in flight finishes everything (the common case): queue the result copy behind it so that a
        // single wait covers the solve and the read-back; redone if stragglers needed more rounds (they rewrite u0)
        if (!on_device) { int rc = copy_u(); if (rc) return rc; u_copied = true; }
        h->sync_after_round = !on_device && want_u;
        int more = 0; int rc = retire_round(h, &more); h->sync_after_round = false; if (rc) return rc;
        if (more) { u_copied = false; rc = finish_solve(h); if (rc) return rc; }
        else if (h->stats.launches && (h->st.count > 0 || !h->cfg.polish)) u_copied = false;   // k_finalize rewrote u0/status
    }
    if (commit_uminus1 && !h->committed) {
        // every kernel that publishes u0 also wrote it into the shadow buffer: committing it as the next u_-1 (mpc.py:330) is a
        // pointer swap, no copy
        double* t = h->um1; h->um1 = h->um1_alt; h->um1_alt = t;
        h->um1_cur = h->um1; h->I.um1 = h->um1; h->I.u0_shadow = h->um1_alt;
        h->committed = true;
    }
    // every instance KKT-verified and none certified infeasible: the status array is all BMPC_SOLVED, no need to fetch it
    const bool all_solved = h->cfg.polish && h->stats.unsolved == 0 && h->stats.infeasible == 0;
    bool need_sync = false;
    if (!u_copied && want_u) { int rc = copy_u(); if (rc) return rc; need_sync = !on_device; }
    if (status) {
        if (all_solved && !on_device) {
            // (a closed loop asks with the same array every step: filled once while it stays all-solved)
            if (h->status_filled != status) { for (size_t i = 0; i < B; i++) status[i] = BMPC_SOLVED; h->status_filled = status; }
        }
        else { BMPC_CUDA(cudaMemcpyAsync(status, h->I.status, sizeof(int32_t) * B, kind, h->stream)); need_sync = !on_device; h->status_filled = nullptr; }
    }
    if (need_sync) BMPC_CUDA(cudaStreamSynchronize(h->stream));
    return BMPC_OK;
}

int bmpc_get_sequences(bmpc_handle* h, double* u_seq, double* x_seq, double* eps_seq, double* obj_val, int32_t* iters) {
    if (!h) return BMPC_ERR_ARG;
    if (!h->solved) { h->err = "bmpc_get_sequences before bmpc_solve"; return BMPC_ERR_STATE; }
    BMPC_CUDA(cudaSetDevice(h->cfg.device));
    if (h->pending) { int rc = finish_solve(h); if (rc) return rc; }
    const BmpcDims& d = h->d; size_t B = h->cfg.batch;
    if (x_seq || eps_seq || obj_val) {
        if (!h->seq_x) {
            BMPC_CUDA(cudaMalloc((void**)&h->seq_x, sizeof(double) * B * d.NX));
            BMPC_CUDA(cudaMalloc((void**)&h->seq_e, sizeof(double) * B * d.NX));
            BMPC_CUDA(cudaMalloc((void**)&h->seq_obj, sizeof(double) * B));
        }
        int wpb = 4;
        size_t sm = (size_t)wpb * (d.NU + d.NX + d.nu + 1) * sizeof(double);
        BMPC_CUDA(cudaFuncSetAttribute(k_sequences, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        condense_stale(h, nullptr, (int)B, nullptr);          // k_sequences reads every instance's condensed block
        k_sequences<<<(int)((B + wpb - 1) / wpb), wpb * 32, sm, h->stream>>>(d, h->o, h->sys, h->I, (int)B, h->xref_mode, h->seq_x, h->seq_e, h->seq_obj);
        BMPC_CUDA(cudaGetLastError());
        if (x_seq) BMPC_CUDA(cudaMemcpyAsync(x_seq, h->seq_x, sizeof(double) * B * d.NX, cudaMemcpyDeviceToHost, h->stream));
        if (eps_seq) BMPC_CUDA(cudaMemcpyAsync(eps_seq, h->seq_e, sizeof(double) * B * d.NX, cudaMemcpyDeviceToHost, h->stream));
        if (obj_val) BMPC_CUDA(cudaMemcpyAsync(obj_val, h->seq_obj, sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream));
    }
    if (u_seq) BMPC_CUDA(cudaMemcpyAsync(u_seq, h->I.Us, sizeof(double) * B * d.NU, cudaMemcpyDeviceToHost, h->stream));
    if (iters) BMPC_CUDA(cudaMemcpyAsync(iters, h->I.iters, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, h->stream));
    BMPC_CUDA(cudaStreamSynchronize(h->stream));
    return BMPC_OK;
}

int bmpc_get_stats(bmpc_handle* h, bmpc_stats* out) {
    if (!h || !out) return BMPC_ERR_ARG;
    if (h->pending) { cudaSetDevice(h->cfg.device); int rc = finish_solve(h); if (rc) return rc; }
    *out = h->stats;    // host-side counters only
    return BMPC_OK;
}

int bmpc_get_sys(bmpc_handle* h, const char* name, double* out, int capacity) {
    if (!h || !name || !out) return BMPC_ERR_ARG;
    if (!h->is_setup) { h->err = "bmpc_get_sys before bmpc_setup"; return BMPC_ERR_STATE; }
    BMPC_CUDA(cudaSetDevice(h->cfg.device));
    const BmpcDims& d = h->d; const BmpcSysOff& o = h->o;
    struct { const char* n; int off; int cnt; } tab[] = {
        {"Bcal", o.Bcal, d.NX * d.NU}, {"Acal", o.Acal, d.NX * d.nx}, {"H", o.H, d.NU * d.NU}, {"Hinv", o.Hinv, d.NU * d.NU},
        {"K", o.K, d.NU * d.NU}, {"Kinv", o.Kinv, d.NU * d.NU}, {"M", o.M, d.mc * d.mc}, {"AHinv", o.AHinv, d.mc * d.NU},
        {"Gx0", o.Gx0, d.NU * d.nx}, {"Gref", o.Gref, d.NU * d.nx}, {"g0", o.g0, d.NU}, {"lo0", o.lo0, d.mc},
        {"hi0", o.hi0, d.mc}, {"rho", o.rho, d.mc}, {"scal", o.scal, BMPC_S_COUNT}};
    for (auto& e : tab) if (strcmp(e.n, name) == 0) {
        if (capacity < e.cnt) { h->err = "bmpc_get_sys: buffer too small"; return BMPC_ERR_ARG; }
        condense_stale(h, nullptr, 1, nullptr);               // the exported block is system 0's
        BMPC_CUDA(cudaGetLastError());
        BMPC_CUDA(cudaMemcpyAsync(out, h->sys + e.off, sizeof(double) * e.cnt, cudaMemcpyDeviceToHost, h->stream));
        BMPC_CUDA(cudaStreamSynchronize(h->stream));
        return e.cnt;
    }
    h->err = std::string("bmpc_get_sys: unknown array ") + name;
    return BMPC_ERR_ARG;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// batched linear state estimator (kalman.py:109-134): one thread per instance, shared matrices in shared memory
__global__ void k_est(int nx, int nu, int ny, int B, const double* __restrict__ mats, double* __restrict__ x, double* __restrict__ y,
                      const double* __restrict__ in, int mode) {
    extern __shared__ double sm[];
    const int nm = nx * nx + nx * nu + ny * nx + nx * ny;
    for (int i = threadIdx.x; i < nm; i += blockDim.x) sm[i] = mats[i];
    __syncthreads();
    const double *A = sm, *Bm = A + nx * nx, *C = Bm + nx * nu, *L = C + ny * nx;
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    double* xb = x + (size_t)b * nx; double* yb = y + (size_t)b * ny;
    double xn[32];
    if (mode == 0) {            // predict: x <- A x + B u ; y <- C x
        const double* u = in + (size_t)b * nu;
        for (int i = 0; i < nx; i++) {
            double acc = 0.0;
            for (int j = 0; j < nx; j++) acc += A[i * nx + j] * xb[j];
            for (int j = 0; j < nu; j++) acc += Bm[i * nu + j] * u[j];
            xn[i] = acc;
        }
        for (int i = 0; i < nx; i++) xb[i] = xn[i];
        for (int i = 0; i < ny; i++) { double acc = 0.0; for (int j = 0; j < nx; j++) acc += C[i * nx + j] * xn[j]; yb[i] = acc; }
    } else {                    // update: x <- x + L (y_meas - y)      (y is NOT refreshed, as in the reference)
        const double* ym = in + (size_t)b * ny;
        for (int i = 0; i < nx; i++) {
            double acc = xb[i];
            for (int j = 0; j < ny; j++) acc += L[i * ny + j] * (ym[j] - yb[j]);
            xn[i] = acc;
        }
        for (int i = 0; i < nx; i++) xb[i] = xn[i];
    }
}

// the same estimator with one (A, B, C, L) per instance: matrices in global memory, FIELD-major (element e of instance b at
// mats[e * B + b]) so that the 32 threads of a warp read 32 consecutive doubles; same operation order as k_est
__global__ void k_est_pi(int nx, int nu, int ny, int B, const double* __restrict__ mats, double* __restrict__ x, double* __restrict__ y,
                         const double* __restrict__ in, int mode) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const double *A = mats + b, *Bm = A + (size_t)nx * nx * B, *C = Bm + (size_t)nx * nu * B, *L = C + (size_t)ny * nx * B;
    double* xb = x + (size_t)b * nx; double* yb = y + (size_t)b * ny;
    double xn[32];
    if (mode == 0) {            // predict: x <- A x + B u ; y <- C x
        const double* u = in + (size_t)b * nu;
        for (int i = 0; i < nx; i++) {
            double acc = 0.0;
            for (int j = 0; j < nx; j++) acc += A[(size_t)(i * nx + j) * B] * xb[j];
            for (int j = 0; j < nu; j++) acc += Bm[(size_t)(i * nu + j) * B] * u[j];
            xn[i] = acc;
        }
        for (int i = 0; i < nx; i++) xb[i] = xn[i];
        for (int i = 0; i < ny; i++) { double acc = 0.0; for (int j = 0; j < nx; j++) acc += C[(size_t)(i * nx + j) * B] * xn[j]; yb[i] = acc; }
    } else {                    // update: x <- x + L (y_meas - y)      (y is NOT refreshed, as in the reference)
        const double* ym = in + (size_t)b * ny;
        for (int i = 0; i < nx; i++) {
            double acc = xb[i];
            for (int j = 0; j < ny; j++) acc += L[(size_t)(i * ny + j) * B] * (ym[j] - yb[j]);
            xn[i] = acc;
        }
        for (int i = 0; i < nx; i++) xb[i] = xn[i];
    }
}

// batched DARE (csrc/bmpc_dare.cuh): one warp per instance, lane = row, the iterates in dynamic shared memory
__global__ void k_dare(int n, int m, int batch, const double* __restrict__ A, const double* __restrict__ B, const double* __restrict__ Q,
                       const double* __restrict__ R, const double* S, double* __restrict__ X, double* __restrict__ G,
                       int* __restrict__ status, int* __restrict__ steps) {
    extern __shared__ double sm[];
    const BmpcDareLayout l = bmpc_dare_layout(n, m);
    const int w = threadIdx.x >> 5;
    const int b = blockIdx.x * (blockDim.x >> 5) + w;
    if (b >= batch) return;                                  // whole warps leave: the team below always has 32 lanes
    WarpTeam t;
    const size_t nn = (size_t)n * n, nm = (size_t)n * m;
    int it = 0;
    const int st = bmpc_dare_solve(t, n, m, l, A + b * nn, B + b * nm, Q + b * nn, R + (size_t)b * m * m, S ? S + b * nm : nullptr,
                                   X + b * nn, G + b * nm, sm + (size_t)w * l.total, it);
    if (t.tid == 0) { status[b] = st; steps[b] = it; }
}

// batched Kalman filter (csrc/bmpc_kf.cuh): one thread per instance; P and the intermediates field-major in global memory.
// k_kf: one shared model, held in shared memory
__global__ void k_kf(int nx, int nu, int ny, int B, const double* __restrict__ mats, double* __restrict__ x, double* __restrict__ y,
                     double* __restrict__ P, double* __restrict__ ws, int* __restrict__ status, const double* __restrict__ in, int mode) {
    extern __shared__ double sm[];
    const BmpcKfLayout l = bmpc_kf_layout(nx, nu, ny);
    for (int i = threadIdx.x; i < l.model; i += blockDim.x) sm[i] = mats[i];
    __syncthreads();
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    bmpc_kf_step(BmpcKfModel<false>{sm, 1, nx, nu, ny, l}, b, B, mode, in, x, y, P, ws, status);
}

// k_kf_pi: one model per instance, field-major in global memory (element e of instance b at mats[e * B + b])
__global__ void k_kf_pi(int nx, int nu, int ny, int B, const double* __restrict__ mats, double* __restrict__ x, double* __restrict__ y,
                        double* __restrict__ P, double* __restrict__ ws, int* __restrict__ status, const double* __restrict__ in, int mode) {
    const BmpcKfLayout l = bmpc_kf_layout(nx, nu, ny);
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    bmpc_kf_step(BmpcKfModel<true>{mats + b, (size_t)B, nx, nu, ny, l}, b, B, mode, in, x, y, P, ws, status);
}

// bmpc_est_set_model of per-instance arrays: src [n, cnt] batch-major -> dst field-major (element k of instance s at dst[k * n + s])
__global__ void k_est_put(const double* __restrict__ src, int cnt, int n, double* __restrict__ dst) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)cnt * n) return;
    const size_t k = i / n, s = i % n;
    dst[i] = src[s * cnt + k];
}

struct bmpc_estimator {
    int nx, nu, ny, B, device, n_sys;
    int kf = 0;                        // 0: fixed gain L (k_est, k_est_pi); 1: Kalman filter (k_kf, k_kf_pi)
    double *mats = nullptr, *x = nullptr, *y = nullptr, *in = nullptr;
    double *P = nullptr, *ws = nullptr, *stage = nullptr;   // Kalman filter: packed P and workspace (field-major); set_model staging
    int* status = nullptr;
    cudaStream_t stream = nullptr, own = nullptr;
    bmpc_handle* mpc = nullptr;        // attached controller: same stream, and its deferred solve is retired before its u0 is read
};

extern "C" {

int bmpc_est_create(int32_t nx, int32_t nu, int32_t ny, int32_t batch, int32_t device, const double* A, const double* B,
                    const double* C, const double* L, const double* x0, bmpc_estimator** out) {
    return bmpc_est_create_ex(nx, nu, ny, batch, 1, device, A, B, C, L, x0, out);
}

// the model's fields in the order of e->mats: fixed gain (A, B, C, L); Kalman filter (A, B, C, Qn, Rn), bmpc_kf_layout's order
static int est_fields(const bmpc_estimator* e, size_t* cnt) {
    const size_t nx = e->nx, nu = e->nu, ny = e->ny;
    cnt[0] = nx * nx; cnt[1] = nx * nu; cnt[2] = ny * nx;
    if (!e->kf) { cnt[3] = nx * ny; return 4; }
    cnt[3] = nx * nx; cnt[4] = ny * ny; return 5;
}

// allocate and upload a new estimator's state: the model's fields (src, in est_fields' order), x0, y = C x0 and, for the Kalman
// filter, P0 and the status.  On failure the caller destroys e.
static int est_init(bmpc_estimator* e, const double* const* src, const double* x0, const double* P0) {
    const int nx = e->nx, ny = e->ny, batch = e->B, n_sys = e->n_sys;
    size_t cnt[5]; const int nf = est_fields(e, cnt);
    size_t nm = 0; for (int f = 0; f < nf; f++) nm += cnt[f];
    const int mx = e->nu > ny ? e->nu : ny;
    bool ok = cudaMalloc((void**)&e->mats, nm * n_sys * 8) == cudaSuccess && cudaMalloc((void**)&e->x, (size_t)batch * nx * 8) == cudaSuccess &&
              cudaMalloc((void**)&e->y, (size_t)batch * ny * 8) == cudaSuccess && cudaMalloc((void**)&e->in, (size_t)batch * mx * 8) == cudaSuccess &&
              cudaStreamCreateWithFlags(&e->own, cudaStreamNonBlocking) == cudaSuccess;
    const BmpcKfLayout l = bmpc_kf_layout(nx, e->nu, ny);
    if (ok && e->kf)
        ok = cudaMalloc((void**)&e->P, (size_t)l.P * batch * 8) == cudaSuccess && cudaMalloc((void**)&e->ws, (size_t)l.ws * batch * 8) == cudaSuccess &&
             cudaMalloc((void**)&e->status, (size_t)batch * 4) == cudaSuccess;
    if (!ok) { g_create_err = "bmpc_est_create: allocation failed"; return BMPC_ERR_CUDA; }
    e->stream = e->own;
    // packed fields of each system; with n_sys = batch transposed to field-major for k_est_pi / k_kf_pi
    std::vector<double> m(nm * n_sys);
    for (int s = 0; s < n_sys; s++) {
        size_t e0 = 0;
        for (int f = 0; f < nf; f++) {
            for (size_t k = 0; k < cnt[f]; k++) m[(e0 + k) * n_sys + s] = src[f][s * cnt[f] + k];
            e0 += cnt[f];
        }
    }
    cudaMemcpyAsync(e->mats, m.data(), m.size() * 8, cudaMemcpyHostToDevice, e->stream);
    cudaMemcpyAsync(e->x, x0, (size_t)batch * nx * 8, cudaMemcpyHostToDevice, e->stream);
    // y = C x0 (kalman.py:113): a predict with A = I, B = 0 would do; compute on the host instead (setup only)
    const double* C = src[2];
    std::vector<double> y0((size_t)batch * ny);
    for (int b = 0; b < batch; b++) {
        const double* Cb = C + (n_sys == 1 ? 0 : (size_t)b * ny * nx);
        for (int i = 0; i < ny; i++) { double acc = 0; for (int j = 0; j < nx; j++) acc += Cb[i * nx + j] * x0[(size_t)b * nx + j]; y0[(size_t)b * ny + i] = acc; }
    }
    cudaMemcpyAsync(e->y, y0.data(), y0.size() * 8, cudaMemcpyHostToDevice, e->stream);
    std::vector<double> Ph; std::vector<int> st;
    if (e->kf) {                       // upper triangle of P0, packed, field-major
        Ph.resize((size_t)l.P * batch); st.assign(batch, BMPC_KF_OK);
        for (int b = 0; b < batch; b++)
            for (int i = 0; i < nx; i++)
                for (int j = i; j < nx; j++) Ph[(size_t)bmpc_kf_pk(nx, i, j) * batch + b] = P0[((size_t)b * nx + i) * nx + j];
        cudaMemcpyAsync(e->P, Ph.data(), Ph.size() * 8, cudaMemcpyHostToDevice, e->stream);
        cudaMemcpyAsync(e->status, st.data(), st.size() * 4, cudaMemcpyHostToDevice, e->stream);
    }
    if (cudaStreamSynchronize(e->stream) != cudaSuccess) { g_create_err = "bmpc_est_create: upload failed"; return BMPC_ERR_CUDA; }
    return BMPC_OK;
}

int bmpc_est_create_ex(int32_t nx, int32_t nu, int32_t ny, int32_t batch, int32_t n_sys, int32_t device, const double* A, const double* B,
                       const double* C, const double* L, const double* x0, bmpc_estimator** out) {
    if (!out || !A || !B || !C || !L || !x0 || nx < 1 || nx > 32 || nu < 1 || ny < 1 || batch < 1) { g_create_err = "bmpc_est_create: bad argument (1 <= nx <= 32)"; return BMPC_ERR_ARG; }
    if (n_sys != 1 && n_sys != batch) { g_create_err = "bmpc_est_create: n_sys must be 1 (shared system) or batch (one system per instance)"; return BMPC_ERR_ARG; }
    *out = nullptr;
    if (bmpc_device_count() <= device) { g_create_err = "no CUDA device visible: libbmpc has no CPU fallback"; return BMPC_ERR_NO_DEVICE; }
    cudaSetDevice(device);
    bmpc_estimator* e = new bmpc_estimator();
    e->nx = nx; e->nu = nu; e->ny = ny; e->B = batch; e->device = device; e->n_sys = n_sys;
    const double* src[4] = {A, B, C, L};
    const int rc = est_init(e, src, x0, nullptr);
    if (rc) { bmpc_est_destroy(e); return rc; }
    *out = e;
    return BMPC_OK;
}

int bmpc_est_create_kf(int32_t nx, int32_t nu, int32_t ny, int32_t batch, int32_t n_sys, int32_t device, const double* A,
                       const double* B, const double* C, const double* Qn, const double* Rn, const double* x0, const double* P0,
                       bmpc_estimator** out) {
    if (!out || !A || !B || !C || !Qn || !Rn || !x0 || !P0 || nx < 1 || nx > BMPC_KF_MAX_DIM || nu < 1 || ny < 1 || ny > BMPC_KF_MAX_DIM || batch < 1) {
        g_create_err = "bmpc_est_create_kf: bad argument (1 <= nx, ny <= 32, nu >= 1)"; return BMPC_ERR_ARG;
    }
    if (n_sys != 1 && n_sys != batch) { g_create_err = "bmpc_est_create_kf: n_sys must be 1 (shared model) or batch (one model per instance)"; return BMPC_ERR_ARG; }
    *out = nullptr;
    if (device < 0 || bmpc_device_count() <= device) { g_create_err = "no CUDA device visible: libbmpc has no CPU fallback"; return BMPC_ERR_NO_DEVICE; }
    cudaSetDevice(device);
    const size_t smem = (size_t)bmpc_kf_layout(nx, nu, ny).model * 8;
    if (n_sys == 1 && smem > 48 * 1024) {              // the shared model of k_kf: large nu needs the opt-in shared memory
        int optin = 0;
        cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
        if (smem > (size_t)optin) { g_create_err = "bmpc_est_create_kf: the shared model exceeds the shared memory of one block (use n_sys = batch)"; return BMPC_ERR_ARG; }
        if (cudaFuncSetAttribute(k_kf, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
            g_create_err = "bmpc_est_create_kf: cannot raise the dynamic shared memory limit"; return BMPC_ERR_CUDA;
        }
    }
    bmpc_estimator* e = new bmpc_estimator();
    e->nx = nx; e->nu = nu; e->ny = ny; e->B = batch; e->device = device; e->n_sys = n_sys; e->kf = 1;
    const double* src[5] = {A, B, C, Qn, Rn};
    const int rc = est_init(e, src, x0, P0);
    if (rc) { bmpc_est_destroy(e); return rc; }
    *out = e;
    return BMPC_OK;
}

void bmpc_est_destroy(bmpc_estimator* e) {
    if (!e) return;
    cudaSetDevice(e->device);
    cudaFree(e->mats); cudaFree(e->x); cudaFree(e->y); cudaFree(e->in); cudaFree(e->P); cudaFree(e->ws); cudaFree(e->stage); cudaFree(e->status);
    if (e->own) cudaStreamDestroy(e->own);
    delete e;
}

static int est_run(bmpc_estimator* e, const double* in, int n, int on_device, int mode) {
    if (!e || !in) return BMPC_ERR_ARG;
    if (cudaSetDevice(e->device) != cudaSuccess) return BMPC_ERR_CUDA;
    if (e->mpc) {
        // on-device chain estimator <-> controller: one stream orders the kernels; a solve whose first round is still in flight may
        // need straggler rounds (host driven) before its u0 is final, so it is retired here
        if (on_device && e->mpc->pending) { int rc = finish_solve(e->mpc); if (rc) return rc; }
        e->stream = e->mpc->stream;
    }
    const double* src = in;
    if (!on_device) {
        if (cudaMemcpyAsync(e->in, in, (size_t)e->B * n * 8, cudaMemcpyHostToDevice, e->stream) != cudaSuccess) return BMPC_ERR_CUDA;
        src = e->in;
    }
    if (e->kf) {
        const BmpcKfLayout l = bmpc_kf_layout(e->nx, e->nu, e->ny);
        if (e->n_sys == 1)
            k_kf<<<(e->B + 127) / 128, 128, (size_t)l.model * 8, e->stream>>>(e->nx, e->nu, e->ny, e->B, e->mats, e->x, e->y, e->P, e->ws, e->status, src, mode);
        else
            k_kf_pi<<<(e->B + 127) / 128, 128, 0, e->stream>>>(e->nx, e->nu, e->ny, e->B, e->mats, e->x, e->y, e->P, e->ws, e->status, src, mode);
        return cudaGetLastError() == cudaSuccess ? BMPC_OK : BMPC_ERR_CUDA;
    }
    const size_t nm = (size_t)e->nx * e->nx + (size_t)e->nx * e->nu + (size_t)e->ny * e->nx + (size_t)e->nx * e->ny;
    if (e->n_sys == 1)
        k_est<<<(e->B + 127) / 128, 128, nm * 8, e->stream>>>(e->nx, e->nu, e->ny, e->B, e->mats, e->x, e->y, src, mode);
    else
        k_est_pi<<<(e->B + 127) / 128, 128, 0, e->stream>>>(e->nx, e->nu, e->ny, e->B, e->mats, e->x, e->y, src, mode);
    return cudaGetLastError() == cudaSuccess ? BMPC_OK : BMPC_ERR_CUDA;
}
int bmpc_est_predict(bmpc_estimator* e, const double* u, int on_device) { return est_run(e, u, e ? e->nu : 0, on_device, 0); }
int bmpc_est_update(bmpc_estimator* e, const double* y_meas, int on_device) { return est_run(e, y_meas, e ? e->ny : 0, on_device, 1); }
int bmpc_est_get(bmpc_estimator* e, double* x, double* y) {
    if (!e) return BMPC_ERR_ARG;
    cudaSetDevice(e->device);
    if (x) cudaMemcpyAsync(x, e->x, (size_t)e->B * e->nx * 8, cudaMemcpyDeviceToHost, e->stream);
    if (y) cudaMemcpyAsync(y, e->y, (size_t)e->B * e->ny * 8, cudaMemcpyDeviceToHost, e->stream);
    return cudaStreamSynchronize(e->stream) == cudaSuccess ? BMPC_OK : BMPC_ERR_CUDA;
}
double* bmpc_est_state_ptr(bmpc_estimator* e) { return e ? e->x : nullptr; }
int bmpc_est_set_stream(bmpc_estimator* e, void* s) { if (!e) return BMPC_ERR_ARG; e->stream = s ? (cudaStream_t)s : e->own; return BMPC_OK; }
int bmpc_est_attach(bmpc_estimator* e, bmpc_handle* h) {
    if (!e) return BMPC_ERR_ARG;
    if (h && h->cfg.device != e->device) return BMPC_ERR_ARG;
    cudaSetDevice(e->device); cudaStreamSynchronize(e->stream);
    e->mpc = h; e->stream = h ? h->stream : e->own;
    return BMPC_OK;
}

int bmpc_est_get_cov(bmpc_estimator* e, double* P, int32_t* status) {
    if (!e || !e->kf) return BMPC_ERR_ARG;
    cudaSetDevice(e->device);
    const int nx = e->nx, B = e->B;
    std::vector<double> Ph;
    if (P) { Ph.resize((size_t)bmpc_kf_layout(nx, e->nu, e->ny).P * B); cudaMemcpyAsync(Ph.data(), e->P, Ph.size() * 8, cudaMemcpyDeviceToHost, e->stream); }
    if (status) cudaMemcpyAsync(status, e->status, (size_t)B * 4, cudaMemcpyDeviceToHost, e->stream);
    if (cudaStreamSynchronize(e->stream) != cudaSuccess) return BMPC_ERR_CUDA;
    if (P)
        for (int b = 0; b < B; b++)
            for (int i = 0; i < nx; i++)
                for (int j = 0; j < nx; j++) P[((size_t)b * nx + i) * nx + j] = Ph[(size_t)bmpc_kf_pk(nx, i, j) * B + b];
    return BMPC_OK;
}

int bmpc_est_set_model(bmpc_estimator* e, const double* A, const double* B, const double* C, const double* L, const double* Qn,
                       const double* Rn, int on_device) {
    if (!e || (e->kf ? L != nullptr : (Qn != nullptr || Rn != nullptr))) return BMPC_ERR_ARG;
    if (cudaSetDevice(e->device) != cudaSuccess) return BMPC_ERR_CUDA;
    if (e->mpc) e->stream = e->mpc->stream;
    size_t cnt[5]; const int nf = est_fields(e, cnt);
    const double* kf_src[5] = {A, B, C, Qn, Rn};
    const double* est_src[4] = {A, B, C, L};
    const double* const* src = e->kf ? kf_src : est_src;
    size_t nm = 0; for (int f = 0; f < nf; f++) nm += cnt[f];
    const size_t n = e->n_sys;
    const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    size_t off = 0;
    for (int f = 0; f < nf; off += cnt[f], f++) {
        if (!src[f]) continue;
        if (n == 1) {                                     // packed: the array is the field
            if (cudaMemcpyAsync(e->mats + off, src[f], cnt[f] * 8, kind, e->stream) != cudaSuccess) return BMPC_ERR_CUDA;
            continue;
        }
        const double* d = src[f];
        if (!on_device) {                                 // host arrays go through a staging copy, one region per field
            if (!e->stage && cudaMalloc((void**)&e->stage, nm * n * 8) != cudaSuccess) return BMPC_ERR_CUDA;
            if (cudaMemcpyAsync(e->stage + off * n, src[f], cnt[f] * n * 8, kind, e->stream) != cudaSuccess) return BMPC_ERR_CUDA;
            d = e->stage + off * n;
        }
        const size_t tot = cnt[f] * n;
        k_est_put<<<(unsigned)((tot + 255) / 256), 256, 0, e->stream>>>(d, (int)cnt[f], (int)n, e->mats + off * n);
        if (cudaGetLastError() != cudaSuccess) return BMPC_ERR_CUDA;
    }
    return BMPC_OK;
}

int bmpc_dare(int32_t n, int32_t m, int32_t batch, int32_t device, const double* A, const double* B, const double* Q,
              const double* R, const double* S, double* X, double* G, int32_t* status, int32_t* iters) {
    if (!A || !B || !Q || !R || !X || !G || !status || !iters || n < 1 || n > BMPC_DARE_MAX_DIM || m < 1 || m > BMPC_DARE_MAX_DIM || batch < 1) {
        g_create_err = "bmpc_dare: bad argument (1 <= n, m <= 32, batch >= 1)"; return BMPC_ERR_ARG;
    }
    if (device < 0 || bmpc_device_count() <= device) { g_create_err = "no CUDA device visible: libbmpc has no CPU fallback"; return BMPC_ERR_NO_DEVICE; }
    if (cudaSetDevice(device) != cudaSuccess) { g_create_err = "bmpc_dare: cudaSetDevice failed"; return BMPC_ERR_CUDA; }
    const BmpcDareLayout l = bmpc_dare_layout(n, m);
    int optin = 0;
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    const size_t per_warp = (size_t)l.total * 8;
    int wpb = (int)((size_t)optin / per_warp);
    if (wpb > 8) wpb = 8;
    if (wpb > batch) wpb = batch;
    if (wpb < 1) { g_create_err = "bmpc_dare: workspace exceeds the shared memory of one block"; return BMPC_ERR_ARG; }
    const size_t smem = per_warp * wpb;
    if (smem > 48 * 1024 && cudaFuncSetAttribute(k_dare, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
        g_create_err = "bmpc_dare: cannot raise the dynamic shared memory limit"; return BMPC_ERR_CUDA;
    }
    const size_t b = (size_t)batch, nn = (size_t)n * n, nm = (size_t)n * m, mm = (size_t)m * m;
    const size_t nd = b * (3 * nn + 3 * nm + mm);                  // A, Q, X | B, S, G | R
    cudaStream_t s = nullptr;
    if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) { g_create_err = "bmpc_dare: stream creation failed"; return BMPC_ERR_CUDA; }
    double* d = nullptr;
    if (cudaMallocAsync((void**)&d, nd * 8 + b * 8, s) != cudaSuccess) {
        cudaStreamDestroy(s); g_create_err = "bmpc_dare: allocation failed"; return BMPC_ERR_CUDA;
    }
    double *dA = d, *dQ = dA + b * nn, *dX = dQ + b * nn, *dB = dX + b * nn, *dS = dB + b * nm, *dG = dS + b * nm, *dR = dG + b * nm;
    int* dst = (int*)(dR + b * mm); int* dit = dst + b;
    bool ok = cudaMemcpyAsync(dA, A, b * nn * 8, cudaMemcpyHostToDevice, s) == cudaSuccess &&
              cudaMemcpyAsync(dQ, Q, b * nn * 8, cudaMemcpyHostToDevice, s) == cudaSuccess &&
              cudaMemcpyAsync(dB, B, b * nm * 8, cudaMemcpyHostToDevice, s) == cudaSuccess &&
              cudaMemcpyAsync(dR, R, b * mm * 8, cudaMemcpyHostToDevice, s) == cudaSuccess &&
              (!S || cudaMemcpyAsync(dS, S, b * nm * 8, cudaMemcpyHostToDevice, s) == cudaSuccess);
    if (ok) {
        k_dare<<<(batch + wpb - 1) / wpb, 32 * wpb, smem, s>>>(n, m, batch, dA, dB, dQ, dR, S ? dS : nullptr, dX, dG, dst, dit);
        ok = cudaGetLastError() == cudaSuccess &&
             cudaMemcpyAsync(X, dX, b * nn * 8, cudaMemcpyDeviceToHost, s) == cudaSuccess &&
             cudaMemcpyAsync(G, dG, b * nm * 8, cudaMemcpyDeviceToHost, s) == cudaSuccess &&
             cudaMemcpyAsync(status, dst, b * 4, cudaMemcpyDeviceToHost, s) == cudaSuccess &&
             cudaMemcpyAsync(iters, dit, b * 4, cudaMemcpyDeviceToHost, s) == cudaSuccess;
    }
    cudaFreeAsync(d, s);
    ok = cudaStreamSynchronize(s) == cudaSuccess && ok;
    cudaStreamDestroy(s);
    if (!ok) { g_create_err = std::string("bmpc_dare: ") + cudaGetErrorString(cudaGetLastError()); return BMPC_ERR_CUDA; }
    return BMPC_OK;
}

}  // extern "C"
