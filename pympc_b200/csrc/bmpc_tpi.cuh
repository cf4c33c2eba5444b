// bmpc_tpi.cuh — thread-per-instance (TPI) fast path for SMALL MPC problems with compile-time shape
// (nx, nu, Np, Nc), e.g. the inverted pendulum (4,1,20,20) and the point mass (2,1,20,20).
//
// Why: the first (team-per-instance) kernels spent ~2700 warp-instructions per ADMM iteration on index
// arithmetic and dense mat-vecs through shared memory (profiles/ncu_r1_summary.txt: fp64 pipe 14 % busy).
// Here ONE THREAD owns one instance, so a warp advances 32 instances per instruction, nothing is exchanged
// between lanes, and the block-Toeplitz structure of the prediction matrix is used as what it is — the
// linear dynamics:   A x̃  = forward simulation  x_{k+1} = Ad x_k + Bd u_k          (Np*(nx^2+nx*nu) FMAs)
//                    A' w  = adjoint sweep       λ_k = w_k + Ad' λ_{k+1}, r_j = Bd' λ_{j+1}
// instead of two dense (Np*nx x Nc*nu) mat-vecs.  All shared matrices (Ad, Bd, K^-1, H^-1, G*) travel in the
// kernel-parameter constant bank (uniform operands, no load instructions); the iterate v lives in shared
// memory as v[row][lane] (conflict-free), x / r / x̃ in registers.  Every loop has compile-time bounds.
//
// Rows handled here: predicted states k = 1..Np (NS = Np*nx rows; the k = 0 block never touches U),
// inputs (NU), the reference's delta-u rows (ND).  The generic layout [B, mc] with mc = NS + nx + NU + ND is
// kept in global memory so the team kernels can take over any instance this path does not finish.
#pragma once
#include "bmpc_core.cuh"

// compiler-only fence between unrolled horizon stages: stops nvcc from hoisting every shared-memory load of an
// iteration to its top (which blew the register file: 1.1 KB of spills, uniform-register spills) while the hardware
// still overlaps neighbouring stages because issue does not wait for completion
#ifdef BMPC_HOSTEMU
#define BMPC_STAGE_FENCE() do {} while (0)
#else
#define BMPC_STAGE_FENCE() asm volatile("" ::: "memory")
#endif

template <int NXc, int NUc, int NPc, int NCc>
struct TpiShape {
    static constexpr int nx = NXc, nu = NUc, Np = NPc, Nc = NCc;
    static constexpr int NS = NPc * NXc;
    static constexpr int NU = NCc * NUc;
    static constexpr int ND = (NCc + 1) * NUc;
    static constexpr int MT = NS + NU + ND;
    static constexpr int NX = (NPc + 1) * NXc;
    static constexpr int mc = NX + NU + ND;
    // dense (Ad, Bd): see TpmSparseShape in bmpc_tpm.cuh for shapes with a compile-time sparsity pattern
    static constexpr unsigned long long amask = ~0ull; static constexpr unsigned bmask = ~0u;
    BMPC_HD static constexpr bool a_nz(int, int) { return true; }
    BMPC_HD static constexpr bool b_nz(int, int) { return true; }
};

template <class S>
struct TpiCommon {
    double Ad[S::nx * S::nx], Bd[S::nx * S::nu];
    double Gx0[S::NU * S::nx], Gref[S::NU * S::nx], g0[S::NU], QDu[S::nu * S::nu];
    double Qx[S::nx * S::nx], QxN[S::nx * S::nx];      // stage / terminal state weights (time-varying reference only)
    double xmin[S::nx], xmax[S::nx], c1x[S::nx], c2x[S::nx], rhox[S::nx];
    double umin[S::nu], umax[S::nu], rhou[S::nu];
    double dmin[S::nu], dmax[S::nu], rhod[S::nu];
    double irhox[S::nx], irhou[S::nu], irhod[S::nu];   // 1 / rho per row class
    double sigma, alpha, inv_rho_e;      // inv_rho_e = 0 -> hard state rows
};

template <class S>
struct TpiAdmmParams {
    TpiCommon<S> c;
    double Kinv[S::NU * S::NU];
    double Gcc[S::NU * S::nx];           // B' R_x Acal : folds the affine offset of the state rows into g
};

// per-thread strided accessor: element i of this thread's private column
struct TpiAcc {
    double* p; int stride;
    BMPC_HD double& operator()(int i) const { return p[i * stride]; }
    BMPC_HD double ld(int i) const { return p[i * stride]; }
    BMPC_HD void st(int i, double v) const { p[i * stride] = v; }
};
#ifndef BMPC_HOSTEMU
// the same column in GLOBAL memory, streamed: loads and stores marked evict-first so that the gain rows (written once, read once
// per refinement) do not push the kernel's local memory out of L1 / L2
struct TpiStreamAcc {
    double* p; int stride;
    __device__ __forceinline__ double ld(int i) const { return __ldcs(p + (size_t)i * stride); }
    __device__ __forceinline__ void st(int i, double v) const { __stcs(p + (size_t)i * stride, v); }
};
#endif

// plain selects (no IEEE fmin/fmax NaN handling: ~3 instructions instead of ~10 in fp64)
BMPC_HD double tpi_clamp(double v, double lo, double hi) { double t = v; t = (v > hi) ? hi : t; t = (v < lo) ? lo : t; return t; }

template <class S>
BMPC_HD double tpi_prox_x(const TpiCommon<S>& c, int a, double v) {
    // soft box: z = v + c2 (clamp(v) - v), c2 = eps_feas / (rho + eps_feas); hard box: c2 = 1.  Branch-free.
    const double t = tpi_clamp(v, c.xmin[a], c.xmax[a]);
    return fma(c.c2x[a], t - v, v);
}

template <class S>
BMPC_HD void tpi_dbounds(const TpiCommon<S>& c, const double* um1, int rr, double& lo, double& hi) {
    lo = c.dmin[rr % S::nu]; hi = c.dmax[rr % S::nu];
    if (rr < S::nu) { lo += um1[rr]; hi += um1[rr]; }
}

// Reference accessor: xr(k, b) = component b of the reference of stage k.  TV = false: one constant reference held in the
// caller's registers (p points at a local array, k is ignored); TV = true: this instance's (Np+1) x nx reference in global
// memory (mpc.py:414-421, SURVEY 8f-2).
template <class S, bool TV_>
struct TpiXref {
    static constexpr bool TV = TV_;
    const double* p;
    BMPC_HD double operator()(int k, int b) const { return TV_ ? p[k * S::nx + b] : p[b]; }
};

// true linear term g (NU) of the condensed QP for this instance
template <class S, class XR>
BMPC_HD void tpi_linear_term(const TpiCommon<S>& c, const double* x0, const double* um1, XR xr, double* g) {
    constexpr int nx = S::nx, nu = S::nu;
#pragma unroll
    for (int a = 0; a < S::NU; a++) {
        double acc = c.g0[a];
#pragma unroll
        for (int q = 0; q < nx; q++) acc += c.Gx0[a * nx + q] * x0[q];
        if (!XR::TV) {
#pragma unroll
            for (int q = 0; q < nx; q++) acc += c.Gref[a * nx + q] * xr(0, q);
        }
        if (a < nu) {
#pragma unroll
            for (int q = 0; q < nu; q++) acc -= c.QDu[a * nu + q] * um1[q];
        }
        g[a] = acc;
    }
}

// time-varying reference: the part -Bcal' P_X xref of g, by the adjoint recursion  lam_k = -Q_k xref_k + Ad' lam_{k+1},
// g_{min(k-1, Nc-1)} += Bd' lam_k;  add(j, value) accumulates into wherever the caller keeps g (dynamic index: not a register array)
template <class S, class XR, class ADD>
BMPC_HD void tpi_linear_term_tv(const TpiCommon<S>& c, XR xr, ADD add) {
    constexpr int nx = S::nx, nu = S::nu;
    double lam[nx];
#pragma unroll
    for (int a = 0; a < nx; a++) lam[a] = 0.0;
#pragma unroll 1
    for (int k = S::Np; k >= 1; k--) {
        double ln[nx];
#pragma unroll
        for (int a = 0; a < nx; a++) {
            double acc = 0.0;
#pragma unroll
            for (int q = 0; q < nx; q++) acc += c.Ad[q * nx + a] * lam[q] - (k == S::Np ? c.QxN[a * nx + q] : c.Qx[a * nx + q]) * xr(k, q);
            ln[a] = acc;
        }
#pragma unroll
        for (int a = 0; a < nx; a++) lam[a] = ln[a];
#pragma unroll
        for (int b = 0; b < nu; b++) {
            double acc = 0.0;
#pragma unroll
            for (int q = 0; q < nx; q++) acc += c.Bd[q * nu + b] * lam[q];
            add(((k - 1 < S::Nc - 1) ? (k - 1) : (S::Nc - 1)) * nu + b, acc);       // stages beyond Nc feed the held last input
        }
    }
}

// ------------------------------------------------------------------------------------------------
// niter ADMM iterations.  V: this thread's iterate v (MT rows).  x: NU registers (in/out).
// G: where g' (NU values, read once per iteration) is parked: rows [MT, MT+NU) of the column, or a per-instance scratch in
// global memory (frees shared memory: one more resident warp per SM)
template <class S, class XR>
BMPC_HD void tpi_admm(const TpiAdmmParams<S>& P, TpiAcc V, TpiAcc G, const double* x0, const double* um1, XR xr,
                      double* x, int niter, bool cold) {
    constexpr int nx = S::nx, nu = S::nu, Np = S::Np, Nc = S::Nc, NS = S::NS, NU = S::NU;
    const TpiCommon<S>& c = P.c;
    // g' = g + B' R_x Acal x0 is parked in G (read once per iteration)
    {
        double gp[NU];
        tpi_linear_term<S>(c, x0, um1, xr, gp);
#pragma unroll
        for (int a = 0; a < NU; a++) {
#pragma unroll
            for (int q = 0; q < nx; q++) gp[a] += P.Gcc[a * nx + q] * x0[q];
            G(a) = gp[a];
        }
        if constexpr (XR::TV) tpi_linear_term_tv<S>(c, xr, [&](int j, double val) { G(j) += val; });
    }
    if (cold) {
        // x = 0, v = A x + cc : free response on the state rows, zeros elsewhere
        double xk[nx];
#pragma unroll
        for (int q = 0; q < nx; q++) xk[q] = x0[q];
#pragma unroll
        for (int k = 1; k <= Np; k++) {
            double xn[nx];
#pragma unroll
            for (int a = 0; a < nx; a++) {
                double acc = 0.0;
#pragma unroll
                for (int q = 0; q < nx; q++) acc += c.Ad[a * nx + q] * xk[q];
                xn[a] = acc;
            }
#pragma unroll
            for (int a = 0; a < nx; a++) { xk[a] = xn[a]; V((k - 1) * nx + a) = xn[a]; }
        }
#pragma unroll
        for (int i = NS; i < S::MT; i++) V(i) = 0.0;
#pragma unroll
        for (int a = 0; a < NU; a++) x[a] = 0.0;
    }
    // One ADMM iteration = two fused sweeps over the horizon (everything unrolled, all register indices static):
    //  backward: lam_k = w_k + Ad' lam_{k+1}; as soon as stage j = k-1 knows lam_{j+1} its r_s is final and is scattered
    //            at once into the NU independent accumulators xt += Kinv[:, s] r_s  (ILP beside the serial lam chain)
    //  forward : x_{k+1} = Ad x_k + Bd xt_k with the row updates v += alpha (zt - prox(v)) riding along
    auto wrow_d = [&](int rr) {                       // w = rho (2 clamp(v) - v) of delta-u row rr
        double lo, hi; tpi_dbounds<S>(c, um1, rr, lo, hi);
        const double v = V(NS + NU + rr);
        return c.rhod[rr % nu] * (2.0 * tpi_clamp(v, lo, hi) - v);
    };
#pragma unroll 1
    for (int it = 0; it < niter; it++) {
        double xt[NU], lam[nx], hold[nu];
#pragma unroll
        for (int a = 0; a < NU; a++) xt[a] = 0.0;
#pragma unroll
        for (int q = 0; q < nx; q++) lam[q] = 0.0;
#pragma unroll
        for (int b = 0; b < nu; b++) hold[b] = 0.0;
        double e_cur = wrow_d(nu + NU - 1);           // row nu+s holds -U[s] + U[s+1]; visited by descending s
#pragma unroll
        for (int k = Np; k >= 1; k--) {
            double ln[nx];
#pragma unroll
            for (int a = 0; a < nx; a++) {
                const double v = V((k - 1) * nx + a);
                double acc = c.rhox[a] * (2.0 * tpi_prox_x<S>(c, a, v) - v);
#pragma unroll
                for (int q = 0; q < nx; q++) acc += c.Ad[q * nx + a] * lam[q];
                ln[a] = acc;
            }
#pragma unroll
            for (int a = 0; a < nx; a++) lam[a] = ln[a];
            if (k - 1 > Nc - 1) {                     // held input (Nc < Np): collect Bd' lam_k
#pragma unroll
                for (int b = 0; b < nu; b++) {
#pragma unroll
                    for (int q = 0; q < nx; q++) hold[b] += c.Bd[q * nu + b] * lam[q];
                }
            } else {
                const int j = k - 1;
#pragma unroll
                for (int b = nu - 1; b >= 0; b--) {
                    const int s2 = j * nu + b;
                    double r = c.sigma * x[s2] - G(s2) + ((j == Nc - 1) ? hold[b] : 0.0);
#pragma unroll
                    for (int q = 0; q < nx; q++) r += c.Bd[q * nu + b] * lam[q];
                    const double vu = V(NS + s2);
                    r += c.rhou[b] * (2.0 * tpi_clamp(vu, c.umin[b], c.umax[b]) - vu);
                    const double e_prev = (s2 >= 1) ? wrow_d(nu + s2 - 1) : 0.0;
                    r += e_prev - e_cur;
                    if (s2 < nu) r += wrow_d(s2);
                    e_cur = e_prev;
#pragma unroll
                    for (int a = 0; a < NU; a++) xt[a] += P.Kinv[a * NU + s2] * r;
                }
            }
            BMPC_STAGE_FENCE();
        }
        double xk[nx];
#pragma unroll
        for (int q = 0; q < nx; q++) xk[q] = x0[q];
#pragma unroll
        for (int k = 1; k <= Np; k++) {
            const int j = (k - 1 < Nc - 1) ? (k - 1) : (Nc - 1);
            double xn[nx];
#pragma unroll
            for (int a = 0; a < nx; a++) {
                double a0 = 0.0, a1 = 0.0;
#pragma unroll
                for (int b = 0; b < nu; b++) a0 += c.Bd[a * nu + b] * xt[j * nu + b];
#pragma unroll
                for (int q = 0; q < nx; q += 2) { a0 += c.Ad[a * nx + q] * xk[q]; if (q + 1 < nx) a1 += c.Ad[a * nx + q + 1] * xk[q + 1]; }
                xn[a] = a0 + a1;
            }
#pragma unroll
            for (int a = 0; a < nx; a++) {
                xk[a] = xn[a];
                const double v = V((k - 1) * nx + a);
                V((k - 1) * nx + a) = v + c.alpha * (xn[a] - tpi_prox_x<S>(c, a, v));
            }
            if (k - 1 <= Nc - 1) {
#pragma unroll
                for (int b = 0; b < nu; b++) {
                    const int s2 = (k - 1) * nu + b;
                    const double vu = V(NS + s2);
                    V(NS + s2) = vu + c.alpha * (xt[s2] - tpi_clamp(vu, c.umin[b], c.umax[b]));
                    {
                        double lo, hi; tpi_dbounds<S>(c, um1, nu + s2, lo, hi);
                        const double v = V(NS + NU + nu + s2);
                        const double zt = -xt[s2] + (s2 + 1 < NU ? xt[s2 + 1] : 0.0);
                        V(NS + NU + nu + s2) = v + c.alpha * (zt - tpi_clamp(v, lo, hi));
                    }
                    if (s2 < nu) {
                        double lo, hi; tpi_dbounds<S>(c, um1, s2, lo, hi);
                        const double v = V(NS + NU + s2);
                        V(NS + NU + s2) = v + c.alpha * (xt[s2] - tpi_clamp(v, lo, hi));
                    }
                    x[s2] += c.alpha * (xt[s2] - x[s2]);
                }
            }
            BMPC_STAGE_FENCE();
        }
    }
}

// Where the forward sweep stages row i of the exact ADMM fixed point v* inside the (already consumed) gain slots of the
// column: stage k owns slots [k*(nx+2), (k+1)*(nx+2)) = its nx state rows, its input row, its delta-u row; the reference's
// spurious last delta-u row goes to the spare slot behind the last stage.
template <class S>
BMPC_HD int tpi_vstar_slot(int i) {
    constexpr int nz1 = S::nx + 2;
    if (i < S::NS) return (i / S::nx) * nz1 + (i % S::nx);
    if (i < S::NS + S::NU) return (i - S::NS) * nz1 + S::nx;
    const int rr = i - S::NS - S::NU;
    return rr < S::Nc ? rr * nz1 + S::nx + 1 : S::Np * nz1;
}

// ------------------------------------------------------------------------------------------------
// host side: fill the parameter blocks from a host copy of the condensed system block
template <class S>
inline void tpi_fill_common(const double* sys, const BmpcSysOff& o, TpiCommon<S>& c) {
    constexpr int nx = S::nx, nu = S::nu, NU = S::NU, NX = S::NX;
    for (int i = 0; i < nx * nx; i++) c.Ad[i] = sys[o.Ad + i];
    for (int i = 0; i < nx * nu; i++) c.Bd[i] = sys[o.Bd + i];
    for (int i = 0; i < NU * nx; i++) { c.Gx0[i] = sys[o.Gx0 + i]; c.Gref[i] = sys[o.Gref + i]; }
    for (int i = 0; i < NU; i++) c.g0[i] = sys[o.g0 + i];
    for (int i = 0; i < nu * nu; i++) c.QDu[i] = sys[o.QDu + i];
    for (int i = 0; i < nx * nx; i++) { c.Qx[i] = sys[o.Qx + i]; c.QxN[i] = sys[o.QxN + i]; }
    const double rho_e = sys[o.scal + BMPC_S_RHOE];
    c.inv_rho_e = rho_e > 0.0 ? 1.0 / rho_e : 0.0;
    c.sigma = sys[o.scal + BMPC_S_SIGMA]; c.alpha = sys[o.scal + BMPC_S_ALPHA];
    for (int a = 0; a < nx; a++) {
        c.xmin[a] = sys[o.lo0 + nx + a]; c.xmax[a] = sys[o.hi0 + nx + a];
        const double rho = sys[o.rho + nx + a]; c.rhox[a] = rho; c.irhox[a] = 1.0 / rho;
        if (rho_e > 0.0) { c.c1x[a] = rho / (rho + rho_e); c.c2x[a] = rho_e / (rho + rho_e); }
        else { c.c1x[a] = 0.0; c.c2x[a] = 1.0; }
    }
    for (int b = 0; b < nu; b++) {
        c.umin[b] = sys[o.lo0 + NX + b]; c.umax[b] = sys[o.hi0 + NX + b]; c.rhou[b] = sys[o.rho + NX + b]; c.irhou[b] = 1.0 / c.rhou[b];
        c.dmin[b] = sys[o.lo0 + NX + NU + b]; c.dmax[b] = sys[o.hi0 + NX + NU + b]; c.rhod[b] = sys[o.rho + NX + NU + b]; c.irhod[b] = 1.0 / c.rhod[b];
    }
}
template <class S>
inline void tpi_fill_admm(const double* sys, const BmpcSysOff& o, TpiAdmmParams<S>& P) {
    constexpr int nx = S::nx, NU = S::NU, NX = S::NX;
    tpi_fill_common<S>(sys, o, P.c);
    for (int i = 0; i < NU * NU; i++) P.Kinv[i] = sys[o.Kinv + i];
    for (int a = 0; a < NU; a++)
        for (int q = 0; q < nx; q++) {
            double acc = 0.0;
            for (int i = 0; i < NX; i++) acc += sys[o.Bcal + i * NU + a] * sys[o.rho + i] * sys[o.Acal + i * nx + q];
            P.Gcc[a * nx + q] = acc;
        }
}

// ================================================================================================
// Riccati polish (nu == 1; Nc < Np: the stages k >= Nc hold the last input, i.e. are pinned to u_k = u_{k-1} without a row
// or a multiplier).  ONE active-set refinement = tpi2_backward + tpi2_forward: the equality-constrained QP of the step is the
// LQ problem
//   min sum_k [ 1/2 x_k' Qt_k x_k - qt_k' x_k ] + sum_j [ 1/2 Qu u_j^2 - Qu uref u_j + 1/2 QDu (u_j - u_{j-1})^2 ]
//   s.t. x_{k+1} = Ad x_k + Bd u_k,  some inputs pinned (u_j = bound, or u_j = u_{j-1} + delta)
// where violated soft rows enter through Qt_k = Q_k + eps_feas diag(mask_k), qt_k = Q_k xref + eps_feas mask_k.*bound.
// It is solved exactly by one backward sweep on the augmented state xi = [x ; u_prev] (cost-to-go 1/2 xi'P xi + p'xi)
// and one forward sweep; multipliers of pinned inputs are -dQ/du of the stage Q-function.  Work and storage are O(Np) and
// independent of the size of the working set (the Schur form of the team kernels needs an r x r factor per instance).
// Workspace: nx + 2 gain slots per stage: free stage -> feedback (k[nx+1], kappa); pinned -> (m[nx+1], m0), dQ/du = m'xi + m0.
//
// Second generation.  What changed against the round-1 sweeps (profiles/ncu_r1_final_summary.txt: 23 % fp64 pipe, the
// forward sweep spent 4 instructions on set bookkeeping per fp64 instruction):
//  * the working sets live as ONE small code word per stage (state rows up / down, input row, delta-u row, the spurious last
//    row) in shared memory next to the gains, and between solves as 2 (nx <= 5) or 4 bytes per stage in global memory: a warm solve reads
//    40 bytes of sets instead of the 968-byte iterate v, shifted by one stage (receding horizon: the plan of step t+1 is the
//    tail of the plan of step t);
//  * both sweeps are branch-free: the pin type of a stage (free / input bound / delta-u bound / spurious row) only selects
//    coefficients, so lanes with different working sets never diverge;
//  * the cost-to-go matrix is kept symmetric (upper triangle), verification thresholds are precomputed constants, the
//    reciprocal of huu is MUFU + two Newton steps (no slow-path branch), the constant-reference term Q xref is hoisted.
// Row / slot conventions are those of the first generation (tpi_vstar_slot): stage k owns gain slots [k (nx+2), (k+1)(nx+2)).
#include <stdint.h>
#include <stddef.h>
#include <type_traits>

template <class S>
struct TpiCode {
    static constexpr unsigned XUP = 0, XDN = S::nx, UUP = 2 * S::nx, UDN = UUP + 1, DUP = UUP + 2, DDN = UUP + 3, QUP = UUP + 4, QDN = UUP + 5;
    static constexpr unsigned BITS = 2 * S::nx + 6;
    using type = typename std::conditional<(BITS <= 16), uint16_t, uint32_t>::type;
    // one 32-bit word holds the sets of nx <= 13 (pympc_b200.build.tpi_shape_supported); wider states run on the team kernels
    static_assert(BITS <= 8 * sizeof(type), "working-set code word wider than 32 bits: the fast path holds nx <= 13");
    static constexpr unsigned XMASK = (1u << (2 * S::nx)) - 1u, UDMASK = 0xFu << UUP, QMASK = 0x3u << QUP;
};

template <class S>
struct TpiPolParams {
    double Ad[S::nx * S::nx], Bd[S::nx];
    double Qx[S::nx * S::nx], QxN[S::nx * S::nx];
    double xlo[S::nx], xhi[S::nx];
    double xlo_m[S::nx], xlo_p[S::nx], xhi_m[S::nx], xhi_p[S::nx];    // bound -/+ 1e-11 (1 + |bound|): soft-row labels
    double cx[S::nx];                                                 // rho_e / rho_x: soft-row multiplier in units of v
    double ulo, uhi, ulo_m, uhi_p, dlo, dhi, dlo_m, dhi_p;            // hard rows: bounds and bound -/+ 1e-9 (1 + |bound|)
    double irhou, irhod, Qu, QDu, quref, rho_e;
    // table-driven decode (dynamic index into the constant bank instead of selects and predicate logic).  Soft rows by label
    // (0 none, 1 above, 2 below): acceptance interval of a consistent candidate [xacc_lo, xacc_hi], penalty weight xm, its
    // linear term xmb = weight * bound, multiplier coefficient xcm = rho_e / rho (in units of v) and bound xbnd
    double xacc_lo[S::nx][4], xacc_hi[S::nx][4], xm[S::nx][4], xmb[S::nx][4], xcm[S::nx][4], xbnd[S::nx][4];
    // pin value of a stage by its pin index (first set bit of the 6 hard-row bits): 0 free, 1/2 input at max/min, 3/4 delta-u at
    // max/min, 5/6 the spurious last row at max/min, 7 held stage (Nc < Np)
    double pintab[8];                                                 // pin value by index
};

#ifdef BMPC_HOSTEMU
BMPC_HD double tpi_rcp(double h) { return 1.0 / h; }
#else
// 1/h for h > 0 in the normal range (a Schur complement of a positive definite Hessian): MUFU seed + two Newton steps
__device__ __forceinline__ double tpi_rcp(double h) {
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(h));
    double e = fma(-h, r, 1.0); r = fma(r, e, r);
    e = fma(-h, r, 1.0); r = fma(r, e, r);
    return r;
}
#endif

// pin index of one stage from its code word (held: a stage k >= Nc of a shape with Nc < Np)
#ifdef BMPC_HOSTEMU
BMPC_HD int tpi_ffs(unsigned b) { return __builtin_ffs((int)b); }
#else
__device__ __forceinline__ int tpi_ffs(unsigned b) { return __ffs((int)b); }
#endif
// first set bit of the 6 hard-row bits = the priority order input bound, delta-u row, spurious row (0: free stage)
template <class S>
BMPC_HD int tpi2_pinidx(unsigned code, bool held) {
    return held ? 7 : tpi_ffs((code >> TpiCode<S>::UUP) & 63u);
}
// soft-row label (0 none, 1 above its bound, 2 below) of state component a
template <class S>
BMPC_HD int tpi2_xlabel(unsigned code, int a) {
    return (int)((code >> (TpiCode<S>::XUP + a)) & 1u) + 2 * (int)((code >> (TpiCode<S>::XDN + a)) & 1u);
}

// Backward sweep: fills the gain slots of W from the working-set codes C(k).
template <class S, class PP, class XR, class CA>
BMPC_HD void tpi2_backward(const PP& P, TpiAcc W, CA C, XR xr) {
    static_assert(S::nu == 1 && S::Nc <= S::Np, "Riccati polish is specialised to nu == 1");
    constexpr int nx = S::nx, N = S::Np, Nc = S::Nc, nz1 = nx + 2;
    double Pm[nx * nx], pxw[nx], px[nx], pww = 0.0, pw = 0.0;          // Pm symmetric: both triangles hold the same values
    double qc[nx];                                                       // Qx xref (constant reference)
    const double P_QDu = P.QDu, P_QuQDu = (double)P.Qu + P_QDu, P_quref = P.quref;   // scalars once (PP may be a view in global memory)
    if (!XR::TV) {
#pragma unroll
        for (int a = 0; a < nx; a++) {
            double q = 0.0;
#pragma unroll
            for (int b = 0; b < nx; b++) q += P.Qx[a * nx + b] * xr(0, b);
            qc[a] = q;
        }
    }
    unsigned code = C(N - 1);
    {   // terminal cost of x_N (its rows are the state bits of stage N-1)
#pragma unroll
        for (int a = 0; a < nx; a++) {
            const int lab = tpi2_xlabel<S>(code, a);
            double q = 0.0;
#pragma unroll
            for (int b = 0; b < nx; b++) { Pm[a * nx + b] = P.QxN[a * nx + b]; q += P.QxN[a * nx + b] * xr(N, b); }
            Pm[a * nx + a] += P.xm[a][lab];
            px[a] = -(q + P.xmb[a][lab]); pxw[a] = 0.0;
        }
    }
#pragma unroll 1
    for (int k = N - 1; k >= 0; k--) {
        const unsigned cprev = C(k >= 1 ? k - 1 : 0);                   // state bits of x_k (x_0 is data: its cost is irrelevant)
        const bool held = (Nc < N) && (k >= Nc);
        const int pi = tpi2_pinidx<S>(code, held);
        const double pin = P.pintab[pi];
        const bool free_ = pi == 0;
        const double dp = (pi == 3 || pi == 4 || pi == 7) ? 1.0 : 0.0;
        double xmk[nx], xmbk[nx];
#pragma unroll
        for (int a = 0; a < nx; a++) { const int lab = tpi2_xlabel<S>(cprev, a); xmk[a] = P.xm[a][lab]; xmbk[a] = P.xmb[a][lab]; }
        double T[nx * nx], PB[nx];
#pragma unroll
        for (int a = 0; a < nx; a++) {
#pragma unroll
            for (int b = 0; b < nx; b++) {
                double acc = Pm[a * nx + 0] * P.Ad[0 * nx + b];
#pragma unroll
                for (int q = 1; q < nx; q++) acc = fma(Pm[a * nx + q], P.Ad[q * nx + b], acc);
                T[a * nx + b] = acc;
            }
            double accb = Pm[a * nx + 0] * P.Bd[0];
#pragma unroll
            for (int q = 1; q < nx; q++) accb = fma(Pm[a * nx + q], P.Bd[q], accb);
            PB[a] = accb;
        }
        double Hxx[nx * nx], hx[nx], gx[nx];
        double huu = pww + P_QuQDu, gu = pw - P_quref;
#pragma unroll
        for (int a = 0; a < nx; a++) { huu = fma(P.Bd[a], PB[a] + 2.0 * pxw[a], huu); gu = fma(P.Bd[a], px[a], gu); }
#pragma unroll
        for (int a = 0; a < nx; a++) {
#pragma unroll
            for (int b = a; b < nx; b++) {                              // upper triangle of A' T (symmetric)
                double acc = P.Ad[0 * nx + a] * T[0 * nx + b];
#pragma unroll
                for (int q = 1; q < nx; q++) acc = fma(P.Ad[q * nx + a], T[q * nx + b], acc);
                Hxx[a * nx + b] = acc + P.Qx[a * nx + b];
            }
            double h = 0.0, g = 0.0;
#pragma unroll
            for (int q = 0; q < nx; q++) { h = fma(P.Ad[q * nx + a], PB[q] + pxw[q], h); g = fma(P.Ad[q * nx + a], px[q], g); }
            hx[a] = h;
            double q;
            if (XR::TV) {
                q = 0.0;
#pragma unroll
                for (int b = 0; b < nx; b++) q = fma(P.Qx[a * nx + b], xr(k, b), q);
            } else q = qc[a];
            Hxx[a * nx + a] += xmk[a];
            gx[a] = g - (q + xmbk[a]);
        }
        const double hw = -P_QDu, Hww = P_QDu;
        const double inv = tpi_rcp(huu);
        const double c1 = free_ ? inv : 0.0, c4 = free_ ? inv : 1.0;
        const double c2 = fma(-c1, gu, pin);                            // free: -gu / huu ; pinned: pin
        const double c3 = fma(-c1, hw, dp);
        const double pinned0 = fma(huu, pin, gu);                       // dQ/du offset of a pinned stage
        const int base = k * nz1;
#pragma unroll
        for (int a = 0; a < nx; a++) W(base + a) = hx[a] * c4;
        W(base + nx) = free_ ? hw * inv : fma(dp, huu, hw);
        W(base + nx + 1) = free_ ? gu * inv : pinned0;
#pragma unroll
        for (int a = 0; a < nx; a++) {
            const double ha = hx[a] * c1;
#pragma unroll
            for (int b = a; b < nx; b++) { const double v = fma(-ha, hx[b], Hxx[a * nx + b]); Pm[a * nx + b] = v; Pm[b * nx + a] = v; }
            px[a] = fma(hx[a], c2, gx[a]);
            pxw[a] = hx[a] * c3;
        }
        pww = fma(dp, fma(2.0, hw, huu), Hww) - c1 * hw * hw;
        pw = fma(hw, c2, dp * pinned0);
        code = cprev;
    }
}

// Forward sweep: rolls the closed loop out, verifies the KKT conditions of the working sets, writes the NEXT working sets
// into C(k), the inputs through outu(k, u), the exact ADMM fixed point v* = z* + y*/rho into the gain slots just consumed
// (the spurious last row into vq) and returns true when the candidate is the minimiser.  mumax: in = scale of the multiplier
// sign tolerance (sum of the multiplier magnitudes of the previous refinement, 0 at first), out = that of this one.
template <class S, class PP, class CA, class FU>
BMPC_HD bool tpi2_forward(const PP& P, TpiAcc W, CA C, const double* x0, double um1, double& mumax, double& vq, FU outu) {
    constexpr int nx = S::nx, N = S::Np, Nc = S::Nc, nz1 = nx + 2;
    using CD = TpiCode<S>;
    const double mutol = -1e-9 * (1.0 + mumax);
    const double ulo_m = P.ulo_m, uhi_p = P.uhi_p, dlo_m = P.dlo_m, dhi_p = P.dhi_p, irhou = P.irhou, irhod = P.irhod;
    double mnew = 0.0;
    unsigned bad = 0u;
    double x[nx], w = um1;
#pragma unroll
    for (int a = 0; a < nx; a++) x[a] = x0[a];
    // KKT check of one hard row with label lab (0 none, 1 at max, 2 at min) and multiplier mu; returns its two bits of the next
    // working set (bit 0 up, bit 1 down).  m = sign(label) * mu must not be negative; the label survives if m > 0.
    auto hard_row = [&](double zi, double lo_m, double hi_p, unsigned lab, double mu) -> unsigned {
        const double m = (double)((int)(lab & 1u) - (int)(lab >> 1)) * mu;
        const unsigned vu = zi > hi_p, vd = zi < lo_m, keep = m > 0.0;
        bad |= vu | vd | (unsigned)(m < mutol);
        const unsigned nu_ = vu | (~vd & keep & lab & 1u);
        const unsigned nd_ = ~nu_ & (vd | (keep & (lab >> 1))) & 1u;
        return (nu_ & 1u) | (nd_ << 1);
    };
    unsigned code = C(0);
    double g[nz1];
#pragma unroll
    for (int a = 0; a < nz1; a++) g[a] = W(a);
#pragma unroll 1
    for (int k = 0; k < N; k++) {
        const int base = k * nz1;
        const bool held = (Nc < N) && (k >= Nc);
        const int pi = tpi2_pinidx<S>(code, held);
        const double pin = P.pintab[pi];
        // soft-row tables of x_{k+1} (independent of the state recursion: issued before it)
        double alo[nx], ahi[nx], cm[nx], bnd[nx];
#pragma unroll
        for (int a = 0; a < nx; a++) { const int lab = tpi2_xlabel<S>(code, a); alo[a] = P.xacc_lo[a][lab]; ahi[a] = P.xacc_hi[a][lab]; cm[a] = P.xcm[a][lab]; bnd[a] = P.xbnd[a][lab]; }
        double lin = g[nx + 1];
#pragma unroll
        for (int a = 0; a < nx; a++) lin = fma(g[a], x[a], lin);
        lin = fma(g[nx], w, lin);
        // next stage's code and gains: in flight while this stage computes
        const int kn = (k + 1 < N) ? k + 1 : k;
        const unsigned code_n = C(kn);
#pragma unroll
        for (int a = 0; a < nz1; a++) g[a] = W(kn * nz1 + a);
        const bool dpin = (pi == 3 || pi == 4 || pi == 7);
        double u = dpin ? w + pin : pin;
        u = (pi == 0) ? -lin : u;
        unsigned ncode = 0u;
        if (!held) {
            const double mu_u = (pi == 1 || pi == 2) ? -lin : 0.0, mu_d = (pi == 3 || pi == 4) ? -lin : 0.0;
            mnew += (pi == 0) ? 0.0 : fabs(lin);
            outu(k, u);
            unsigned hb = hard_row(u, ulo_m, uhi_p, (code >> CD::UUP) & 3u, mu_u);
            ncode |= hb << CD::UUP;
            W(base + nx) = fma(mu_u, irhou, u);
            const double dz = u - w;                                    // row 0: u_0 against bounds shifted by u_-1 = the same test
            hb = hard_row(dz, dlo_m, dhi_p, (code >> CD::DUP) & 3u, mu_d);
            ncode |= hb << CD::DUP;
            W(base + nx + 1) = fma(mu_d, irhod, (k == 0) ? u : dz);
            if (k == Nc - 1) {
                const double mu_q = (pi == 5 || pi == 6) ? lin : 0.0;
                hb = hard_row(-u, dlo_m, dhi_p, (code >> CD::QUP) & 3u, mu_q);
                ncode |= hb << CD::QUP;
                vq = fma(mu_q, irhod, -u);
            }
        }
        double xn[nx];
#pragma unroll
        for (int a = 0; a < nx; a++) {
            double a0 = P.Bd[a] * u, a1 = 0.0;
#pragma unroll
            for (int q = 0; q < nx; q += 2) { a0 = fma(P.Ad[a * nx + q], x[q], a0); if (q + 1 < nx) a1 = fma(P.Ad[a * nx + q + 1], x[q + 1], a1); }
            xn[a] = a0 + a1;
        }
        w = u;
#pragma unroll
        for (int a = 0; a < nx; a++) {
            const double zi = xn[a];
            x[a] = zi;
            // a label may differ from the side the candidate is on only if the row sits on that bound (to 1e-11 relative): the
            // candidate is consistent iff zi lies in the acceptance interval of the row's label
            bad |= (unsigned)(zi < alo[a]) | (unsigned)(zi > ahi[a]);
            const unsigned nu_ = zi > P.xhi_p[a], nd_ = zi < P.xlo_m[a];
            W(base + a) = fma(cm[a], zi - bnd[a], zi);
            ncode |= nu_ << (CD::XUP + a);
            ncode |= (nd_ & ~nu_ & 1u) << (CD::XDN + a);
        }
        C(k) = (typename CD::type)ncode;
        code = code_n;
    }
    mumax = mnew;
    return bad == 0u;
}

// first working sets from an ADMM iterate v (TPI rows; after a cold start or a straggler round): as tpi_sets_from_v
template <class S, class PP, class Acc, class CA>
BMPC_HD void tpi2_codes_from_v(const PP& P, double um1, Acc V, double vlast, CA C) {
    constexpr int nx = S::nx, Np = S::Np, Nc = S::Nc, NS = S::NS, NU = S::NU;
    using CD = TpiCode<S>;
    auto over = [](double v, double hi) { return v > hi + 1e-9 * (1.0 + fabs(hi)); };
    auto under = [](double v, double lo) { return v < lo - 1e-9 * (1.0 + fabs(lo)); };
    const double uhi = P.uhi, ulo = P.ulo, dhi = P.dhi, dlo = P.dlo;
#pragma unroll 1
    for (int k = 0; k < Np; k++) {
        unsigned c = 0u;
#pragma unroll
        for (int a = 0; a < nx; a++) {
            const double v = V(k * nx + a), xh = P.xhi[a], xl = P.xlo[a];
            c |= (over(v, xh) ? 1u : 0u) << (CD::XUP + a); c |= (under(v, xl) ? 1u : 0u) << (CD::XDN + a);
        }
        if (k < Nc) {
            const double vu = V(NS + k);
            c |= (over(vu, uhi) ? 1u : 0u) << CD::UUP; c |= (under(vu, ulo) ? 1u : 0u) << CD::UDN;
            const double vd = V(NS + NU + k), sh = (k == 0) ? um1 : 0.0;
            c |= (over(vd, dhi + sh) ? 1u : 0u) << CD::DUP; c |= (under(vd, dlo + sh) ? 1u : 0u) << CD::DDN;
            if (k == Nc - 1) { c |= (over(vlast, dhi) ? 1u : 0u) << CD::QUP; c |= (under(vlast, dlo) ? 1u : 0u) << CD::QDN; }
        }
        C(k) = (typename CD::type)c;
    }
}

// receding-horizon shift of stored working sets: stage k takes the sets of stage k + 1 (the last stage keeps its own)
template <class S>
BMPC_HD unsigned tpi2_shifted_code(const typename TpiCode<S>::type* stored, int k, bool shift) {
    using CD = TpiCode<S>;
    constexpr int Np = S::Np, Nc = S::Nc;
    if (!shift) return stored[k];
    const int ks = (k + 1 < Np) ? k + 1 : Np - 1, ku = (k + 1 < Nc) ? k + 1 : Nc - 1;
    unsigned c = stored[ks] & CD::XMASK;
    if (k < Nc) c |= stored[ku] & CD::UDMASK;
    if (k == Nc - 1) c |= stored[Nc - 1] & CD::QMASK;
    return c;
}

// The polish parameters of one system.  Reads only the system's inputs (Ad .. uref) and scal[RHO], scal[RHOE], never the condensed
// arrays: the rows' bounds are the raw bounds (lo0 / hi0 copy them) and a row's rho follows the condense's rule (bmpc_row_rho).
// So the fill stays valid on a block whose condensed part predates its inputs (per-instance systems after bmpc_update_problem,
// k_fill_view), and gives bit for bit the block a fill from a freshly condensed system gives.
template <class S>
BMPC_HOSTDEV void tpi_fill_pol(const double* sys, const BmpcSysOff& o, TpiPolParams<S>& P) {
    constexpr int nx = S::nx;
    for (int i = 0; i < nx * nx; i++) { P.Ad[i] = sys[o.Ad + i]; P.Qx[i] = sys[o.Qx + i]; P.QxN[i] = sys[o.QxN + i]; }
    for (int i = 0; i < nx; i++) P.Bd[i] = sys[o.Bd + i];
    const double rho_e = sys[o.scal + BMPC_S_RHOE], rho = sys[o.scal + BMPC_S_RHO];
    auto tol = [](double b, double rel, double sgn) { return (fabs(b) > 1e300) ? b : b + sgn * rel * (1.0 + fabs(b)); };
    for (int a = 0; a < nx; a++) {
        const double lo = sys[o.xmin + a], hi = sys[o.xmax + a];          // the state rows of stage 1 (condensed rows nx + a)
        P.xlo[a] = lo; P.xhi[a] = hi;
        P.xlo_m[a] = tol(lo, 1e-11, -1.0); P.xlo_p[a] = tol(lo, 1e-11, 1.0); P.xhi_m[a] = tol(hi, 1e-11, -1.0); P.xhi_p[a] = tol(hi, 1e-11, 1.0);
        P.cx[a] = rho_e / bmpc_row_rho(lo, hi, rho);
    }
    // the input row and the delta-u rows (condensed rows NX and NX + NU; nu == 1)
    P.ulo = sys[o.umin]; P.uhi = sys[o.umax]; P.ulo_m = tol(P.ulo, 1e-9, -1.0); P.uhi_p = tol(P.uhi, 1e-9, 1.0);
    P.dlo = sys[o.Dumin]; P.dhi = sys[o.Dumax]; P.dlo_m = tol(P.dlo, 1e-9, -1.0); P.dhi_p = tol(P.dhi, 1e-9, 1.0);
    P.irhou = 1.0 / bmpc_row_rho(P.ulo, P.uhi, rho); P.irhod = 1.0 / bmpc_row_rho(P.dlo, P.dhi, rho);
    P.Qu = sys[o.Qu]; P.QDu = sys[o.QDu]; P.quref = sys[o.Qu] * sys[o.uref]; P.rho_e = rho_e;
    const double inf = 1.0 / 0.0;
    for (int a = 0; a < nx; a++) {
        const double lo = P.xlo[a], hi = P.xhi[a];
        const double al[4] = {P.xlo_m[a], P.xhi_m[a], -inf, -inf}, ah[4] = {P.xhi_p[a], inf, P.xlo_p[a], inf};
        const double m[4] = {0.0, rho_e, rho_e, 0.0}, bd[4] = {0.0, hi, lo, 0.0};
        for (int l = 0; l < 4; l++) {
            P.xacc_lo[a][l] = al[l]; P.xacc_hi[a][l] = ah[l]; P.xm[a][l] = m[l]; P.xbnd[a][l] = (fabs(bd[l]) > 1e300) ? 0.0 : bd[l];
            P.xmb[a][l] = m[l] * P.xbnd[a][l]; P.xcm[a][l] = (l == 1 || l == 2) ? P.cx[a] : 0.0;
        }
    }
    const double pt[8] = {0.0, P.uhi, P.ulo, P.dhi, P.dlo, -P.dhi, -P.dlo, 0.0};
    for (int i = 0; i < 8; i++) P.pintab[i] = pt[i];
}

// ------------------------------------------------------------------------------------------------
// Per-instance systems (SURVEY 8f-3) on the fast path: the same parameter block, one per instance, in GLOBAL memory stored
// field-major — double number f of instance i at pg[f * B + i] — so that the 32 lanes of a warp (32 consecutive instances)
// read every field with one coalesced access.  TpiPolView offers the member names of TpiPolParams (P.Ad[i], P.xm[a][lab],
// P.uhi_p, ...), so the sweeps above compile unchanged against either.
struct TpiGScalar { const double* p; BMPC_HD operator double() const { return *p; } };
struct TpiGArr { const double* p; size_t B; BMPC_HD double operator[](int i) const { return p[(size_t)i * B]; } };
struct TpiGArr2 { const double* p; size_t B; BMPC_HD TpiGArr operator[](int a) const { return TpiGArr{p + (size_t)a * 4 * B, B}; } };
template <class S>
struct TpiPolView {
    using PS = TpiPolParams<S>;
    TpiGArr Ad, Bd, Qx, QxN, xlo, xhi, xlo_m, xlo_p, xhi_m, xhi_p, cx, pintab;
    TpiGArr2 xacc_lo, xacc_hi, xm, xmb, xcm, xbnd;
    TpiGScalar ulo, uhi, ulo_m, uhi_p, dlo, dhi, dlo_m, dhi_p, irhou, irhod, Qu, QDu, quref, rho_e;
    static constexpr int NF = (int)(sizeof(PS) / sizeof(double));
#define BMPC_VF(m) (p + (offsetof(PS, m) / sizeof(double)) * B)
    BMPC_HD TpiPolView(const double* p, size_t B)
        : Ad{BMPC_VF(Ad), B}, Bd{BMPC_VF(Bd), B}, Qx{BMPC_VF(Qx), B}, QxN{BMPC_VF(QxN), B}, xlo{BMPC_VF(xlo), B}, xhi{BMPC_VF(xhi), B},
          xlo_m{BMPC_VF(xlo_m), B}, xlo_p{BMPC_VF(xlo_p), B}, xhi_m{BMPC_VF(xhi_m), B}, xhi_p{BMPC_VF(xhi_p), B}, cx{BMPC_VF(cx), B},
          pintab{BMPC_VF(pintab), B}, xacc_lo{BMPC_VF(xacc_lo), B}, xacc_hi{BMPC_VF(xacc_hi), B}, xm{BMPC_VF(xm), B}, xmb{BMPC_VF(xmb), B},
          xcm{BMPC_VF(xcm), B}, xbnd{BMPC_VF(xbnd), B}, ulo{BMPC_VF(ulo)}, uhi{BMPC_VF(uhi)}, ulo_m{BMPC_VF(ulo_m)}, uhi_p{BMPC_VF(uhi_p)},
          dlo{BMPC_VF(dlo)}, dhi{BMPC_VF(dhi)}, dlo_m{BMPC_VF(dlo_m)}, dhi_p{BMPC_VF(dhi_p)}, irhou{BMPC_VF(irhou)}, irhod{BMPC_VF(irhod)},
          Qu{BMPC_VF(Qu)}, QDu{BMPC_VF(QDu)}, quref{BMPC_VF(quref)}, rho_e{BMPC_VF(rho_e)} {}
#undef BMPC_VF
};
