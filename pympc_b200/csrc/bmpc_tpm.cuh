// bmpc_tpm.cuh — constrained Riccati polish for multi-input shapes (nu >= 1), one THREAD per instance.
//
// The multi-input counterpart of the second-generation polish in bmpc_tpi.cuh (same verification rules; mpc.py:166-240 and
// :456-615 build the QP these sweeps solve exactly for a guessed working set).  The reference's delta-u block is "-I + eye(k=1)"
// on the SCALAR stacking of U (mpc.py:569-571): its rows chain u_k[j] - u_k[j-1] inside a stage and u_k[0] - u_{k-1}[nu-1] across
// stages.  The sweeps therefore treat every scalar input as a sub-step of its own:
//  * sub-step (k, j) applies u = u_k[j] through column j of Bd to the partial next state y (y = Ad x_k before sub-step 0, x_{k+1}
//    after sub-step nu-1) and overwrites entry j of the register r of most recent inputs (r[j] = u_{k-1}[j] before, u_k[j] after:
//    the delta-u COST of mpc.py:510-524 pairs u with r[j], the chain ROW pairs it with the previously written entry);
//  * cost-to-go over s = (y, r), n = nx + nu: V(s) = 1/2 s'P s + p's; a sub-step is a scalar-input Riccati step (rank-1 update),
//    the state map y = Ad x is applied once per stage;
//  * rows of a sub-step: input bound, first-block row u_0[j] - u_-1[j] (k = 0), chain row, spurious last row -u_{Nc-1}[nu-1]
//    (mpc.py:216-221): two code bits each (at max / at min), 8 bits per channel after the 2 nx soft state-row bits.  The first
//    set bit is the sub-step's pin (u = bound, u = r[j] + d, u = previous scalar + d, u = -d); stages k >= Nc hold (u = r[j]);
//  * per sub-step ONE row of n + 1 numbers (+ the resolved pin type and value) is stored: free: the feedback row (u = -row . (s, 1)); pinned: the gradient row
//    dQ/du along the policy (the multiplier of the pinning row is -row . (s, 1)).  Mask arithmetic, no divergence between lanes;
//  * forward sweep: rolls the closed loop out, checks primal feasibility and multiplier signs of every row (KKT: the candidate is
//    then THE minimiser of the strictly convex QP), builds the next working sets (primal-dual active-set update), stages
//    v* = z* + y*/rho (the ADMM fixed point, the warm start of the fallback rounds) in the slots it has consumed.
//  * anchored runs: a run of active chain rows that ends at a scalar fixed by another row (its bound, the first-block row, the
//    spurious last row — the usual end of a horizon: -u_{Nc-1}[nu-1] within the delta-u box drags the tail of the plan down at the
//    maximum rate) determines the EARLIER scalars of the run: u_t = a_{t+1} - d.  The backward sweep resolves this while it
//    walks the scalars in descending order (pin type 5, absolute value a_t); the multipliers of such a run follow from
//    stationarity scalar by scalar, y_{t+1} = dQ/du_t + y_t, which the forward sweep accumulates.
// Working sets with two anchors in one run are degenerate (the surplus row is treated as inactive); an instance that cannot be
// verified takes the team path (Schur-form polish, any working set).
// Requires a diagonal QDu (the register keeps one previous value per channel).  Gain rows live in GLOBAL memory
// (nu nz Np doubles per instance: 16.6 KB at nx=8, nu=4, Np=40 — beyond shared memory), lane-interleaved.
#pragma once
#include "bmpc_tpi.cuh"

// A shape with the sparsity pattern of (Ad, Bd) fixed at compile time (bit q nx + b of AM: Ad[q][b] may be non-zero, bit a nu + j of
// BM: Bd[a][j]): the sweeps skip the structural zeros — the MIMO reference governor's Ad is block diagonal (12 of 64 entries), its
// Bd has one entry per channel.  A system whose pattern is contained in the masks runs on this instantiation; the plain TpiShape
// is dense.  (nx nx <= 64, nx nu <= 32.)
template <int NXc, int NUc, int NPc, int NCc, unsigned long long AM, unsigned BM>
struct TpmSparseShape : TpiShape<NXc, NUc, NPc, NCc> {
    static_assert(NXc * NXc <= 64 && NXc * NUc <= 32, "pattern masks hold nx nx <= 64 and nx nu <= 32 bits");
    static constexpr unsigned long long amask = AM; static constexpr unsigned bmask = BM;
    BMPC_HD static constexpr bool a_nz(int q, int b) { return (AM >> (q * NXc + b)) & 1ull; }
    BMPC_HD static constexpr bool b_nz(int a, int j) { return (BM >> (a * NUc + j)) & 1u; }
};

template <class S>
struct TpmCode {
    // channel j: bits CH0 + 8 j + {0 u max, 1 u min, 2 first max, 3 first min, 4 chain max, 5 chain min, 6 last max, 7 last min}
    // + hints of the forward sweep for the next resolution: bit 8 "let the chain row pin this scalar", bit 9 "let the next chain row pin it"
    static constexpr unsigned XUP = 0, XDN = S::nx, CH0 = 2 * S::nx, CHS = 10;
    static constexpr unsigned BITS = 2 * S::nx + CHS * S::nu;
    static_assert(BITS <= 64, "working-set code word exceeds 64 bits");
    using type = uint64_t;
    static constexpr uint64_t XMASK = (1ull << (2 * S::nx)) - 1ull;
    BMPC_HD static constexpr uint64_t chmask(unsigned bits) { uint64_t m = 0; for (int j = 0; j < S::nu; j++) m |= (uint64_t)bits << (CH0 + CHS * j); return m; }
};

template <class S>
struct TpmParams {
    static constexpr int nx = S::nx, nu = S::nu;
    double Ad[nx * nx], Bd[nx * nu];
    double Qx[nx * nx], QxN[nx * nx];
    double Qu[nu * nu], QDu[nu], quref[nu];                           // Qu (full), diag QDu, Qu uref
    double xlo[nx], xhi[nx], xlo_m[nx], xhi_p[nx];
    double xacc_lo[nx][4], xacc_hi[nx][4], xm[nx][4], xmb[nx][4], xcm[nx][4], xbnd[nx][4];     // soft rows by label: as TpiPolParams
    double ulo[nu], uhi[nu], ulo_m[nu], uhi_p[nu], irhou[nu];         // input rows of channel j
    double flo[nu], fhi[nu], flo_m[nu], fhi_p[nu], irhof[nu];         // first-block rows (unshifted bounds: those of channel j)
    double clo[nu], chi[nu], clo_m[nu], chi_p[nu], irhoc[nu];         // chain row that ENDS at channel j: bounds of channel (j-1) mod nu
};

template <class S>
struct TpmLayout {
    static constexpr int n = S::nx + S::nu, nz = n + 3, per_stage = S::nu * nz, slots = S::Np * per_stage;
    // v* staged in a consumed stage block: sub-step j: input row at 2 j, chain row at 2 j + 1; then the nx rows of x_{k+1}
    static_assert(per_stage >= S::nx + 2 * S::nu, "stage block too small for the staged v*");
    // the domain of pympc_b200.build.tpm_shape_supported (the code word is checked by TpmCode): wider states or longer horizons
    // make the per-thread stack frame of k_tpm_pol grow to tens of KB
    static_assert(S::nx >= 1 && S::nx <= 13 && S::Np >= 2 && S::Np <= 64 && S::Nc >= 1 && S::Nc <= S::Np,
                  "multi-input fast-path shapes need nx <= 13, Np <= 64, 1 <= Nc <= Np");
};

// index of (a, b) in a packed upper triangle of order n (either order of the arguments)
BMPC_HD constexpr int tpm_tri(int n, int a, int b) { return a <= b ? a * n - a * (a - 1) / 2 + (b - a) : b * n - b * (b - 1) / 2 + (a - b); }

// resolved pin types of a sub-step
enum { TPM_FREE = 0, TPM_INPUT = 1, TPM_FIRST = 2, TPM_CHAIN = 3, TPM_LAST = 4, TPM_BACK = 5, TPM_HELD = 9 };
template <class S>
BMPC_HD int tpm_xlabel(uint64_t code, int a) {
    return (int)((code >> (TpmCode<S>::XUP + a)) & 1ull) + 2 * (int)((code >> (TpmCode<S>::XDN + a)) & 1ull);
}

// Backward sweep: fills the gain rows of W from the working-set codes C(k).
template <class S, class PP, class WA, class CA, class XR>
BMPC_HD void tpm_backward(const PP& P, WA W, CA C, XR xr, const double* um1) {
    constexpr int nx = S::nx, nu = S::nu, N = S::Np, Nc = S::Nc, n = TpmLayout<S>::n, nz = TpmLayout<S>::nz, PS = TpmLayout<S>::per_stage;
    double Pu[n * (n + 1) / 2], p[n];                                   // cost-to-go matrix: packed upper triangle (PM(a, b), any order)
#define PM(a_, b_) Pu[tpm_tri(n, (a_), (b_))]
    double qc[nx];
    if (!XR::TV) {
#pragma unroll
        for (int a = 0; a < nx; a++) {
            double q = 0.0;
#pragma unroll
            for (int b = 0; b < nx; b++) q = fma(P.Qx[a * nx + b], xr(0, b), q);
            qc[a] = q;
        }
    }
    uint64_t code = C(N - 1), code_next = 0ull;
    bool abs_next = false;                                              // the scalar after the current one is fixed to a value ...
    double a_next = 0.0;                                                // ... this one
#pragma unroll
    for (int t = 0; t < n * (n + 1) / 2; t++) Pu[t] = 0.0;
#pragma unroll
    for (int a = 0; a < nx; a++) {
        const int lab = tpm_xlabel<S>(code, a);
        double q = 0.0;
#pragma unroll
        for (int b = 0; b < nx; b++) { if (b >= a) PM(a, b) = P.QxN[a * nx + b]; q = fma(P.QxN[a * nx + b], xr(N, b), q); }
        PM(a, a) += P.xm[a][lab];
        p[a] = -(q + P.xmb[a][lab]);
    }
#pragma unroll
    for (int j = 0; j < nu; j++) p[nx + j] = 0.0;
#pragma unroll 1
    for (int k = N - 1; k >= 0; k--) {
        const uint64_t cprev = C(k >= 1 ? k - 1 : 0);
        const bool held = (Nc < N) && (k >= Nc);
        const int base = k * PS;
#pragma unroll
        for (int j = nu - 1; j >= 0; j--) {
            const int io = nx + j, in_ = nx + (j > 0 ? j - 1 : nu - 1);    // register entries: this channel's previous value, the previous scalar
            // resolve the pin of scalar t = k nu + j from the row labels (see the header)
            const unsigned cbh = (unsigned)(code >> (TpmCode<S>::CH0 + TpmCode<S>::CHS * j)) & 1023u, cb = cbh & 255u;
            const bool want_chain = (cbh >> 8) & 1u, want_back = (cbh >> 9) & 1u;
            const unsigned labn = (j + 1 < nu) ? ((unsigned)(code >> (TpmCode<S>::CH0 + TpmCode<S>::CHS * (j + 1) + 4)) & 3u)
                                               : ((k + 1 < Nc) ? ((unsigned)(code_next >> (TpmCode<S>::CH0 + 4)) & 3u) : 0u);
            const int jn = (j + 1 < nu) ? j + 1 : 0;
            int tau = TPM_FREE; double pin = 0.0;
            if (held) tau = TPM_HELD;
            else if (want_back && labn != 0u && abs_next) { tau = TPM_BACK; pin = a_next - ((labn & 1u) ? P.chi[jn] : P.clo[jn]); }
            else if (want_chain && ((cb >> 4) & 3u)) { tau = TPM_CHAIN; pin = ((cb >> 4) & 1u) ? P.chi[j] : P.clo[j]; }
            else if (cb & 3u) { tau = TPM_INPUT; pin = (cb & 1u) ? P.uhi[j] : P.ulo[j]; }
            else if ((cb >> 2) & 3u) { tau = TPM_FIRST; pin = um1[j] + (((cb >> 2) & 1u) ? P.fhi[j] : P.flo[j]); }
            else if ((cb >> 6) & 3u) { tau = TPM_LAST; pin = -(((cb >> 6) & 1u) ? P.chi[0] : P.clo[0]); }
            else if (labn != 0u && abs_next) { tau = TPM_BACK; pin = a_next - ((labn & 1u) ? P.chi[jn] : P.clo[jn]); }
            else if ((cb >> 4) & 3u) { tau = TPM_CHAIN; pin = ((cb >> 4) & 1u) ? P.chi[j] : P.clo[j]; }
            abs_next = (tau == TPM_INPUT || tau == TPM_FIRST || tau == TPM_LAST || tau == TPM_BACK); a_next = pin;
            const bool free_ = tau == TPM_FREE;
            const double so = (tau == TPM_HELD) ? 1.0 : 0.0, sn = (tau == TPM_CHAIN) ? 1.0 : 0.0;
            double Pb[n];
#pragma unroll
            for (int t = 0; t < n; t++) {
                double acc = PM(t, io);
#pragma unroll
                for (int a = 0; a < nx; a++) if (S::b_nz(a, j)) acc = fma(PM(t, a), P.Bd[a * nu + j], acc);
                Pb[t] = acc;
            }
            double huu = Pb[io] + P.Qu[j * nu + j] + P.QDu[j], gu = p[io] - P.quref[j];
#pragma unroll
            for (int a = 0; a < nx; a++) if (S::b_nz(a, j)) { huu = fma(P.Bd[a * nu + j], Pb[a], huu); gu = fma(P.Bd[a * nu + j], p[a], gu); }
            double hus[n];
#pragma unroll
            for (int t = 0; t < n; t++) hus[t] = Pb[t];
            hus[io] = -P.QDu[j];
#pragma unroll
            for (int i = 0; i < j; i++) hus[nx + i] += P.Qu[j * nu + i];
            // the old r[j] leaves the state: its row / column keep only this sub-step's delta-u cost
#pragma unroll
            for (int t = 0; t < n; t++) PM(t, io) = 0.0;
            PM(io, io) = P.QDu[j];
            p[io] = 0.0;
            const double inv = tpi_rcp(huu);
            const double kap = free_ ? inv : 0.0;
            const double k0 = fma(-kap, gu, pin);                      // constant of the policy u = k's + k0
            const double y0 = fma(huu, k0, gu);                        // gradient along the policy (zero when free)
            // stored row: free: hus / huu, gu / huu ; pinned: y = hus + huu (so e_io + sn e_in), y0
            double yrow[n];
#pragma unroll
            for (int t = 0; t < n; t++) yrow[t] = hus[t];
            yrow[io] = fma(huu, so, yrow[io]); yrow[in_] = fma(huu, sn, yrow[in_]);
#pragma unroll
            for (int t = 0; t < n; t++) W.st(base + j * nz + t, free_ ? hus[t] * inv : yrow[t]);
            W.st(base + j * nz + n, free_ ? gu * inv : y0);
            W.st(base + j * nz + n + 1, pin); W.st(base + j * nz + n + 2, (double)tau);
            // P' = Hss - kap hus hus' + (so e_io + sn e_in) y~' + hus (so e_io + sn e_in)'   with y~ = y of the pinned policy
            // p' = gs + hus k0 + k (gu + huu k0)
#pragma unroll
            for (int a = 0; a < n; a++) {
                const double ha = hus[a] * kap;
#pragma unroll
                for (int b = a; b < n; b++) PM(a, b) = fma(-ha, hus[b], PM(a, b));
                p[a] = fma(hus[a], k0, p[a]);
            }
            // pinned-policy terms (so, sn are zero when free): rows / columns io and in_
#pragma unroll
            for (int t = 0; t < n; t++) {
                const double add_o = so * hus[t], add_n = sn * hus[t];
                PM(io, t) += (t == io) ? 2.0 * add_o : add_o;             // e hus' + hus e'
                PM(in_, t) += (t == in_) ? 2.0 * add_n : add_n;
            }
            PM(io, io) = fma(so, huu, PM(io, io));
            PM(in_, in_) = fma(sn, huu, PM(in_, in_));
            p[io] = fma(so, y0, p[io]); p[in_] = fma(sn, y0, p[in_]);
        }
        // state map y = Ad x_k: Pyy <- A'Pyy A, Pyr <- A'Pyr, py <- A'py; then the cost of x_k (labels: state bits of stage k-1)
        {
            double T[nx * nx];
#pragma unroll
            for (int a = 0; a < nx; a++)
#pragma unroll
                for (int b = 0; b < nx; b++) {
                    double acc = 0.0;
#pragma unroll
                    for (int q = 0; q < nx; q++) if (S::a_nz(q, b)) acc = fma(PM(a, q), P.Ad[q * nx + b], acc);
                    T[a * nx + b] = acc;
                }
            double pyn[nx], Pyr[nx * nu];
#pragma unroll
            for (int a = 0; a < nx; a++) {
                double g = 0.0;
#pragma unroll
                for (int q = 0; q < nx; q++) if (S::a_nz(q, a)) g = fma(P.Ad[q * nx + a], p[q], g);
                pyn[a] = g;
#pragma unroll
                for (int j = 0; j < nu; j++) {
                    double acc = 0.0;
#pragma unroll
                    for (int q = 0; q < nx; q++) if (S::a_nz(q, a)) acc = fma(P.Ad[q * nx + a], PM(q, nx + j), acc);
                    Pyr[a * nu + j] = acc;
                }
            }
#pragma unroll
            for (int a = 0; a < nx; a++) {
                const int lab = tpm_xlabel<S>(cprev, a);
#pragma unroll
                for (int b = a; b < nx; b++) {
                    double acc = 0.0;
#pragma unroll
                    for (int q = 0; q < nx; q++) if (S::a_nz(q, a)) acc = fma(P.Ad[q * nx + a], T[q * nx + b], acc);
                    acc += P.Qx[a * nx + b];
                    PM(a, b) = acc;
                }
                PM(a, a) += P.xm[a][lab];
#pragma unroll
                for (int j = 0; j < nu; j++) PM(a, nx + j) = Pyr[a * nu + j];
                double q;
                if (XR::TV) {
                    q = 0.0;
#pragma unroll
                    for (int b = 0; b < nx; b++) q = fma(P.Qx[a * nx + b], xr(k, b), q);
                } else q = qc[a];
                p[a] = pyn[a] - (q + P.xmb[a][lab]);
            }
        }
        code_next = code; code = cprev;
    }
#undef PM
}

// Forward sweep: see the header.  x0 [nx], um1 [nu]; vfirst [nu]: v* of the first-block rows, vq: of the spurious last row;
// outu(k, j, u).  mumax: in = multiplier scale of the previous refinement (0 at first), out = this one's.  True when verified.
// Verification of the dual side.  At a degenerate vertex (more rows at their bounds than scalars they fix — the rule in a
// rate-limited transient, where every value sits on the lattice of the rate bound) the multipliers are not unique and the ones
// the elimination order happens to produce may carry wrong signs although the point is optimal.  The rows form a path
// (row t couples scalars t-1 and t, own rows touch one scalar), so stationarity reads y_{t+1} = gamma_t + mu_t + y_t with
// gamma_t = dJ/du_t at the candidate, and "do multipliers with the right signs exist" is an interval propagation along the
// path: Y_{t+1} = (Y_t + gamma_t + M_t) ∩ S_{t+1}, M_t / S_t = the sign sets of the rows that sit at a bound ({0} otherwise).
// gamma_t = G_t - [scalar t+1 forward chain-pinned] G_{t+1}, G = the stored total derivative along the policy.
struct TpmInterval {
    double lo, hi;
    // sign set of a row with OSQP's convention (y >= 0 at the upper bound, <= 0 at the lower bound)
    BMPC_HD static TpmInterval row(bool at_hi, bool at_lo) { return TpmInterval{at_lo ? -1e300 : 0.0, at_hi ? 1e300 : 0.0}; }
};

// Forward sweep: see the header.  x0 [nx], um1 [nu]; vfirst [nu]: v* of the first-block rows, vq: of the spurious last row;
// outu(k, j, u).  mumax: in = multiplier scale of the previous refinement (0 at first), out = this one's.  Returns 0 when verified
// (bit 0: a row violated or a soft-row label inconsistent, bit 1: no multipliers with the right signs exist).
// C(k): in = the working sets, out = the primal-dual active-set update; CB(k): out = the rows AT a bound at this candidate
// (the description of a verified, possibly degenerate, vertex: what the next solve should start from); CK(k): out = the update without dual
// drops (violated rows join, labelled rows stay while they sit at their bound).
// EX (exchange mode, the straggler rounds): the soft-row labels follow the candidate as always, but the hard-row labels change by
// single exchanges — per refinement the most violated row enters and the PINNING row with the largest wrong-signed multiplier
// leaves; labels of rows that pin nothing (no multiplier) still go.  The all-rows-at-once update of the default mode settles an
// ordinary solve in 3 - 4 refinements but cycles on ~6 % of the MIMO transient's warm solves; single exchanges do not (host study
// tools/tpm_search_study.py: every one of those stragglers verifies within 12 refinements after their ADMM chunk; 54 % with the
// default update capped at 4).  A separate instantiation: the code of the default mode is unchanged.
template <class S, bool EX, class PP, class WA, class CA, class CB_, class CK_, class FU>
BMPC_HD int tpm_forward(const PP& P, WA W, CA C, CB_ CB, CK_ CK, const double* x0, const double* um1, double& mumax, double* vfirst, double& vq, FU outu) {
    constexpr int nx = S::nx, nu = S::nu, N = S::Np, Nc = S::Nc, n = TpmLayout<S>::n, nz = TpmLayout<S>::nz, PS = TpmLayout<S>::per_stage;
    using CD = TpmCode<S>;
    const double mutol = 1e-9 * (1.0 + mumax);
    double mnew = 0.0, carry = 0.0, prev_mag = 0.0;
    bool carry_on = false;
    int prev_tau = TPM_FREE;
    unsigned pbad = 0u, ibad = 0u;                                      // primal / label failures, dual (interval) failures
    int tr_k = 0; (void)tr_k;
    double s[n];                                                        // (y, r)
#pragma unroll
    for (int a = 0; a < nx; a++) s[a] = x0[a];
#pragma unroll
    for (int j = 0; j < nu; j++) s[nx + j] = um1[j];
    // one hard row: primal check, next label by the primal-dual rule (bits 0-1), at-bound label (bits 2-3), label without dual drops (bits 4-5), violated (bit 6)
    double x_add = -1.0, x_drop = 0.0; int xk_add = -1, xk_drop = -1; unsigned xp_add = 0u, xp_drop = 0u, xl_add = 0u;     // (EX only)
    auto hard_row = [&](double zi, double lo_m, double hi_p, double lo, double hi, unsigned lab, double mu, unsigned pos) -> unsigned {
        const double m = (double)((int)(lab & 1u) - (int)(lab >> 1)) * mu;
        const unsigned vu = zi > hi_p, vd = zi < lo_m, keep = m > 0.0;
        pbad |= vu | vd;
        if (EX) {
            // pos: bit position of the row's label in the code word of stage tr_k
            const unsigned au = zi >= hi - (hi_p - hi), ad = (zi <= lo + (lo - lo_m)) & ~au & 1u;
            const unsigned ku = vu | (lab & au & 1u), kd = ~ku & (vd | ((lab >> 1) & ad)) & 1u;
            unsigned nl = lab;
            if (vu | vd) {
                const unsigned want = vu ? 1u : 2u;
                if (want != lab) {
                    const double sc = (vu ? zi - hi : lo - zi) / (1.0 + fabs(vu ? hi : lo));
                    if (sc > x_add) { x_add = sc; xk_add = tr_k; xp_add = pos; xl_add = want; }
                }
            } else if (lab != 0u && !keep) {
                if (m < 0.0) { if (-m > x_drop) { x_drop = -m; xk_drop = tr_k; xp_drop = pos; } }
                else nl = 0u;
            }
            return (nl & 3u) | (au << 2) | (ad << 3) | (ku << 4) | (kd << 5) | ((vu | vd) << 6);
        }
#ifdef TPM_TRACE
        if (vu | vd) printf("  hard row violated (k %d): z %.6g [%.6g, %.6g] lab %u mu %.6g\n", tr_k, zi, lo_m, hi_p, lab, mu);
#endif
        const unsigned nu_ = vu | (~vd & keep & lab & 1u);
        const unsigned nd_ = ~nu_ & (vd | (keep & (lab >> 1))) & 1u;
        const unsigned au = zi >= hi - (hi_p - hi), ad = (zi <= lo + (lo - lo_m)) & ~au & 1u;
        const unsigned ku = vu | (lab & au & 1u), kd = ~ku & (vd | ((lab >> 1) & ad)) & 1u;    // no dual drops: labels stay while the row sits at its bound
        return (nu_ & 1u) | (nd_ << 1) | (au << 2) | (ad << 3) | (ku << 4) | (kd << 5) | ((vu | vd) << 6);
    };
    // v* of a hard row: z + mu / rho when the multiplier of the elimination order has the sign of its label; otherwise (a surplus row
    // of a degenerate vertex, or a row that merely touches its bound) the bound pushed outward by just more than the label threshold,
    // so that working sets derived from v* are the rows AT their bounds — the description the verified vertex is stored under
    auto stage_v = [&](double zi, double mu, double irho, unsigned lab, unsigned r, double lo, double hi) -> double {
        const double m = (double)((int)(lab & 1u) - (int)(lab >> 1)) * mu;
        const double vb = ((r >> 2) & 1u) ? hi + 4e-9 * (1.0 + fabs(hi)) : (((r >> 3) & 1u) ? lo - 4e-9 * (1.0 + fabs(lo)) : zi);
        return (m > 0.0) ? fma(mu, irho, zi) : vb;
    };
    TpmInterval Y{0.0, 0.0}, pend{0.0, 0.0};                            // multiplier of the chain row into the current scalar; Y + M + G of the previous one
    auto meet = [&](TpmInterval I, TpmInterval Sg) -> TpmInterval {
        double lo = I.lo > Sg.lo ? I.lo : Sg.lo, hi = I.hi < Sg.hi ? I.hi : Sg.hi;
        if (lo > hi) {
            ibad |= (unsigned)(lo - hi > mutol);
#ifdef TPM_TRACE
            if (lo - hi > mutol) printf("  no multipliers (k %d): [%.6g, %.6g] vs sign set [%.3g, %.3g]\n", tr_k, I.lo, I.hi, Sg.lo, Sg.hi);
#endif
            lo = hi = 0.5 * (lo + hi);
        }
        return TpmInterval{lo, hi};
    };
#pragma unroll 1
    for (int k = 0; k < N; k++) {
        const int base = k * PS;
        const uint64_t code = C(k);
        tr_k = k;
        const bool held = (Nc < N) && (k >= Nc);
        {   // y = Ad x_k
            double y[nx];
#pragma unroll
            for (int a = 0; a < nx; a++) {
                double acc = 0.0;
#pragma unroll
                for (int q = 0; q < nx; q++) if (S::a_nz(a, q)) acc = fma(P.Ad[a * nx + q], s[q], acc);
                y[a] = acc;
            }
#pragma unroll
            for (int a = 0; a < nx; a++) s[a] = y[a];
        }
        uint64_t ncode = 0ull, acode = 0ull, kcode = 0ull;
        // the stage's rows, all requested before the first use (the staging stores below alias them: the compiler would not hoist)
        double g[nu * nz];
#pragma unroll
        for (int i = 0; i < nu * nz; i++) g[i] = W.ld(base + i);
#pragma unroll
        for (int j = 0; j < nu; j++) {
            const int io = nx + j, in_ = nx + (j > 0 ? j - 1 : nu - 1);
            double lin = g[j * nz + n];
#pragma unroll
            for (int t = 0; t < n; t++) lin = fma(g[j * nz + t], s[t], lin);
            const double pin = g[j * nz + n + 1];
            const int tau = (int)g[j * nz + n + 2];
            const double rold = s[io], prev = s[in_];
            double u = pin;                                             // absolute pins
            u = (tau == TPM_HELD) ? rold : u;
            u = (tau == TPM_CHAIN) ? prev + pin : u;
            u = (tau == TPM_FREE) ? -lin : u;
            if (!held) {
                const unsigned cb = (unsigned)(code >> (CD::CH0 + CD::CHS * j)) & 255u;
                // multipliers by the elimination order (they drive the active-set update): chain row ending here: carried in from a
                // backward-pinned predecessor, or -lin of a forward pin; own anchor row: closes the stationarity of this scalar
                const double mu_c = carry_on ? carry : ((tau == TPM_CHAIN) ? -lin : 0.0);
                const double tot = lin + (carry_on ? carry : 0.0);
                const double mu_u = (tau == TPM_INPUT) ? -tot : 0.0, mu_f = (tau == TPM_FIRST) ? -tot : 0.0;
                mnew += (tau == TPM_FREE) ? 0.0 : fabs(lin);
                outu(k, j, u);
                unsigned nb = 0u, ab = 0u, kb = 0u, r;                 // (nb: 10 bits: labels + hints)
                r = hard_row(u, P.ulo_m[j], P.uhi_p[j], P.ulo[j], P.uhi[j], cb & 3u, mu_u, CD::CH0 + CD::CHS * j);
                nb |= r & 3u; ab |= (r >> 2) & 3u; kb |= (r >> 4) & 3u;
                TpmInterval M = TpmInterval::row((r >> 2) & 1u, (r >> 3) & 1u);
                W.st(base + 2 * j, stage_v(u, mu_u, P.irhou[j], cb & 3u, r, P.ulo[j], P.uhi[j]));
                if (k == 0) {
                    r = hard_row(u - rold, P.flo_m[j], P.fhi_p[j], P.flo[j], P.fhi[j], (cb >> 2) & 3u, mu_f, CD::CH0 + CD::CHS * j + 2);
                    nb |= (r & 3u) << 2; ab |= ((r >> 2) & 3u) << 2; kb |= ((r >> 4) & 3u) << 2;
                    const TpmInterval Mf = TpmInterval::row((r >> 2) & 1u, (r >> 3) & 1u);
                    M.lo += Mf.lo; M.hi += Mf.hi;
                    vfirst[j] = stage_v(u - rold, mu_f, P.irhof[j], (cb >> 2) & 3u, r, P.flo[j], P.fhi[j]) + rold;   // the row is u_0[j] itself against bounds shifted by u_-1[j]
                }
                if (k > 0 || j > 0) {
                    r = hard_row(u - prev, P.clo_m[j], P.chi_p[j], P.clo[j], P.chi[j], (cb >> 4) & 3u, mu_c, CD::CH0 + CD::CHS * j + 4);
                    nb |= (r & 3u) << 4; ab |= ((r >> 2) & 3u) << 4; kb |= ((r >> 4) & 3u) << 4;
                    W.st(base + 2 * j + 1, stage_v(u - prev, mu_c, P.irhoc[j], (cb >> 4) & 3u, r, P.clo[j], P.chi[j]));
                    // violated although both of its scalars are held by other rows: two anchors in one run.  Next resolution lets this row
                    // pin the scalar whose anchor carries the smaller multiplier (hint bits 8 / 9 of the channel field)
                    if (((r >> 6) & 1u) && !carry_on && tau != TPM_CHAIN && tau != TPM_FREE && prev_tau != TPM_FREE && prev_tau != TPM_HELD) {
                        if (prev_mag <= fabs(tot)) {
                            if (j > 0) ncode |= 1ull << (CD::CH0 + CD::CHS * (j - 1) + 9);
                            else C(k - 1) |= 1ull << (CD::CH0 + CD::CHS * (nu - 1) + 9);
                        } else nb |= 1u << 8;
                    }
                    // close the previous scalar: gamma_{t-1} = G_{t-1} - [this one forward chain-pinned] G_t
                    const double corr = (tau == TPM_CHAIN) ? lin : 0.0;
                    Y = meet(TpmInterval{pend.lo - corr, pend.hi - corr}, TpmInterval::row((r >> 2) & 1u, (r >> 3) & 1u));
                }
                const double G = (tau == TPM_FREE) ? 0.0 : lin;        // a free scalar's row is its feedback law: gradient zero
                pend.lo = Y.lo + M.lo + G; pend.hi = Y.hi + M.hi + G;
                if (k == Nc - 1 && j == nu - 1) {
                    const double mu_q = (tau == TPM_LAST) ? tot : 0.0;
                    r = hard_row(-u, P.clo_m[0], P.chi_p[0], P.clo[0], P.chi[0], (cb >> 6) & 3u, mu_q, CD::CH0 + CD::CHS * j + 6);     // bounds of channel nu-1 = those of the chain row ending at channel 0
                    nb |= (r & 3u) << 6; ab |= ((r >> 2) & 3u) << 6; kb |= ((r >> 4) & 3u) << 6;
                    vq = stage_v(-u, mu_q, P.irhoc[0], (cb >> 6) & 3u, r, P.clo[0], P.chi[0]);
                    (void)meet(pend, TpmInterval::row((r >> 2) & 1u, (r >> 3) & 1u));    // 0 = gamma + mu + y - mu_q
                }
                ncode |= (uint64_t)nb << (CD::CH0 + CD::CHS * j);
                acode |= (uint64_t)ab << (CD::CH0 + CD::CHS * j);
                kcode |= (uint64_t)kb << (CD::CH0 + CD::CHS * j);
                carry = tot; carry_on = (tau == TPM_BACK);              // y_{t+1} = dQ/du_t + y_t
                prev_tau = tau; prev_mag = fabs(tot);
            }
#pragma unroll
            for (int a = 0; a < nx; a++) if (S::b_nz(a, j)) s[a] = fma(P.Bd[a * nu + j], u, s[a]);
            s[io] = u;
        }
#pragma unroll
        for (int a = 0; a < nx; a++) {
            const int lab = tpm_xlabel<S>(code, a);
            const double zi = s[a];
            pbad |= (unsigned)(zi < P.xacc_lo[a][lab]) | (unsigned)(zi > P.xacc_hi[a][lab]);
            const uint64_t nu_ = zi > P.xhi_p[a], nd_ = zi < P.xlo_m[a];
            W.st(base + 2 * nu + a, fma(P.xcm[a][lab], zi - P.xbnd[a][lab], zi));
            ncode |= nu_ << (CD::XUP + a);
            ncode |= (nd_ & ~nu_ & 1ull) << (CD::XDN + a);
        }
        acode |= ncode & CD::XMASK; kcode |= ncode & CD::XMASK;
        C(k) = ncode; CB(k) = acode; CK(k) = kcode;
    }
    mumax = mnew;
    if (EX && (pbad | ibad)) {
        if (xk_add >= 0) C(xk_add) = (C(xk_add) & ~(3ull << xp_add)) | ((uint64_t)xl_add << xp_add);
        if (xk_drop >= 0) C(xk_drop) &= ~(3ull << xp_drop);
    }
    return (int)(pbad != 0u) | ((int)(ibad != 0u) << 1);                // 0: verified
}

// first working sets from an ADMM iterate v in the standard row order (x_0..x_N | u_0..u_{Nc-1} | first block | NU chain rows).
// shift = 1: v belongs to the PREVIOUS problem of a receding-horizon loop: stage k takes the rows of stage k + 1 (the first-block
// rows, which have no predecessor there, from the time difference u_1[j] - u_0[j] of the rows' primal parts)
template <class S, class PP, class VA, class CA>
BMPC_HD void tpm_codes_from_v(const PP& P, const double* um1, VA V, CA C, int shift = 0) {
    constexpr int nx = S::nx, nu = S::nu, Np = S::Np, Nc = S::Nc, NX = S::NX, NU = S::NU;
    using CD = TpmCode<S>;
    auto over = [](double v, double hi) { return v > hi + 1e-9 * (1.0 + fabs(hi)); };
    auto under = [](double v, double lo) { return v < lo - 1e-9 * (1.0 + fabs(lo)); };
#pragma unroll 1
    for (int k = 0; k < Np; k++) {
        const int ks = (k + shift < Np) ? k + shift : Np - 1, ku = (k + shift < Nc) ? k + shift : Nc - 1;
        uint64_t c = 0ull;
#pragma unroll
        for (int a = 0; a < nx; a++) {
            const double v = V((ks + 1) * nx + a);
            c |= (uint64_t)(over(v, P.xhi[a]) ? 1u : 0u) << (CD::XUP + a); c |= (uint64_t)(under(v, P.xlo[a]) ? 1u : 0u) << (CD::XDN + a);
        }
        if (k < Nc) {
#pragma unroll
            for (int j = 0; j < nu; j++) {
                unsigned b = 0u;
                const double vu = V(NX + ku * nu + j);
                b |= over(vu, P.uhi[j]) ? 1u : 0u; b |= under(vu, P.ulo[j]) ? 2u : 0u;
                if (k == 0) {
                    if (shift == 0) {
                        const double vf = V(NX + NU + j);
                        b |= over(vf, P.fhi[j] + um1[j]) ? 4u : 0u; b |= under(vf, P.flo[j] + um1[j]) ? 8u : 0u;
                    } else if (Nc > 1) {
                        // time difference of the previous plan, sharpened by the multipliers of the input rows' iterate
                        const double dv = V(NX + nu + j) - V(NX + j);
                        b |= (dv >= P.fhi[j] - 1e-9 * (1.0 + fabs(P.fhi[j]))) ? 4u : 0u; b |= (dv <= P.flo[j] + 1e-9 * (1.0 + fabs(P.flo[j]))) ? 8u : 0u;
                    }
                }
                const int i = ku * nu + j;                              // scalar index of the source sub-step
                if ((k > 0 || j > 0) && i >= 1) {
                    const double vc = V(NX + NU + nu + i - 1);
                    b |= over(vc, P.chi[j]) ? 16u : 0u; b |= under(vc, P.clo[j]) ? 32u : 0u;
                }
                if (k == Nc - 1 && j == nu - 1) {
                    const double vl = V(NX + NU + nu + NU - 1);
                    b |= over(vl, P.chi[0]) ? 64u : 0u; b |= under(vl, P.clo[0]) ? 128u : 0u;
                }
                c |= (uint64_t)b << (CD::CH0 + CD::CHS * j);
            }
        }
        C(k) = c;
    }
}

// first scalar of the horizon-anchored tail of a stored working set.  The end of a plan is shaped by the end of the horizon (the
// spurious last row -u_{Nc-1}[nu-1] within the delta-u box drags the last inputs down at the maximum rate): those labels stay where
// they are when the horizon recedes, the rest moves one stage.  Tail = the trailing block of stages that carry input-row labels,
// up to the last label-free stage (at most min(8, Nc/2) stages; a plan labelled throughout has only the run hanging on the last row as tail)
template <class S>
BMPC_HD int tpm_tail_start(const uint64_t* stored) {
    using CD = TpmCode<S>;
    constexpr int Nc = S::Nc, nu = S::nu, NU = S::NU;
    constexpr int LMAX = (Nc / 2 < 8) ? Nc / 2 : 8;
    int k = Nc - 1;
    while (k >= 0 && Nc - 1 - k < LMAX && (stored[k] & ~CD::XMASK) != 0ull) k--;
    if (k >= 0 && (stored[k] & ~CD::XMASK) == 0ull) return k * nu;     // the label-free stage stays label-free (nothing is shifted into it)
    if (((stored[Nc - 1] >> (CD::CH0 + CD::CHS * (nu - 1) + 6)) & 3ull) == 0ull) return NU;
    int i = NU - 1;
    while (i >= 1 && ((stored[i / nu] >> (CD::CH0 + CD::CHS * (i % nu) + 4)) & 3ull) != 0ull) i--;
    return i;
}

// receding-horizon shift of stored working sets (as tpi2_shifted_code): stage k takes the state, input and chain bits of stage
// k + 1, except for the scalars of the terminal run (index >= tail), which keep theirs; the first-block bits of stage 0 come from
// the caller (first: 2 bits per channel, from the previous plan's time difference)
template <class S>
BMPC_HD uint64_t tpm_shifted_code(const uint64_t* stored, int k, bool shift, const unsigned* first = nullptr, int tail = S::NU) {
    using CD = TpmCode<S>;
    constexpr int Np = S::Np, Nc = S::Nc, nu = S::nu;
    if (!shift) return stored[k];
    const int ks = (k + 1 < Np) ? k + 1 : Np - 1, ku = (k + 1 < Nc) ? k + 1 : Nc - 1;
    uint64_t c = stored[ks] & CD::XMASK;
    if (k < Nc) {
        for (int j = 0; j < nu; j++) {
            const uint64_t m = (uint64_t)0x33u << (CD::CH0 + CD::CHS * j);   // input and chain bits
            c |= ((k * nu + j >= tail) ? stored[k] : stored[ku]) & m;
        }
    }
    if (k == 0) {
        c &= ~((uint64_t)0x30u << CD::CH0);                             // sub-step (0, 0) has no chain row
        if (first) for (int j = 0; j < nu; j++) c |= (uint64_t)(first[j] & 3u) << (CD::CH0 + CD::CHS * j + 2);
    }
    if (k == Nc - 1) c |= stored[Nc - 1] & ((uint64_t)0xC0u << (CD::CH0 + CD::CHS * (nu - 1)));
    return c;
}

// first-block labels of the next problem's stage 0 from the plan U of this one: the time difference u_1[j] - u_0[j]
template <class S, class PP>
BMPC_HD unsigned tpm_first_label(const PP& P, int j, double u0j, double u1j) {
    const double dv = u1j - u0j, hi = P.fhi[j], lo = P.flo[j];
    return ((dv >= hi - 1e-9 * (1.0 + fabs(hi))) ? 1u : 0u) | ((dv <= lo + 1e-9 * (1.0 + fabs(lo))) ? 2u : 0u);
}

// standard-layout row of the v* value staged at (stage k, position p of the stage block) — the inverse of the staging above;
// -1: position unused at this stage
template <class S>
BMPC_HD int tpm_vstar_row(int k, int p) {
    constexpr int nx = S::nx, nu = S::nu, NX = S::NX, NU = S::NU, Nc = S::Nc;
    if (p >= 2 * nu) return (p < 2 * nu + nx) ? (k + 1) * nx + (p - 2 * nu) : -1;
    if (k >= Nc) return -1;
    const int j = p >> 1, i = k * nu + j;
    if ((p & 1) == 0) return NX + i;
    return (i >= 1) ? NX + NU + nu + i - 1 : -1;
}

// The parameters of one system; returns "QDu diagonal" (the sweeps need it).  Reads only the system's inputs (Ad .. uref) and
// scal[RHO], scal[RHOE], never the condensed arrays: the rows' bounds are the raw bounds (lo0 / hi0 copy them, periodic in nu) and a
// row's rho follows the condense's rule (bmpc_row_rho).  So the fill stays valid on a block whose condensed part predates its inputs
// (per-instance systems after bmpc_update_problem, k_fill_view) and gives bit for bit what a fill of the freshly condensed block gives.
template <class S>
BMPC_HOSTDEV bool tpm_fill(const double* sys, const BmpcSysOff& o, TpmParams<S>& P) {
    constexpr int nx = S::nx, nu = S::nu;
    bool diag = true;
    for (int i = 0; i < nx * nx; i++) { P.Ad[i] = sys[o.Ad + i]; P.Qx[i] = sys[o.Qx + i]; P.QxN[i] = sys[o.QxN + i]; }
    for (int i = 0; i < nx * nu; i++) P.Bd[i] = sys[o.Bd + i];
    for (int i = 0; i < nu; i++)
        for (int j = 0; j < nu; j++) { P.Qu[i * nu + j] = sys[o.Qu + i * nu + j]; if (i != j && sys[o.QDu + i * nu + j] != 0.0) diag = false; }
    for (int i = 0; i < nu; i++) {
        P.QDu[i] = sys[o.QDu + i * nu + i];
        double q = 0.0; for (int j = 0; j < nu; j++) q += sys[o.Qu + i * nu + j] * sys[o.uref + j]; P.quref[i] = q;
    }
    const double rho_e = sys[o.scal + BMPC_S_RHOE], rho = sys[o.scal + BMPC_S_RHO];
    auto tol = [](double b, double rel, double sgn) { return (fabs(b) > 1e300) ? b : b + sgn * rel * (1.0 + fabs(b)); };
    const double inf = 1.0 / 0.0;
    for (int a = 0; a < nx; a++) {
        const double lo = sys[o.xmin + a], hi = sys[o.xmax + a];          // the state rows of stage 1 (condensed rows nx + a)
        P.xlo[a] = lo; P.xhi[a] = hi; P.xlo_m[a] = tol(lo, 1e-11, -1.0); P.xhi_p[a] = tol(hi, 1e-11, 1.0);
        const double xlo_p = tol(lo, 1e-11, 1.0), xhi_m = tol(hi, 1e-11, -1.0), cx = rho_e / bmpc_row_rho(lo, hi, rho);
        const double al[4] = {P.xlo_m[a], xhi_m, -inf, -inf}, ah[4] = {P.xhi_p[a], inf, xlo_p, inf};
        const double m[4] = {0.0, rho_e, rho_e, 0.0}, bd[4] = {0.0, hi, lo, 0.0};
        for (int l = 0; l < 4; l++) {
            P.xacc_lo[a][l] = al[l]; P.xacc_hi[a][l] = ah[l]; P.xm[a][l] = m[l]; P.xbnd[a][l] = (fabs(bd[l]) > 1e300) ? 0.0 : bd[l];
            P.xmb[a][l] = m[l] * P.xbnd[a][l]; P.xcm[a][l] = (l == 1 || l == 2) ? cx : 0.0;
        }
    }
    for (int j = 0; j < nu; j++) {
        const int jc = (j + nu - 1) % nu;                               // channel whose bounds the chain row ending at j carries
        P.ulo[j] = sys[o.umin + j]; P.uhi[j] = sys[o.umax + j];        // input row (condensed row NX + j)
        P.flo[j] = sys[o.Dumin + j]; P.fhi[j] = sys[o.Dumax + j];      // first-block row (NX + NU + j)
        P.clo[j] = sys[o.Dumin + jc]; P.chi[j] = sys[o.Dumax + jc];    // chain row (NX + NU + nu + jc)
        P.ulo_m[j] = tol(P.ulo[j], 1e-9, -1.0); P.uhi_p[j] = tol(P.uhi[j], 1e-9, 1.0);
        P.flo_m[j] = tol(P.flo[j], 1e-9, -1.0); P.fhi_p[j] = tol(P.fhi[j], 1e-9, 1.0);
        P.clo_m[j] = tol(P.clo[j], 1e-9, -1.0); P.chi_p[j] = tol(P.chi[j], 1e-9, 1.0);
        P.irhou[j] = 1.0 / bmpc_row_rho(P.ulo[j], P.uhi[j], rho); P.irhof[j] = 1.0 / bmpc_row_rho(P.flo[j], P.fhi[j], rho);
        P.irhoc[j] = 1.0 / bmpc_row_rho(P.clo[j], P.chi[j], rho);
    }
    return diag;
}

// ------------------------------------------------------------------------------------------------
// Per-instance systems (n_sys = batch) on the multi-input fast path: one TpmParams<S> per instance in GLOBAL memory, field-major —
// double number f of instance i at pg[f * B + i] — so that a warp's 32 consecutive instances read a field with one coalesced access.
// TpmPolView offers the member names of TpmParams (P.Ad[i], P.xm[a][lab], P.ulo_m[j], ...), so the sweeps above compile unchanged
// against either.  Unlike TpiPolView it keeps no pointer per field: every field is addressed from the one base pointer and the
// stride, at an offset fixed at compile time (k_tpm_pol runs at the register limit; 30 field pointers would not fit beside it).
template <int OFF>
struct TpmVF { const double* p; size_t B; BMPC_HD double operator[](int i) const { return TpiGArr{p + (size_t)OFF * B, B}[i]; } };
template <int OFF>
struct TpmVF2 { const double* p; size_t B; BMPC_HD TpiGArr operator[](int a) const { return TpiGArr2{p + (size_t)OFF * B, B}[a]; } };
template <class S>
struct TpmPolView {
    using PS = TpmParams<S>;
    static constexpr int NF = (int)(sizeof(PS) / sizeof(double));
#define BMPC_TVF(m) TpmVF<(int)(offsetof(PS, m) / sizeof(double))> m
#define BMPC_TVF2(m) TpmVF2<(int)(offsetof(PS, m) / sizeof(double))> m
    BMPC_TVF(Ad); BMPC_TVF(Bd); BMPC_TVF(Qx); BMPC_TVF(QxN); BMPC_TVF(Qu); BMPC_TVF(QDu); BMPC_TVF(quref);
    BMPC_TVF(xlo); BMPC_TVF(xhi); BMPC_TVF(xlo_m); BMPC_TVF(xhi_p);
    BMPC_TVF2(xacc_lo); BMPC_TVF2(xacc_hi); BMPC_TVF2(xm); BMPC_TVF2(xmb); BMPC_TVF2(xcm); BMPC_TVF2(xbnd);
    BMPC_TVF(ulo); BMPC_TVF(uhi); BMPC_TVF(ulo_m); BMPC_TVF(uhi_p); BMPC_TVF(irhou);
    BMPC_TVF(flo); BMPC_TVF(fhi); BMPC_TVF(flo_m); BMPC_TVF(fhi_p); BMPC_TVF(irhof);
    BMPC_TVF(clo); BMPC_TVF(chi); BMPC_TVF(clo_m); BMPC_TVF(chi_p); BMPC_TVF(irhoc);
#undef BMPC_TVF
#undef BMPC_TVF2
    BMPC_HD TpmPolView(const double* p, size_t B)
        : Ad{p, B}, Bd{p, B}, Qx{p, B}, QxN{p, B}, Qu{p, B}, QDu{p, B}, quref{p, B}, xlo{p, B}, xhi{p, B}, xlo_m{p, B}, xhi_p{p, B},
          xacc_lo{p, B}, xacc_hi{p, B}, xm{p, B}, xmb{p, B}, xcm{p, B}, xbnd{p, B},
          ulo{p, B}, uhi{p, B}, ulo_m{p, B}, uhi_p{p, B}, irhou{p, B}, flo{p, B}, fhi{p, B}, flo_m{p, B}, fhi_p{p, B}, irhof{p, B},
          clo{p, B}, chi{p, B}, clo_m{p, B}, chi_p{p, B}, irhoc{p, B} {}
};
