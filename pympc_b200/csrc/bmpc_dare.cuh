// bmpc_dare.cuh — batched discrete algebraic Riccati equation (fp64), the design step of pyMPC.kalman
// (kalman_design / kalman_design_simple call control.dare, /root/reference/pyMPC/kalman.py:67, 96).
//
// Solves the control-form DARE with cross term (python-control's dare(A, B, Q, R, S), E = I)
//     X = A'XA - (A'XB + S)(R + B'XB)^-1 (B'XA + S') + Q,      G = (R + B'XB)^-1 (B'XA + S')
// for one instance, n <= 32 states, m <= 32 inputs, written once against the team abstraction of bmpc_core.cuh:
// WarpTeam on the device (k_dare: one warp per instance, lane = row), SeqTeam in the host emulation of the tests.
//
// Algorithm: structured doubling (SDA).  The cross term is eliminated first (A <- A - B R^-1 S', Q <- Q - S R^-1 S'), then
//     A_0 = A, G_0 = B R^-1 B', H_0 = Q,     W = I + G_k H_k,
//     A_{k+1} = A_k W^-1 A_k,   G_{k+1} = G_k + A_k W^-1 G_k A_k',   H_{k+1} = H_k + A_k' H_k W^-1 A_k
// with H and G symmetrised after every step; H_k -> X.  W is not symmetric: it is solved by Gauss-Jordan with partial pivoting.
// Acceptance: A_k is the closed-loop matrix raised to the power 2^k, so an instance is solved only when, within
// BMPC_DARE_MAX_STEPS doublings, both the relative change of X is below BMPC_DARE_TOL and ||A_k||_inf <= 1e-8 max(1, ||A_0||_inf):
// the decay certifies that X is the STABILISING solution.  Without it an unstable mode that neither B reaches nor Q sees
// converges in a few steps to a non-stabilising X.
#pragma once
#include "../../include/bmpc.h"   // BMPC_DARE_SOLVED, BMPC_DARE_NO_SOLUTION, BMPC_DARE_R_NOT_PD

enum { BMPC_DARE_MAX_STEPS = 64, BMPC_DARE_MAX_DIM = 32 };
#define BMPC_DARE_TOL 1e-14
#define BMPC_DARE_DECAY 1e-8

// Offsets (in doubles) inside one instance's workspace.  Odd leading dimensions keep a lane-per-row access free of bank conflicts.
// A, G, H live through the whole solve; the scratch area after them is reused by the three phases (set-up, doubling, gain).
struct BmpcDareLayout {
    int ldn, lda, ldb, ldm;
    int A, G, H;
    int aug, T;                      // doubling: [W | A_k | G_k] (n x 3n) and one n x n product
    int Ri, cb, rb, BRi, SRi;        // set-up: R^-1 (m x m, dense), two pivot buffers, B R^-1 and S R^-1 (n x m)
    int XB, aug2;                    // gain: X B (n x m) and [R + B'XB | B'XA + S'] (m x (m + n))
    int total;
};

BMPC_HOSTDEV BmpcDareLayout bmpc_dare_layout(int n, int m) {
    BmpcDareLayout l;
    l.ldn = n | 1; l.lda = (3 * n) | 1; l.ldb = m | 1; l.ldm = (m + n) | 1;
    l.A = 0; l.G = n * l.ldn; l.H = 2 * n * l.ldn;
    const int s0 = 3 * n * l.ldn;
    l.aug = s0; l.T = s0 + n * l.lda;
    l.Ri = s0; l.cb = l.Ri + m * m; l.rb = l.cb + m; l.BRi = l.rb + m; l.SRi = l.BRi + n * l.ldb;
    l.XB = s0; l.aug2 = s0 + n * l.ldb;
    int s = n * l.lda + n * l.ldn;
    if (m * m + 2 * m + 2 * n * l.ldb > s) s = m * m + 2 * m + 2 * n * l.ldb;
    if (n * l.ldb + m * l.ldm > s) s = n * l.ldb + m * l.ldm;
    l.total = (s0 + s + 1) & ~1;
    return l;
}

// In-place Gauss-Jordan with partial pivoting on the row-major block aug[rows x cols] (leading dimension ld): the first `rows`
// columns hold the (square) matrix, the columns after them the right-hand sides, which hold the solution afterwards.  The columns of
// the matrix itself are left partly reduced.  Returns false (the same on every lane) on a zero or non-finite pivot.
template <class Team>
BMPC_HD bool bmpc_gj_solve(Team& t, double* aug, int rows, int cols, int ld) {
    for (int k = 0; k < rows; k++) {
        double best = -1.0; int bi = rows;
        for (int i = k + t.tid; i < rows; i += t.n) {
            const double v = fabs(aug[i * ld + k]);
            if (v > best) { best = v; bi = i; }
        }
        const double gmax = t.max(best);
        if (!(gmax > 0.0) || !isfinite(gmax)) return false;
        const int p = (int)(-t.max(best == gmax && bi < rows ? -(double)bi : -1e9));   // lowest row index holding the maximum
        if (p != k) {
            for (int j = k + t.tid; j < cols; j += t.n) { const double a = aug[k * ld + j]; aug[k * ld + j] = aug[p * ld + j]; aug[p * ld + j] = a; }
            t.sync();
        }
        const double inv = 1.0 / aug[k * ld + k];
        for (int j = k + 1 + t.tid; j < cols; j += t.n) aug[k * ld + j] *= inv;
        t.sync();
        for (int i = t.tid; i < rows; i += t.n) {
            if (i == k) continue;
            const double f = aug[i * ld + k];
            if (f != 0.0)
                for (int j = k + 1; j < cols; j++) aug[i * ld + j] -= f * aug[k * ld + j];
        }
        t.sync();
    }
    return true;
}

// One instance.  A [n x n], B [n x m], Q [n x n], R [m x m], S [n x m] (nullptr: no cross term) are row-major inputs (global memory on
// the device); X [n x n] and G [m x n] receive the solution; ws holds bmpc_dare_layout(n, m).total doubles.  Returns the status
// (BMPC_DARE_*) and the number of doubling steps in `steps`; X and G are NaN when the status is not BMPC_DARE_SOLVED.
template <class Team>
BMPC_HD int bmpc_dare_solve(Team& t, int n, int m, const BmpcDareLayout& l, const double* A, const double* B, const double* Q,
                            const double* R, const double* S, double* X, double* G, double* ws, int& steps) {
    steps = 0;
    const int ldn = l.ldn, ldb = l.ldb;
    double *Ak = ws + l.A, *Gk = ws + l.G, *Hk = ws + l.H;
    // ---- set-up: R^-1 (its pivots are those of a Cholesky factorisation: all positive iff R is positive definite), then the
    // cross term is folded into A and Q
    double *Ri = ws + l.Ri, *BRi = ws + l.BRi, *SRi = ws + l.SRi;
    for (int e = t.tid; e < m * m; e += t.n) Ri[e] = R[e];
    t.sync();
    if (!bmpc_spd_inverse(t, Ri, m, ws + l.cb, ws + l.rb)) {
        for (int e = t.tid; e < n * n; e += t.n) X[e] = NAN;
        for (int e = t.tid; e < m * n; e += t.n) G[e] = NAN;
        return BMPC_DARE_R_NOT_PD;
    }
    for (int i = t.tid; i < n; i += t.n)
        for (int j = 0; j < m; j++) {
            double b = 0.0, s = 0.0;
            for (int k = 0; k < m; k++) { b += B[i * m + k] * Ri[k * m + j]; if (S) s += S[i * m + k] * Ri[k * m + j]; }
            BRi[i * ldb + j] = b; SRi[i * ldb + j] = s;
        }
    t.sync();
    double an0 = 0.0;
    for (int i = t.tid; i < n; i += t.n) {
        double rs = 0.0;
        for (int j = 0; j < n; j++) {
            double a = A[i * n + j], q = Q[i * n + j], g = 0.0;
            for (int k = 0; k < m; k++) {
                g += BRi[i * ldb + k] * B[j * m + k];
                if (S) { a -= BRi[i * ldb + k] * S[j * m + k]; q -= SRi[i * ldb + k] * S[j * m + k]; }
            }
            Ak[i * ldn + j] = a; Hk[i * ldn + j] = q; Gk[i * ldn + j] = g;
            rs += fabs(a);
        }
        an0 = rs > an0 ? rs : an0;
    }
    t.sync();
    const double decay = BMPC_DARE_DECAY * fmax(1.0, t.max(an0));
    auto symmetrise = [&](double* M) {
        for (int i = t.tid; i < n; i += t.n)
            for (int j = i + 1; j < n; j++) { const double v = 0.5 * (M[i * ldn + j] + M[j * ldn + i]); M[i * ldn + j] = v; M[j * ldn + i] = v; }
    };
    symmetrise(Gk); symmetrise(Hk);
    t.sync();
    // ---- doubling
    double *aug = ws + l.aug, *T = ws + l.T;
    const int lda = l.lda;
    int status = BMPC_DARE_NO_SOLUTION;
    for (int k = 0; k < BMPC_DARE_MAX_STEPS; k++) {
        for (int i = t.tid; i < n; i += t.n)
            for (int j = 0; j < n; j++) {
                double w = i == j ? 1.0 : 0.0;
                for (int c = 0; c < n; c++) w += Gk[i * ldn + c] * Hk[c * ldn + j];
                aug[i * lda + j] = w; aug[i * lda + n + j] = Ak[i * ldn + j]; aug[i * lda + 2 * n + j] = Gk[i * ldn + j];
            }
        t.sync();
        if (!bmpc_gj_solve(t, aug, n, 3 * n, lda)) break;            // Y1 = W^-1 A_k in columns [n, 2n), Y2 = W^-1 G_k in [2n, 3n)
        steps = k + 1;
        for (int i = t.tid; i < n; i += t.n)                         // T = A_k Y2
            for (int j = 0; j < n; j++) { double s = 0.0; for (int c = 0; c < n; c++) s += Ak[i * ldn + c] * aug[c * lda + 2 * n + j]; T[i * ldn + j] = s; }
        t.sync();
        for (int i = t.tid; i < n; i += t.n)                         // G += T A_k'
            for (int j = 0; j < n; j++) { double s = 0.0; for (int c = 0; c < n; c++) s += T[i * ldn + c] * Ak[j * ldn + c]; Gk[i * ldn + j] += s; }
        t.sync();
        for (int i = t.tid; i < n; i += t.n)                         // T = H_k Y1
            for (int j = 0; j < n; j++) { double s = 0.0; for (int c = 0; c < n; c++) s += Hk[i * ldn + c] * aug[c * lda + n + j]; T[i * ldn + j] = s; }
        t.sync();
        double dmax = 0.0, hmax = 0.0;
        for (int i = t.tid; i < n; i += t.n)                         // H += A_k' T
            for (int j = 0; j < n; j++) {
                double s = 0.0; for (int c = 0; c < n; c++) s += Ak[c * ldn + i] * T[c * ldn + j];
                const double h = Hk[i * ldn + j] + s;
                Hk[i * ldn + j] = h;
                dmax = fmax(dmax, fabs(s)); hmax = fmax(hmax, fabs(h));
                if (!isfinite(h)) dmax = INFINITY;
            }
        t.sync();
        for (int i = t.tid; i < n; i += t.n)                         // T = A_k Y1 = A_{k+1}
            for (int j = 0; j < n; j++) { double s = 0.0; for (int c = 0; c < n; c++) s += Ak[i * ldn + c] * aug[c * lda + n + j]; T[i * ldn + j] = s; }
        t.sync();
        double an = 0.0;
        for (int i = t.tid; i < n; i += t.n) {
            double rs = 0.0;
            for (int j = 0; j < n; j++) { Ak[i * ldn + j] = T[i * ldn + j]; rs += fabs(T[i * ldn + j]); }
            an = isfinite(rs) ? fmax(an, rs) : INFINITY;
        }
        symmetrise(Gk); symmetrise(Hk);
        t.sync();
        const double dm = t.max(dmax), hm = t.max(hmax), am = t.max(an);
        if (!isfinite(dm) || !isfinite(am)) break;
        if (dm <= BMPC_DARE_TOL * hm && am <= decay) { status = BMPC_DARE_SOLVED; break; }
    }
    // ---- X and the gain G = (R + B'XB)^-1 (B'XA + S') from the ORIGINAL A, B, R, S
    if (status != BMPC_DARE_SOLVED) {
        for (int e = t.tid; e < n * n; e += t.n) X[e] = NAN;
        for (int e = t.tid; e < m * n; e += t.n) G[e] = NAN;
        return status;
    }
    double *XB = ws + l.XB, *aug2 = ws + l.aug2;
    const int ldm = l.ldm;
    for (int i = t.tid; i < n; i += t.n)
        for (int j = 0; j < m; j++) { double s = 0.0; for (int c = 0; c < n; c++) s += Hk[i * ldn + c] * B[c * m + j]; XB[i * ldb + j] = s; }
    t.sync();
    for (int i = t.tid; i < m; i += t.n) {
        for (int j = 0; j < m; j++) { double s = R[i * m + j]; for (int c = 0; c < n; c++) s += B[c * m + i] * XB[c * ldb + j]; aug2[i * ldm + j] = s; }
        for (int j = 0; j < n; j++) {
            double s = S ? S[j * m + i] : 0.0;
            for (int c = 0; c < n; c++) s += XB[c * ldb + i] * A[c * n + j];
            aug2[i * ldm + m + j] = s;
        }
    }
    t.sync();
    if (!bmpc_gj_solve(t, aug2, m, m + n, ldm)) {
        for (int e = t.tid; e < n * n; e += t.n) X[e] = NAN;
        for (int e = t.tid; e < m * n; e += t.n) G[e] = NAN;
        return BMPC_DARE_NO_SOLUTION;
    }
    for (int e = t.tid; e < n * n; e += t.n) X[e] = Hk[(e / n) * ldn + e % n];
    for (int e = t.tid; e < m * n; e += t.n) G[e] = aug2[(e / n) * ldm + m + e % n];
    return BMPC_DARE_SOLVED;
}
