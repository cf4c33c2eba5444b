// bmpc_core.cuh — numerical core of the batched linear-MPC solver (fp64), written once against a
// "team" abstraction so that the same code runs as
//   * WarpTeam  : one warp per MPC instance (small problems: pendulum, point mass),
//   * BlockTeam : one CTA per MPC instance (large problems: MIMO nx=8,nu=4,Np=40),
//   * SeqTeam   : one host thread (tests/hostemu only — index-logic checks without a GPU; never
//                 linked into the product library).
//
// What is computed (reference: /root/reference/pyMPC/mpc.py; math: doc/latex/main.tex:535-671):
//   K1  condense   Ad^k, block-Toeplitz prediction matrix, H = B'P_X B + P_U, K = H + sigma I + A'RA,
//                  their inverses, and the dual operators A H^-1, A H^-1 A' used by the polish
//                  (replaces _compute_QP_matrices_, mpc.py:456-615, + OSQP setup)
//   K3  prep       per-step linear term g and affine offset cc from (x0, u_-1, xref)
//                  (replaces _update_QP_matrices_, mpc.py:386-454)
//   K4  admm       OSQP-form ADMM iterations on the condensed QP with the slack block eliminated in
//                  closed form (soft box = prox of a squared distance)      (replaces OSQP.solve, mpc.py:369)
//   K5  polish     primal-dual active-set refinement with KKT verification -> exact minimiser
//
// The condensed problem has the SAME minimiser (u-block) as the QP the reference assembles:
//   variables U (NU = Nc*nu), rows z = A U + cc,  A = [Bcal ; I ; D]  (mc = NX + NU + (Nc+1)*nu rows)
//   rows [0,NX)      : predicted states x_k, SOFT box [xmin,xmax] with weight eps_feas  (mpc.py:555-559)
//   rows [NX,NX+NU)  : inputs, hard box [umin,umax]                                     (mpc.py:561-565)
//   rows [NX+NU,mc)  : the reference's "delta-u" rows, reproduced with its scalar-shift quirk (mpc.py:569-580)
#pragma once
#include <math.h>

#ifdef BMPC_HOSTEMU
#define BMPC_HD inline
#define BMPC_HOSTDEV inline
#else
#define BMPC_HD __device__ __forceinline__
#define BMPC_HOSTDEV __host__ __device__ __forceinline__
#endif

struct BmpcDims {
    int nx, nu, Np, Nc, NX, NU, ND, mc;
};

// Offsets (in doubles) of every array inside one system block.
struct BmpcSysOff {
    // inputs (copied from the host by bmpc_setup)
    int Ad, Bd, Qx, QxN, Qu, QDu, xmin, xmax, umin, umax, Dumin, Dumax, uref;
    // derived by the condense kernel
    int pw, Acal, Bcal, BcalT, PB, H, Hinv, K, Kinv, AHinv, M, Gx0, Gref, GrefFull, g0, lo0, hi0, rho, scal, KinvL;
    int total;
};

// scal[] slots
// adaptive-rho table: level l uses rho * 10^((l - BMPC_LEV0)/2) and its own K^-1 (OSQP refactors on a rho change; with shared
// matrices the factors for a fixed ladder are precomputed once instead)
enum { BMPC_NLEV = 11, BMPC_LEV0 = 2 };
// polish: active-set steps that update all rows at once before the hard rows switch to single exchanges
enum { BMPC_PDAS_FULL = 3 };
// the round policy of a solve (host code; bmpc_polish_steps: refinements allowed per Schur-form polish attempt), shared by everything
// that runs the core: the library's host loop and the host emulation
#include "bmpc_rounds.cuh"
BMPC_HOSTDEV double bmpc_level_factor(int l) {
    const double f[BMPC_NLEV] = {0.1, 0.31622776601683794, 1.0, 3.1622776601683795, 10.0, 31.622776601683793, 100.0,
                                 316.22776601683796, 1000.0, 3162.2776601683795, 10000.0};
    return f[l];
}

enum { BMPC_S_RHO = 0, BMPC_S_SIGMA, BMPC_S_ALPHA, BMPC_S_RHOE, BMPC_S_ERR, BMPC_S_TRH, BMPC_S_TRA, BMPC_S_COUNT = 8 };

BMPC_HOSTDEV BmpcDims bmpc_make_dims(int nx, int nu, int Np, int Nc) {
    BmpcDims d;
    d.nx = nx; d.nu = nu; d.Np = Np; d.Nc = Nc;
    d.NX = (Np + 1) * nx; d.NU = Nc * nu; d.ND = (Nc + 1) * nu; d.mc = d.NX + d.NU + d.ND;
    return d;
}

BMPC_HOSTDEV BmpcSysOff bmpc_make_off(const BmpcDims& d) {
    BmpcSysOff o; int p = 0;
#define BMPC_TAKE(f, cnt) o.f = p; p += (cnt)
    BMPC_TAKE(Ad, d.nx * d.nx); BMPC_TAKE(Bd, d.nx * d.nu); BMPC_TAKE(Qx, d.nx * d.nx); BMPC_TAKE(QxN, d.nx * d.nx);
    BMPC_TAKE(Qu, d.nu * d.nu); BMPC_TAKE(QDu, d.nu * d.nu);
    BMPC_TAKE(xmin, d.nx); BMPC_TAKE(xmax, d.nx); BMPC_TAKE(umin, d.nu); BMPC_TAKE(umax, d.nu);
    BMPC_TAKE(Dumin, d.nu); BMPC_TAKE(Dumax, d.nu); BMPC_TAKE(uref, d.nu);
    BMPC_TAKE(pw, (d.Np + 1) * d.nx * d.nx); BMPC_TAKE(Acal, d.NX * d.nx);
    BMPC_TAKE(Bcal, d.NX * d.NU); BMPC_TAKE(BcalT, d.NX * d.NU); BMPC_TAKE(PB, d.NX * d.NU);
    BMPC_TAKE(H, d.NU * d.NU); BMPC_TAKE(Hinv, d.NU * d.NU); BMPC_TAKE(K, d.NU * d.NU); BMPC_TAKE(Kinv, d.NU * d.NU);
    BMPC_TAKE(AHinv, d.mc * d.NU); BMPC_TAKE(M, d.mc * d.mc);
    BMPC_TAKE(Gx0, d.NU * d.nx); BMPC_TAKE(Gref, d.NU * d.nx); BMPC_TAKE(GrefFull, d.NU * d.NX); BMPC_TAKE(g0, d.NU);
    BMPC_TAKE(lo0, d.mc); BMPC_TAKE(hi0, d.mc); BMPC_TAKE(rho, d.mc); BMPC_TAKE(scal, BMPC_S_COUNT);
    BMPC_TAKE(KinvL, BMPC_NLEV * d.NU * d.NU);
#undef BMPC_TAKE
    o.total = (p + 1) & ~1;
    return o;
}

// ------------------------------------------------------------------------------------------------
// Sequential team (host emulation / one thread).  Warp and block teams live in bmpc_kernels.cu.
struct SeqTeam {
    int tid; int n;
    BMPC_HD SeqTeam() : tid(0), n(1) {}
    BMPC_HD void sync() {}
    BMPC_HD bool all(bool p) { return p; }
    BMPC_HD double max(double v) { return v; }
    BMPC_HD double sum(double v) { return v; }
    BMPC_HD int excl_scan(int f, int& total) { total = f; return 0; }
    // sub-team topology used by the row-parallel mat-vecs: rows go to warps, columns to lanes
    BMPC_HD int warp() const { return 0; }
    BMPC_HD int nwarps() const { return 1; }
    BMPC_HD int lane() const { return 0; }
    BMPC_HD int lanes() const { return 1; }
    BMPC_HD double wsum(double v) { return v; }
    BMPC_HD void wsync() {}
};

// y_r = sum_{c in [c0(r), c1(r))} M[r*ld + c] x[c]; rows striped over the team's warps, columns over the lanes of a
// warp (coalesced row reads, shuffle reduction); out(r, y_r) is called by lane 0 of the owning warp.
template <class Team, class C0, class C1, class Out>
BMPC_HD void bmpc_gemv(Team& t, const double* M, int ld, int nrows, const double* x, C0 c0, C1 c1, Out out) {
    for (int r = t.warp(); r < nrows; r += t.nwarps()) {
        const double* row = M + (size_t)r * ld;
        double a0 = 0.0, a1 = 0.0;
        int c = c0(r) + t.lane();
        const int ce = c1(r), st = t.lanes();
        for (; c + st < ce; c += 2 * st) { a0 += row[c] * x[c]; a1 += row[c + st] * x[c + st]; }
        if (c < ce) a0 += row[c] * x[c];
        const double acc = t.wsum(a0 + a1);
        if (t.lane() == 0) out(r, acc);
    }
}

// ------------------------------------------------------------------------------------------------
// Row helpers
// per-row rho of a constraint row with bounds [lo, hi]: rows with both bounds infinite get rho_min like OSQP, the others the
// scalar rho (bmpc_condense; the fast path's fill applies it to the raw bounds, tpi_fill_pol)
BMPC_HOSTDEV double bmpc_row_rho(double lo, double hi, double rho) {
    const bool free_row = (lo < -1e29) && (hi > 1e29);
    return free_row ? 1e-6 : rho;
}

BMPC_HD void bmpc_row_bounds(const BmpcDims& d, const double* lo0, const double* hi0, const double* um1, int i,
                             double& lo, double& hi) {
    lo = lo0[i]; hi = hi0[i];
    int r = i - (d.NX + d.NU);
    if (r >= 0 && r < d.nu) { lo += um1[r]; hi += um1[r]; }
}

// prox of the row function: hard box -> projection; soft box with weight rho_e -> pulled toward the bound
BMPC_HD double bmpc_prox(double v, double lo, double hi, bool soft, double rho, double rho_e) {
    if (v > hi) return soft ? (rho * v + rho_e * hi) / (rho + rho_e) : hi;
    if (v < lo) return soft ? (rho * v + rho_e * lo) / (rho + rho_e) : lo;
    return v;
}

// (A x)_i for the structured A = [Bcal ; I ; D]   (without the affine offset)
BMPC_HD double bmpc_Arow_dot(const BmpcDims& d, const double* BcalT, const double* x, int i) {
    if (i < d.NX) {
        int k = i / d.nx;
        int jend = (k < d.Nc ? k : d.Nc) * d.nu;          // block-lower-triangular: x_k depends on u_j, j < k
        double a0 = 0.0, a1 = 0.0;
        int a = 0;
        for (; a + 1 < jend; a += 2) { a0 += BcalT[a * d.NX + i] * x[a]; a1 += BcalT[(a + 1) * d.NX + i] * x[a + 1]; }
        if (a < jend) a0 += BcalT[a * d.NX + i] * x[a];
        return a0 + a1;
    }
    if (i < d.NX + d.NU) return x[i - d.NX];
    int r = i - d.NX - d.NU;
    if (r < d.nu) return x[r];
    int s = r - d.nu;
    return -x[s] + (s + 1 < d.NU ? x[s + 1] : 0.0);
}

// (A' w)_a
BMPC_HD double bmpc_ATcol_dot(const BmpcDims& d, const double* Bcal, const double* w, int a) {
    int j = a / d.nu;
    int i0 = (j + 1) * d.nx;                               // first state row that sees u_j
    double a0 = 0.0, a1 = 0.0;
    int i = i0;
    for (; i + 1 < d.NX; i += 2) { a0 += Bcal[i * d.NU + a] * w[i]; a1 += Bcal[(i + 1) * d.NU + a] * w[i + 1]; }
    if (i < d.NX) a0 += Bcal[i * d.NU + a] * w[i];
    const double* wd = w + d.NX + d.NU;
    double acc = a0 + a1 + w[d.NX + a];
    if (a < d.nu) acc += wd[a];
    acc -= wd[d.nu + a];
    if (a >= 1) acc += wd[d.nu + a - 1];
    return acc;
}

// ------------------------------------------------------------------------------------------------
// K1: condense one system.  `sys` points at the system block (inputs already filled in).
// In-place Gauss-Jordan inversion of an SPD matrix (no pivoting needed for SPD); returns false if a
// pivot is not positive.  Row/column k are staged in colbuf/rowbuf so the rank-1 update is race-free.
template <class Team>
BMPC_HD bool bmpc_spd_inverse(Team& t, double* A, int n, double* colbuf, double* rowbuf) {
    bool ok = true;
    for (int k = 0; k < n; k++) {
        double p = A[k * n + k];
        if (!(p > 0.0)) ok = false;
        double pinv = 1.0 / p;
        for (int i = t.tid; i < n; i += t.n) { colbuf[i] = A[i * n + k]; rowbuf[i] = A[k * n + i]; }
        t.sync();
        for (int idx = t.tid; idx < n * n; idx += t.n) {
            int i = idx / n, j = idx % n;
            double v;
            if (i == k && j == k) v = pinv;
            else if (i == k) v = rowbuf[j] * pinv;
            else if (j == k) v = -colbuf[i] * pinv;
            else v = A[idx] - colbuf[i] * rowbuf[j] * pinv;
            A[idx] = v;
        }
        t.sync();
    }
    return ok;
}

// rho_in <= 0 -> automatic rho = sqrt(trace(H) / trace(A'A))
template <class Team>
BMPC_HD void bmpc_condense(Team& t, const BmpcDims& d, const BmpcSysOff& o, double* sys, double rho_in, double sigma,
                           double alpha, double eps_feas, int soft_on) {
    const int nx = d.nx, nu = d.nu, Np = d.Np, Nc = d.Nc, NX = d.NX, NU = d.NU, mc = d.mc;
    const double *Ad = sys + o.Ad, *Bd = sys + o.Bd, *Qx = sys + o.Qx, *QxN = sys + o.QxN, *Qu = sys + o.Qu, *QDu = sys + o.QDu;
    double *pw = sys + o.pw, *Acal = sys + o.Acal, *Bcal = sys + o.Bcal, *BcalT = sys + o.BcalT, *PB = sys + o.PB;
    double *H = sys + o.H, *Hinv = sys + o.Hinv, *K = sys + o.K, *Kinv = sys + o.Kinv, *AHinv = sys + o.AHinv, *M = sys + o.M;
    double *Gx0 = sys + o.Gx0, *Gref = sys + o.Gref, *GrefFull = sys + o.GrefFull, *g0 = sys + o.g0;
    double *lo0 = sys + o.lo0, *hi0 = sys + o.hi0, *rhov = sys + o.rho, *scal = sys + o.scal;

    // powers of Ad: pw[k] = Ad^k, k = 0..Np
    for (int idx = t.tid; idx < nx * nx; idx += t.n) pw[idx] = (idx / nx == idx % nx) ? 1.0 : 0.0;
    t.sync();
    for (int k = 1; k <= Np; k++) {
        for (int idx = t.tid; idx < nx * nx; idx += t.n) {
            int r = idx / nx, c = idx % nx; double acc = 0.0;
            for (int q = 0; q < nx; q++) acc += Ad[r * nx + q] * pw[(k - 1) * nx * nx + q * nx + c];
            pw[k * nx * nx + idx] = acc;
        }
        t.sync();
    }
    // Acal = [I; Ad; ...; Ad^Np]
    for (int idx = t.tid; idx < NX * nx; idx += t.n) Acal[idx] = pw[idx];
    // Bcal[(k,a),(j,b)] = sum_{j' < k, min(j',Nc-1) = j} (Ad^(k-1-j') Bd)[a,b]      (mpc.py:537-544)
    for (int idx = t.tid; idx < NX * NU; idx += t.n) {
        int i = idx / NU, c = idx % NU;
        int k = i / nx, a = i % nx, j = c / nu, b = c % nu;
        double acc = 0.0;
        int jlo = j, jhi = (j == Nc - 1) ? (k - 1) : j;   // held input collects j' = Nc-1 .. k-1
        for (int jp = jlo; jp <= jhi && jp < k; jp++) {
            const double* P = pw + (k - 1 - jp) * nx * nx;
            for (int q = 0; q < nx; q++) acc += P[a * nx + q] * Bd[q * nu + b];
        }
        Bcal[idx] = acc; BcalT[c * NX + i] = acc;
    }
    t.sync();
    // PB = P_X Bcal  (P_X = blkdiag(Qx x Np, QxN), mpc.py:486-487)
    for (int idx = t.tid; idx < NX * NU; idx += t.n) {
        int i = idx / NU, c = idx % NU, k = i / nx, a = i % nx;
        const double* Q = (k < Np) ? Qx : QxN; double acc = 0.0;
        for (int q = 0; q < nx; q++) acc += Q[a * nx + q] * Bcal[(k * nx + q) * NU + c];
        PB[idx] = acc;
    }
    t.sync();
    // H = Bcal' PB + P_U ;  P_U = kron(diag(w), Qu) + kron(T, QDu)   (mpc.py:510-524)
    for (int idx = t.tid; idx < NU * NU; idx += t.n) {
        int r = idx / NU, c = idx % NU; double acc = 0.0;
        for (int i = 0; i < NX; i++) acc += BcalT[r * NX + i] * PB[i * NU + c];
        int jr = r / nu, br = r % nu, jc = c / nu, bc = c % nu;
        if (jr == jc) {
            double wq = (jr == Nc - 1) ? (double)(Np - Nc + 1) : 1.0;
            double tdiag = (jr == Nc - 1) ? 1.0 : 2.0;
            acc += wq * Qu[br * nu + bc] + tdiag * QDu[br * nu + bc];
        } else if (jr == jc + 1 || jc == jr + 1) {
            acc -= QDu[br * nu + bc];
        }
        H[idx] = acc;
    }
    t.sync();
    // symmetrise, copy
    for (int idx = t.tid; idx < NU * NU; idx += t.n) { int r = idx / NU, c = idx % NU; Hinv[idx] = 0.5 * (H[idx] + H[c * NU + r]); }
    t.sync();
    for (int idx = t.tid; idx < NU * NU; idx += t.n) H[idx] = Hinv[idx];
    t.sync();
    // traces for the automatic rho
    if (t.tid == 0) {
        double trH = 0.0, trA = 0.0;
        for (int a = 0; a < NU; a++) trH += H[a * NU + a];
        for (int idx = 0; idx < NX * NU; idx++) trA += Bcal[idx] * Bcal[idx];
        trA += (double)NU + (double)nu + 2.0 * (double)NU - 1.0;     // ||I||_F^2 + ||D||_F^2
        scal[BMPC_S_TRH] = trH; scal[BMPC_S_TRA] = trA;
        double rho = rho_in > 0.0 ? rho_in : sqrt(trH / trA);
        if (!(rho > 1e-6)) rho = 1e-6;
        if (rho > 1e6) rho = 1e6;
        scal[BMPC_S_RHO] = rho; scal[BMPC_S_SIGMA] = sigma; scal[BMPC_S_ALPHA] = alpha;
        scal[BMPC_S_RHOE] = soft_on ? eps_feas : 0.0; scal[BMPC_S_ERR] = 0.0;
    }
    t.sync();
    const double rho = scal[BMPC_S_RHO];
    // bounds and per-row rho (rows with both bounds infinite get rho_min like OSQP)
    for (int i = t.tid; i < mc; i += t.n) {
        double lo, hi;
        if (i < NX) { lo = sys[o.xmin + i % nx]; hi = sys[o.xmax + i % nx]; }
        else if (i < NX + NU) { lo = sys[o.umin + (i - NX) % nu]; hi = sys[o.umax + (i - NX) % nu]; }
        else { int r = i - NX - NU; lo = sys[o.Dumin + r % nu]; hi = sys[o.Dumax + r % nu]; }
        lo0[i] = lo; hi0[i] = hi;
        rhov[i] = bmpc_row_rho(lo, hi, rho);
    }
    t.sync();
    // K = H + sigma I + Bcal' Rx Bcal + Ru + D' Rd D
    for (int idx = t.tid; idx < NU * NU; idx += t.n) {
        int r = idx / NU, c = idx % NU;
        double acc = H[idx];
        for (int i = 0; i < NX; i++) acc += rhov[i] * BcalT[r * NX + i] * BcalT[c * NX + i];
        const double* rd = rhov + NX + NU;
        if (r == c) {
            acc += sigma + rhov[NX + r];
            if (r < nu) acc += rd[r];
            acc += rd[nu + r];                       // row nu+r has -1 at column r
            if (r >= 1) acc += rd[nu + r - 1];       // row nu+r-1 has +1 at column r
        } else if (c == r + 1) acc -= rd[nu + r];    // row nu+r: (-1 at r)(+1 at r+1)
        else if (r == c + 1) acc -= rd[nu + c];
        K[idx] = acc; Kinv[idx] = acc;
    }
    t.sync();
    // inverses (scratch: g0 / GrefFull are not yet in use)
    bool okH = bmpc_spd_inverse(t, Hinv, NU, GrefFull, GrefFull + NU);
    bool okK = bmpc_spd_inverse(t, Kinv, NU, GrefFull, GrefFull + NU);
    if (t.tid == 0 && !(okH && okK)) scal[BMPC_S_ERR] = okH ? 2.0 : 1.0;
    t.sync();
    // ladder of K^-1 for the adaptive rho: K_l = H + sigma I + f_l (K - H - sigma I)
    {
        double* KinvL = sys + o.KinvL;
        for (int l = 0; l < BMPC_NLEV; l++) {
            double* Kl = KinvL + (size_t)l * NU * NU;
            const double f = bmpc_level_factor(l);
            for (int idx = t.tid; idx < NU * NU; idx += t.n) {
                const double hs = H[idx] + ((idx / NU == idx % NU) ? sigma : 0.0);
                Kl[idx] = hs + f * (K[idx] - hs);
            }
            t.sync();
            bmpc_spd_inverse(t, Kl, NU, GrefFull, GrefFull + NU);
        }
    }
    // AHinv = A Hinv  (rows: Bcal Hinv ; Hinv ; D Hinv)
    for (int idx = t.tid; idx < mc * NU; idx += t.n) {
        int i = idx / NU, c = idx % NU; double acc = 0.0;
        if (i < NX) { for (int a = 0; a < NU; a++) acc += Bcal[i * NU + a] * Hinv[a * NU + c]; }
        else if (i < NX + NU) acc = Hinv[(i - NX) * NU + c];
        else {
            int r = i - NX - NU;
            if (r < nu) acc = Hinv[r * NU + c];
            else { int s = r - nu; acc = -Hinv[s * NU + c] + (s + 1 < NU ? Hinv[(s + 1) * NU + c] : 0.0); }
        }
        AHinv[idx] = acc;
    }
    t.sync();
    // M = AHinv A'
    for (int idx = t.tid; idx < mc * mc; idx += t.n) {
        int i = idx / mc, c = idx % mc; const double* row = AHinv + i * NU; double acc = 0.0;
        if (c < NX) { for (int a = 0; a < NU; a++) acc += row[a] * Bcal[c * NU + a]; }
        else if (c < NX + NU) acc = row[c - NX];
        else {
            int r = c - NX - NU;
            if (r < nu) acc = row[r];
            else { int s = r - nu; acc = -row[s] + (s + 1 < NU ? row[s + 1] : 0.0); }
        }
        M[idx] = acc;
    }
    // linear-term operators:  g = Gx0 x0 + Gref xref (or GrefFull vec(Xref)) + g0 + [-QDu u_-1 ; 0]
    for (int idx = t.tid; idx < NU * nx; idx += t.n) {
        int a = idx / nx, c = idx % nx; double acc = 0.0, accr = 0.0;
        for (int i = 0; i < NX; i++) { acc += PB[i * NU + a] * Acal[i * nx + c]; if (i % nx == c) accr -= PB[i * NU + a]; }
        Gx0[idx] = acc; Gref[idx] = accr;
    }
    for (int idx = t.tid; idx < NU * NX; idx += t.n) { int a = idx / NX, i = idx % NX; GrefFull[idx] = -PB[i * NU + a]; }
    for (int a = t.tid; a < NU; a += t.n) {
        int j = a / nu, b = a % nu; double wq = (j == Nc - 1) ? (double)(Np - Nc + 1) : 1.0, acc = 0.0;
        for (int q = 0; q < nu; q++) acc += Qu[b * nu + q] * sys[o.uref + q];
        g0[a] = -wq * acc;
    }
    t.sync();
}

// ------------------------------------------------------------------------------------------------
// K3: per-step data.  xref_mode 0: xref is (nx) ; 1: xref is ((Np+1)*nx) time-varying (mpc.py:414-421)
template <class Team>
BMPC_HD void bmpc_prep(Team& t, const BmpcDims& d, const BmpcSysOff& o, const double* sys, const double* x0,
                       const double* um1, const double* xref, int xref_mode, double* g, double* cc) {
    const double *Gx0 = sys + o.Gx0, *Gref = sys + o.Gref, *GrefFull = sys + o.GrefFull, *g0 = sys + o.g0, *QDu = sys + o.QDu;
    const double* Acal = sys + o.Acal;
    for (int a = t.tid; a < d.NU; a += t.n) {
        double acc = g0[a];
        for (int c = 0; c < d.nx; c++) acc += Gx0[a * d.nx + c] * x0[c];
        if (xref_mode == 0) { for (int c = 0; c < d.nx; c++) acc += Gref[a * d.nx + c] * xref[c]; }
        else { for (int i = 0; i < d.NX; i++) acc += GrefFull[a * d.NX + i] * xref[i]; }
        if (a < d.nu) { for (int q = 0; q < d.nu; q++) acc -= QDu[a * d.nu + q] * um1[q]; }
        g[a] = acc;
    }
    for (int i = t.tid; i < d.NX; i += t.n) {
        double acc = 0.0;
        for (int c = 0; c < d.nx; c++) acc += Acal[i * d.nx + c] * x0[c];
        cc[i] = acc;
    }
    t.sync();
}

// ------------------------------------------------------------------------------------------------
// K4: `niter` ADMM iterations in Douglas-Rachford form.  State: x (NU), v (mc) with z = prox(v),
// y = rho (v - z).  One iteration (equivalent to OSQP's Algorithm 1 with the KKT system reduced to
// (H + sigma I + A'RA) xt = sigma x - g + A'(rho z - y)):
//     z  = prox(v);  w = rho (2 z - v - cc)
//     xt = Kinv (sigma x - g + A' w);  zt = A xt + cc
//     x += alpha (xt - x);  v += alpha (zt - z)
// On return res[0] = ||zt - z||_inf, res[1] = ||sigma (xt-x) + A' rho (zt - z)||_inf of the LAST
// iteration, res[2], res[3] = the OSQP normalisers max(||zt||,||z||), max(||H xt||,||A'y||,||g||).
// ---- variant 1 (one warp per instance): lanes own rows / columns, mat-vec loops run along the other dimension ----
template <class Team>
BMPC_HD void bmpc_admm_lanes(Team& t, const BmpcDims& d, const BmpcSysOff& o, const double* sys, const double* um1,
                       const double* g, const double* cc, double* x, double* v, double* w, double* xt, double* r,
                       int niter, double* res, int lvl) {
    const double *Bcal = sys + o.Bcal, *BcalT = sys + o.BcalT, *Kinv = sys + o.KinvL + (size_t)lvl * d.NU * d.NU, *H = sys + o.H;
    const double *lo0 = sys + o.lo0, *hi0 = sys + o.hi0, *rhov = sys + o.rho, *scal = sys + o.scal;
    const double sigma = scal[BMPC_S_SIGMA], alpha = scal[BMPC_S_ALPHA], rho_e = scal[BMPC_S_RHOE];
    const double fac = bmpc_level_factor(lvl);
    const bool soft_on = rho_e > 0.0;
    const int NX = d.NX, NU = d.NU, mc = d.mc;
    double rp = 0.0, rd = 0.0, np_ = 0.0, nd_ = 0.0;
    for (int it = 0; it < niter; it++) {
        const bool last = (it == niter - 1);
        // A: rows
        for (int i = t.tid; i < mc; i += t.n) {
            double lo, hi; bmpc_row_bounds(d, lo0, hi0, um1, i, lo, hi);
            double vi = v[i], rho = fac * rhov[i];
            double z = bmpc_prox(vi, lo, hi, soft_on && i < NX, rho, rho_e);
            double ci = i < NX ? cc[i] : 0.0;
            w[i] = rho * (2.0 * z - vi - ci);
        }
        t.sync();
        // B: columns  r = sigma x - g + A' w
        for (int a = t.tid; a < NU; a += t.n) r[a] = sigma * x[a] - g[a] + bmpc_ATcol_dot(d, Bcal, w, a);
        t.sync();
        // C: columns  xt = Kinv r
        for (int a = t.tid; a < NU; a += t.n) {
            const double* row = Kinv + a * NU; double a0 = 0.0, a1 = 0.0; int b = 0;
            for (; b + 1 < NU; b += 2) { a0 += row[b] * r[b]; a1 += row[b + 1] * r[b + 1]; }
            if (b < NU) a0 += row[b] * r[b];
            xt[a] = a0 + a1;
        }
        t.sync();
        // D: rows  v += alpha (zt - z)   (w is reused for rho*(zt - z) on the last iteration)
        double lrp = 0.0, lnp = 0.0;
        for (int i = t.tid; i < mc; i += t.n) {
            double lo, hi; bmpc_row_bounds(d, lo0, hi0, um1, i, lo, hi);
            double vi = v[i], rho = fac * rhov[i];
            double z = bmpc_prox(vi, lo, hi, soft_on && i < NX, rho, rho_e);
            double zt = bmpc_Arow_dot(d, BcalT, xt, i) + (i < NX ? cc[i] : 0.0);
            double dz = zt - z;
            v[i] = vi + alpha * dz;
            if (last) {
                w[i] = rho * dz;
                lrp = fmax(lrp, fabs(dz)); lnp = fmax(lnp, fmax(fabs(zt), fabs(z)));
            }
        }
        if (last) {
            t.sync();
            // dual residual sigma dx + A' rho dz ; normaliser pieces ||H xt||, ||g||
            double lrd = 0.0, lnd = 0.0;
            for (int a = t.tid; a < NU; a += t.n) {
                double dx = xt[a] - x[a];
                lrd = fmax(lrd, fabs(sigma * dx + bmpc_ATcol_dot(d, Bcal, w, a)));
                const double* row = H + a * NU; double hx = 0.0;
                for (int b = 0; b < NU; b++) hx += row[b] * xt[b];
                lnd = fmax(lnd, fmax(fabs(hx), fabs(g[a])));
            }
            t.sync();
            // ||A'y|| with y = rho (v_new - prox(v_new))
            for (int i = t.tid; i < mc; i += t.n) {
                double lo, hi; bmpc_row_bounds(d, lo0, hi0, um1, i, lo, hi);
                double vi = v[i], rho = fac * rhov[i];
                w[i] = rho * (vi - bmpc_prox(vi, lo, hi, soft_on && i < NX, rho, rho_e));
            }
            t.sync();
            for (int a = t.tid; a < NU; a += t.n) lnd = fmax(lnd, fabs(bmpc_ATcol_dot(d, Bcal, w, a)));
            rp = t.max(lrp); np_ = t.max(lnp); rd = t.max(lrd); nd_ = t.max(lnd);
        }
        for (int a = t.tid; a < NU; a += t.n) x[a] += alpha * (xt[a] - x[a]);
        t.sync();
    }
    if (res && t.tid == 0) { res[0] = rp; res[1] = rd; res[2] = np_; res[3] = nd_; }
    t.sync();
}

// ---- variant 2 (one CTA per instance): rows striped over warps, columns over lanes, shuffle reductions ----
template <class Team>
BMPC_HD void bmpc_admm_rows(Team& t, const BmpcDims& d, const BmpcSysOff& o, const double* sys, const double* um1,
                       const double* g, const double* cc, double* x, double* v, double* w, double* xt, double* r,
                       int niter, double* res, int lvl) {
    const double *Bcal = sys + o.Bcal, *BcalT = sys + o.BcalT, *Kinv = sys + o.KinvL + (size_t)lvl * d.NU * d.NU, *H = sys + o.H;
    const double *lo0 = sys + o.lo0, *hi0 = sys + o.hi0, *rhov = sys + o.rho, *scal = sys + o.scal;
    const double sigma = scal[BMPC_S_SIGMA], alpha = scal[BMPC_S_ALPHA], rho_e = scal[BMPC_S_RHOE];
    const double fac = bmpc_level_factor(lvl);
    const bool soft_on = rho_e > 0.0;
    const int nx = d.nx, nu = d.nu, Nc = d.Nc, NX = d.NX, NU = d.NU, mc = d.mc;
    // (A' w)_a beyond the dense state block: input row + the reference's delta-u rows
    auto at_tail = [&](const double* ww, int a) {
        const double* wd = ww + NX + NU;
        double acc = ww[NX + a] - wd[nu + a];
        if (a < nu) acc += wd[a];
        if (a >= 1) acc += wd[nu + a - 1];
        return acc;
    };
    auto col0 = [&](int a) { return (a / nu + 1) * nx; };          // first state row that sees input a
    auto colN = [&](int) { return NX; };
    auto zero = [&](int) { return 0; };
    auto allU = [&](int) { return NU; };
    auto rowend = [&](int i) { int k = i / nx; return (k < Nc ? k : Nc) * nu; };   // x_k depends on u_j, j < k
    double rp = 0.0, rd = 0.0, np_ = 0.0, nd_ = 0.0;
    for (int it = 0; it < niter; it++) {
        const bool last = (it == niter - 1);
        // A: rows  w = rho (2 prox(v) - v - cc)
        for (int i = t.tid; i < mc; i += t.n) {
            double lo, hi; bmpc_row_bounds(d, lo0, hi0, um1, i, lo, hi);
            const double vi = v[i], rho = fac * rhov[i];
            const double z = bmpc_prox(vi, lo, hi, soft_on && i < NX, rho, rho_e);
            w[i] = rho * (2.0 * z - vi - (i < NX ? cc[i] : 0.0));
        }
        t.sync();
        // B: r = sigma x - g + A' w      (rows of B' striped over warps, lanes over the horizon)
        bmpc_gemv(t, BcalT, NX, NU, w, col0, colN, [&](int a, double acc) { r[a] = sigma * x[a] - g[a] + acc + at_tail(w, a); });
        t.sync();
        // C: xt = Kinv r
        bmpc_gemv(t, Kinv, NU, NU, r, zero, allU, [&](int a, double acc) { xt[a] = acc; });
        t.sync();
        // D1: zt on the state rows (kept in w, which is dead now)
        bmpc_gemv(t, Bcal, NU, NX, xt, zero, rowend, [&](int i, double acc) { w[i] = acc + cc[i]; });
        t.sync();
        // D2: rows  v += alpha (zt - prox(v))
        double lrp = 0.0, lnp = 0.0;
        for (int i = t.tid; i < mc; i += t.n) {
            double lo, hi; bmpc_row_bounds(d, lo0, hi0, um1, i, lo, hi);
            const double vi = v[i], rho = fac * rhov[i];
            const double z = bmpc_prox(vi, lo, hi, soft_on && i < NX, rho, rho_e);
            double zt;
            if (i < NX) zt = w[i];
            else if (i < NX + NU) zt = xt[i - NX];
            else {
                const int rr = i - NX - NU;
                if (rr < nu) zt = xt[rr];
                else { const int s2 = rr - nu; zt = -xt[s2] + (s2 + 1 < NU ? xt[s2 + 1] : 0.0); }
            }
            const double dz = zt - z;
            v[i] = vi + alpha * dz;
            if (last) { lrp = fmax(lrp, fabs(dz)); lnp = fmax(lnp, fmax(fabs(zt), fabs(z))); }
            if (last) w[i] = rho * dz;            // safe: every state row's zt was consumed by this same thread above
        }
        if (last) {
            t.sync();
            // OSQP residuals of the last iteration: r_prim = ||zt - z||, r_dual = ||sigma (xt - x) + A' rho (zt - z)||
            double lrd = 0.0, lnd = 0.0;
            bmpc_gemv(t, BcalT, NX, NU, w, col0, colN, [&](int a, double acc) { r[a] = sigma * (xt[a] - x[a]) + acc + at_tail(w, a); });
            t.sync();
            for (int a = t.tid; a < NU; a += t.n) { lrd = fmax(lrd, fabs(r[a])); lnd = fmax(lnd, fabs(g[a])); }
            t.sync();
            bmpc_gemv(t, H, NU, NU, xt, zero, allU, [&](int a, double acc) { r[a] = acc; });
            // y = rho (v_new - prox(v_new)) for ||A'y||
            for (int i = t.tid; i < mc; i += t.n) {
                double lo, hi; bmpc_row_bounds(d, lo0, hi0, um1, i, lo, hi);
                const double vi = v[i], rho = fac * rhov[i];
                w[i] = rho * (vi - bmpc_prox(vi, lo, hi, soft_on && i < NX, rho, rho_e));
            }
            t.sync();
            for (int a = t.tid; a < NU; a += t.n) lnd = fmax(lnd, fabs(r[a]));
            t.sync();
            bmpc_gemv(t, BcalT, NX, NU, w, col0, colN, [&](int a, double acc) { r[a] = acc + at_tail(w, a); });
            t.sync();
            for (int a = t.tid; a < NU; a += t.n) lnd = fmax(lnd, fabs(r[a]));
            rp = t.max(lrp); np_ = t.max(lnp); rd = t.max(lrd); nd_ = t.max(lnd);
        }
        for (int a = t.tid; a < NU; a += t.n) x[a] += alpha * (xt[a] - x[a]);
        t.sync();
    }
    if (res && t.tid == 0) { res[0] = rp; res[1] = rd; res[2] = np_; res[3] = nd_; }
    t.sync();
}

// dispatcher: a lone warp is better off with variant 1 (measured 5x), a CTA with variant 2
template <class Team>
BMPC_HD void bmpc_admm(Team& t, const BmpcDims& d, const BmpcSysOff& o, const double* sys, const double* um1,
                       const double* g, const double* cc, double* x, double* v, double* w, double* xt, double* r,
                       int niter, double* res, int lvl) {
    if (t.nwarps() > 1) bmpc_admm_rows(t, d, o, sys, um1, g, cc, x, v, w, xt, r, niter, res, lvl);
    else bmpc_admm_lanes(t, d, o, sys, um1, g, cc, x, v, w, xt, r, niter, res, lvl);
}

// OSQP's adaptive-rho rule (OSQP paper 5.2) on a fixed ladder: estimate rho sqrt((r_prim/n_prim)/(r_dual/n_dual)),
// move to the nearest ladder level if that is at least one decade away (OSQP's 5x test, coarsened), and rescale
// v = z + y/rho so that (z, y) are unchanged.  Returns the new level.
template <class Team>
BMPC_HD int bmpc_adapt_level(Team& t, const BmpcDims& d, const BmpcSysOff& o, const double* sys, const double* um1,
                             double* v, const double* res, int lvl) {
    const double rp = res[0] / fmax(res[2], 1e-12), rd = res[1] / fmax(res[3], 1e-12);
    int nl = lvl;
    if (rp > 0.0 && rd > 0.0) {
        const double steps = log10(rp / rd);               // sqrt(ratio) in half-decade steps = log10(ratio)
        int mv = (int)(steps >= 0.0 ? steps + 0.5 : steps - 0.5);
        if (mv >= 1 || mv <= -1) nl = lvl + mv;
        if (nl < 0) nl = 0;
        if (nl > BMPC_NLEV - 1) nl = BMPC_NLEV - 1;
    }
    if (nl != lvl) {
        const double *lo0 = sys + o.lo0, *hi0 = sys + o.hi0, *rhov = sys + o.rho;
        const double rho_e = sys[o.scal + BMPC_S_RHOE];
        const bool soft_on = rho_e > 0.0;
        const double fo = bmpc_level_factor(lvl), ratio = fo / bmpc_level_factor(nl);
        for (int i = t.tid; i < d.mc; i += t.n) {
            double lo, hi; bmpc_row_bounds(d, lo0, hi0, um1, i, lo, hi);
            const double vi = v[i];
            const double z = bmpc_prox(vi, lo, hi, soft_on && i < d.NX, fo * rhov[i], rho_e);
            v[i] = z + (vi - z) * ratio;
        }
        t.sync();
    }
    return nl;
}

// ------------------------------------------------------------------------------------------------
// What to do with a polish candidate that did not verify (the active-set iteration cycles on degenerate vertices).
// Its multipliers are still worth a lot to ADMM when a soft row is strongly violated: the row's multiplier eps_feas * d
// would otherwise be built in steps of rho * residual (eps_feas * d / rho iterations; the reference's OSQP path, with
// explicit slack and equilibration, needs ~700).  Policy (DESIGN.md section 7, round-1 host study): take the candidate as
// the new ADMM state v = zz + mu / rho only if its hard rows are feasible to 1e-2 (relative) — a wild candidate is
// worse than the iterate it would replace.
template <class Team>
BMPC_HD bool bmpc_candidate_usable(Team& t, const BmpcDims& d, const BmpcSysOff& o, const double* sys, const double* um1,
                                   const double* zz, const double* murow) {
    const double *lo0 = sys + o.lo0, *hi0 = sys + o.hi0;
    const bool soft_on = sys[o.scal + BMPC_S_RHOE] > 0.0;
    bool ok = true;
    for (int i = t.tid; i < d.mc; i += t.n) {
        if (soft_on && i < d.NX) continue;
        double lo, hi; bmpc_row_bounds(d, lo0, hi0, um1, i, lo, hi);
        const double zi = zz[i];
        if (zi > hi + 1e-2 * (1.0 + fabs(hi)) || zi < lo - 1e-2 * (1.0 + fabs(lo)) || !(fabs(murow[i]) < 1e300)) ok = false;
    }
    return t.all(ok);
}
template <class Team>
BMPC_HD void bmpc_warm_from_candidate(Team& t, const BmpcDims& d, const BmpcSysOff& o, const double* sys, const double* zz,
                                      const double* murow, const double* U, double* x, double* v, int lvl) {
    const double* rhov = sys + o.rho; const double fac = bmpc_level_factor(lvl);
    for (int i = t.tid; i < d.mc; i += t.n) v[i] = zz[i] + murow[i] / (fac * rhov[i]);
    for (int a = t.tid; a < d.NU; a += t.n) x[a] = U[a];
    t.sync();
}
// ADMM residuals far below any tolerance a caller can ask for: the iterate IS the solution to ~1e-8 even if the polish cannot
// certify it (degenerate vertex): stop iterating, status "solved" (unpolished).  res as written by bmpc_admm.  Only after 1600
// iterations (seven polish attempts): until then the instance keeps its chances of a KKT-verified answer — at 200 one instance
// of a 65 536 batch lost it.
BMPC_HD bool bmpc_residuals_tight(const double* res, int iters) {
    return iters >= 1600 && res[0] <= 1e-9 * (1.0 + res[2]) && res[1] <= 1e-9 * (1.0 + res[3]);
}
// ... and the candidate replaces the ADMM state only while ADMM itself is far from converged (relative primal residual above
// 1e-2 after at least 25 iterations: the slow-multiplier regime); an iteration that is converging is left alone — overwriting
// it round after round would throw its progress away.
BMPC_HD bool bmpc_admm_stalled(const double* res, int iters) {
    return iters >= 25 && res[0] > 1e-2 * fmax(res[2], 1e-12);
}

// ------------------------------------------------------------------------------------------------
// Primal infeasibility (OSQP paper 3.4) from two ADMM states (v0 on ladder level lvl0, v1 on lvl1) of the same problem:
// dy = y1 - y0 on the hard rows (soft rows are penalties, not constraints), projected on the polar of the recession cone
// of the row box like OSQP does; a certificate needs  ||A' dy|| < eps ||dy||  and a negative support function
// sum_i (hi_i - cc_i) dy_i^+ + (lo_i - cc_i) dy_i^-  < -eps ||dy||   (rows are z = A U + cc).  dy: mc doubles of scratch.
template <class Team>
BMPC_HD bool bmpc_primal_infeasible(Team& t, const BmpcDims& d, const BmpcSysOff& o, const double* sys, const double* um1,
                                    const double* cc, const double* v0, int lvl0, const double* v1, int lvl1, double* dy, double eps) {
    const double *lo0 = sys + o.lo0, *hi0 = sys + o.hi0, *rhov = sys + o.rho, *Bcal = sys + o.Bcal;
    const double rho_e = sys[o.scal + BMPC_S_RHOE];
    const bool soft_on = rho_e > 0.0;
    const double f0 = bmpc_level_factor(lvl0), f1 = bmpc_level_factor(lvl1);
    double ln = 0.0, ls = 0.0;
    for (int i = t.tid; i < d.mc; i += t.n) {
        double lo, hi; bmpc_row_bounds(d, lo0, hi0, um1, i, lo, hi);
        const bool soft = soft_on && i < d.NX;
        const double a0 = v0[i], a1 = v1[i], r0 = f0 * rhov[i], r1 = f1 * rhov[i];
        double dyi = soft ? 0.0 : r1 * (a1 - bmpc_prox(a1, lo, hi, false, r1, rho_e)) - r0 * (a0 - bmpc_prox(a0, lo, hi, false, r0, rho_e));
        if (hi > 1e29 && dyi > 0.0) dyi = 0.0;
        if (lo < -1e29 && dyi < 0.0) dyi = 0.0;
        dy[i] = dyi;
        ln = fmax(ln, fabs(dyi));
        const double ci = i < d.NX ? cc[i] : 0.0;
        ls += dyi > 0.0 ? (hi - ci) * dyi : (dyi < 0.0 ? (lo - ci) * dyi : 0.0);
    }
    const double ndy = t.max(ln);
    const double supp = t.sum(ls);
    if (!(ndy > 1e-30) || !(supp < -eps * ndy)) return false;      // uniform across the team
    t.sync();
    double la = 0.0;
    for (int a = t.tid; a < d.NU; a += t.n) la = fmax(la, fabs(bmpc_ATcol_dot(d, Bcal, dy, a)));
    return t.max(la) < eps * ndy;
}

// triangular solves with the packed unit-lower factor of S = L D L' (dv = 1/d_j), in place, by ONE warp (warp-level barriers
// only): L y = t, z = D^-1 y, L' mu = z
template <class Team>
BMPC_HD void bmpc_ldl_solve(Team& t, const double* S, const double* dv, double* tt, int r) {
    #define BMPC_TRI_(k, l) ((size_t)(k) * ((k) + 1) / 2 + (l))
    for (int j = 0; j < r; j++) {
        const double sj = dv[j] * tt[j];
        for (int i = j + 1 + t.lane(); i < r; i += t.lanes()) tt[i] -= S[BMPC_TRI_(i, j)] * sj;
        t.wsync();
    }
    for (int j = t.lane(); j < r; j += t.lanes()) tt[j] *= dv[j];
    t.wsync();
    for (int j = r - 1; j > 0; j--) {
        const double mj = tt[j];
        for (int i = t.lane(); i < j; i += t.lanes()) tt[i] -= S[BMPC_TRI_(j, i)] * dv[i] * mj;
        t.wsync();
    }
    #undef BMPC_TRI_
}

// ------------------------------------------------------------------------------------------------
// K5: polish.  Primal-dual active-set refinement on the condensed QP, in dual (Schur) form:
// with R the current set of "working" rows (violated soft rows + active hard rows, bound b_R),
//     S mu = A_R U0 + cc_R - b_R,   S = (A H^-1 A')[R,R] + diag(1/rho_e on soft rows, delta on hard rows)
//     U = U0 - H^-1 A_R' mu,        zz = A U + cc = W0 - (A H^-1 A')[:,R] mu
// where U0 = -H^-1 g and W0 = A U0 + cc.  A candidate is accepted only if it satisfies the KKT
// conditions of the condensed QP (primal feasibility of hard rows, multiplier signs, soft rows on the
// side their set says) — then it is THE minimiser.  Otherwise the sets are updated from the candidate
// (primal-dual active-set step) and the solve repeated, up to max_steps times.
// Returns the number of steps used (>0) on success, 0 if not verified, -1 if the working set outgrew rmax.
template <class Team>
BMPC_HD int bmpc_polish(Team& t, const BmpcDims& d, const BmpcSysOff& o, const double* sys, const double* um1,
                        const double* g, const double* cc, const double* v, double* W0, double* zz, double* murow,
                        int* st, double* S, double* tt, int* R, double* U0, double* U, int rmax, int max_steps) {
    const double *Hinv = sys + o.Hinv, *AHinv = sys + o.AHinv, *M = sys + o.M, *BcalT = sys + o.BcalT;
    const double *lo0 = sys + o.lo0, *hi0 = sys + o.hi0, *scal = sys + o.scal;
    const double rho_e = scal[BMPC_S_RHOE];
    const bool soft_on = rho_e > 0.0;
    const double inv_rho_e = soft_on ? 1.0 / rho_e : 0.0;
    const int NX = d.NX, NU = d.NU, mc = d.mc;
    // S is stored packed (lower triangle by rows): element (k,l), l <= k, at k(k+1)/2 + l
    #define BMPC_TRI(k, l) ((size_t)(k) * ((k) + 1) / 2 + (l))
    const double delta = 1e-13;

    // U0 = -H^-1 g (H^-1 symmetric: column reads are coalesced over a), W0 = A U0 + cc through the structured A
    for (int a = t.tid; a < NU; a += t.n) {
        const double* col = Hinv + a; double a0 = 0.0, a1 = 0.0; int b = 0;
        for (; b + 1 < NU; b += 2) { a0 += col[(size_t)b * NU] * g[b]; a1 += col[(size_t)(b + 1) * NU] * g[b + 1]; }
        if (b < NU) a0 += col[(size_t)b * NU] * g[b];
        U0[a] = -(a0 + a1);
    }
    t.sync();
    for (int i = t.tid; i < mc; i += t.n) {
        W0[i] = bmpc_Arow_dot(d, BcalT, U0, i) + ((i < NX) ? cc[i] : 0.0);
        double lo, hi; bmpc_row_bounds(d, lo0, hi0, um1, i, lo, hi);
        // rows sitting on a bound to rounding level (steady state at xref = xmax, say) stay out of the first guess
        st[i] = v[i] > hi + 1e-9 * (1.0 + fabs(hi)) ? 1 : (v[i] < lo - 1e-9 * (1.0 + fabs(lo)) ? 2 : 0);
    }
    t.sync();

    for (int step = 0; step < max_steps; step++) {
        // working set R (ordered compaction)
        int cnt = 0;
        for (int base = 0; base < mc; base += t.n) {
            int i = base + t.tid;
            int f = (i < mc && st[i] != 0) ? 1 : 0;
            int total; int pos = t.excl_scan(f, total);
            if (f && cnt + pos < rmax) R[cnt + pos] = i;
            cnt += total;
        }
        if (cnt > rmax) return -1;
        t.sync();
        const int r = cnt;
        double mumax = 0.0;
        if (r > 0) {
            for (int k = t.tid; k < r; k += t.n) {
                int i = R[k]; double lo, hi; bmpc_row_bounds(d, lo0, hi0, um1, i, lo, hi);
                tt[k] = W0[i] - (st[i] == 1 ? hi : lo);
            }
            for (int e = t.tid; e < r * (r + 1) / 2; e += t.n) {       // all threads share the r(r+1)/2 gathers
                int k = (int)((sqrt(8.0 * (double)e + 1.0) - 1.0) * 0.5);
                while ((k + 1) * (k + 2) / 2 <= e) k++;
                while (k * (k + 1) / 2 > e) k--;
                const int l = e - k * (k + 1) / 2;
                double val = M[(size_t)R[k] * mc + R[l]];
                if (k == l) val += (soft_on && R[k] < NX) ? inv_rho_e : delta * (1.0 + fabs(val));
                S[e] = val;
            }
            t.sync();
            // S = L D L' (unit lower L).  The pivot column is left untouched and its scale 1/d_j kept aside (dv), so a column
            // costs ONE barrier and one reciprocal (no square root, no scaling pass); rows go to warps, columns to lanes.
            double* dv = zz;                                   // zz is free until the candidate rows are formed
            for (int j = 0; j < r; j++) {
                double djj = S[BMPC_TRI(j, j)];
                if (!(djj > 1e-300)) djj = 1e-300;           // dependent working rows: candidate will fail verification
                const double dinv = 1.0 / djj;
                if (t.tid == 0) dv[j] = dinv;
                for (int i = j + 1 + t.warp(); i < r; i += t.nwarps()) {
                    const double lij = S[BMPC_TRI(i, j)] * dinv;
                    for (int k = j + 1 + t.lane(); k <= i; k += t.lanes()) S[BMPC_TRI(i, k)] -= lij * S[BMPC_TRI(k, j)];
                }
                t.sync();
            }
            // triangular solves by one warp (warp-level barriers only): L y = t, z = D^-1 y, L' mu = z
            if (t.warp() == 0) bmpc_ldl_solve(t, S, dv, tt, r);
            t.sync();
            // Large multipliers (a state far outside its soft box with a big eps_feas: mu ~ eps_feas * distance, balanced by the
            // active hard rows) make the hard-row regularisation visible: the candidate's active hard rows miss their bounds by
            // delta (1 + M_kk) mu_k (4e-8 at mu = 3e5) and fail the 1e-9 feasibility test although the working set is the right
            // one — 70 % of such instances then never verify.  One step of iterative refinement against the unregularised system
            // removes it: S e = Delta mu, mu += e.  Only when that miss comes near the tolerance: with ordinary multipliers the
            // correction is below rounding, and on dependent working rows (degenerate vertices) it would amplify the null-space
            // component the regularisation keeps small.
            double* mu0 = murow;                               // free until the multipliers are scattered below
            double lm0 = 0.0;
            for (int k = t.tid; k < r; k += t.n) {
                const int i = R[k]; const double m = tt[k];
                const double miss = (soft_on && i < NX) ? 0.0 : delta * (1.0 + fabs(M[(size_t)i * mc + i])) * m;
                mu0[k] = miss; lm0 = fmax(lm0, fabs(miss));
            }
            if (t.max(lm0) > 2e-10) {
                for (int k = t.tid; k < r; k += t.n) { const double m = tt[k]; tt[k] = mu0[k]; mu0[k] = m; }
                t.sync();
                if (t.warp() == 0) bmpc_ldl_solve(t, S, dv, tt, r);
                t.sync();
                for (int k = t.tid; k < r; k += t.n) tt[k] += mu0[k];
                t.sync();
            }
        }
        for (int i = t.tid; i < mc; i += t.n) murow[i] = 0.0;
        t.sync();
        double lm = 0.0;
        for (int k = t.tid; k < r; k += t.n) { murow[R[k]] = tt[k]; lm = fmax(lm, fabs(tt[k])); }
        mumax = t.max(lm);
        t.sync();
        // candidate: U = U0 - (A H^-1)[R,:]' mu (rows of A H^-1: coalesced), rows zz = A U + cc through the structured A
        // (BcalT read coalesced over the rows; an M[:,R] gather would touch one 32-byte sector per 8-byte entry)
        for (int a = t.tid; a < NU; a += t.n) {
            double acc = U0[a];
            for (int k = 0; k < r; k++) acc -= AHinv[R[k] * NU + a] * tt[k];
            U[a] = acc;
        }
        t.sync();
        for (int i = t.tid; i < mc; i += t.n) zz[i] = bmpc_Arow_dot(d, BcalT, U, i) + (i < NX ? cc[i] : 0.0);
        // verification + next sets.  The first BMPC_PDAS_FULL steps update every row at once (primal-dual active-set step: two or
        // three of them settle an ordinary solve).  That update can cycle when many hard rows are active at once; from then on the
        // soft-row labels still follow the candidate, but the hard rows change by single exchanges — per step the most violated
        // row enters and the row with the largest wrong-signed multiplier leaves — which does not cycle in practice (host study,
        // tools/soft_row_study.py: instances ending as max-iter 5 % -> 0.5 %, ADMM iterations per solve 553 -> 63).
        bool ok = true;
        const double mutol = 1e-9 * (1.0 + mumax);
        const bool exchange = step >= BMPC_PDAS_FULL;
        double best_add = -1.0, best_drop = -1.0; int i_add = -1, i_drop = -1, s_add = 0;
        for (int i = t.tid; i < mc; i += t.n) {
            double lo, hi; bmpc_row_bounds(d, lo0, hi0, um1, i, lo, hi);
            int s = st[i], ns; double zi = zz[i];
            if (soft_on && i < NX) {
                ns = zi > hi + 1e-11 * (1.0 + fabs(hi)) ? 1 : (zi < lo - 1e-11 * (1.0 + fabs(lo)) ? 2 : 0);
                if (ns != s) {
                    // tolerated only if the row sits on the boundary the two labels disagree about
                    bool same_hi = (s == 1 || ns == 1) && !(s == 2 || ns == 2);
                    bool same_lo = (s == 2 || ns == 2) && !(s == 1 || ns == 1);
                    double gap = same_hi ? fabs(zi - hi) : (same_lo ? fabs(zi - lo) : 1e300);
                    double bnd = same_hi ? hi : lo;
                    if (!(gap <= 1e-11 * (1.0 + fabs(bnd)))) ok = false;
                }
            } else {
                double mu = murow[i];
                bool vu = zi > hi + 1e-9 * (1.0 + fabs(hi));
                bool vd = zi < lo - 1e-9 * (1.0 + fabs(lo));
                bool bad = vu || vd || (s == 1 && mu < -mutol) || (s == 2 && mu > mutol);
                if (bad) ok = false;
                ns = vu ? 1 : (vd ? 2 : ((s == 1 && mu > 0.0) ? 1 : ((s == 2 && mu < 0.0) ? 2 : 0)));
                if (exchange && ns != s) {
                    if (ns == 0) { const double sc = fabs(mu); if (sc > best_drop) { best_drop = sc; i_drop = i; } }
                    else {
                        const double sc = fmax(zi - hi, lo - zi) / (1.0 + fmin(fabs(hi), fabs(lo)));
                        if (sc > best_add) { best_add = sc; i_add = i; s_add = ns; }
                    }
                    ns = s;
                }
            }
            st[i] = ns;
        }
        if (exchange) {
            const double g_add = t.max(best_add), g_drop = t.max(best_drop);
            if (i_add >= 0 && best_add == g_add) st[i_add] = s_add;
            if (i_drop >= 0 && best_drop == g_drop) st[i_drop] = 0;
        }
        ok = t.all(ok);
        t.sync();
        if (ok) return step + 1;
    }
    return 0;
}
