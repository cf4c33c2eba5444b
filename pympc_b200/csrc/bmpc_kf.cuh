// bmpc_kf.cuh — one step of the batched Kalman filter (fp64) for a model that may change between steps.
//
// The model of kalman_design_simple (/root/reference/pyMPC/kalman.py:73-106):
//     x+ = A x + B u + w,   E[ww'] = Qn (nx x nx);      y = C x + v,   E[vv'] = Rn (ny x ny);   no cross covariance.
// The filter holds the a-priori estimate x[k|k-1] and its covariance P, where the reference's LinearStateEstimator sits after
// its construction or predict:
//     predict(u):       x <- A x + B u;   P <- A P A' + Qn;   y <- C x
//     update(y_meas):   S = C P C' + Rn (Cholesky);   K = P C' S^-1;   x <- x + K (y_meas - y);
//                       P <- sym((I - K C) P (I - K C)' + K Rn K')      (Joseph form, then (X + X') / 2)
// y is refreshed by predict only, as in the reference (kalman.py:128).  With a constant model the recursion settles on the
// fixed point of dare(A', C', Qn, Rn), whose gain is kalman_design_simple(..., type='filter')'s L.
//
// One thread runs one instance (k_kf, k_kf_pi in bmpc.cu; the host emulation of the tests runs the same functions in a loop).
// P (packed upper triangle) and the intermediates live FIELD-major in global memory: element k of instance b at [k * B + b], so
// the threads of a warp touch consecutive doubles and no per-thread array sized by the largest dimension is needed (the driver
// reserves a stack frame for every resident thread).  x, y, u and y_meas are batch-major ([B, n]), the layout the controller reads.
// Only the addressing of the model differs between the shared model (packed, stride 1, k_kf holds it in shared memory) and the
// per-instance one (field-major, stride B, k_kf_pi): BmpcKfModel carries the model's names for both.
#pragma once
#include "bmpc_core.cuh"
#include "../../include/bmpc.h"   // BMPC_KF_OK, BMPC_KF_S_NOT_PD

enum { BMPC_KF_MAX_DIM = 32 };

// Offsets (in elements) of the model's fields and of one instance's workspace.
struct BmpcKfLayout {
    int A, B, C, Qn, Rn, model;      // model: A (nx x nx), B (nx x nu), C (ny x nx), Qn (nx x nx), Rn (ny x ny), row-major
    int P;                           // packed upper triangle of P: nx (nx + 1) / 2
    int M, T, K, KR, S, xn, ws;      // workspace: M = A P or I - K C, T = M P (nx x nx); K = P C' then the gain, KR = K Rn (nx x ny);
                                     // the factor of S (packed lower, ny (ny + 1) / 2); the new x (nx)
};

BMPC_HOSTDEV BmpcKfLayout bmpc_kf_layout(int nx, int nu, int ny) {
    BmpcKfLayout l;
    l.A = 0; l.B = nx * nx; l.C = l.B + nx * nu; l.Qn = l.C + ny * nx; l.Rn = l.Qn + nx * nx; l.model = l.Rn + ny * ny;
    l.P = nx * (nx + 1) / 2;
    l.M = 0; l.T = nx * nx; l.K = 2 * nx * nx; l.KR = l.K + nx * ny; l.S = l.KR + nx * ny; l.xn = l.S + ny * (ny + 1) / 2;
    l.ws = l.xn + nx;
    return l;
}

// one instance's view of a field-major array: element k at p[k * s]
struct BmpcKfCol {
    double* p; size_t s;
    BMPC_HD double& operator[](int k) const { return p[(size_t)k * s]; }
};

// one instance's model: PI = false packed (stride 1), PI = true field-major (stride s)
template <bool PI>
struct BmpcKfModel {
    const double* p; size_t s; int nx, nu, ny; BmpcKfLayout l;
    BMPC_HD double el(int e) const { return PI ? p[(size_t)e * s] : p[e]; }
    BMPC_HD double A(int i, int j) const { return el(l.A + i * nx + j); }
    BMPC_HD double B(int i, int j) const { return el(l.B + i * nu + j); }
    BMPC_HD double C(int i, int j) const { return el(l.C + i * nx + j); }
    BMPC_HD double Qn(int i, int j) const { return el(l.Qn + i * nx + j); }
    BMPC_HD double Rn(int i, int j) const { return el(l.Rn + i * ny + j); }
};

// index of P(i, j) in the packed upper triangle (row by row)
BMPC_HOSTDEV int bmpc_kf_pk(int n, int i, int j) {
    if (i > j) { const int t = i; i = j; j = t; }
    return i * n - i * (i - 1) / 2 + (j - i);
}

// predict(u): x <- A x + B u;  P <- A P A' + Qn (upper triangle of Qn);  y <- C x
template <class Mod>
BMPC_HD void bmpc_kf_predict(const Mod& m, const double* u, double* x, double* y, BmpcKfCol P, BmpcKfCol w) {
    const int nx = m.nx, nu = m.nu, ny = m.ny;
    const BmpcKfLayout& l = m.l;
    for (int i = 0; i < nx; i++) {
        double acc = 0.0;
        for (int j = 0; j < nx; j++) acc += m.A(i, j) * x[j];
        for (int j = 0; j < nu; j++) acc += m.B(i, j) * u[j];
        w[l.xn + i] = acc;
    }
    for (int i = 0; i < nx; i++) x[i] = w[l.xn + i];
    for (int i = 0; i < ny; i++) { double acc = 0.0; for (int j = 0; j < nx; j++) acc += m.C(i, j) * x[j]; y[i] = acc; }
    for (int i = 0; i < nx; i++)                                       // M = A P
        for (int j = 0; j < nx; j++) {
            double acc = 0.0;
            for (int k = 0; k < nx; k++) acc += m.A(i, k) * P[bmpc_kf_pk(nx, k, j)];
            w[l.M + i * nx + j] = acc;
        }
    for (int i = 0; i < nx; i++)                                       // P = M A' + Qn
        for (int j = i; j < nx; j++) {
            double acc = 0.0;
            for (int k = 0; k < nx; k++) acc += w[l.M + i * nx + k] * m.A(j, k);
            P[bmpc_kf_pk(nx, i, j)] = acc + m.Qn(i, j);
        }
}

// update(y_meas) with the y of the last predict.  Returns BMPC_KF_OK, or BMPC_KF_S_NOT_PD when a pivot of the Cholesky
// factorisation of S is not positive and finite: x and P are then left as they were.  Rn: the lower triangle forms S.
template <class Mod>
BMPC_HD int bmpc_kf_update(const Mod& m, const double* ym, double* x, const double* y, BmpcKfCol P, BmpcKfCol w) {
    const int nx = m.nx, ny = m.ny;
    const BmpcKfLayout& l = m.l;
    for (int i = 0; i < nx; i++)                                       // K = P C'
        for (int a = 0; a < ny; a++) {
            double acc = 0.0;
            for (int k = 0; k < nx; k++) acc += P[bmpc_kf_pk(nx, i, k)] * m.C(a, k);
            w[l.K + i * ny + a] = acc;
        }
    for (int i = 0; i < ny; i++)                                       // S = C P C' + Rn, lower triangle
        for (int j = 0; j <= i; j++) {
            double acc = 0.0;
            for (int k = 0; k < nx; k++) acc += m.C(i, k) * w[l.K + k * ny + j];
            w[l.S + i * (i + 1) / 2 + j] = acc + m.Rn(i, j);
        }
    for (int j = 0; j < ny; j++) {                                     // S = G G' in place
        double d = w[l.S + j * (j + 1) / 2 + j];
        for (int k = 0; k < j; k++) { const double g = w[l.S + j * (j + 1) / 2 + k]; d -= g * g; }
        if (!(d > 0.0) || !isfinite(d)) return BMPC_KF_S_NOT_PD;
        d = sqrt(d);
        w[l.S + j * (j + 1) / 2 + j] = d;
        for (int i = j + 1; i < ny; i++) {
            double s = w[l.S + i * (i + 1) / 2 + j];
            for (int k = 0; k < j; k++) s -= w[l.S + i * (i + 1) / 2 + k] * w[l.S + j * (j + 1) / 2 + k];
            w[l.S + i * (i + 1) / 2 + j] = s / d;
        }
    }
    for (int i = 0; i < nx; i++) {                                     // row i of K: S k' = (P C')_i'  (G z = ., then G' k' = z)
        for (int a = 0; a < ny; a++) {
            double s = w[l.K + i * ny + a];
            for (int b = 0; b < a; b++) s -= w[l.S + a * (a + 1) / 2 + b] * w[l.K + i * ny + b];
            w[l.K + i * ny + a] = s / w[l.S + a * (a + 1) / 2 + a];
        }
        for (int a = ny - 1; a >= 0; a--) {
            double s = w[l.K + i * ny + a];
            for (int b = a + 1; b < ny; b++) s -= w[l.S + b * (b + 1) / 2 + a] * w[l.K + i * ny + b];
            w[l.K + i * ny + a] = s / w[l.S + a * (a + 1) / 2 + a];
        }
    }
    for (int i = 0; i < nx; i++) {                                     // x <- x + K (y_meas - y)
        double acc = x[i];
        for (int a = 0; a < ny; a++) acc += w[l.K + i * ny + a] * (ym[a] - y[a]);
        x[i] = acc;
    }
    for (int i = 0; i < nx; i++)                                       // M = I - K C
        for (int j = 0; j < nx; j++) {
            double acc = i == j ? 1.0 : 0.0;
            for (int a = 0; a < ny; a++) acc -= w[l.K + i * ny + a] * m.C(a, j);
            w[l.M + i * nx + j] = acc;
        }
    for (int i = 0; i < nx; i++)                                       // T = M P
        for (int j = 0; j < nx; j++) {
            double acc = 0.0;
            for (int k = 0; k < nx; k++) acc += w[l.M + i * nx + k] * P[bmpc_kf_pk(nx, k, j)];
            w[l.T + i * nx + j] = acc;
        }
    for (int i = 0; i < nx; i++)                                       // KR = K Rn
        for (int a = 0; a < ny; a++) {
            double acc = 0.0;
            for (int b = 0; b < ny; b++) acc += w[l.K + i * ny + b] * m.Rn(b, a);
            w[l.KR + i * ny + a] = acc;
        }
    for (int i = 0; i < nx; i++)                                       // P = sym(T M' + KR K')
        for (int j = i; j < nx; j++) {
            double pij = 0.0, pji = 0.0;
            for (int k = 0; k < nx; k++) { pij += w[l.T + i * nx + k] * w[l.M + j * nx + k]; pji += w[l.T + j * nx + k] * w[l.M + i * nx + k]; }
            for (int a = 0; a < ny; a++) { pij += w[l.KR + i * ny + a] * w[l.K + j * ny + a]; pji += w[l.KR + j * ny + a] * w[l.K + i * ny + a]; }
            P[bmpc_kf_pk(nx, i, j)] = 0.5 * (pij + pji);
        }
    return BMPC_KF_OK;
}

// the per-instance step both kernels and the host emulation run: mode 0 = predict(in = u), 1 = update(in = y_meas)
template <class Mod>
BMPC_HD void bmpc_kf_step(const Mod& m, int b, int B, int mode, const double* in, double* x, double* y, double* P, double* ws,
                          int* status) {
    const BmpcKfCol Pc{P + b, (size_t)B}, wc{ws + b, (size_t)B};
    double* xb = x + (size_t)b * m.nx; double* yb = y + (size_t)b * m.ny;
    if (mode == 0) bmpc_kf_predict(m, in + (size_t)b * m.nu, xb, yb, Pc, wc);
    else status[b] = bmpc_kf_update(m, in + (size_t)b * m.ny, xb, yb, Pc, wc);
}
