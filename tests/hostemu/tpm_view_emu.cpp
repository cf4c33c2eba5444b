// Host build of the multi-input fast path's parameter fill and sweeps (TEST INFRASTRUCTURE ONLY): tpm_fill and the sweeps of
// pympc_b200/csrc/bmpc_tpm.cuh compiled for the CPU against either parameter type — the TpmParams block the shared-system kernel
// reads from the constant bank, or the field-major TpmPolView of per-instance systems — so that tests/test_mimo_view_cpu.py can
// compare them bit for bit.  Built by that test with g++; pympc_b200 never loads it.
#define BMPC_HOSTEMU 1
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../../pympc_b200/csrc/bmpc_core.cuh"
#include "../../pympc_b200/csrc/bmpc_tpm.cuh"

// The in-tree entries (csrc/tpm_shapes.inc): 0 the MIMO reference governor's pattern, 1 dense (8,4,40,40), 2 dense (8,4,12,5)
using TpmE0 = TpmSparseShape<8, 4, 40, 40, 0x40c01030040c0103ull, 0x8040201u>;
using TpmE1 = TpiShape<8, 4, 40, 40>;
using TpmE2 = TpiShape<8, 4, 12, 5>;

// tpm_fill of one system block: the parameter block as doubles; returns the number written (-1 out too small), *diag "QDu diagonal"
template <class S>
static int fill_t(const double* sys, double* out, int capacity, int* diag) {
    constexpr int nf = TpmPolView<S>::NF;
    if (capacity < nf) return -1;
    BmpcDims d = bmpc_make_dims(S::nx, S::nu, S::Np, S::Nc); BmpcSysOff o = bmpc_make_off(d);
    TpmParams<S>* P = new TpmParams<S>();
    *diag = tpm_fill<S>(sys, o, *P) ? 1 : 0;
    memcpy(out, P, sizeof(TpmParams<S>));
    delete P;
    return nf;
}

// up to max_ref refinements (as hostemu.cpp's emu_tpm_run: mode 0 codes as stored, 1 shifted one stage — Uout holds the previous
// plan —, 2 from v; exchange_from >= 0: single-exchange refinements from that index on) against the parameters P of either type.
// codes [Np] in/out, v [mc] in/out, Uout [NU] in/out, mumax in/out; out: W column [slots] after the last refinement.  Returns
// the refinements used (> 0 verified, 0 not verified).
template <class S, bool TV, class PP>
static int run_t(const PP& P, const double* x0, const double* um1, const double* xref, uint64_t* codes, int mode, double* v, double* Uout,
                 int max_ref, double* mumax_io, int exchange_from, double* col) {
    using L = TpmLayout<S>;
    const TpiXref<S, TV> xr{xref};
    uint64_t cur[S::Np], atb[S::Np], keep[S::Np];
    TpiAcc W{col, 1};
    auto C = [&](int k) -> uint64_t& { return cur[k]; };
    auto CB = [&](int k) -> uint64_t& { return atb[k]; };
    auto CK = [&](int k) -> uint64_t& { return keep[k]; };
    if (mode >= 2) { TpiAcc V{v, 1}; tpm_codes_from_v<S>(P, um1, V, C, mode == 3); }
    else {
        unsigned first[S::nu];
        for (int j = 0; j < S::nu; j++) first[j] = (mode == 1 && S::Nc > 1) ? tpm_first_label<S>(P, j, Uout[j], Uout[S::nu + j]) : 0u;
        const int tail = tpm_tail_start<S>(codes);
        for (int k = 0; k < S::Np; k++) cur[k] = tpm_shifted_code<S>(codes, k, mode == 1, first, tail);
    }
    double mumax = *mumax_io, vfirst[S::nu], vq = 0.0, U[S::NU];
    int used = 0;
    for (int r = 0; r < max_ref; r++) {
        tpm_backward<S>(P, W, C, xr, um1);
        auto outu = [&](int k, int j, double u) { U[k * S::nu + j] = u; };
        const bool ex = exchange_from >= 0 && r >= exchange_from;
        const int fl = ex ? tpm_forward<S, true>(P, W, C, CB, CK, x0, um1, mumax, vfirst, vq, outu)
                          : tpm_forward<S, false>(P, W, C, CB, CK, x0, um1, mumax, vfirst, vq, outu);
        if (fl == 0) { used = r + 1; break; }
    }
    if (used > 0) {
        for (int k = 0; k < S::Np; k++)
            for (int p = 0; p < 2 * S::nu + S::nx; p++) { const int row = tpm_vstar_row<S>(k, p); if (row >= 0) v[row] = col[k * L::per_stage + p]; }
        for (int j = 0; j < S::nu; j++) v[S::NX + S::NU + j] = vfirst[j];
        v[S::mc - 1] = vq;
        for (int q = 0; q < S::nx; q++) v[q] = x0[q];
    }
    for (int j = 0; j < S::NU; j++) Uout[j] = U[j];                    // (the last candidate when not verified)
    for (int k = 0; k < S::Np; k++) codes[k] = (used > 0) ? atb[k] : cur[k];
    *mumax_io = mumax;
    return used;
}

// view = 0: the sweeps read the TpmParams block of sys; view = 1: they read a TpmPolView of a field-major array of B instances in
// which instance idx holds the same block and every other instance NaN
template <class S, bool TV>
static int step_t(int view, int B, int idx, const double* sys, const double* x0, const double* um1, const double* xref, uint64_t* codes,
                  int mode, double* v, double* Uout, int max_ref, double* mumax_io, int exchange_from, double* col) {
    BmpcDims d = bmpc_make_dims(S::nx, S::nu, S::Np, S::Nc); BmpcSysOff o = bmpc_make_off(d);
    TpmParams<S>* P = new TpmParams<S>();
    if (!tpm_fill<S>(sys, o, *P)) { delete P; return -101; }
    int rc;
    if (!view) rc = run_t<S, TV>(*P, x0, um1, xref, codes, mode, v, Uout, max_ref, mumax_io, exchange_from, col);
    else {
        constexpr int nf = TpmPolView<S>::NF;
        double* pg = (double*)malloc(sizeof(double) * (size_t)nf * B);
        for (size_t i = 0; i < (size_t)nf * B; i++) pg[i] = NAN;
        const double* src = (const double*)P;
        for (int f = 0; f < nf; f++) pg[(size_t)f * B + idx] = src[f];
        const TpmPolView<S> Pv(pg + idx, (size_t)B);
        rc = run_t<S, TV>(Pv, x0, um1, xref, codes, mode, v, Uout, max_ref, mumax_io, exchange_from, col);
        free(pg);
    }
    delete P;
    return rc;
}

#define TPM_ENTRY_SWITCH(CALL)                  \
    switch (entry) {                            \
    case 0: return CALL(TpmE0);                 \
    case 1: return CALL(TpmE1);                 \
    case 2: return CALL(TpmE2);                 \
    default: return -100;                       \
    }

extern "C" int emu_tpm_fill(int entry, const double* sys, double* out, int capacity, int* diag) {
#define FILL(S) fill_t<S>(sys, out, capacity, diag)
    TPM_ENTRY_SWITCH(FILL)
#undef FILL
}

extern "C" int emu_tpm_view_step(int entry, int view, int B, int idx, const double* sys, const double* x0, const double* um1,
                                 const double* xref, int xref_mode, uint64_t* codes, int mode, double* v, double* Uout, int max_ref,
                                 double* mumax_io, int exchange_from, double* col) {
#define STEP(S) (xref_mode ? step_t<S, true>(view, B, idx, sys, x0, um1, xref, codes, mode, v, Uout, max_ref, mumax_io, exchange_from, col) \
                           : step_t<S, false>(view, B, idx, sys, x0, um1, xref, codes, mode, v, Uout, max_ref, mumax_io, exchange_from, col))
    TPM_ENTRY_SWITCH(STEP)
#undef STEP
}

extern "C" int emu_tpm_slots(int entry) {
#define SLOTS(S) TpmLayout<S>::slots
    TPM_ENTRY_SWITCH(SLOTS)
#undef SLOTS
}
