// Host build of the fast path's parameter fill (TEST INFRASTRUCTURE ONLY): tpi_fill_pol of pympc_b200/csrc/bmpc_tpi.cuh compiled
// for the CPU, so that tests/test_tv_params_cpu.py can compare the parameter block of a stale system block with that of a freshly
// condensed one bit for bit.  Built by that test with g++; pympc_b200 never loads it.
#define BMPC_HOSTEMU 1
#include <stdlib.h>
#include <stdio.h>
#include <string.h>
#include "../../pympc_b200/csrc/bmpc_core.cuh"
#include "../../pympc_b200/csrc/bmpc_tpi.cuh"

// The polish parameter block (TpiPolParams<S> as doubles) of one system block; returns the number of doubles written (-100 shape
// not compiled here, -1 out too small).  For the in-tree single-input shapes (csrc/tpi_shapes.inc).
template <class S>
static int emu_tpi_fill_pol_t(const double* sys, double* out, int capacity) {
    constexpr int nf = (int)(sizeof(TpiPolParams<S>) / sizeof(double));
    if (capacity < nf) return -1;
    BmpcDims d = bmpc_make_dims(S::nx, S::nu, S::Np, S::Nc); BmpcSysOff o = bmpc_make_off(d);
    TpiPolParams<S>* P = new TpiPolParams<S>();
    tpi_fill_pol<S>(sys, o, *P);
    memcpy(out, P, sizeof(TpiPolParams<S>));
    delete P;
    return nf;
}

extern "C" int emu_tpi_fill_pol(int nx, int nu, int Np, int Nc, const double* sys, double* out, int capacity) {
    if (nx == 4 && nu == 1 && Np == 20 && Nc == 20) return emu_tpi_fill_pol_t<TpiShape<4, 1, 20, 20>>(sys, out, capacity);
    if (nx == 2 && nu == 1 && Np == 20 && Nc == 20) return emu_tpi_fill_pol_t<TpiShape<2, 1, 20, 20>>(sys, out, capacity);
    if (nx == 4 && nu == 1 && Np == 10 && Nc == 10) return emu_tpi_fill_pol_t<TpiShape<4, 1, 10, 10>>(sys, out, capacity);
    if (nx == 4 && nu == 1 && Np == 20 && Nc == 10) return emu_tpi_fill_pol_t<TpiShape<4, 1, 20, 10>>(sys, out, capacity);
    return -100;
}
