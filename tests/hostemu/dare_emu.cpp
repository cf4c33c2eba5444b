// Host emulation of the batched DARE core (TEST INFRASTRUCTURE ONLY).
// Compiles pympc_b200/csrc/bmpc_dare.cuh for the CPU with the one-thread SeqTeam of bmpc_core.cuh, so that the structured-doubling
// algorithm and its acceptance rule can be checked against scipy without a GPU.  This is NOT a CPU fallback: pympc_b200 never
// loads this library; it lives under tests/ and is built by the tests.
#define BMPC_HOSTEMU 1
#include <math.h>
#include <stdlib.h>
#include <vector>
#include "../../pympc_b200/csrc/bmpc_core.cuh"
#include "../../pympc_b200/csrc/bmpc_dare.cuh"

extern "C" {

// same arguments and layout as bmpc_dare (include/bmpc.h), minus the device
void emu_dare(int n, int m, int batch, const double* A, const double* B, const double* Q, const double* R, const double* S,
              double* X, double* G, int* status, int* iters) {
    const BmpcDareLayout l = bmpc_dare_layout(n, m);
    std::vector<double> ws(l.total);
    const size_t nn = (size_t)n * n, nm = (size_t)n * m, mm = (size_t)m * m;
    for (int b = 0; b < batch; b++) {
        SeqTeam t;
        status[b] = bmpc_dare_solve(t, n, m, l, A + b * nn, B + b * nm, Q + b * nn, R + b * mm, S ? S + b * nm : nullptr,
                                    X + b * nn, G + b * nm, ws.data(), iters[b]);
    }
}

}
