// Host emulation of the batched Kalman filter step (TEST INFRASTRUCTURE ONLY).
// Compiles pympc_b200/csrc/bmpc_kf.cuh for the CPU and runs the per-instance step of k_kf / k_kf_pi over a batch, with the
// library's layouts: the model packed (shared) or field-major (per instance), P packed upper and field-major, the workspace
// field-major.  This is NOT a CPU fallback: pympc_b200 never loads this library; it lives under tests/ and is built by the tests.
#define BMPC_HOSTEMU 1
#include <math.h>
#include <vector>
#include "../../pympc_b200/csrc/bmpc_core.cuh"
#include "../../pympc_b200/csrc/bmpc_kf.cuh"

extern "C" {

int emu_kf_layout(int nx, int nu, int ny, int* out) {   // model, P and workspace sizes per instance
    const BmpcKfLayout l = bmpc_kf_layout(nx, nu, ny);
    out[0] = l.model; out[1] = l.P; out[2] = l.ws;
    return 0;
}

// one predict (mode 0, in = u [B,nu]) or update (mode 1, in = y_meas [B,ny]) over the batch.  mats: n_sys = 1 packed
// [A|B|C|Qn|Rn], n_sys = B field-major; x [B,nx], y [B,ny], P [l.P,B], ws [l.ws,B], status [B] as in the library.
void emu_kf_step(int nx, int nu, int ny, int B, int n_sys, int mode, const double* mats, const double* in, double* x, double* y,
                 double* P, double* ws, int* status) {
    const BmpcKfLayout l = bmpc_kf_layout(nx, nu, ny);
    for (int b = 0; b < B; b++) {
        if (n_sys == 1) bmpc_kf_step(BmpcKfModel<false>{mats, 1, nx, nu, ny, l}, b, B, mode, in, x, y, P, ws, status);
        else bmpc_kf_step(BmpcKfModel<true>{mats + b, (size_t)B, nx, nu, ny, l}, b, B, mode, in, x, y, P, ws, status);
    }
}

}
