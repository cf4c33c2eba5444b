/*
 * bmpc.h — C ABI of the H100-native batched linear-MPC solver (libbmpc.so).
 *
 * The reference (forgi86/pyMPC) has no FFI of its own: its hot path is the Python class
 * MPCController (/root/reference/pyMPC/mpc.py:27-615) driving the third-party OSQP object through
 * three calls (mpc.py:266 setup, :454 update, :369 solve) and slicing the result (mpc.py:301-304).
 * Each entry point below replaces one of those steps for a BATCH of B independent MPC instances
 * that live on one CUDA device; pympc_b200/mpc.py binds them with ctypes (see INTEGRATION.md).
 *
 * Conventions: plain pointers and sizes, row-major fp64, batch-major [B, ...]; every call returns 0
 * on success or a negative bmpc_error; the message is available from bmpc_last_error().  The
 * library owns all device state; callers own every buffer they pass.  HOST buffers handed to bmpc_update / bmpc_est_* are read by
 * an asynchronous copy queued on the handle's stream: leave them untouched until the next call that waits for the device
 * (bmpc_output to host memory, bmpc_synchronize, bmpc_get_*); pympc_b200.MPCController double-buffers its staging arrays.
 * One handle <-> one device + one stream; a handle is not thread-safe.
 */
#ifndef BMPC_H
#define BMPC_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct bmpc_handle bmpc_handle;

typedef enum {
    BMPC_OK = 0,
    BMPC_ERR_ARG = -1,        /* bad argument (reference: ValueError in MPCController.__init__, mpc.py:82-223) */
    BMPC_ERR_CUDA = -2,       /* CUDA runtime failure */
    BMPC_ERR_STATE = -3,      /* call order violated (e.g. solve before setup) */
    BMPC_ERR_NOT_PD = -4,     /* condensed Hessian not positive definite (QP not strictly convex in U) */
    BMPC_ERR_NO_DEVICE = -5   /* no usable CUDA device: there is NO CPU fallback */
} bmpc_error;

/* per-instance solver status written by bmpc_output (mirrors OSQP's status_val where it exists) */
enum {
    BMPC_SOLVED = 1,            /* KKT-verified minimiser (polished)            -> reference 'solved' */
    BMPC_SOLVED_UNPOLISHED = 2, /* ADMM met eps_abs/eps_rel (OSQP's criterion), polish not verified -> 'solved' */
    BMPC_PRIMAL_INFEASIBLE = -3, /* OSQP 'primal infeasible' (certificate found on the hard rows) -> reference falls back to u_failure */
    BMPC_MAX_ITER = -2,         /* OSQP 'maximum iterations reached'            -> reference falls back to u_failure */
    BMPC_UNSOLVED = -10
};

/* per-instance status written by bmpc_dare */
enum {
    BMPC_DARE_SOLVED = 1,       /* stabilising solution: X converged and the closed-loop powers decayed */
    BMPC_DARE_NO_SOLUTION = -1, /* no stabilising solution (64 doubling steps without convergence and decay, or a non-finite iterate) */
    BMPC_DARE_R_NOT_PD = -2     /* R is not positive definite */
};

typedef struct {
    int32_t nx, nu, Np, Nc;     /* Nc <= 0 means Nc = Np            (mpc.py:76-108) */
    int32_t batch;              /* instances on this device */
    int32_t device;             /* CUDA ordinal */
    int32_t soft_on;            /* SOFT_ON flag (mpc.py:237); 0 = hard state bounds */
    int32_t max_iter;           /* ADMM iteration cap per solve (OSQP default 4000) */
    int32_t first_iters;        /* ADMM iterations before the first polish attempt (0 = auto: none on a warm fast-path solve — the polish starts from the previous solution's working sets —, 25 on a cold one, 10 on the team kernels; later rounds reach 25, 50, 100, ... cumulative) */
    int32_t pdas_steps;         /* active-set refinements per polish attempt */
    int32_t rmax;               /* working-set capacity of the polish (0 = auto) */
    int32_t polish;             /* 1 = ADMM + polish (exact), 0 = pure ADMM to eps (OSQP-like) */
    int32_t team_threads;       /* 0 = auto; 32 = one warp per instance; >32 = one CTA of that size per instance */
    int32_t warps_per_block;    /* 0 = auto (warp team only) */
    int32_t fast_path;          /* 1 = use the thread-per-instance kernels when the shape has one (default), 0 = team kernels only */
    int32_t n_sys;              /* 1 = every instance shares (Ad,Bd,weights,bounds); batch = one system per instance (SURVEY 8f-3) */
    int32_t shift_warm;         /* 1 (default) = a warm fast-path solve starts from the previous working sets shifted by one stage (receding horizon: update() is one sample later); 0 = unshifted */
    int32_t candidate_warm;     /* 1 = an instance the polish could not verify AND whose ADMM is stalled (relative primal residual > 1e-2 after >= 25 iterations) continues its ADMM rounds from the last candidate (rows and multipliers) when that candidate's hard rows are feasible to 1e-2: the remedy for strongly violated soft rows with a large eps_feas (DESIGN.md section 7); 0 (default) = from its own ADMM state: on regular transients replacing the iterate costs a few instances their verification */
    int32_t cold_iters;         /* ADMM iterations before the first polish attempt of a COLD solve on the team / tile kernels (0 = auto: 50; 25 on multi-input fast-path shapes) */
    double eps_feas;            /* slack weight (mpc.py:226) */
    double rho;                 /* <= 0: automatic sqrt(trace H / trace A'A) */
    double sigma, alpha;        /* OSQP defaults 1e-6, 1.6 */
    double eps_abs, eps_rel;    /* OSQP termination tolerances (mpc.py:266) */
} bmpc_config;

typedef struct {
    int64_t admm_iters;         /* sum over instances of ADMM iterations in the last solve */
    int32_t rounds;             /* ADMM/polish rounds of the last solve */
    int32_t unsolved;           /* instances the polish never verified (status 2 or -2); -1 in pure-ADMM mode */
    int64_t polish_steps;       /* sum of active-set refinements */
    float ms_admm;              /* device time of the ADMM kernels in the last solve (CUDA events) */
    float ms_polish;            /* device time of the polish kernels */
    int32_t launches;           /* kernels launched by the last solve */
    int32_t infeasible;         /* instances certified primal infeasible (status -3) in the last solve */
    int32_t recondensed;        /* per-instance systems: condensed blocks the last solve brought up to date after bmpc_update_system */
} bmpc_stats;

void bmpc_default_config(bmpc_config* cfg);

/* replaces MPCController.__init__'s solver object creation (mpc.py:241) */
int bmpc_create(const bmpc_config* cfg, bmpc_handle** out);
void bmpc_destroy(bmpc_handle* h);
const char* bmpc_last_error(const bmpc_handle* h);   /* h may be NULL: error of the last failed bmpc_create */

/* replaces _compute_QP_matrices_ + OSQP.setup (mpc.py:254-269, 456-615): condense + factor on device (K1).
 * All pointers are HOST pointers; each array carries a leading n_sys dimension (n_sys = 1: one shared system).
 * BMPC_ERR_NOT_PD on a handle set up before: the handle holds the new arrays and bmpc_solve returns BMPC_ERR_STATE until a
 * successful bmpc_setup or update. */
int bmpc_setup(bmpc_handle* h, const double* Ad, const double* Bd, const double* Qx, const double* QxN,
               const double* Qu, const double* QDu, const double* xmin, const double* xmax, const double* umin,
               const double* umax, const double* Dumin, const double* Dumax, const double* uref);

/* replaces update()/_update_QP_matrices_/OSQP.update (mpc.py:338-364, 386-454).
 * x0 [B,nx]; uminus1 [B,nu] or NULL (keep: the previously committed output, quirk Q9);
 * xref [B,nx] (xref_rows = 1) or [B,Np+1,nx] (xref_rows = Np+1) or NULL (keep).
 * on_device = 1: the pointers are device pointers on this handle's device (copied, stream-ordered);
 * on_device = 2: device pointers that are BORROWED — the solver kernels read x0 / uminus1 in place, no copy; the caller leaves
 * them unchanged until the next solve has been retired (bmpc_output, bmpc_synchronize); xref is always copied. */
int bmpc_update(bmpc_handle* h, const double* x0, const double* uminus1, const double* xref, int xref_rows, int on_device);

/* time-varying system matrices (doc/latex/main.tex:505-511: with time-varying Ad and Bd the prediction matrices have to be
 * updated at every MPC iteration): replace (Ad, Bd) of every system of an already set-up handle; weights, bounds, uref and rho are unchanged.
 * Ad [n_sys,nx,nx], Bd [n_sys,nx,nu], row-major, batch-major; either may be NULL (keep).  on_device = 0: host pointers, 1: device
 * pointers on this handle's device (stream-ordered; the caller keeps them unchanged until the next solve has been retired).
 * A pending solve is retired first.  The warm-start state — working sets, v*, the per-instance rho level, the committed u_-1, the
 * cold/warm flag — is kept: the next bmpc_solve is a WARM solve of the QP the reference would assemble with the new matrices.
 * rho keeps the value the setup chose (the exact answer does not depend on it).
 * n_sys = 1: the system is condensed again at once and checked like bmpc_setup.  n_sys = batch: when P_X >= 0 and P_U > 0 (decided
 * at setup) H is positive definite for any (Ad, Bd) and each instance is condensed again only before the first launch that reads its
 * condensed block — a warm solve that the fast-path polish finishes alone condenses nothing; otherwise all instances at once.
 * BMPC_ERR_NOT_PD: bmpc_solve returns BMPC_ERR_STATE until a successful bmpc_update_system or bmpc_setup. */
int bmpc_update_system(bmpc_handle* h, const double* Ad, const double* Bd, int on_device);

/* time-varying problem data (gain scheduling, successive linearisation, derated actuator limits, tightened constraints): replace
 * any of the arrays of bmpc_setup of an already set-up handle without a new setup.  Arguments and layout as bmpc_setup's, each with
 * its leading n_sys dimension (n_sys = 1: one set shared by every instance; n_sys = batch: one set per instance); a NULL array keeps
 * its current value.  on_device = 0: host pointers, 1: device pointers on this handle's device (stream-ordered; the caller keeps
 * them unchanged until the next solve has been retired).  bmpc_update_system(h, Ad, Bd, d) is this call with the other arrays NULL.
 * A pending solve is retired first.  Kept: the working sets, v*, the per-instance rho level, the committed u_-1, the cold/warm flag
 * and the scalar rho the setup chose; the next bmpc_solve is a WARM solve of the QP the reference would assemble with the new arrays.
 * The per-row rho follows the setup's rule (rows with both bounds infinite: 1e-6): a row that changes between free and bounded
 * changes its rho, its K^-1 ladder and the fast path's row parameters.  The answer stays exact (it does not depend on rho); the
 * staged v* of such a row may be a poor warm start, which costs iterations only.  eps_feas, soft_on, the shapes and the solver
 * options stay as set up; u_failure (the output of an instance that fails) follows the new uref.
 * n_sys = 1: the system is condensed again at once and checked like bmpc_setup; the fast paths' constant-bank parameters are refilled
 * and the multi-input entry is chosen again (a QDu that stops being diagonal moves the handle to the team kernels).
 * n_sys = batch: the arrays go into every instance's block and the fast path's parameter view; each instance is condensed again only
 * before the first launch that reads its condensed block (a warm solve that the fast-path polish finishes alone condenses nothing).
 * New weights decide again whether H stays positive definite for any (Ad, Bd) (host weights: Qx, QxN, Qu, QDu >= 0 and Qu or
 * QDu > 0 on every instance); if not, or when the weights are device pointers, every instance is condensed at once and checked.
 * Bounds and uref never affect definiteness.
 * BMPC_ERR_NOT_PD: the handle holds the new arrays and bmpc_solve returns BMPC_ERR_STATE until a successful update or bmpc_setup. */
int bmpc_update_problem(bmpc_handle* h, const double* Ad, const double* Bd, const double* Qx, const double* QxN,
                        const double* Qu, const double* QDu, const double* xmin, const double* xmax, const double* umin,
                        const double* umax, const double* Dumin, const double* Dumax, const double* uref, int on_device);

/* replaces OSQP.solve (mpc.py:366-375): K3 + K4 + K5 */
int bmpc_solve(bmpc_handle* h);

/* replaces output() (mpc.py:271-336): u0 [B,nu] (u_failure = uref where status < 0), status [B] (nullable);
 * commit_uminus1 != 0 makes u0 the next uminus1 (mpc.py:330): every kernel that publishes u0 also writes a shadow copy, so the
 * commit is a pointer swap, not a copy. */
int bmpc_output(bmpc_handle* h, double* u0, int32_t* status, int commit_uminus1, int on_device);

/* optional info of output(): u_seq [B,Nc*nu], x_seq [B,(Np+1)*nx], eps_seq [B,(Np+1)*nx], obj_val [B]
 * (QP objective WITHOUT the reference's J_CNST), iters [B]; any pointer may be NULL.  Host pointers. */
int bmpc_get_sequences(bmpc_handle* h, double* u_seq, double* x_seq, double* eps_seq, double* obj_val, int32_t* iters);

/* let the polish epilogue write u0 straight into a caller-owned DEVICE buffer [B,nu]
 * (e.g. this rank's slice of an all-gather buffer); NULL restores the internal buffer. */
int bmpc_bind_output(bmpc_handle* h, double* dev_u0);
/* K6 fused: additionally store u0 into up to 8 PEER device buffers (each already offset to this rank's slice of the
 * peer's gathered [B_total, nu] buffer, e.g. torch symmetric-memory pointers): the epilogue's NVLink peer stores replace
 * the all-gather collective; the caller only needs a cross-rank barrier before reading.  n = 0 unbinds. */
int bmpc_bind_output_peers(bmpc_handle* h, double* const* peer_u0, int n);
/* K6 arrival: my_flags is this rank's DEVICE array of `world` int64 counters (zero-initialised), peer_flags[p] the same array
 * of peer p as mapped into this process (symmetric memory).  From then on every bmpc_solve is one arrival epoch (base_epoch + 1,
 * + 2, ...; all ranks solve in lockstep).  Arrival = store the epoch into slot `rank` of every peer's array and wait until every
 * peer's slot here holds a value >= epoch: then every peer's u* of this step has landed in the buffer bound with
 * bmpc_bind_output_peers.  A warm fast-path solve that finishes every instance does this in the last warp of the solver kernel
 * itself (no launch); otherwise bmpc_gather_arrive launches one small kernel behind the straggler rounds.  Call
 * bmpc_gather_arrive after bmpc_output in every step (it is a no-op when the kernel already arrived); its epoch argument is
 * ignored.  Rebinding (a new handle) continues at base_epoch = the number of solves the ranks have gathered so far.  Use two
 * gathered buffers alternately (step parity) so that the stores of step t+1 cannot overwrite data a slower peer is still
 * reading from step t. */
int bmpc_bind_gather_flags(bmpc_handle* h, int64_t* my_flags, int64_t* const* peer_flags, int n_peers, int rank, int world, int64_t base_epoch);
int bmpc_gather_arrive(bmpc_handle* h, int64_t epoch);
int bmpc_set_stream(bmpc_handle* h, void* cuda_stream);   /* NULL = handle-owned stream */
int bmpc_synchronize(bmpc_handle* h);

int bmpc_get_stats(bmpc_handle* h, bmpc_stats* out);
/* export one array of the condensed system for parity tests: name in {"Bcal","H","Hinv","K","Kinv","M","AHinv",
 * "Gx0","Gref","g0","lo0","hi0","rho","scal"}; out must hold `capacity` doubles; returns the element count. */
int bmpc_get_sys(bmpc_handle* h, const char* name, double* out, int capacity);
/* problem sizes: dims[0..7] = nx, nu, Np, Nc, NX, NU, mc, team_threads */
int bmpc_get_dims(const bmpc_handle* h, int32_t* dims);

/* ---- batched linear state estimator: the step on the INPUT side of the path (SURVEY.md 8f-4).
 * Replaces LinearStateEstimator.predict/update (/root/reference/pyMPC/kalman.py:109-134) for B instances sharing
 * (A,B,C,L):  predict  x <- A x + B u, y <- C x   (kalman.py:126-129);   update  x <- x + L (y_meas - y)  (:131-133).
 * The state lives on the device; bmpc_est_state_ptr() can be handed to bmpc_update(..., on_device=1) so the whole
 * control loop (estimate -> MPC -> plant input) stays on the GPU. */
typedef struct bmpc_estimator bmpc_estimator;
/* one (A,B,C,L) shared by every instance: bmpc_est_create_ex(..., n_sys = 1, ...) */
int bmpc_est_create(int32_t nx, int32_t nu, int32_t ny, int32_t batch, int32_t device, const double* A, const double* B,
                    const double* C, const double* L, const double* x0 /* [batch,nx] host */, bmpc_estimator** out);
/* n_sys = 1: shared (A,B,C,L); n_sys = batch: one system per instance, each array with a leading batch dimension (host pointers,
 * batch-major, row-major).  Per-instance systems run one thread per instance with the matrices in global memory. */
int bmpc_est_create_ex(int32_t nx, int32_t nu, int32_t ny, int32_t batch, int32_t n_sys, int32_t device, const double* A,
                       const double* B, const double* C, const double* L, const double* x0, bmpc_estimator** out);
void bmpc_est_destroy(bmpc_estimator* e);
int bmpc_est_predict(bmpc_estimator* e, const double* u /* [batch,nu] */, int on_device);
int bmpc_est_update(bmpc_estimator* e, const double* y_meas /* [batch,ny] */, int on_device);
int bmpc_est_get(bmpc_estimator* e, double* x /* [batch,nx] or NULL */, double* y /* [batch,ny] or NULL */);
double* bmpc_est_state_ptr(bmpc_estimator* e);           /* device pointer to x [batch,nx] */
int bmpc_est_set_stream(bmpc_estimator* e, void* cuda_stream);
/* on-device chain estimator <-> controller without host reads in between: the estimator runs on the controller's stream (its
 * kernels are ordered against bmpc_update(on_device=1) reading bmpc_est_state_ptr() and against the solver writing u0), and
 * a predict/update that takes a device pointer first retires the controller's deferred solve.  h = NULL detaches. */
int bmpc_est_attach(bmpc_estimator* e, bmpc_handle* h);

/* ---- batched Kalman filter: an estimator whose gain is computed every step (csrc/bmpc_kf.cuh), for models that change between
 * steps.  Model of kalman_design_simple (kalman.py:73-106): x+ = A x + B u + w, E[ww'] = Qn; y = C x + v, E[vv'] = Rn.
 *   predict(u):       x <- A x + B u;  P <- A P A' + Qn;  y <- C x
 *   update(y_meas):   S = C P C' + Rn;  K = P C' S^-1 (Cholesky of S);  x <- x + K (y_meas - y);
 *                     P <- (I - K C) P (I - K C)' + K Rn K', symmetrised
 * x is the a-priori estimate x[k|k-1], where the reference's estimator sits after construction or predict; y is refreshed by
 * predict only.  bmpc_est_predict / update / get / state_ptr / set_stream / attach / destroy apply unchanged.  1 <= nx, ny <= 32,
 * nu >= 1; n_sys = 1 (shared model, held in shared memory) or batch (one model per instance).  A [n_sys,nx,nx], B [n_sys,nx,nu],
 * C [n_sys,ny,nx], Qn [n_sys,nx,nx], Rn [n_sys,ny,ny], x0 [batch,nx], P0 [batch,nx,nx]: host pointers, row-major, batch-major.
 * Qn, Rn and P0 are symmetric: their upper triangles (Rn: lower) are read.  The per-instance status of the last update is
 * BMPC_KF_OK, or BMPC_KF_S_NOT_PD when S is not positive definite (a non-positive or non-finite Cholesky pivot): that instance's x
 * and P are left as they were; the others are unaffected.  Before the first update the status is BMPC_KF_OK. */
enum {
    BMPC_KF_OK = 1,
    BMPC_KF_S_NOT_PD = -2       /* innovation covariance S = C P C' + Rn not positive definite */
};
int bmpc_est_create_kf(int32_t nx, int32_t nu, int32_t ny, int32_t batch, int32_t n_sys, int32_t device, const double* A,
                       const double* B, const double* C, const double* Qn, const double* Rn, const double* x0, const double* P0,
                       bmpc_estimator** out);
/* P [batch,nx,nx] (full, symmetric) and status [batch] of a Kalman filter; either may be NULL.  Synchronises.  BMPC_ERR_ARG on a
 * fixed-gain estimator. */
int bmpc_est_get_cov(bmpc_estimator* e, double* P, int32_t* status);
/* replace any of the matrices of a created estimator between steps (time-varying model); NULL keeps an array.  L applies to the
 * fixed-gain estimator only, Qn and Rn to the Kalman filter only: the wrong kind returns BMPC_ERR_ARG.  Layout and leading n_sys
 * dimension as at creation; on_device = 0: host pointers, 1: device pointers on the estimator's device.  Stream-ordered on the
 * estimator's stream (the controller's once attached): whatever wrote device arrays must be ordered before it, and they stay
 * unchanged until that stream has passed this call.  A, B and Qn act from the next predict, C and Rn (and L) from the next update;
 * y is not recomputed. */
int bmpc_est_set_model(bmpc_estimator* e, const double* A, const double* B, const double* C, const double* L, const double* Qn,
                       const double* Rn, int on_device);

/* ---- batched DARE, the design step of kalman_design / kalman_design_simple (kalman.py:67, 96: control.dare):
 *   X = A'XA - (A'XB + S)(R + B'XB)^-1 (B'XA + S') + Q,   G = (R + B'XB)^-1 (B'XA + S')
 * for `batch` independent instances, 1 <= n, m <= 32, by structured doubling in fp64 (csrc/bmpc_dare.cuh).
 * A [batch,n,n], B [batch,n,m], Q [batch,n,n], R [batch,m,m], S [batch,n,m] (NULL: no cross term) in; X [batch,n,n],
 * G [batch,m,n], status [batch] (BMPC_DARE_*), iters [batch] (doubling steps) out.  Host pointers; synchronises before it returns.
 * X and G of an instance with status < 0 are NaN. */
int bmpc_dare(int32_t n, int32_t m, int32_t batch, int32_t device, const double* A, const double* B, const double* Q,
              const double* R, const double* S, double* X, double* G, int32_t* status, int32_t* iters);

/* pinned host memory for the end-to-end path (cudaHostAlloc mapped + portable / cudaFreeHost): the GPU can read and write it in place,
 * so such a buffer may be passed to bmpc_update(..., on_device = 2) and to bmpc_bind_output — the solver kernels then fetch x0 / u_-1
 * over PCIe while they compute and store u* straight into host memory: no H2D / D2H copy phases around the solve */
void* bmpc_host_alloc(uint64_t bytes);
void bmpc_host_free(void* p);
/* 1 if this build of the library holds the thread-per-instance fast path for the shape (nu == 1; Nc <= 0 means Nc = Np) */
int bmpc_has_fast_path(int nx, int nu, int Np, int Nc);

/* 1 when this build holds a thread-per-instance instantiation of the multi-input Riccati polish (csrc/bmpc_tpm.cuh) for the shape
 * (any sparsity pattern; bmpc_setup picks the entry whose compile-time (Ad, Bd) pattern contains the system's, or none).  Such a
 * controller starts every warm solve with that polish alone — no ADMM — and falls back to the ADMM rounds per instance. */
int bmpc_has_multi_input_fast_path(int nx, int nu, int Np, int Nc);
/* number of visible CUDA devices (0 if none / driver missing) */
int bmpc_device_count(void);

#ifdef __cplusplus
}
#endif
#endif
