/*
 * tinympc_b200.h — C ABI of the H100-native (sm_90a) batched TinyMPC solve path.
 *
 * This is the drop-in boundary for the hot path of TinyMPC/TinyMPC:
 *     tiny_solve()  (reference src/tinympc/tiny_api.cpp:384-386)
 *       -> solve()  (reference src/tinympc/admm.cpp:331-455)
 * run for B independent MPC instances per call on one H100.
 *
 * Plain C: POD structs, raw pointers, sizes.  No Eigen, no torch types.
 * The reference's own "C" API (src/tinympc/tiny_api.hpp:10-62) passes Eigen
 * objects by value and therefore cannot be bound from C; each entry point
 * below cites the reference interface it replaces.  INTEGRATION.md shows the
 * reference-side binding (the C++ shim with the reference's names/signatures
 * lives in tinympc_b200/shim/).
 *
 * Conventions
 *   - every matrix is COLUMN-MAJOR, exactly like the reference's dynamic
 *     Eigen matrices (types.hpp:16-17): M(i,j) at M[i + rows*j].
 *   - a per-instance trajectory is the reference's nx x N (or nu x (N-1))
 *     column-major matrix, i.e. time-major / state-minor: X[k*nx + i];
 *     a batch is that block repeated B times, instance-major:
 *     X[(b*N + k)*nx + i].
 *   - dtype selects the arithmetic type of ALL floating-point buffers
 *     (TINYMPC_F32 = float, TINYMPC_F64 = double = the reference's
 *     `tinytype`, types.hpp:15).
 *   - return value: 0 = ok; negative = error (see tinympc_b200_last_error);
 *     nothing is ever printed.
 */
#ifndef TINYMPC_B200_H
#define TINYMPC_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TINYMPC_F32 0
#define TINYMPC_F64 1

/* arithmetic mode of the device kernels */
#define TINYMPC_MODE_STRICT 0 /* separate mul/add, ascending-k sums: bit-identical to the pinned oracle */
#define TINYMPC_MODE_FAST 1   /* FMA contraction allowed (fp32/fp64); same operation order otherwise  */

/* kernel family selection (TINYMPC_KERNEL_AUTO picks the fastest that fits) */
#define TINYMPC_KERNEL_AUTO 0
#define TINYMPC_KERNEL_TPI 1 /* thread-per-instance, state streamed through HBM/L2 (any feature set)   */
#define TINYMPC_KERNEL_GPI 2 /* lane-group-per-instance: state resident on chip (shared memory) when the            */
                             /* problem is box-constrained and fits, else the streamed variant below               */
/* 3 was an experimental split of a batch between the GPI and TPI kernels; removed (it never won) */
#define TINYMPC_KERNEL_GPS 4 /* lane-group-per-instance, state streamed through an L2/HBM workspace by TMA bulk     */
                             /* copies (any feature set: box, cones, hyperplanes; fp32 and fp64)                   */

/* error codes */
#define TINYMPC_OK 0
#define TINYMPC_ERR_ARG (-1)         /* null pointer / bad size / inconsistent description            */
#define TINYMPC_ERR_UNSUPPORTED (-2) /* (nx,nu,dtype,features) has no compiled kernel                   */
#define TINYMPC_ERR_CUDA (-3)        /* CUDA runtime error (message in tinympc_b200_last_error)        */
#define TINYMPC_ERR_NO_BOUNDS (-4)   /* en_*_bound set but bounds were never provided (UB in the ref.) */
#define TINYMPC_ERR_CONE_DIM (-5)    /* cone dimension != 3 (the reference only supports 3, admm.cpp:53)*/
#define TINYMPC_ERR_SINGULAR (-6)    /* batched precompute: R + B'PB singular for some instance (index in last_error) */

/*
 * Problem description = the read-only part of the reference's
 * TinyWorkspace + TinyCache (types.hpp:43-59, 88-208), host pointers.
 * Everything is copied at create(); the caller may free it afterwards.
 */
typedef struct tinympc_problem {
    int32_t nx, nu, N; /* work->nx, nu, N (types.hpp:89-91) */
    int32_t dtype;     /* TINYMPC_F32 / TINYMPC_F64 */
    double rho;        /* cache->rho (types.hpp:44); exact for float inputs */

    /* model, types.hpp:186-190 */
    const void *Adyn; /* nx x nx */
    const void *Bdyn; /* nx x nu */
    const void *fdyn; /* nx */
    const void *Q;    /* nx  : work->Q  = diag(Q_user) + rho  (tiny_api.cpp:117) */
    const void *R;    /* nu  : work->R  = diag(R_user) + rho  (tiny_api.cpp:118) */

    /* precomputed cache, types.hpp:43-51 (layout kept: column-major) */
    const void *Kinf;    /* nu x nx */
    const void *Pinf;    /* nx x nx */
    const void *Quu_inv; /* nu x nu */
    const void *AmBKt;   /* nx x nx */
    const void *APf;     /* nx */
    const void *BPf;     /* nu */

    /* box bounds (tiny_set_bound_constraints, tiny_api.hpp:13-15); NULL = never set */
    const void *x_min, *x_max; /* nx x N     */
    const void *u_min, *u_max; /* nu x (N-1) */

    /* second-order cones (tiny_set_cone_constraints, tiny_api.cpp:176-208).
     * STATE triple first — this is the order of the reference DEFINITION; its header
     * (tiny_api.hpp:16-18) names the parameters the other way round. */
    int32_t num_state_cones, num_input_cones; /* work->numStateCones / numInputCones */
    const int32_t *Acx, *qcx;                 /* start index, dimension per state cone */
    const void *cx;                           /* mu per state cone */
    const int32_t *Acu, *qcu;
    const void *cu;

    /* static hyperplanes (tiny_set_linear_constraints, tiny_api.hpp:19-21) */
    int32_t num_state_linear, num_input_linear;
    const void *Alin_x; /* num_state_linear x nx */
    const void *blin_x; /* num_state_linear */
    const void *Alin_u; /* num_input_linear x nu */
    const void *blin_u;

    /* time-varying hyperplanes (tiny_set_tv_linear_constraints, tiny_api.hpp:22-24) */
    int32_t num_tv_state_linear, num_tv_input_linear;
    const void *tv_Alin_x; /* (num_tv_state_linear*N) x nx     */
    const void *tv_blin_x; /* num_tv_state_linear x N          */
    const void *tv_Alin_u; /* (num_tv_input_linear*(N-1)) x nu */
    const void *tv_blin_u; /* num_tv_input_linear x (N-1)      */
} tinympc_problem_t;

/* TinySettings (types.hpp:63-82) without the adaptive-rho fields: adaptive rho is a separate call
 * (tinympc_b200_solve_adaptive, tinympc_adaptive_rho_t below). */
typedef struct tinympc_settings {
    double abs_pri_tol;
    double abs_dua_tol;
    int32_t max_iter;
    int32_t check_termination;
    int32_t en_state_bound;
    int32_t en_input_bound;
    int32_t en_state_soc;
    int32_t en_input_soc;
    int32_t en_state_linear;
    int32_t en_input_linear;
    int32_t en_tv_state_linear;
    int32_t en_tv_input_linear;
} tinympc_settings_t;

/*
 * The mutable part of TinyWorkspace that survives between tiny_solve() calls (warm start,
 * SURVEY §5 "checkpoint/resume").  Every pointer is [B] x (nx x N) or [B] x (nu x (N-1));
 * any pointer may be NULL: on input NULL reads as zeros (the state right after tiny_setup,
 * tiny_api.cpp:68-115), on output NULL is simply not written.  The slack / dual fields of a constraint
 * family the settings leave disabled (cones, hyperplanes, time-varying hyperplanes) are neither read
 * nor written by any kernel.  tinympc_b200_solve returns such buffers unchanged, also on a cold start;
 * tinympc_b200_solve_host returns them unchanged on a warm start (they are staged to the device and
 * copied back as they were), but on a cold start their contents on return are unspecified.
 */
typedef struct tinympc_state {
    void *x, *u;         /* work->x, work->u   (rollout; x[:,0] is overwritten by x0)        */
    void *v, *z;         /* work->v, work->z   (slack of the previous iteration)             */
    void *vnew, *znew;   /* work->vnew, znew                                                  */
    void *g, *y;         /* work->g, work->y   (box duals)                                    */
    void *vcnew, *zcnew; /* cone slacks  (types.hpp:136-138)                                 */
    void *gc, *yc;       /* cone duals                                                        */
    void *vlnew, *zlnew; /* static-hyperplane slacks                                          */
    void *gl, *yl;
    void *vlnew_tv, *zlnew_tv; /* time-varying-hyperplane slacks                              */
    void *gl_tv, *yl_tv;
} tinympc_state_t;

/* One batched tiny_solve(): inputs, warm-start state (in/out) and outputs. */
typedef struct tinympc_batch {
    int64_t B; /* number of independent instances */

    const void *x0; /* [B][nx]          -> work->x.col(0)   (tiny_set_x0, tiny_api.cpp:443-453)   */
    const void *Xref; /* work->Xref (tiny_set_x_ref): [B][N][nx] if xref_per_instance else [N][nx] */
    int32_t xref_per_instance;
    const void *Uref; /* work->Uref: [B][N-1][nu] / [N-1][nu]; NULL = zeros                        */
    int32_t uref_per_instance;

    int32_t cold_start; /* 1: ignore the contents of `state` on input (all zeros)                 */
    tinympc_state_t state;

    void *sol_x;  /* [B][N][nx]    solution->x = vnew   (admm.cpp:436,452)  may be NULL (e.g. when state.vnew is given) */
    void *sol_u;  /* [B][N-1][nu]  solution->u = znew   (admm.cpp:437,453)  may be NULL */
    int32_t *iter;   /* [B] solution->iter                                           */
    int32_t *solved; /* [B] solution->solved (tiny_solve returns !solved)            */
    void *residuals; /* [B][4]: primal_state, dual_state, primal_input, dual_input (types.hpp:202-205); may be NULL */
    void *u0;        /* [B][nu] optional: work->u.col(0), the control every example applies (e.g. quadrotor_hovering.cpp:92) */
    /* Heterogeneous batch (optional, SURVEY §8f-2): one model + cache per instance instead of the handle's shared one.
     * [B][tinympc_b200_model_blob_elems(nx,nu)] elements of the problem dtype, each blob =
     *   Adyn | Bdyn | fdyn | Q | R | Kinf | Pinf | Quu_inv | AmBKt | APf | BPf | rho      (column-major pieces, as in
     * tinympc_problem_t); build it with tinympc_b200_precompute_cache_batch.  Time-varying hyperplanes, the cone structure
     * and settings stay shared; box bounds, cone coefficients and static hyperplanes are the handle's unless the batch brings
     * its own (bounds_per_instance, cones_per_instance, planes_per_instance below).  Served by the lane-group
     * kernels: the on-chip (GPI) kernel when the family is AUTO or GPI, the problem has box constraints only and the
     * horizon fits in shared memory; otherwise (explicit GPS, cones or hyperplanes, a horizon off chip) the streamed (GPS)
     * kernel, one instance per lane group.  TPI returns TINYMPC_ERR_UNSUPPORTED. */
    const void *models;
    /* Per-instance box bounds (optional): instance b clamps with its own x_min, x_max, u_min, u_max, as a TinySolver whose
     * tiny_set_bound_constraints was called with them would.  Arrays of the problem dtype, selected per call by
     * bounds_per_instance:
     *   0: the handle's bounds (the pointers are ignored; what every zero-initialised batch gets);
     *   1: x_min / x_max [B][nx], u_min / u_max [B][nu]: one column per instance, the same at every knot point;
     *   2: x_min / x_max [B][N][nx], u_min / u_max [B][N-1][nu]: the full nx x N / nu x (N-1) matrices per instance
     *      (the layout of a per-instance Xref / Uref).
     * With 1 or 2 they replace the handle's bounds on both sides, and the handle needs no bounds of its own.  A side the
     * settings enable (en_state_bound, en_input_bound) needs both pointers of its pair (else TINYMPC_ERR_NO_BOUNDS); a pair
     * for a disabled side is never read.  One pointer of a pair without the other, any other mode value or a non-zero
     * reserved2 return TINYMPC_ERR_ARG.  DEVICE pointers for tinympc_b200_solve, HOST pointers (staged per chunk) for
     * tinympc_b200_solve_host.  Routed like `models` (lane-group kernels only; explicit TPI returns
     * TINYMPC_ERR_UNSUPPORTED) and STRICT only: FAST mode, adaptive rho and rollouts return TINYMPC_ERR_UNSUPPORTED. */
    const void *x_min, *x_max; /* per-instance state bounds (see bounds_per_instance), or NULL */
    const void *u_min, *u_max; /* per-instance input bounds, or NULL                         */
    int32_t bounds_per_instance; /* 0: the handle's bounds; 1: one column per instance; 2: full horizon per instance */
    int32_t reserved2;           /* must be 0 */
    /* Per-instance cone coefficients (optional): instance b projects its cones with its own mu, as a TinySolver whose
     * tiny_set_cone_constraints got these cx / cu would.  The cone structure (Acx, qcx, Acu, qcu) stays the handle's.
     * Arrays of the problem dtype, named positionally as in tinympc_problem_t: cone_x_mu goes with Acx / qcx (the state
     * cones), cone_u_mu with Acu / qcu (the input cones).  With cones_per_instance = 1 a side whose cone loop runs
     * (en_state_soc / en_input_soc set and the handle has cones on that side) needs its pointer (else TINYMPC_ERR_ARG); a
     * side whose loop does not run is never read, and when neither runs the solve is the one without per-instance cones.
     * Any other mode value or a non-zero reserved3 return TINYMPC_ERR_ARG.  DEVICE pointers for tinympc_b200_solve, HOST
     * pointers (staged per chunk) for tinympc_b200_solve_host.  Served by the streamed (GPS) kernel, the one that runs
     * cones, with two instances per lane group where the shared solve has two; combines with models and bounds.  STRICT
     * only: FAST mode, explicit TPI, adaptive rho and rollouts return TINYMPC_ERR_UNSUPPORTED. */
    const void *cone_x_mu;      /* [B][num_state_cones]: state-cone mu per instance (replaces problem->cx), or NULL */
    const void *cone_u_mu;      /* [B][num_input_cones]: input-cone mu per instance (replaces problem->cu), or NULL */
    int32_t cones_per_instance; /* 0: the handle's cx / cu (every zero-initialised batch); 1: the arrays above */
    int32_t reserved3;          /* must be 0 */
    /* Per-instance static hyperplanes (optional): instance b projects its static linear constraints with its own Alin_x,
     * blin_x, Alin_u, blin_u, as a TinySolver whose tiny_set_linear_constraints got them would.  The hyperplane structure
     * (num_state_linear, num_input_linear, en_state_linear, en_input_linear), the time-varying hyperplanes, the cones, the
     * bounds and the model stay the handle's.  Arrays of the problem dtype, each instance's matrix column-major as in
     * tinympc_problem_t.  A row a = 0, b = 0 never projects, so an instance with fewer planes pads its rows with zeros.  With
     * planes_per_instance = 1 a side whose static hyperplane loop runs (en_state_linear / en_input_linear set and the handle
     * has rows on that side) needs both pointers of its pair (else TINYMPC_ERR_ARG); a side whose loop does not run is never
     * read, and when neither runs the solve is the one without per-instance planes.  Any other mode value or a non-zero
     * reserved4 return TINYMPC_ERR_ARG.  DEVICE pointers for tinympc_b200_solve, HOST pointers (staged per chunk) for
     * tinympc_b200_solve_host.  Served by the streamed (GPS) kernel, the one that runs hyperplanes, with two instances per
     * lane group where the shared solve has two; combines with models only.  STRICT only: FAST mode, explicit TPI, adaptive
     * rho, rollouts and per-instance bounds or cones in the same batch return TINYMPC_ERR_UNSUPPORTED. */
    const void *Alin_x;   /* [B][nx][num_state_linear]: instance b's Alin_x, column-major like tinympc_problem_t.Alin_x */
    const void *blin_x;   /* [B][num_state_linear] */
    const void *Alin_u;   /* [B][nu][num_input_linear] */
    const void *blin_u;   /* [B][num_input_linear] */
    int32_t planes_per_instance; /* 0: the handle's hyperplanes; 1: the arrays above */
    int32_t reserved4;           /* must be 0 */
} tinympc_batch_t;

typedef struct tinympc_b200_solver tinympc_b200_solver_t;

/* aggregated counters of the last solve on a handle */
typedef struct tinympc_b200_stats {
    int64_t instances;
    int64_t kernel_launches; /* launches of this library's kernels in the last solve call */
    float kernel_ms;         /* device time of the solve kernel(s), CUDA events on the launch stream */
    int32_t kernel_family;   /* TINYMPC_KERNEL_TPI / _GPI / _GPS actually used */
    int32_t lanes_per_instance;
    int32_t instances_per_cta;
    int32_t smem_bytes_per_cta;
    int32_t ctas;
    int32_t threads_per_cta;
    int64_t gpi_instances; /* instances of the batch solved by a lane-group kernel (GPI or GPS) */
    int32_t tmem_cols_per_cta; /* always 0: the state of every kernel family lives in shared / global memory on sm_90   */
    int32_t reserved0;
    int64_t workspace_bytes; /* GPS / TPI: bytes of streamed-state workspace behind the last solve (0 = state on chip) */
} tinympc_b200_stats_t;

/* tiny_set_default_settings (tiny_api.cpp:413-441, tiny_api_constants.hpp:5-16) */
int tinympc_b200_default_settings(tinympc_settings_t *s);

/*
 * tiny_precompute_and_set_cache (tiny_api.cpp:307-381) on the host, fp64 or fp32 per `dtype`:
 * Riccati fixed point started at P = rho*I, at most 1000 sweeps, stop when max|K - K_prev| < 1e-5.
 * Q, R are the vectors the reference passes in (work->Q, work->R — they already contain +rho,
 * and rho is added once more inside: the "double rho" quirk, SURVEY A.3-1).
 * Outputs (caller-allocated, column-major): Kinf nu*nx, Pinf nx*nx, Quu_inv nu*nu, AmBKt nx*nx,
 * APf nx, BPf nu.  Returns the number of sweeps used (>0) or a negative error.
 */
int tinympc_b200_precompute_cache(int32_t dtype, int32_t nx, int32_t nu, double rho, const void *Adyn,
                                  const void *Bdyn, const void *fdyn, const void *Q, const void *R, void *Kinf,
                                  void *Pinf, void *Quu_inv, void *AmBKt, void *APf, void *BPf);

/* number of elements of one per-instance model blob (see tinympc_batch_t.models) */
int64_t tinympc_b200_model_blob_elems(int32_t nx, int32_t nu);

/*
 * tiny_setup's arithmetic for B different models at once, on the host with `nthreads` threads: for instance b
 *   Q_b = Qdiag[b] + rho[b], R_b = Rdiag[b] + rho[b]            (tiny_api.cpp:117-118)
 *   cache_b = tiny_precompute_and_set_cache(A[b], B[b], f[b], Q_b, R_b, rho[b])   (tiny_api.cpp:307-381)
 * packed into models_out[b] (layout: tinympc_batch_t.models).  A [B][nx*nx], Bm [B][nx*nu] column-major, f [B][nx],
 * Qdiag [B][nx], Rdiag [B][nu] (the USER's diagonals, without rho), rho [B]; all in `dtype`.
 * Returns 0, or TINYMPC_ERR_SINGULAR when some instance's Riccati recursion hit a singular matrix (the index of the
 * first such instance is in tinympc_b200_last_error()).
 */
int tinympc_b200_precompute_cache_batch(int32_t dtype, int32_t nx, int32_t nu, int64_t B, const void *A, const void *Bm,
                                        const void *f, const void *Qdiag, const void *Rdiag, const void *rho,
                                        void *models_out, int32_t nthreads);

/*
 * The same computation ON THE DEVICE of handle `h` (one warp per instance, riccati.cuh: riccati_kernel), for batches whose
 * models change often (per-instance re-linearisation): all pointers are device pointers of the handle's dtype, layouts
 * as above; nx, nu are the handle's.  Asynchronous on `stream`.  The blobs are bit-identical to the host routine's.
 * sweeps_out (optional, [B]): Riccati sweeps used per instance, -1 where a matrix was singular (that blob's cache is
 * then undefined).  models_out can be passed straight to tinympc_b200_solve as tinympc_batch_t.models.
 */
int tinympc_b200_precompute_cache_batch_device(tinympc_b200_solver_t *h, int64_t B, const void *A, const void *Bm, const void *f,
                                               const void *Qdiag, const void *Rdiag, const void *rho, void *models_out,
                                               int32_t *sweeps_out, void *stream);

/*
 * Sensitivity tables for adaptive rho (tinympc_adaptive_rho_t below), for B different models at once, on the host with
 * `nthreads` threads.  The reference ships one hard-coded pair for one quadrotor (tiny_api.cpp:479-540, applied by
 * update_matrices_with_derivatives, rho_benchmark.cpp:215-229); here the tables of model b are DEFINED as the forward-mode
 * derivative, with respect to rho[b], of tinympc_b200_precompute_cache_batch as it runs: the Riccati recursion of
 * tiny_precompute_and_set_cache (tiny_api.cpp:307-381) with its tangent carried alongside,
 *     Q1 = Qdiag + 2 rho, R1 = Rdiag + 2 rho (the "double rho"):  dQ1 = dR1 = 2 I;    P <- rho I:  dP = I
 *     per sweep, S = R1 + B'PB, K = S^-1 B'PA:
 *         dS = dR1 + B'dP B;   dK = S^-1 (B'dP A - dS K);   dP+ = (dQ1 + A'dP (A - BK)) - A'P (B dK)
 * for exactly the sweeps the primal recursion of that model takes (the primal's stop test ends both), so the tables are
 * the derivative of the Kinf / Pinf the cache call returns, sweep count held fixed.  Ascending-k sums, separate multiply
 * and add, like the cache.  Inputs as in tinympc_b200_precompute_cache_batch (f is accepted for symmetry and not read: it
 * does not enter Kinf / Pinf).  dK_out [B][nu*nx], dP_out [B][nx*nx], column-major per instance, in `dtype`.
 * In fp32 a model whose recursion never meets the stop test (typically few inputs for many states) runs all 1000 sweeps, and
 * its tangent can overflow to Inf / NaN on the way; compute such tables in fp64 and round them.
 * Returns 0, or TINYMPC_ERR_SINGULAR under the same condition, and with the same message, as the cache call.
 */
int tinympc_b200_precompute_sensitivity_batch(int32_t dtype, int32_t nx, int32_t nu, int64_t B, const void *A, const void *Bm,
                                              const void *f, const void *Qdiag, const void *Rdiag, const void *rho, void *dK_out,
                                              void *dP_out, int32_t nthreads);

/*
 * The same tables ON THE DEVICE of handle `h` (one warp per instance, riccati.cuh: riccati_kernel): device pointers of the
 * handle's dtype, nx, nu are the handle's, asynchronous on `stream`.  Bit-identical to the host routine's.  sweeps_out
 * (optional, [B]): sweeps used per instance, -1 where a matrix was singular (the same instances as in
 * tinympc_b200_precompute_cache_batch_device; their tables are not written).  dK_out / dP_out can be passed straight to
 * tinympc_b200_solve_adaptive with tables_per_instance = 1.
 */
int tinympc_b200_precompute_sensitivity_batch_device(tinympc_b200_solver_t *h, int64_t B, const void *A, const void *Bm, const void *f,
                                                     const void *Qdiag, const void *Rdiag, const void *rho, void *dK_out, void *dP_out,
                                                     int32_t *sweeps_out, void *stream);

/* tiny_setup (tiny_api.hpp:10-12) minus the precompute: uploads the problem to `device`. */
int tinympc_b200_create(const tinympc_problem_t *problem, int32_t device, tinympc_b200_solver_t **out);
int tinympc_b200_destroy(tinympc_b200_solver_t *s);

/* tiny_update_settings (tiny_api.hpp:36-42) */
int tinympc_b200_update_settings(tinympc_b200_solver_t *s, const tinympc_settings_t *settings);
int tinympc_b200_get_settings(const tinympc_b200_solver_t *s, tinympc_settings_t *settings);

/* arithmetic mode / kernel family (see the defines above); both default to STRICT / AUTO */
int tinympc_b200_set_mode(tinympc_b200_solver_t *s, int32_t mode, int32_t kernel_family);

/*
 * Batched tiny_solve (tiny_api.hpp:34).  All pointers in `io` are DEVICE pointers on the
 * handle's device.  Asynchronous on `cuda_stream` (a cudaStream_t, NULL = legacy default stream).
 * Returns 0 when the work was enqueued; per-instance success is io->solved.
 */
int tinympc_b200_solve(tinympc_b200_solver_t *s, const tinympc_batch_t *io, void *cuda_stream);

/*
 * Same call with HOST pointers: stages the inputs to the device, solves, and copies every
 * requested output back; synchronous.  This is the call the reference-facing shim uses and what
 * bench.py times as `e2e`.
 */
int tinympc_b200_solve_host(tinympc_b200_solver_t *s, const tinympc_batch_t *io);

int tinympc_b200_get_stats(const tinympc_b200_solver_t *s, tinympc_b200_stats_t *stats);

/*
 * Adaptive rho (admm.cpp:397-423, rho_benchmark.cpp), per instance.  After the dual update of loop index i with
 * i > 0 && i % 5 == 0, the residuals of format_matrices / compute_residuals (Eigen's summation order) give
 *     new = rho * sqrt((pri / (pri_norm + 1e-10)) / ((dual / (dual_norm + 1e-10)) + 1e-10)),
 * clipped to [rho_min, rho_max] when enable_clipping != 0, and update_matrices_with_derivatives runs twice:
 *     Kinf += (new - rho) * dKinf_drho;  Pinf += (new - rho) * dPinf_drho;  rho = new.
 * The same iteration's termination check and every later iteration use the new rho / Kinf / Pinf.  Quu_inv, AmBKt,
 * APf, BPf, Q, R stay as they are (as in the reference); C1 / C2 are never read by a solve and are not modelled.
 * The reference declares its RhoAdapter uninitialised (admm.cpp:340) and then reads it (rho_benchmark.cpp:56), which
 * makes its adaptive solve undefined behaviour; this library implements the value-initialised adapter.
 *
 *   dKinf_drho (nu x nx), dPinf_drho (nx x nx): HOST pointers of the handle's dtype, column-major, read during the call
 *           (tables_per_instance = 0: one pair adapts every instance, right when all instances share one model).
 *           tables_per_instance = 1: dKinf_drho is [B][nu*nx] and dPinf_drho [B][nx*nx], instance b adapts with its own
 *           pair (a fleet of different models; build them with tinympc_b200_precompute_sensitivity_batch[_device]).  They
 *           are then DEVICE pointers for tinympc_b200_solve_adaptive (read by the kernel, like `models`) and host pointers
 *           for tinympc_b200_solve_adaptive_host (chunked and staged with the models).
 *   models: [B][tinympc_b200_model_blob_elems(nx,nu)] (layout: tinympc_batch_t.models), IN/OUT: every instance starts from
 *           its blob's model, cache and rho, and its adapted rho / Kinf / Pinf are written back, so passing the same
 *           buffer to the next solve continues the adaptation (the reference's one-TinySolver-per-robot semantics).
 * Served by the on-chip (GPI) kernel in STRICT mode with box constraints only; io->models must be NULL.
 */
typedef struct tinympc_adaptive_rho {
    double rho_min, rho_max;  /* settings->adaptive_rho_min / max (rounded to the dtype) */
    int32_t enable_clipping;  /* settings->adaptive_rho_enable_clipping */
    int32_t reserved;         /* must be 0 */
    const void *dKinf_drho;   /* nu x nx */
    const void *dPinf_drho;   /* nx x nx */
    void *models;             /* [B][blob] in/out */
    int32_t tables_per_instance; /* 0: one table pair for the batch; 1: one pair per instance */
    int32_t reserved1;
} tinympc_adaptive_rho_t;

/* tinympc_b200_solve with adaptive rho: io and ar->models are DEVICE pointers; asynchronous on `cuda_stream` */
int tinympc_b200_solve_adaptive(tinympc_b200_solver_t *s, const tinympc_batch_t *io, const tinympc_adaptive_rho_t *ar,
                                void *cuda_stream);
/* the same with HOST pointers (chunked like tinympc_b200_solve_host; ar->models is copied back); synchronous */
int tinympc_b200_solve_adaptive_host(tinympc_b200_solver_t *s, const tinympc_batch_t *io, const tinympc_adaptive_rho_t *ar);

/*
 * Closed-loop rollout: T warm-started MPC steps per instance in one launch, the loop of the reference's examples
 * (examples/quadrotor_tracking.cpp:77-106).  For every instance b and step t = 0 ... T-1 the result is bit-identical to
 *     solve (warm start from step t-1; the first step is cold or warm from io->state per io->cold_start) with
 *         x0 = the plant state, Xref = knot points t ... t+N-1 of Xref, Uref = knot points t ... t+N-2 of Uref;
 *     u0 = work->u.col(0);  x0 <- (Adyn x0 + Bdyn u0) + fdyn  (tinympc_b200_advance[_models]);  x0 <- x0 + w[b][t]
 * with the warm state kept on chip from one step to the next.  reset_duals = 1 zeroes g, y before every step after the first
 * (zero io->state.g / y yourself to reset them before the first).  carry_v = 1 carries work->v / work->z (the slack of the
 * previous iteration, which feeds the first iteration's dual residual) from one step to the next, as a solve with state.v / z
 * would; carry_v = 0 reads them as zeros at every step and needs io->state.v / z NULL.
 *
 *   io: B, x0 (the initial plant states, not modified), cold_start, state (in: the first step's warm start; out: the state
 *       after the last step; x and u must be NULL), models (a fleet: every instance solves and advances with its own blob),
 *       optional sol_x / sol_u (solution of the last step).  Xref, Uref, iter, solved, residuals and u0 must be NULL.
 *   Xref: [B][T+N-1][nx] (xref_per_instance) or [T+N-1][nx]; Uref: [B][T+N-2][nu] / [T+N-2][nu], or NULL = zeros.
 *   Outputs, each may be NULL: x_traj [B][T+1][nx] the plant state before step t and after the last one; u_traj [B][T][nu];
 *   iter_traj, solved_traj [B][T]; residuals_traj [B][T][4].  T = 0 writes nothing.
 * All pointers are DEVICE pointers; asynchronous on `cuda_stream`.  Served by the on-chip (GPI) kernel in STRICT mode with box
 * constraints only, with the launch plan a solve of the same batch gets on it (stats() reports it); FAST mode, cones,
 * hyperplanes, a horizon that does not fit on chip and an explicit TPI or GPS family return TINYMPC_ERR_UNSUPPORTED.
 */
typedef struct tinympc_rollout {
    int32_t T;            /* steps per instance, >= 0 */
    int32_t reset_duals;  /* 0 / 1 */
    int32_t carry_v;      /* 0 / 1 */
    int32_t xref_per_instance;
    const void *Xref;
    const void *Uref;
    int32_t uref_per_instance;
    int32_t reserved;     /* must be 0 */
    const void *w;        /* [B][T][nx] disturbance, or NULL */
    void *x_traj;         /* [B][T+1][nx] */
    void *u_traj;         /* [B][T][nu] */
    int32_t *iter_traj;   /* [B][T] */
    int32_t *solved_traj; /* [B][T] */
    void *residuals_traj; /* [B][T][4] */
    int64_t reserved1[2]; /* must be 0 */
    /*
     * A plant of their own and measurement noise (a robustness study: every robot heavier, lighter or pushed by wind, seeing its
     * state through a noisy sensor).  Instance b's plant P_b = (A_p, B_p, f_p) is the controller's model (the handle's, or
     * io->models[b]) when plant is NULL, else the record `plant` (plant_per_instance = 0) or plant[b] (= 1).  Step t then runs
     *     x^_t = x_t + noise[b][t]  (no add at all when noise is NULL);  solve from x^_t;  u0 = work->u.col(0);
     *     x_{t+1} = (A_p x_t + B_p u0) + f_p  (tinympc_b200_advance_plant);  x_{t+1} = x_{t+1} + w[b][t]
     * and x_traj records the true states x_t.  plant == NULL with noise == NULL is the rollout above.
     */
    const void *plant;          /* A | B | f column-major, nx*nx + nx*nu + nx elements (the start of a model blob), or [B][record] */
    int32_t plant_per_instance; /* 0: one record for the batch; 1: one per instance (plant required) */
    int32_t reserved2;          /* must be 0 */
    const void *noise;          /* [B][T][nx] measurement noise, or NULL */
} tinympc_rollout_t;

int tinympc_b200_rollout(tinympc_b200_solver_t *s, const tinympc_batch_t *io, const tinympc_rollout_t *ro, void *cuda_stream);

/*
 * Closed-loop helper (the caller of the hot path, e.g. examples/quadrotor_tracking.cpp:105):
 *     x0[b] <- (Adyn * x0[b] + Bdyn * u[b][:,0]) + fdyn        for b in [0, B)
 * with x0 [B][nx] (in/out) and u pointing at the first control of instance 0, consecutive instances `u_stride`
 * elements apart (nu for a tinympc_batch_t.u0 buffer, (N-1)*nu for a work->u buffer); DEVICE pointers;
 * ascending-k sums, no FMA.  Lets thousands of simulated plants step without a host round trip between two
 * tinympc_b200_solve calls.
 */
int tinympc_b200_advance(tinympc_b200_solver_t *s, int64_t B, void *x0, const void *u, int64_t u_stride, void *cuda_stream);

/*
 * The same step for a heterogeneous batch: instance b is advanced with Adyn, Bdyn, fdyn of its own blob models[b]
 * ([B][tinympc_b200_model_blob_elems(nx,nu)], layout: tinympc_batch_t.models, DEVICE pointer), same arithmetic.
 */
int tinympc_b200_advance_models(tinympc_b200_solver_t *s, int64_t B, void *x0, const void *u, int64_t u_stride, const void *models,
                                void *cuda_stream);

/*
 * The same step against plants that are not the controller's model: instance b is advanced with the plant record `plant`
 * (plant_per_instance = 0) or plant[b] (= 1), each A | B | f column-major, nx*nx + nx*nu + nx elements of the handle's dtype
 * (the first pieces of a model blob), DEVICE pointer; same arithmetic.  The plant step of tinympc_rollout_t.plant.
 */
int tinympc_b200_advance_plant(tinympc_b200_solver_t *s, int64_t B, void *x0, const void *u, int64_t u_stride, const void *plant,
                               int32_t plant_per_instance, void *cuda_stream);

/* 1 if a kernel is compiled for (dtype,nx,nu); used by callers to fail early */
int tinympc_b200_supported(int32_t dtype, int32_t nx, int32_t nu);

const char *tinympc_b200_last_error(void);
const char *tinympc_b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* TINYMPC_B200_H */
