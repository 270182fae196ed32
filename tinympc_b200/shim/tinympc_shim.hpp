// tinympc_shim.hpp — source-compatible C++ front end of the reference's solver interface on top of the
// H100 C ABI (include/tinympc_b200.h).
//
// A program written against the reference (#include <tinympc/tiny_api.hpp>, TinySolver struct tree, tiny_setup /
// tiny_set_* / tiny_solve) compiles unchanged against this header and links tinympc_shim.cpp +
// libtinympc_b200.so; tiny_solve() then runs on the GPU (a batch of one through tinympc_b200_solve_host —
// Eigen's dynamic matrices are contiguous column-major, so the struct tree's buffers are handed to the C ABI
// without copies).  Names, argument order and return codes follow TinyMPC src/tinympc/tiny_api.hpp:10-62
// and types.hpp:32-218, including the known quirks (SURVEY §8b / A.3): the cone setter's positional semantics,
// the "double rho" in the cache, tiny_set_bound_constraints returning 0 on a dimension mismatch, and the
// "Solver converged in N iterations" line on stdout (admm.cpp:439).
//
// Needs an Eigen 3.4 include path supplied by the user (the reference vendors one under include/Eigen).
// The reference's batched use is NOT expressible through this interface (it is single-instance by design);
// batched callers use the C ABI directly or tiny_solve_batch() below.
#pragma once

#if __has_include(<Eigen.h>)
#include <Eigen.h>  // the reference's vendored wrapper (include/Eigen/Eigen.h)
#else
#include <Eigen/Core>
#include <Eigen/LU>
#endif

#include <iostream>

using namespace Eigen;

extern "C" {

typedef double tinytype;  // the shim mirrors the reference as shipped (types.hpp:15); fp32 goes through the C ABI
typedef Matrix<tinytype, Dynamic, Dynamic> tinyMatrix;
typedef Matrix<tinytype, Dynamic, 1> tinyVector;

// ---- struct tree (field names = the reference's: they ARE its API; every example pokes them directly) ----
typedef struct {
    int iter, solved;
    tinyMatrix x, u;  // nx x N, nu x (N-1): the projected slacks vnew / znew
} TinySolution;

typedef struct {
    tinytype rho;
    tinyMatrix Kinf, Pinf, Quu_inv, AmBKt;
    tinyVector APf, BPf;
    tinyMatrix C1, C2;                                     // = Quu_inv, AmBKt (adaptive rho leftovers)
    tinyMatrix dKinf_drho, dPinf_drho, dC1_drho, dC2_drho;  // filled by tiny_initialize_sensitivity_matrices only
} TinyCache;

typedef struct {
    tinytype abs_pri_tol, abs_dua_tol;
    int max_iter, check_termination;
    int en_state_bound, en_input_bound, en_state_soc, en_input_soc;
    int en_state_linear, en_input_linear, en_tv_state_linear, en_tv_input_linear;
    int adaptive_rho;  // must stay 0
    tinytype adaptive_rho_min, adaptive_rho_max;
    int adaptive_rho_enable_clipping;
} TinySettings;

typedef struct {
    int nx, nu, N;
    tinyMatrix x, u, q, r, p, d;
    tinyMatrix v, vnew, z, znew, g, y;
    tinyMatrix x_min, x_max, u_min, u_max;
    int numStateCones, numInputCones;
    tinyVector cx, cu;
    VectorXi Acx, Acu, qcx, qcu;
    tinyMatrix vc, vcnew, zc, zcnew, gc, yc;
    int numStateLinear, numInputLinear;
    tinyMatrix Alin_x;
    tinyVector blin_x;
    tinyMatrix Alin_u;
    tinyVector blin_u;
    tinyMatrix vl, vlnew, zl, zlnew, gl, yl;
    int numtvStateLinear, numtvInputLinear;
    tinyMatrix tv_Alin_x, tv_blin_x, tv_Alin_u, tv_blin_u;
    tinyMatrix vl_tv, vlnew_tv, zl_tv, zlnew_tv, gl_tv, yl_tv;
    tinyVector Q, R;  // diag + rho
    tinyMatrix Adyn, Bdyn;
    tinyVector fdyn;
    tinyMatrix Xref, Uref;
    tinyVector Qu;
    tinytype primal_residual_state, primal_residual_input, dual_residual_state, dual_residual_input;
    int status, iter;
} TinyWorkspace;

typedef struct {
    TinySolution *solution;
    TinySettings *settings;
    TinyCache *cache;
    TinyWorkspace *work;
} TinySolver;

// ---- tiny_api.hpp:10-62 ----
int tiny_setup(TinySolver **solverp, tinyMatrix Adyn, tinyMatrix Bdyn, tinyMatrix fdyn, tinyMatrix Q, tinyMatrix R,
               tinytype rho, int nx, int nu, int N, int verbose);
int tiny_set_bound_constraints(TinySolver *solver, tinyMatrix x_min, tinyMatrix x_max, tinyMatrix u_min, tinyMatrix u_max);
// NOTE: declared with the reference header's parameter NAMES; the first triple is bound to the STATE cones,
// exactly as the reference's definition does (tiny_api.cpp:176-178).
int tiny_set_cone_constraints(TinySolver *solver, VectorXi Acu, VectorXi qcu, tinyVector cu, VectorXi Acx, VectorXi qcx,
                              tinyVector cx);
int tiny_set_linear_constraints(TinySolver *solver, tinyMatrix Alin_x, tinyVector blin_x, tinyMatrix Alin_u, tinyVector blin_u);
int tiny_set_tv_linear_constraints(TinySolver *solver, tinyMatrix tv_Alin_x, tinyMatrix tv_blin_x, tinyMatrix tv_Alin_u,
                                   tinyMatrix tv_blin_u);
int tiny_precompute_and_set_cache(TinyCache *cache, tinyMatrix Adyn, tinyMatrix Bdyn, tinyMatrix fdyn, tinyMatrix Q,
                                  tinyMatrix R, int nx, int nu, tinytype rho, int verbose);
int tiny_solve(TinySolver *solver);
int tiny_update_settings(TinySettings *settings, tinytype abs_pri_tol, tinytype abs_dua_tol, int max_iter,
                         int check_termination, int en_state_bound, int en_input_bound, int en_state_soc, int en_input_soc,
                         int en_state_linear, int en_input_linear, int en_tv_state_linear, int en_tv_input_linear);
int tiny_set_default_settings(TinySettings *settings);
int tiny_set_x0(TinySolver *solver, tinyVector x0);
int tiny_set_x_ref(TinySolver *solver, tinyMatrix x_ref);
int tiny_set_u_ref(TinySolver *solver, tinyMatrix u_ref);

void tiny_initialize_sensitivity_matrices(TinySolver *solver);  // tiny_api.hpp:54 (table data, see tinympc_shim.cpp)

// ---- admm.hpp:9-34 ----
int solve(TinySolver *solver);  // one whole ADMM solve on the GPU (tiny_solve forwards here, as in the reference)
// The stage functions are fused into the solve kernel; the symbols exist for link compatibility and abort with a message.
void update_linear_cost(TinySolver *solver);
void backward_pass_grad(TinySolver *solver);
void forward_pass(TinySolver *solver);
void update_slack(TinySolver *solver);
void update_dual(TinySolver *solver);
bool termination_condition(TinySolver *solver);

// ---- additions (not in the reference) ----
int tinympc_shim_sensitivity_tables(double *dKinf, double *dPinf, double *dC1, double *dC2);
int tiny_destroy(TinySolver *solver);  // the reference has no destroy function (leaks by design)
// Same problem, B instances: x0 is nx x B, Xref is (nx*N) x B (one column-major trajectory per column);
// cold start; outputs: u0 (nu x B) = first rollout input of every instance, iter/solved (B).
int tiny_solve_batch(TinySolver *solver, const tinyMatrix &x0, const tinyMatrix &Xref, tinyMatrix &u0, VectorXi &iter,
                     VectorXi &solved);

}  // extern "C"
