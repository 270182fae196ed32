/*
 * tests/adaptive/adaptive_oracle.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C restatement of the reference's adaptive-rho solve (admm.cpp:331-455 with the branch :397-423, and
 * rho_benchmark.cpp), with the RhoAdapter value-initialised (the reference leaves it uninitialised: admm.cpp:340,
 * read at rho_benchmark.cpp:56).  The stage functions are the pinned restatement's (oracle/tinympc_oracle_impl.h,
 * included unchanged); this file adds the residuals of format_matrices / compute_residuals in Eigen's summation order
 * (GeneralMatrixVector.h), predict_rho and update_matrices_with_derivatives.
 *
 * Compiled by the tests (tests/adaptive_common.py) with  gcc -O2 -ffp-contract=off -fopenmp -shared -fPIC.
 * tests/adaptive/ref_adaptive_driver.cpp runs the same loop on the compiled reference; the golden fixtures
 * fixtures under tests/golden/adaptive hold its outputs.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "tinympc_b200.h"

#define T double
#define SUFFIX _f64
#define SQRT sqrt
#define FABS fabs
#include "tinympc_oracle_impl.h"
#include "adaptive_impl.h"
#undef T
#undef SUFFIX
#undef SQRT
#undef FABS

#define T float
#define SUFFIX _f32
#define SQRT sqrtf
#define FABS fabsf
#include "tinympc_oracle_impl.h"
#include "adaptive_impl.h"
#undef T
#undef SUFFIX
#undef SQRT
#undef FABS

/* Batched adaptive-rho solve on host buffers; same contract as tinympc_b200_solve_adaptive_host.  Only the box-constraint
 * state fields (x, u, v, z, vnew, znew, g, y) are read and written. */
int tinympc_adaptive_oracle_solve_batch(const tinympc_problem_t *pr, const tinympc_settings_t *st, const tinympc_batch_t *io,
                                        const tinympc_adaptive_rho_t *ar, int32_t nthreads) {
    if (!pr || !st || !io || !ar || !io->x0 || !io->Xref || !ar->models || !ar->dKinf_drho || !ar->dPinf_drho) return TINYMPC_ERR_ARG;
    if (pr->dtype == TINYMPC_F64) return adaptive_solve_batch_f64(pr, st, io, ar, nthreads);
    if (pr->dtype == TINYMPC_F32) return adaptive_solve_batch_f32(pr, st, io, ar, nthreads);
    return TINYMPC_ERR_ARG;
}

/* The residual quadruple of one compute_residuals call (pri, dual, pri_norm, dual_norm) for the given iterates, so that the
 * tests can pin the summation order on its own. */
int tinympc_adaptive_oracle_residuals(int32_t dtype, int32_t nx, int32_t nu, int32_t N, const void *A, const void *B,
                                      const void *Qd, const void *Rd, const void *Pinf, const void *x, const void *u,
                                      const void *vnew, const void *znew, const void *g, const void *y, double *out4) {
    if (dtype == TINYMPC_F64) {
        double r[4];
        adapt_residuals_f64(nx, nu, N, A, B, Qd, Rd, Pinf, x, u, vnew, znew, g, y, r);
        for (int i = 0; i < 4; ++i) out4[i] = r[i];
        return 0;
    }
    if (dtype == TINYMPC_F32) {
        float r[4];
        adapt_residuals_f32(nx, nu, N, A, B, Qd, Rd, Pinf, x, u, vnew, znew, g, y, r);
        for (int i = 0; i < 4; ++i) out4[i] = r[i];
        return 0;
    }
    return TINYMPC_ERR_ARG;
}
