/*
 * tests/adaptive/adaptive_oracle_per_instance.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The adaptive-rho restatement of adaptive_oracle.c (included unchanged) for per-instance sensitivity tables
 * (tinympc_adaptive_rho_t.tables_per_instance = 1: dKinf_drho [B][nu*nx], dPinf_drho [B][nx*nx], host pointers): instance b is
 * solved by the shared-table entry point as a batch of one, with its own table pair.  tables_per_instance = 0 passes the one
 * shared pair to every instance, which must reproduce tinympc_adaptive_oracle_solve_batch bit for bit.
 *
 * Compiled by the tests (tests/sensitivity_common.py) with the flags of adaptive_oracle.c.
 */
#include "adaptive_oracle.c"

int tinympc_adaptive_oracle_solve_batch_per_instance(const tinympc_problem_t *pr, const tinympc_settings_t *st,
                                                     const tinympc_batch_t *io, const tinympc_adaptive_rho_t *ar) {
    if (!pr || !st || !io || !ar || !io->x0 || !io->Xref || !ar->models || !ar->dKinf_drho || !ar->dPinf_drho) return TINYMPC_ERR_ARG;
    if (pr->dtype != TINYMPC_F64 && pr->dtype != TINYMPC_F32) return TINYMPC_ERR_ARG;
    const size_t es = pr->dtype == TINYMPC_F64 ? 8 : 4;
    const size_t nx = pr->nx, nu = pr->nu, nN = nx * pr->N, mN = nu * (pr->N - 1);
    const size_t blob = 3 * nx * nx + 2 * nx * nu + nu * nu + 3 * nx + 2 * nu + 1; /* tinympc_b200/csrc/model_blob.h */
    int rc = 0;
#pragma omp parallel for schedule(static)
    for (int64_t b = 0; b < io->B; ++b) {
        /* instance b of a [B][n] array of elements es bytes wide (NULL stays NULL) */
#define AT(p, n, es_) ((p) ? (void *)((char *)(p) + (size_t)b * (n) * (es_)) : NULL)
        tinympc_batch_t one = *io;
        one.B = 1;
        one.x0 = AT(io->x0, nx, es);
        if (io->xref_per_instance) one.Xref = AT(io->Xref, nN, es);
        if (io->uref_per_instance) one.Uref = AT(io->Uref, mN, es);
        void *const *src = (void *const *)&io->state;
        void **dst = (void **)&one.state;
        for (size_t i = 0; i < sizeof(tinympc_state_t) / sizeof(void *); ++i)
            dst[i] = AT(src[i], (i % 2 == 0) ? nN : mN, es); /* x, v, vnew, g, ... alternate with u, z, znew, y, ... */
        one.sol_x = AT(io->sol_x, nN, es);
        one.sol_u = AT(io->sol_u, mN, es);
        one.iter = (int32_t *)AT(io->iter, 1, sizeof(int32_t));
        one.solved = (int32_t *)AT(io->solved, 1, sizeof(int32_t));
        one.residuals = AT(io->residuals, 4, es);
        one.u0 = AT(io->u0, nu, es);
        tinympc_adaptive_rho_t a1 = *ar;
        a1.models = AT(ar->models, blob, es);
        a1.tables_per_instance = 0;
        if (ar->tables_per_instance) {
            a1.dKinf_drho = AT(ar->dKinf_drho, nu * nx, es);
            a1.dPinf_drho = AT(ar->dPinf_drho, nx * nx, es);
        }
#undef AT
        if (tinympc_adaptive_oracle_solve_batch(pr, st, &one, &a1, 1)) {
#pragma omp atomic write
            rc = TINYMPC_ERR_ARG;
        }
    }
    return rc;
}
