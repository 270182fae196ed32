/*
 * tests/adaptive/adaptive_impl.h — TEST INFRASTRUCTURE.  Included by adaptive_oracle.c once per T, right after
 * oracle/tinympc_oracle_impl.h (whose FN(work), stage functions and solve-loop helpers it uses).
 */
#define CAT_(a, b) a##b
#define CAT(a, b) CAT_(a, b)
#define FN(name) CAT(name, SUFFIX)

/* Eigen's maxCoeff of cwiseAbs(): res = (res < |v|) ? |v| : res  (res starts at 0, which no |v| lowers) */
#define AMAX(m, v)                 \
    do {                           \
        T a_ = FABS(v);            \
        if ((m) < a_) (m) = a_;    \
    } while (0)

/* One output of Eigen's column-major GEMV (GeneralMatrixVector.h:149-284) restricted to the nonzero columns of a row:
 * the row is a sum of column-block partials ((0 + blk0) + blk1) + ..., each partial an ascending c = a*b + c chain from 0,
 * blocks bw columns wide at absolute column indices.  The terms come in ascending column order; the skipped (structurally
 * zero) columns contribute products +-0, which change at most the sign of an exact-zero sum. */
typedef struct {
    T res, c;
    long blk, bw;
} FN(gemv_row);
static void FN(gr_init)(FN(gemv_row) * g, long bw) {
    g->res = 0;
    g->c = 0;
    g->blk = -1;
    g->bw = bw;
}
static void FN(gr_add)(FN(gemv_row) * g, long col, T prod) {
    const long b = col / g->bw;
    if (b != g->blk) {
        if (g->blk >= 0) g->res = g->res + g->c;
        g->c = 0;
        g->blk = b;
    }
    g->c = prod + g->c;
}
static T FN(gr_done)(FN(gemv_row) * g) { return g->blk >= 0 ? g->res + g->c : g->res; }

/* format_matrices + compute_residuals (rho_benchmark.cpp:47-188) for the iterates x (nx x N), u (nu x N-1) and
 * vnew, znew, g, y.  out = {pri_res, dual_res, pri_norm, dual_norm}. */
static void FN(adapt_residuals)(int nx, int nu, int N, const T *A, const T *B, const T *Qd, const T *Rd, const T *Pinf,
                                const T *x, const T *u, const T *vnew, const T *znew, const T *g, const T *y, T *out) {
    const long cols = (long)nx * N + (long)nu * (N - 1), rowsA = (long)(nx + nu) * (N - 1), S = nx + nu;
    const long bwA = cols < 128 ? cols : (rowsA * (long)sizeof(T) < 32000 ? 16 : 4);
    const long bwP = cols < 128 ? cols : (cols * (long)sizeof(T) < 32000 ? 16 : 4);
    T ax_m = 0, z_m = 0, rp_m = 0, px_m = 0, aty_m = 0, q_m = 0, rd_m = 0;
    /* A x - z: input rows (identity on u_k against znew_k), then dynamics rows A x_k + B u_k - x_{k+1} against vnew_{k+1} */
    for (int k = 0; k < N - 1; ++k)
        for (int j = 0; j < nu; ++j) {
            const T ax = u[(size_t)k * nu + j], z = znew[(size_t)k * nu + j];
            AMAX(ax_m, ax);
            AMAX(z_m, z);
            AMAX(rp_m, ax - z);
        }
    for (int k = 0; k < N - 1; ++k)
        for (int r = 0; r < nx; ++r) {
            FN(gemv_row) gr;
            FN(gr_init)(&gr, bwA);
            const long c0 = (long)k * S;
            for (int j = 0; j < nx; ++j) FN(gr_add)(&gr, c0 + j, A[r + (size_t)nx * j] * x[(size_t)k * nx + j]);
            for (int j = 0; j < nu; ++j) FN(gr_add)(&gr, c0 + nx + j, B[r + (size_t)nx * j] * u[(size_t)k * nu + j]);
            FN(gr_add)(&gr, c0 + S + r, (T)(-1) * x[(size_t)(k + 1) * nx + r]);
            const T ax = FN(gr_done)(&gr), z = vnew[(size_t)(k + 1) * nx + r];
            AMAX(ax_m, ax);
            AMAX(z_m, z);
            AMAX(rp_m, ax - z);
        }
    /* P x, q, A^T y and r_dual = (P x + q) + A^T y per decision element (x_k rows, then u_k rows) */
    for (int k = 0; k < N; ++k) {
        const long c0 = (long)k * S;
        for (int r = 0; r < nx; ++r) {
            const T xv = x[(size_t)k * nx + r];
            T px;
            if (k == N - 1) {
                FN(gemv_row) gr;
                FN(gr_init)(&gr, bwP);
                for (int j = 0; j < nx; ++j) FN(gr_add)(&gr, c0 + j, Pinf[r + (size_t)nx * j] * x[(size_t)k * nx + j]);
                px = FN(gr_done)(&gr);
            } else {
                px = Qd[r] * xv;
            }
            const T q = Qd[r] * xv;
            /* row-major GEMV (A^T y): one ascending chain over the rows of A from 0 */
            T aty = 0;
            if (k >= 1) aty = ((T)(-1) * g[(size_t)k * nx + r]) + aty;
            if (k <= N - 2)
                for (int i = 0; i < nx; ++i) aty = (A[i + (size_t)nx * r] * g[(size_t)(k + 1) * nx + i]) + aty;
            AMAX(px_m, px);
            AMAX(q_m, q);
            AMAX(aty_m, aty);
            AMAX(rd_m, (px + q) + aty);
        }
        if (k == N - 1) break;
        for (int j = 0; j < nu; ++j) {
            const T uv = u[(size_t)k * nu + j];
            const T px = Rd[j] * uv, q = Rd[j] * uv;
            T aty = 0;
            aty = ((T)1 * y[(size_t)k * nu + j]) + aty;
            for (int i = 0; i < nx; ++i) aty = (B[i + (size_t)nx * j] * g[(size_t)(k + 1) * nx + i]) + aty;
            AMAX(px_m, px);
            AMAX(q_m, q);
            AMAX(aty_m, aty);
            AMAX(rd_m, (px + q) + aty);
        }
    }
    out[0] = rp_m;
    out[1] = rd_m;
    out[2] = (ax_m < z_m) ? z_m : ax_m;                                  /* std::max(a, b) = (a < b) ? b : a */
    {
        const T m1 = (px_m < aty_m) ? aty_m : px_m;
        out[3] = (m1 < q_m) ? q_m : m1;
    }
}

/* predict_rho (rho_benchmark.cpp:190-213) */
static T FN(predict_rho)(const T *res, T rho, int clip, T rho_min, T rho_max) {
    const T eps = (T)1e-10;
    const T np = res[0] / (res[2] + eps);
    const T nd = res[1] / (res[3] + eps);
    const T ratio = np / (nd + eps);
    T nr = rho * SQRT(ratio);
    if (clip) {
        nr = (nr < rho_min) ? rho_min : nr; /* std::max(nr, rho_min) */
        nr = (rho_max < nr) ? rho_max : nr; /* std::min(nr, rho_max) */
    }
    return nr;
}

/* update_matrices_with_derivatives (rho_benchmark.cpp:215-229) */
static void FN(update_with_derivatives)(int nx, int nu, T *Kinf, T *Pinf, T *rho, const T *dK, const T *dP, T new_rho) {
    const T delta = new_rho - *rho;
    for (int e = 0; e < nu * nx; ++e) Kinf[e] = Kinf[e] + delta * dK[e];
    for (int e = 0; e < nx * nx; ++e) Pinf[e] = Pinf[e] + delta * dP[e];
    *rho = new_rho;
}

/* admm.cpp:331-455 with adaptive rho on (box constraints); the adapted rho / Kinf / Pinf are in *pr / Kinf / Pinf */
static int FN(solve_one_adaptive)(tinympc_problem_t *pr, const tinympc_settings_t *st, FN(work) * w, T *Kinf, T *Pinf,
                                  const T *dK, const T *dP, int clip, T rho_min, T rho_max) {
    const int nx = pr->nx, nu = pr->nu, N = pr->N;
    const size_t nN = (size_t)nx * N, mN = (size_t)nu * (N - 1);
    w->solved = 0;
    w->iter = 0;
    w->status = 11;
    for (int i = 0; i < st->max_iter; ++i) {
        FN(update_linear_cost)(pr, st, w);
        FN(backward_pass)(pr, w);
        FN(forward_pass)(pr, w);
        FN(update_slack)(pr, st, w);
        FN(update_dual)(pr, st, w);
        w->iter += 1;
        if (i > 0 && i % 5 == 0) {
            T res[4], rho = (T)pr->rho;
            FN(adapt_residuals)(nx, nu, N, (const T *)pr->Adyn, (const T *)pr->Bdyn, (const T *)pr->Q, (const T *)pr->R, Pinf,
                                w->x, w->u, w->vnew, w->znew, w->g, w->y, res);
            const T nr = FN(predict_rho)(res, rho, clip, rho_min, rho_max);
            FN(update_with_derivatives)(nx, nu, Kinf, Pinf, &rho, dK, dP, nr); /* rho_benchmark.cpp:240 */
            FN(update_with_derivatives)(nx, nu, Kinf, Pinf, &rho, dK, dP, nr); /* admm.cpp:421 */
            pr->rho = (double)rho;
        }
        if (FN(termination)(pr, st, w)) {
            w->status = 1;
            w->solved = 1;
            return 0;
        }
        memcpy(w->v, w->vnew, sizeof(T) * nN);
        memcpy(w->z, w->znew, sizeof(T) * mN);
    }
    w->solved = 0;
    return 1;
}

static int FN(adaptive_solve_batch)(const tinympc_problem_t *pr0, const tinympc_settings_t *st, const tinympc_batch_t *io,
                                    const tinympc_adaptive_rho_t *ar, int nthreads) {
    const int nx = pr0->nx, nu = pr0->nu, N = pr0->N;
    const size_t nN = (size_t)nx * N, mN = (size_t)nu * (N - 1);
    if (nx > 64 || nu > 64) return -1;
    /* model blob layout (tinympc_b200/csrc/model_blob.h) */
    const size_t oA = 0, oB = oA + (size_t)nx * nx, of = oB + (size_t)nx * nu, oQ = of + nx, oR = oQ + nx, oK = oR + nu;
    const size_t oP = oK + (size_t)nu * nx, oQuu = oP + (size_t)nx * nx, oAm = oQuu + (size_t)nu * nu, oAPf = oAm + (size_t)nx * nx;
    const size_t oBPf = oAPf + nx, orho = oBPf + nu, blob = orho + 1;
    const T *dK = (const T *)ar->dKinf_drho, *dP = (const T *)ar->dPinf_drho;
    const T rho_min = (T)ar->rho_min, rho_max = (T)ar->rho_max;
    const int clip = ar->enable_clipping != 0;
    if (nthreads < 1) nthreads = 1;
#pragma omp parallel num_threads(nthreads)
    {
        T *buf = (T *)malloc(sizeof(T) * (14 * nN + 12 * mN));
        FN(work) w;
        T *c = buf;
#define TAKE(field, n) w.field = c; c += (n)
        TAKE(x, nN); TAKE(q, nN); TAKE(p, nN); TAKE(v, nN); TAKE(vnew, nN); TAKE(g, nN);
        TAKE(vcnew, nN); TAKE(gc, nN); TAKE(vlnew, nN); TAKE(gl, nN); TAKE(vlnew_tv, nN); TAKE(gl_tv, nN);
        TAKE(Xref, nN); c += nN;
        TAKE(u, mN); TAKE(r, mN); TAKE(d, mN); TAKE(z, mN); TAKE(znew, mN); TAKE(y, mN);
        TAKE(zcnew, mN); TAKE(yc, mN); TAKE(zlnew, mN); TAKE(yl, mN); TAKE(zlnew_tv, mN); TAKE(yl_tv, mN);
#undef TAKE
        T *Uref_buf = (T *)malloc(sizeof(T) * (mN ? mN : 1));
        w.Uref = Uref_buf;
        const tinympc_state_t *S = &io->state;
        const int cold = io->cold_start != 0;
#pragma omp for schedule(static)
        for (int64_t b = 0; b < io->B; ++b) {
            T *mb = (T *)ar->models + (size_t)b * blob;
            tinympc_problem_t pr = *pr0;
            pr.Adyn = mb + oA; pr.Bdyn = mb + oB; pr.fdyn = mb + of; pr.Q = mb + oQ; pr.R = mb + oR;
            pr.Kinf = mb + oK; pr.Pinf = mb + oP; pr.Quu_inv = mb + oQuu; pr.AmBKt = mb + oAm; pr.APf = mb + oAPf; pr.BPf = mb + oBPf;
            pr.rho = (double)mb[orho];
            FN(ld)(w.x, cold ? NULL : S->x, b, nN);
            FN(ld)(w.u, cold ? NULL : S->u, b, mN);
            FN(ld)(w.v, cold ? NULL : S->v, b, nN);
            FN(ld)(w.z, cold ? NULL : S->z, b, mN);
            FN(ld)(w.vnew, cold ? NULL : S->vnew, b, nN);
            FN(ld)(w.znew, cold ? NULL : S->znew, b, mN);
            FN(ld)(w.g, cold ? NULL : S->g, b, nN);
            FN(ld)(w.y, cold ? NULL : S->y, b, mN);
            FN(ld)(w.Xref, io->Xref, io->xref_per_instance ? b : 0, nN);
            FN(ld)(w.Uref, io->Uref, io->uref_per_instance ? b : 0, mN);
            memset(w.q, 0, sizeof(T) * nN);
            memset(w.p, 0, sizeof(T) * nN);
            w.pri_x = w.dua_x = w.pri_u = w.dua_u = 0;
            memcpy(w.x, (const T *)io->x0 + (size_t)b * nx, sizeof(T) * nx);

            FN(solve_one_adaptive)(&pr, st, &w, mb + oK, mb + oP, dK, dP, clip, rho_min, rho_max);
            mb[orho] = (T)pr.rho;

            FN(st)(io->sol_x, b, w.vnew, nN);
            FN(st)(io->sol_u, b, w.znew, mN);
            if (io->iter) io->iter[b] = w.iter;
            if (io->solved) io->solved[b] = w.solved;
            if (io->residuals) {
                T *rr = (T *)io->residuals + 4 * (size_t)b;
                rr[0] = w.pri_x; rr[1] = w.dua_x; rr[2] = w.pri_u; rr[3] = w.dua_u;
            }
            if (io->u0) memcpy((T *)io->u0 + (size_t)b * nu, w.u, sizeof(T) * nu);
            FN(st)(S->x, b, w.x, nN);
            FN(st)(S->u, b, w.u, mN);
            FN(st)(S->v, b, w.v, nN);
            FN(st)(S->z, b, w.z, mN);
            FN(st)(S->vnew, b, w.vnew, nN);
            FN(st)(S->znew, b, w.znew, mN);
            FN(st)(S->g, b, w.g, nN);
            FN(st)(S->y, b, w.y, mN);
        }
        free(buf);
        free(Uref_buf);
    }
    return 0;
}

#undef AMAX
#undef FN
#undef CAT
#undef CAT_
