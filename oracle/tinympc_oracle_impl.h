/*
 * oracle/tinympc_oracle_impl.h — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C CPU restatement of the reference's solve path, included twice by tinympc_oracle.c
 * (once with T = double, once with T = float).  Each function cites the reference lines it follows
 * (paths relative to the TinyMPC checkout).  Arithmetic contract (SURVEY Appendix A/B.2, validated there
 * and re-validated by tests/test_oracle_vs_reference.py against oracle/_ref):
 *   - every dot product is  s = a0*b0; s = s + ak*bk  for k ascending, separate multiply and add
 *     (compile with -ffp-contract=off);
 *   - Eigen expression association is preserved left to right;
 *   - box clamp: m = (lo < a) ? a : lo;  r = (m < hi) ? m : hi;
 *   - project_soc narrows mu and the norm to float even when T is double.
 * It is bit-identical to the reference built with
 *   -O3 -DNDEBUG -DEIGEN_DONT_VECTORIZE -ffp-contract=off      (the "pinned" oracle build, oracle/Makefile).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may use this.
 */

#define CAT_(a, b) a##b
#define CAT(a, b) CAT_(a, b)
#define FN(name) CAT(name, SUFFIX)

typedef struct {
    /* per-instance arrays, column-major nx x N / nu x (N-1) */
    T *x, *u, *q, *r, *p, *d, *v, *vnew, *z, *znew, *g, *y;
    T *vcnew, *zcnew, *gc, *yc;
    T *vlnew, *zlnew, *gl, *yl;
    T *vlnew_tv, *zlnew_tv, *gl_tv, *yl_tv;
    T *Xref, *Uref;
    T pri_x, dua_x, pri_u, dua_u;
    int iter, solved, status;
} FN(work);

/* admm.cpp:39-60 exactly as executed (SURVEY A.4); only 3-dimensional cones are defined */
static void FN(project_soc3)(T *s, T mu_T) {
    float mu = (float)mu_T;              /* parameter type is float (admm.cpp:39)          */
    T u0 = s[2] * (T)mu;                 /* tinytype * float -> tinytype       (:40)        */
    T sq = s[0] * s[0];
    sq = sq + s[1] * s[1];
    float a = (float)SQRT(sq);           /* float a = u1.norm()                (:42)        */
    if ((T)a <= -u0) {                   /* below cone                          (:46)        */
        s[0] = 0; s[1] = 0; s[2] = 0;
        return;
    }
    if ((T)a <= u0) return;              /* in cone                             (:49)        */
    {
        T third = (T)(a / mu);           /* float division                      (:54)        */
        T c = (T)0.5 * ((T)1 + u0 / (T)a);   /* (:55) */
        s[0] = c * s[0];
        s[1] = c * s[1];
        s[2] = c * third;
    }
}

static T FN(dot)(const T *a, int sa, const T *b, int sb, int n) {
    T s = a[0] * b[0];
    for (int k = 1; k < n; ++k) s = s + a[(size_t)k * sa] * b[(size_t)k * sb];
    return s;
}

/* admm.cpp:70-73,148-157 (SURVEY A.5): sequential projections, row k of A (rows x n, column-major, ld = lda) */
static void FN(project_rows)(T *zcol, int n, const T *A, int lda, int row0, int nrows, const T *b, int sb) {
    for (int k = 0; k < nrows; ++k) {
        const T *a = A + row0 + k; /* element j at a[j*lda] */
        T cv = FN(dot)(a, lda, zcol, 1, n);
        if (cv > b[(size_t)k * sb]) {
            T num = FN(dot)(a, lda, zcol, 1, n) - b[(size_t)k * sb];
            T den = FN(dot)(a, lda, a, lda, n);
            T dist = num / den;
            for (int j = 0; j < n; ++j) zcol[j] = zcol[j] - dist * a[(size_t)j * lda];
        }
    }
}

/* admm.cpp:262-304 */
static void FN(update_linear_cost)(const tinympc_problem_t *pr, const tinympc_settings_t *st, FN(work) * w) {
    const int nx = pr->nx, nu = pr->nu, N = pr->N;
    const T rho = (T)pr->rho;
    const T *Q = (const T *)pr->Q, *R = (const T *)pr->R, *Pinf = (const T *)pr->Pinf;
    const int soc_x = st->en_state_soc && pr->num_state_cones > 0;
    const int soc_u = st->en_input_soc && pr->num_input_cones > 0;
    for (int k = 0; k < N; ++k)
        for (int i = 0; i < nx; ++i) {
            size_t e = (size_t)k * nx + i;
            T qv = -(w->Xref[e] * Q[i]);
            qv = qv - rho * (w->vnew[e] - w->g[e]);
            if (soc_x) qv = qv - rho * (w->vcnew[e] - w->gc[e]);
            if (st->en_state_linear) qv = qv - rho * (w->vlnew[e] - w->gl[e]);
            if (st->en_tv_state_linear) qv = qv - rho * (w->vlnew_tv[e] - w->gl_tv[e]);
            w->q[e] = qv;
        }
    for (int k = 0; k < N - 1; ++k)
        for (int j = 0; j < nu; ++j) {
            size_t e = (size_t)k * nu + j;
            T rv = -(w->Uref[e] * R[j]);
            rv = rv - rho * (w->znew[e] - w->y[e]);
            if (soc_u) rv = rv - rho * (w->zcnew[e] - w->yc[e]);
            if (st->en_input_linear) rv = rv - rho * (w->zlnew[e] - w->yl[e]);
            if (st->en_tv_input_linear) rv = rv - rho * (w->zlnew_tv[e] - w->yl_tv[e]);
            w->r[e] = rv;
        }
    {
        const size_t c = (size_t)(N - 1) * nx;
        for (int j = 0; j < nx; ++j) {
            size_t e = c + j;
            T pv = -FN(dot)(w->Xref + c, 1, Pinf + (size_t)j * nx, 1, nx); /* (Xref_col^T * Pinf)(j) */
            pv = pv - rho * (w->vnew[e] - w->g[e]);
            if (soc_x) pv = pv - rho * (w->vcnew[e] - w->gc[e]);
            if (st->en_state_linear) pv = pv - rho * (w->vlnew[e] - w->gl[e]);
            if (st->en_tv_state_linear) pv = pv - rho * (w->vlnew_tv[e] - w->gl_tv[e]);
            w->p[e] = pv;
        }
    }
}

/* admm.cpp:13-20 */
static void FN(backward_pass)(const tinympc_problem_t *pr, FN(work) * w) {
    const int nx = pr->nx, nu = pr->nu, N = pr->N;
    const T *B = (const T *)pr->Bdyn, *Quu = (const T *)pr->Quu_inv, *AmBKt = (const T *)pr->AmBKt;
    const T *Kinf = (const T *)pr->Kinf, *APf = (const T *)pr->APf, *BPf = (const T *)pr->BPf;
    T s[64];
    for (int k = N - 2; k >= 0; --k) {
        const T *pn = w->p + (size_t)(k + 1) * nx;
        const T *rk = w->r + (size_t)k * nu;
        for (int j = 0; j < nu; ++j) {
            T t = FN(dot)(B + (size_t)j * nx, 1, pn, 1, nx); /* (B^T p)(j) */
            s[j] = (t + rk[j]) + BPf[j];
        }
        for (int j = 0; j < nu; ++j) w->d[(size_t)k * nu + j] = FN(dot)(Quu + j, nu, s, 1, nu);
        for (int i = 0; i < nx; ++i) {
            T a = FN(dot)(AmBKt + i, nx, pn, 1, nx);
            T kr = FN(dot)(Kinf + (size_t)i * nu, 1, rk, 1, nu); /* (Kinf^T r)(i) = sum_j Kinf(j,i) r_j */
            w->p[(size_t)k * nx + i] = ((w->q[(size_t)k * nx + i] + a) - kr) + APf[i];
        }
    }
}

/* admm.cpp:25-32 */
static void FN(forward_pass)(const tinympc_problem_t *pr, FN(work) * w) {
    const int nx = pr->nx, nu = pr->nu, N = pr->N;
    const T *A = (const T *)pr->Adyn, *B = (const T *)pr->Bdyn, *f = (const T *)pr->fdyn;
    const T *Kinf = (const T *)pr->Kinf;
    for (int k = 0; k < N - 1; ++k) {
        const T *xk = w->x + (size_t)k * nx;
        T *uk = w->u + (size_t)k * nu;
        for (int j = 0; j < nu; ++j) uk[j] = (-FN(dot)(Kinf + j, nu, xk, 1, nx)) - w->d[(size_t)k * nu + j];
        for (int i = 0; i < nx; ++i) {
            T ax = FN(dot)(A + i, nx, xk, 1, nx);
            T bu = FN(dot)(B + i, nx, uk, 1, nu);
            w->x[(size_t)(k + 1) * nx + i] = (ax + bu) + f[i];
        }
    }
}

/* admm.cpp:81-213 */
static void FN(update_slack)(const tinympc_problem_t *pr, const tinympc_settings_t *st, FN(work) * w) {
    const int nx = pr->nx, nu = pr->nu, N = pr->N;
    const size_t nN = (size_t)nx * N, mN = (size_t)nu * (N - 1);
    for (size_t e = 0; e < nN; ++e) w->vnew[e] = w->x[e] + w->g[e];
    for (size_t e = 0; e < mN; ++e) w->znew[e] = w->u[e] + w->y[e];
    if (st->en_state_bound) {
        const T *lo = (const T *)pr->x_min, *hi = (const T *)pr->x_max;
        for (size_t e = 0; e < nN; ++e) {
            T m = (lo[e] < w->vnew[e]) ? w->vnew[e] : lo[e];
            w->vnew[e] = (m < hi[e]) ? m : hi[e];
        }
    }
    if (st->en_input_bound) {
        const T *lo = (const T *)pr->u_min, *hi = (const T *)pr->u_max;
        for (size_t e = 0; e < mN; ++e) {
            T m = (lo[e] < w->znew[e]) ? w->znew[e] : lo[e];
            w->znew[e] = (m < hi[e]) ? m : hi[e];
        }
    }
    if (st->en_state_soc && pr->num_state_cones > 0)
        for (size_t e = 0; e < nN; ++e) w->vcnew[e] = w->x[e] + w->gc[e];
    if (st->en_input_soc && pr->num_input_cones > 0)
        for (size_t e = 0; e < mN; ++e) w->zcnew[e] = w->u[e] + w->yc[e];
    if (st->en_state_soc)
        for (int k = 0; k < N; ++k)
            for (int c = 0; c < pr->num_state_cones; ++c)
                FN(project_soc3)(w->vcnew + (size_t)k * nx + pr->Acx[c], ((const T *)pr->cx)[c]);
    if (st->en_input_soc)
        for (int k = 0; k < N - 1; ++k)
            for (int c = 0; c < pr->num_input_cones; ++c)
                FN(project_soc3)(w->zcnew + (size_t)k * nu + pr->Acu[c], ((const T *)pr->cu)[c]);
    if (st->en_state_linear) {
        for (size_t e = 0; e < nN; ++e) w->vlnew[e] = w->x[e] + w->gl[e];
    }
    if (st->en_input_linear) {
        for (size_t e = 0; e < mN; ++e) w->zlnew[e] = w->u[e] + w->yl[e];
    }
    if (st->en_state_linear)
        for (int k = 0; k < N; ++k)
            FN(project_rows)(w->vlnew + (size_t)k * nx, nx, (const T *)pr->Alin_x, pr->num_state_linear, 0,
                             pr->num_state_linear, (const T *)pr->blin_x, 1);
    if (st->en_input_linear)
        for (int k = 0; k < N - 1; ++k)
            FN(project_rows)(w->zlnew + (size_t)k * nu, nu, (const T *)pr->Alin_u, pr->num_input_linear, 0,
                             pr->num_input_linear, (const T *)pr->blin_u, 1);
    if (st->en_tv_state_linear) {
        for (size_t e = 0; e < nN; ++e) w->vlnew_tv[e] = w->x[e] + w->gl_tv[e];
    }
    if (st->en_tv_input_linear) {
        for (size_t e = 0; e < mN; ++e) w->zlnew_tv[e] = w->u[e] + w->yl_tv[e];
    }
    if (st->en_tv_state_linear) {
        const int n = pr->num_tv_state_linear;
        for (int k = 0; k < N; ++k)
            FN(project_rows)(w->vlnew_tv + (size_t)k * nx, nx, (const T *)pr->tv_Alin_x, n * N, n * k, n,
                             (const T *)pr->tv_blin_x + (size_t)k * n, 1);
    }
    if (st->en_tv_input_linear) {
        const int n = pr->num_tv_input_linear;
        for (int k = 0; k < N - 1; ++k)
            FN(project_rows)(w->zlnew_tv + (size_t)k * nu, nu, (const T *)pr->tv_Alin_u, n * (N - 1), n * k, n,
                             (const T *)pr->tv_blin_u + (size_t)k * n, 1);
    }
}

/* admm.cpp:219-256 */
static void FN(update_dual)(const tinympc_problem_t *pr, const tinympc_settings_t *st, FN(work) * w) {
    const size_t nN = (size_t)pr->nx * pr->N, mN = (size_t)pr->nu * (pr->N - 1);
    for (size_t e = 0; e < nN; ++e) w->g[e] = (w->g[e] + w->x[e]) - w->vnew[e];
    for (size_t e = 0; e < mN; ++e) w->y[e] = (w->y[e] + w->u[e]) - w->znew[e];
    if (st->en_state_soc && pr->num_state_cones > 0)
        for (size_t e = 0; e < nN; ++e) w->gc[e] = (w->gc[e] + w->x[e]) - w->vcnew[e];
    if (st->en_input_soc && pr->num_input_cones > 0)
        for (size_t e = 0; e < mN; ++e) w->yc[e] = (w->yc[e] + w->u[e]) - w->zcnew[e];
    if (st->en_state_linear)
        for (size_t e = 0; e < nN; ++e) w->gl[e] = (w->gl[e] + w->x[e]) - w->vlnew[e];
    if (st->en_input_linear)
        for (size_t e = 0; e < mN; ++e) w->yl[e] = (w->yl[e] + w->u[e]) - w->zlnew[e];
    if (st->en_tv_state_linear)
        for (size_t e = 0; e < nN; ++e) w->gl_tv[e] = (w->gl_tv[e] + w->x[e]) - w->vlnew_tv[e];
    if (st->en_tv_input_linear)
        for (size_t e = 0; e < mN; ++e) w->yl_tv[e] = (w->yl_tv[e] + w->u[e]) - w->zlnew_tv[e];
}

static T FN(max_abs_diff)(const T *a, const T *b, size_t n) {
    T m = FABS(a[0] - b[0]);
    for (size_t e = 1; e < n; ++e) {
        T d = FABS(a[e] - b[e]);
        if (d > m) m = d;
    }
    return m;
}

/* admm.cpp:310-328 */
static int FN(termination)(const tinympc_problem_t *pr, const tinympc_settings_t *st, FN(work) * w) {
    const size_t nN = (size_t)pr->nx * pr->N, mN = (size_t)pr->nu * (pr->N - 1);
    if (w->iter % st->check_termination == 0) {
        const T rho = (T)pr->rho;
        w->pri_x = FN(max_abs_diff)(w->x, w->vnew, nN);
        w->dua_x = FN(max_abs_diff)(w->v, w->vnew, nN) * rho;
        w->pri_u = FN(max_abs_diff)(w->u, w->znew, mN);
        w->dua_u = FN(max_abs_diff)(w->z, w->znew, mN) * rho;
        if (w->pri_x < (T)st->abs_pri_tol && w->pri_u < (T)st->abs_pri_tol && w->dua_x < (T)st->abs_dua_tol &&
            w->dua_u < (T)st->abs_dua_tol)
            return 1;
    }
    return 0;
}

/* admm.cpp:331-455 (adaptive-rho branch :397-423 omitted: disabled by default and out of scope) */
static int FN(solve_one)(const tinympc_problem_t *pr, const tinympc_settings_t *st, FN(work) * w) {
    const size_t nN = (size_t)pr->nx * pr->N, mN = (size_t)pr->nu * (pr->N - 1);
    w->solved = 0;
    w->iter = 0;
    w->status = 11;
    if (st->en_state_soc && pr->num_state_cones > 0) memcpy(w->vcnew, w->x, sizeof(T) * nN);
    if (st->en_input_soc && pr->num_input_cones > 0) memcpy(w->zcnew, w->u, sizeof(T) * mN);
    if (st->en_state_linear) memcpy(w->vlnew, w->x, sizeof(T) * nN);
    if (st->en_input_linear) memcpy(w->zlnew, w->u, sizeof(T) * mN);
    if (st->en_tv_state_linear) memcpy(w->vlnew_tv, w->x, sizeof(T) * nN);
    if (st->en_tv_input_linear) memcpy(w->zlnew_tv, w->u, sizeof(T) * mN);
    for (int i = 0; i < st->max_iter; ++i) {
        FN(update_linear_cost)(pr, st, w);
        FN(backward_pass)(pr, w);
        FN(forward_pass)(pr, w);
        FN(update_slack)(pr, st, w);
        FN(update_dual)(pr, st, w);
        w->iter += 1;
        if (FN(termination)(pr, st, w)) {
            w->status = 1;
            w->solved = 1;
            return 0; /* returns BEFORE v = vnew (admm.cpp:441 precedes :445) */
        }
        memcpy(w->v, w->vnew, sizeof(T) * nN);
        memcpy(w->z, w->znew, sizeof(T) * mN);
    }
    w->solved = 0;
    return 1;
}

static void FN(ld)(T *dst, const void *base, int64_t b, size_t n) {
    if (base)
        memcpy(dst, (const T *)base + (size_t)b * n, sizeof(T) * n);
    else
        memset(dst, 0, sizeof(T) * n);
}
static void FN(st)(void *base, int64_t b, const T *src, size_t n) {
    if (base) memcpy((T *)base + (size_t)b * n, src, sizeof(T) * n);
}

static int FN(solve_batch)(const tinympc_problem_t *pr, const tinympc_settings_t *st, const tinympc_batch_t *io,
                           int nthreads) {
    const int nx = pr->nx, nu = pr->nu, N = pr->N;
    const size_t nN = (size_t)nx * N, mN = (size_t)nu * (N - 1);
    if (nx > 64 || nu > 64) return -1;
    for (int c = 0; c < pr->num_state_cones; ++c)
        if (pr->qcx[c] != 3) return TINYMPC_ERR_CONE_DIM;
    for (int c = 0; c < pr->num_input_cones; ++c)
        if (pr->qcu[c] != 3) return TINYMPC_ERR_CONE_DIM;
    if (nthreads < 1) nthreads = 1;
    int rc = 0;
#pragma omp parallel num_threads(nthreads)
    {
        const size_t total = 14 * nN + 12 * mN;
        T *buf = (T *)malloc(sizeof(T) * total);
        FN(work) w;
        T *c = buf;
#define TAKE(field, n) w.field = c; c += (n)
        TAKE(x, nN); TAKE(q, nN); TAKE(p, nN); TAKE(v, nN); TAKE(vnew, nN); TAKE(g, nN);
        TAKE(vcnew, nN); TAKE(gc, nN); TAKE(vlnew, nN); TAKE(gl, nN); TAKE(vlnew_tv, nN); TAKE(gl_tv, nN);
        TAKE(Xref, nN); c += nN; /* spare */
        TAKE(u, mN); TAKE(r, mN); TAKE(d, mN); TAKE(z, mN); TAKE(znew, mN); TAKE(y, mN);
        TAKE(zcnew, mN); TAKE(yc, mN); TAKE(zlnew, mN); TAKE(yl, mN); TAKE(zlnew_tv, mN); TAKE(yl_tv, mN);
#undef TAKE
        T *Uref_buf = (T *)malloc(sizeof(T) * (mN ? mN : 1));
        w.Uref = Uref_buf;
        const tinympc_state_t *S = &io->state;
        const int cold = io->cold_start != 0;
#pragma omp for schedule(static)
        for (int64_t b = 0; b < io->B; ++b) {
            FN(ld)(w.x, cold ? NULL : S->x, b, nN);
            FN(ld)(w.u, cold ? NULL : S->u, b, mN);
            FN(ld)(w.v, cold ? NULL : S->v, b, nN);
            FN(ld)(w.z, cold ? NULL : S->z, b, mN);
            FN(ld)(w.vnew, cold ? NULL : S->vnew, b, nN);
            FN(ld)(w.znew, cold ? NULL : S->znew, b, mN);
            FN(ld)(w.g, cold ? NULL : S->g, b, nN);
            FN(ld)(w.y, cold ? NULL : S->y, b, mN);
            FN(ld)(w.vcnew, cold ? NULL : S->vcnew, b, nN);
            FN(ld)(w.zcnew, cold ? NULL : S->zcnew, b, mN);
            FN(ld)(w.gc, cold ? NULL : S->gc, b, nN);
            FN(ld)(w.yc, cold ? NULL : S->yc, b, mN);
            FN(ld)(w.vlnew, cold ? NULL : S->vlnew, b, nN);
            FN(ld)(w.zlnew, cold ? NULL : S->zlnew, b, mN);
            FN(ld)(w.gl, cold ? NULL : S->gl, b, nN);
            FN(ld)(w.yl, cold ? NULL : S->yl, b, mN);
            FN(ld)(w.vlnew_tv, cold ? NULL : S->vlnew_tv, b, nN);
            FN(ld)(w.zlnew_tv, cold ? NULL : S->zlnew_tv, b, mN);
            FN(ld)(w.gl_tv, cold ? NULL : S->gl_tv, b, nN);
            FN(ld)(w.yl_tv, cold ? NULL : S->yl_tv, b, mN);
            FN(ld)(w.Xref, io->Xref, io->xref_per_instance ? b : 0, nN);
            FN(ld)(w.Uref, io->Uref, io->uref_per_instance ? b : 0, mN);
            memset(w.q, 0, sizeof(T) * nN);
            memset(w.p, 0, sizeof(T) * nN);
            w.pri_x = w.dua_x = w.pri_u = w.dua_u = 0;
            memcpy(w.x, (const T *)io->x0 + (size_t)b * nx, sizeof(T) * nx); /* tiny_set_x0, tiny_api.cpp:451 */

            FN(solve_one)(pr, st, &w);

            FN(st)(io->sol_x, b, w.vnew, nN); /* solution->x = vnew (admm.cpp:436,452) */
            FN(st)(io->sol_u, b, w.znew, mN);
            if (io->iter) io->iter[b] = w.iter;
            if (io->solved) io->solved[b] = w.solved;
            if (io->residuals) {
                T *rr = (T *)io->residuals + 4 * (size_t)b;
                rr[0] = w.pri_x; rr[1] = w.dua_x; rr[2] = w.pri_u; rr[3] = w.dua_u;
            }
            FN(st)(S->x, b, w.x, nN);
            FN(st)(S->u, b, w.u, mN);
            FN(st)(S->v, b, w.v, nN);
            FN(st)(S->z, b, w.z, mN);
            FN(st)(S->vnew, b, w.vnew, nN);
            FN(st)(S->znew, b, w.znew, mN);
            FN(st)(S->g, b, w.g, nN);
            FN(st)(S->y, b, w.y, mN);
            FN(st)(S->vcnew, b, w.vcnew, nN);
            FN(st)(S->zcnew, b, w.zcnew, mN);
            FN(st)(S->gc, b, w.gc, nN);
            FN(st)(S->yc, b, w.yc, mN);
            FN(st)(S->vlnew, b, w.vlnew, nN);
            FN(st)(S->zlnew, b, w.zlnew, mN);
            FN(st)(S->gl, b, w.gl, nN);
            FN(st)(S->yl, b, w.yl, mN);
            FN(st)(S->vlnew_tv, b, w.vlnew_tv, nN);
            FN(st)(S->zlnew_tv, b, w.zlnew_tv, mN);
            FN(st)(S->gl_tv, b, w.gl_tv, nN);
            FN(st)(S->yl_tv, b, w.yl_tv, mN);
        }
        free(buf);
        free(Uref_buf);
    }
    return rc;
}

/* ---- tiny_precompute_and_set_cache restated (tiny_api.cpp:307-381); tolerance-level vs Eigen ---- */

static void FN(matmul)(const T *A, const T *B, T *C, int m, int k, int n) { /* C(m x n) = A(m x k) B(k x n) */
    for (int j = 0; j < n; ++j)
        for (int i = 0; i < m; ++i) {
            T s = 0;
            for (int l = 0; l < k; ++l) s += A[i + (size_t)l * m] * B[l + (size_t)j * k];
            C[i + (size_t)j * m] = s;
        }
}
static void FN(transpose)(const T *A, T *At, int m, int n) {
    for (int j = 0; j < n; ++j)
        for (int i = 0; i < m; ++i) At[j + (size_t)i * n] = A[i + (size_t)j * m];
}
/* inverse by LU with partial pivoting (what Eigen's PartialPivLU::inverse does mathematically) */
static int FN(inverse)(const T *Ain, T *inv, int n) {
    T *a = (T *)malloc(sizeof(T) * n * n);
    memcpy(a, Ain, sizeof(T) * n * n);
    for (int j = 0; j < n; ++j)
        for (int i = 0; i < n; ++i) inv[i + (size_t)j * n] = (i == j) ? (T)1 : (T)0;
    for (int c = 0; c < n; ++c) {
        int piv = c;
        T best = FABS(a[c + (size_t)c * n]);
        for (int i = c + 1; i < n; ++i)
            if (FABS(a[i + (size_t)c * n]) > best) { best = FABS(a[i + (size_t)c * n]); piv = i; }
        if (best == 0) { free(a); return -1; }
        if (piv != c)
            for (int j = 0; j < n; ++j) {
                T t = a[c + (size_t)j * n]; a[c + (size_t)j * n] = a[piv + (size_t)j * n]; a[piv + (size_t)j * n] = t;
                t = inv[c + (size_t)j * n]; inv[c + (size_t)j * n] = inv[piv + (size_t)j * n]; inv[piv + (size_t)j * n] = t;
            }
        T d = a[c + (size_t)c * n];
        for (int i = 0; i < n; ++i) {
            if (i == c) continue;
            T fct = a[i + (size_t)c * n] / d;
            if (fct == 0) continue;
            for (int j = 0; j < n; ++j) {
                a[i + (size_t)j * n] -= fct * a[c + (size_t)j * n];
                inv[i + (size_t)j * n] -= fct * inv[c + (size_t)j * n];
            }
        }
    }
    for (int i = 0; i < n; ++i) {
        T d = a[i + (size_t)i * n];
        for (int j = 0; j < n; ++j) inv[i + (size_t)j * n] /= d;
    }
    free(a);
    return 0;
}

static int FN(precompute)(int nx, int nu, double rho_d, const T *A, const T *B, const T *f, const T *Q, const T *R,
                          T *Kinf, T *Pinf, T *Quu_inv, T *AmBKt, T *APf, T *BPf) {
    const T rho = (T)rho_d;
    const size_t xx = (size_t)nx * nx, xu = (size_t)nx * nu, uu = (size_t)nu * nu;
    T *Q1 = calloc(xx, sizeof(T)), *R1 = calloc(uu, sizeof(T)), *P = calloc(xx, sizeof(T));
    T *Kp = calloc(xu, sizeof(T)), *Bt = malloc(sizeof(T) * xu), *At = malloc(sizeof(T) * xx);
    T *BtP = malloc(sizeof(T) * xu), *S = malloc(sizeof(T) * uu), *Si = malloc(sizeof(T) * uu);
    T *BtPA = malloc(sizeof(T) * xu), *BK = malloc(sizeof(T) * xx), *AmBK = malloc(sizeof(T) * xx);
    T *AtP = malloc(sizeof(T) * xx), *tmp = malloc(sizeof(T) * xx), *Pf = malloc(sizeof(T) * nx);
    int iters = 0, rc = 0;
    for (int i = 0; i < nx; ++i) { Q1[i + (size_t)i * nx] = Q[i] + rho; P[i + (size_t)i * nx] = rho; }  /* :317,:331 */
    for (int j = 0; j < nu; ++j) R1[j + (size_t)j * nu] = R[j] + rho;                                    /* :318 */
    FN(transpose)(B, Bt, nx, nu);
    FN(transpose)(A, At, nx, nx);
    for (int it = 0; it < 1000; ++it) { /* :335-349 */
        FN(matmul)(Bt, P, BtP, nu, nx, nx);
        FN(matmul)(BtP, B, S, nu, nx, nu);
        for (size_t e = 0; e < uu; ++e) S[e] += R1[e];
        if (FN(inverse)(S, Si, nu)) { rc = -1; break; }
        FN(matmul)(BtP, A, BtPA, nu, nx, nx);
        FN(matmul)(Si, BtPA, Kinf, nu, nu, nx);
        FN(matmul)(B, Kinf, BK, nx, nu, nx);
        for (size_t e = 0; e < xx; ++e) AmBK[e] = A[e] - BK[e];
        FN(matmul)(At, P, AtP, nx, nx, nx);
        FN(matmul)(AtP, AmBK, tmp, nx, nx, nx);
        for (size_t e = 0; e < xx; ++e) Pinf[e] = Q1[e] + tmp[e];
        iters = it + 1;
        T md = 0;
        for (size_t e = 0; e < xu; ++e) { T dlt = FABS(Kinf[e] - Kp[e]); if (dlt > md) md = dlt; }
        if (md < (T)1e-5) break;
        memcpy(Kp, Kinf, sizeof(T) * xu);
        memcpy(P, Pinf, sizeof(T) * xx);
    }
    if (!rc) { /* :352-357 */
        FN(matmul)(Bt, Pinf, BtP, nu, nx, nx);
        FN(matmul)(BtP, B, S, nu, nx, nu);
        for (size_t e = 0; e < uu; ++e) S[e] += R1[e];
        if (FN(inverse)(S, Quu_inv, nu)) rc = -1;
        FN(matmul)(B, Kinf, BK, nx, nu, nx);
        for (size_t e = 0; e < xx; ++e) AmBK[e] = A[e] - BK[e];
        FN(transpose)(AmBK, AmBKt, nx, nx);
        FN(matmul)(Pinf, f, Pf, nx, nx, 1);
        FN(matmul)(AmBKt, Pf, APf, nx, nx, 1);
        FN(matmul)(Bt, Pf, BPf, nu, nx, 1);
    }
    free(Q1); free(R1); free(P); free(Kp); free(Bt); free(At); free(BtP); free(S); free(Si); free(BtPA);
    free(BK); free(AmBK); free(AtP); free(tmp); free(Pf);
    return rc ? rc : iters;
}

#undef FN
#undef CAT
#undef CAT_
