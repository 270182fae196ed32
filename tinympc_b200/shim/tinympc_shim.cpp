// tinympc_shim.cpp — implementation of the reference-compatible front end (tinympc_shim.hpp) over the C ABI.
// Host-side bookkeeping only; every tiny_solve() is one tinympc_b200_solve_host() call (batch of one), or with
// settings->adaptive_rho one tinympc_b200_solve_adaptive_host() call.
#include "tinympc_shim.hpp"

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/tinympc_b200.h"

namespace {

IOFormat kFmt(4, 0, ", ", "\n", "[", "]");  // the reference prints its setup matrices with 4 significant digits

int check_dim(const std::string &what, const char *axis, long actual, long expected) {
    if (actual != expected) {
        std::cout << what << " has " << actual << " " << axis << ". Expected " << expected << "." << std::endl;
        return 1;
    }
    return 0;
}

struct Impl {
    tinympc_b200_solver_t *h = nullptr;
    uint64_t fingerprint = 0;
};
std::map<TinySolver *, Impl> &table() {
    static std::map<TinySolver *, Impl> t;
    return t;
}
// The reference is safe with one TinySolver per thread (SURVEY §8b "Threading"): the handle table is the only state
// shared between solvers, so look-ups / inserts / erases take this lock.  std::map nodes are stable, so the Impl& a
// thread obtained stays valid while other threads insert.
std::mutex &table_mutex() {
    static std::mutex m;
    return m;
}
Impl &impl_of(TinySolver *s) {
    std::lock_guard<std::mutex> lk(table_mutex());
    return table()[s];
}

#include "sensitivity_tables.inc"

[[noreturn]] void fused_stage(const char *name) {
    std::fprintf(stderr,
                 "tinympc_b200 shim: %s() is not available as a separate call - the ADMM stages (admm.hpp:9-34) are fused into one "
                 "batched GPU kernel; call tiny_solve()/solve() (one whole solve) or the C ABI (tinympc_b200_solve).\n",
                 name);
    std::abort();
}

uint64_t fnv(uint64_t h, const void *p, size_t n) {
    const unsigned char *c = static_cast<const unsigned char *>(p);
    for (size_t i = 0; i < n; ++i) h = (h ^ c[i]) * 1099511628211ULL;
    return h;
}
template <class M>
uint64_t fnv_m(uint64_t h, const M &m) {
    long d[2] = {(long)m.rows(), (long)m.cols()};
    h = fnv(h, d, sizeof(d));
    return m.size() ? fnv(h, m.data(), sizeof(typename M::Scalar) * m.size()) : h;
}

// adaptive: rho, Kinf and Pinf travel in the solve's model blob (adaptive rho rewrites them after every solve), so they do not
// key the handle
uint64_t fingerprint(const TinySolver *s, bool adaptive) {
    const TinyWorkspace *w = s->work;
    const TinyCache *c = s->cache;
    uint64_t h = 1469598103934665603ULL;
    // the counts key the handle too: a program may lower one directly and keep its matrices (the reference loops to the counts)
    int dims[10] = {w->nx, w->nu, w->N, (int)adaptive, w->numStateCones, w->numInputCones, w->numStateLinear, w->numInputLinear,
                    w->numtvStateLinear, w->numtvInputLinear};
    h = fnv(h, dims, sizeof(dims));
    if (!adaptive) h = fnv(h, &c->rho, sizeof(c->rho));
    h = fnv_m(h, w->Adyn); h = fnv_m(h, w->Bdyn); h = fnv_m(h, w->fdyn); h = fnv_m(h, w->Q); h = fnv_m(h, w->R);
    if (!adaptive) {
        h = fnv_m(h, c->Kinf);
        h = fnv_m(h, c->Pinf);
    }
    h = fnv_m(h, c->Quu_inv); h = fnv_m(h, c->AmBKt); h = fnv_m(h, c->APf); h = fnv_m(h, c->BPf);
    h = fnv_m(h, w->x_min); h = fnv_m(h, w->x_max); h = fnv_m(h, w->u_min); h = fnv_m(h, w->u_max);
    h = fnv_m(h, w->Acx); h = fnv_m(h, w->qcx); h = fnv_m(h, w->cx); h = fnv_m(h, w->Acu); h = fnv_m(h, w->qcu); h = fnv_m(h, w->cu);
    h = fnv_m(h, w->Alin_x); h = fnv_m(h, w->blin_x); h = fnv_m(h, w->Alin_u); h = fnv_m(h, w->blin_u);
    h = fnv_m(h, w->tv_Alin_x); h = fnv_m(h, w->tv_blin_x); h = fnv_m(h, w->tv_Alin_u); h = fnv_m(h, w->tv_blin_u);
    return h;
}

template <class M>
const void *ptr(const M &m) {
    return m.size() ? static_cast<const void *>(m.data()) : nullptr;
}

// A count the program raised above the rows of its arrays, on a family a solve would run: the reference would read past
// them, so the solve is refused instead.  (With the family switched off the reference never reads them.)
int check_counts(const TinySolver *s) {
    const TinyWorkspace *w = s->work;
    const TinySettings *t = s->settings;
    const long N = w->N;
    const char *bad = nullptr;
    if (t->en_state_soc && (w->numStateCones > w->Acx.size() || w->numStateCones > w->qcx.size() || w->numStateCones > w->cx.size()))
        bad = "numStateCones";
    else if (t->en_input_soc && (w->numInputCones > w->Acu.size() || w->numInputCones > w->qcu.size() || w->numInputCones > w->cu.size()))
        bad = "numInputCones";
    else if (t->en_state_linear && (w->numStateLinear > w->Alin_x.rows() || w->numStateLinear > w->blin_x.size()))
        bad = "numStateLinear";
    else if (t->en_input_linear && (w->numInputLinear > w->Alin_u.rows() || w->numInputLinear > w->blin_u.size()))
        bad = "numInputLinear";
    else if (t->en_tv_state_linear && (w->numtvStateLinear * N > w->tv_Alin_x.rows() || w->numtvStateLinear > w->tv_blin_x.rows()))
        bad = "numtvStateLinear";
    else if (t->en_tv_input_linear &&
             (w->numtvInputLinear * (N - 1) > w->tv_Alin_u.rows() || w->numtvInputLinear > w->tv_blin_u.rows()))
        bad = "numtvInputLinear";
    if (!bad) return 0;
    std::cout << "tinympc_b200 shim: work->" << bad << " exceeds the constraint arrays it counts" << std::endl;
    return 1;
}

// the first `rows` rows of m (at most all of them) as their own column-major matrix: what the reference reads of a
// constraint matrix whose count was lowered below its row count
tinyMatrix top_rows(const tinyMatrix &m, long rows) { return m.topRows(std::min<long>(rows, m.rows())); }

int ensure_handle(TinySolver *s, Impl &im) {
    const uint64_t fp = fingerprint(s, s->settings && s->settings->adaptive_rho);
    if (im.h && fp == im.fingerprint) return 0;
    if (im.h) tinympc_b200_destroy(im.h);
    im.h = nullptr;
    const TinyWorkspace *w = s->work;
    const TinyCache *c = s->cache;
    const long N = w->N;
    // counts above their arrays only reach here on a family that is off (check_counts), where they are never read
    const int ncx = std::min<long>(w->numStateCones, std::min<long>(w->Acx.size(), std::min<long>(w->qcx.size(), w->cx.size())));
    const int ncu = std::min<long>(w->numInputCones, std::min<long>(w->Acu.size(), std::min<long>(w->qcu.size(), w->cu.size())));
    const tinyMatrix Ax = top_rows(w->Alin_x, w->numStateLinear), bx = top_rows(w->blin_x, Ax.rows());
    const tinyMatrix Au = top_rows(w->Alin_u, w->numInputLinear), bu = top_rows(w->blin_u, Au.rows());
    const int ntx = std::min<long>(w->numtvStateLinear, std::min<long>(w->tv_Alin_x.rows() / N, w->tv_blin_x.rows()));
    const int ntu = std::min<long>(w->numtvInputLinear, std::min<long>(w->tv_Alin_u.rows() / (N - 1), w->tv_blin_u.rows()));
    const tinyMatrix tAx = top_rows(w->tv_Alin_x, ntx * N), tbx = top_rows(w->tv_blin_x, ntx);
    const tinyMatrix tAu = top_rows(w->tv_Alin_u, ntu * (N - 1)), tbu = top_rows(w->tv_blin_u, ntu);
    tinympc_problem_t p;
    std::memset(&p, 0, sizeof(p));
    p.nx = w->nx; p.nu = w->nu; p.N = w->N; p.dtype = TINYMPC_F64; p.rho = c->rho;
    p.Adyn = ptr(w->Adyn); p.Bdyn = ptr(w->Bdyn); p.fdyn = ptr(w->fdyn); p.Q = ptr(w->Q); p.R = ptr(w->R);
    p.Kinf = ptr(c->Kinf); p.Pinf = ptr(c->Pinf); p.Quu_inv = ptr(c->Quu_inv); p.AmBKt = ptr(c->AmBKt);
    p.APf = ptr(c->APf); p.BPf = ptr(c->BPf);
    const bool xb = w->x_min.rows() == w->nx && w->x_min.cols() == w->N && w->x_max.rows() == w->nx && w->x_max.cols() == w->N;
    const bool ub = w->u_min.rows() == w->nu && w->u_min.cols() == w->N - 1 && w->u_max.rows() == w->nu && w->u_max.cols() == w->N - 1;
    if (xb) { p.x_min = ptr(w->x_min); p.x_max = ptr(w->x_max); }
    if (ub) { p.u_min = ptr(w->u_min); p.u_max = ptr(w->u_max); }
    p.num_state_cones = ncx; p.num_input_cones = ncu;
    p.Acx = w->Acx.data(); p.qcx = w->qcx.data(); p.cx = ptr(w->cx);
    p.Acu = w->Acu.data(); p.qcu = w->qcu.data(); p.cu = ptr(w->cu);
    p.num_state_linear = (int)Ax.rows(); p.num_input_linear = (int)Au.rows();
    p.Alin_x = ptr(Ax); p.blin_x = ptr(bx); p.Alin_u = ptr(Au); p.blin_u = ptr(bu);
    p.num_tv_state_linear = ntx; p.num_tv_input_linear = ntu;
    p.tv_Alin_x = ptr(tAx); p.tv_blin_x = ptr(tbx); p.tv_Alin_u = ptr(tAu); p.tv_blin_u = ptr(tbu);
    int rc = tinympc_b200_create(&p, 0, &im.h);
    if (rc) {
        std::cout << "tinympc_b200 shim: " << tinympc_b200_last_error() << std::endl;
        return rc;
    }
    im.fingerprint = fp;
    return 0;
}

// a rejected update (check_termination <= 0) is an error of the solve: the handle would otherwise keep the previous settings
int push_settings(const TinySolver *s, Impl &im) {
    const TinySettings *t = s->settings;
    tinympc_settings_t st;
    st.abs_pri_tol = t->abs_pri_tol; st.abs_dua_tol = t->abs_dua_tol; st.max_iter = t->max_iter;
    st.check_termination = t->check_termination; st.en_state_bound = t->en_state_bound; st.en_input_bound = t->en_input_bound;
    st.en_state_soc = t->en_state_soc; st.en_input_soc = t->en_input_soc; st.en_state_linear = t->en_state_linear;
    st.en_input_linear = t->en_input_linear; st.en_tv_state_linear = t->en_tv_state_linear; st.en_tv_input_linear = t->en_tv_input_linear;
    if (tinympc_b200_update_settings(im.h, &st)) {
        std::cout << "tinympc_b200 shim: " << tinympc_b200_last_error() << std::endl;
        return 1;
    }
    return 0;
}

template <class M>
void *mptr(M &m, long rows, long cols) {  // a state buffer the C ABI may read and write in place
    if (m.rows() != rows || m.cols() != cols) m = M::Zero(rows, cols);
    return m.data();
}

}  // namespace

extern "C" {

int tiny_set_default_settings(TinySettings *s) {
    if (!s) {
        std::cout << "Error in tiny_set_default_settings: settings is nullptr" << std::endl;
        return 1;
    }
    tinympc_settings_t d;
    tinympc_b200_default_settings(&d);
    s->abs_pri_tol = d.abs_pri_tol; s->abs_dua_tol = d.abs_dua_tol; s->max_iter = d.max_iter;
    s->check_termination = d.check_termination; s->en_state_bound = d.en_state_bound; s->en_input_bound = d.en_input_bound;
    s->en_state_soc = d.en_state_soc; s->en_input_soc = d.en_input_soc; s->en_state_linear = d.en_state_linear;
    s->en_input_linear = d.en_input_linear; s->en_tv_state_linear = d.en_tv_state_linear; s->en_tv_input_linear = d.en_tv_input_linear;
    s->adaptive_rho = 0; s->adaptive_rho_min = 1.0; s->adaptive_rho_max = 100.0; s->adaptive_rho_enable_clipping = 1;
    return 0;
}

int tiny_update_settings(TinySettings *s, tinytype abs_pri_tol, tinytype abs_dua_tol, int max_iter, int check_termination,
                         int en_state_bound, int en_input_bound, int en_state_soc, int en_input_soc, int en_state_linear,
                         int en_input_linear, int en_tv_state_linear, int en_tv_input_linear) {
    if (!s) {
        std::cout << "Error in tiny_update_settings: settings is nullptr" << std::endl;
        return 1;
    }
    s->abs_pri_tol = abs_pri_tol; s->abs_dua_tol = abs_dua_tol; s->max_iter = max_iter; s->check_termination = check_termination;
    s->en_state_bound = en_state_bound; s->en_input_bound = en_input_bound; s->en_state_soc = en_state_soc; s->en_input_soc = en_input_soc;
    s->en_state_linear = en_state_linear; s->en_input_linear = en_input_linear; s->en_tv_state_linear = en_tv_state_linear;
    s->en_tv_input_linear = en_tv_input_linear;
    return 0;
}

int tiny_precompute_and_set_cache(TinyCache *cache, tinyMatrix A, tinyMatrix B, tinyMatrix f, tinyMatrix Q, tinyMatrix R, int nx,
                                  int nu, tinytype rho, int verbose) {
    if (!cache) {
        std::cout << "Error in tiny_precompute_and_set_cache: cache is nullptr" << std::endl;
        return 1;
    }
    // Q, R arrive as (diagonal) matrices that already contain +rho; rho is added once more inside (A.3-1)
    tinyVector Qd = Q.diagonal(), Rd = R.diagonal();
    tinyVector fv = f;
    if (verbose) {
        tinyMatrix Q1 = Q + rho * tinyMatrix::Identity(nx, nx), R1 = R + rho * tinyMatrix::Identity(nu, nu);
        std::cout << "A = " << A.format(kFmt) << std::endl;
        std::cout << "B = " << B.format(kFmt) << std::endl;
        std::cout << "Q = " << Q1.format(kFmt) << std::endl;
        std::cout << "R = " << R1.format(kFmt) << std::endl;
        std::cout << "rho = " << rho << std::endl;
    }
    cache->Kinf = tinyMatrix::Zero(nu, nx); cache->Pinf = tinyMatrix::Zero(nx, nx); cache->Quu_inv = tinyMatrix::Zero(nu, nu);
    cache->AmBKt = tinyMatrix::Zero(nx, nx); cache->APf = tinyVector::Zero(nx); cache->BPf = tinyVector::Zero(nu);
    int sweeps = tinympc_b200_precompute_cache(TINYMPC_F64, nx, nu, rho, A.data(), B.data(), fv.data(), Qd.data(), Rd.data(),
                                               cache->Kinf.data(), cache->Pinf.data(), cache->Quu_inv.data(), cache->AmBKt.data(),
                                               cache->APf.data(), cache->BPf.data());
    if (sweeps < 0) return 1;
    if (verbose) {
        if (sweeps < 1000) std::cout << "Kinf converged after " << sweeps << " iterations" << std::endl;
        std::cout << "Kinf = " << cache->Kinf.format(kFmt) << std::endl;
        std::cout << "Pinf = " << cache->Pinf.format(kFmt) << std::endl;
        std::cout << "Quu_inv = " << cache->Quu_inv.format(kFmt) << std::endl;
        std::cout << "AmBKt = " << cache->AmBKt.format(kFmt) << std::endl;
        std::cout << "APf = " << cache->APf.format(kFmt) << std::endl;
        std::cout << "BPf = " << cache->BPf.format(kFmt) << std::endl;
        std::cout << "\nPrecomputation finished!\n" << std::endl;
    }
    cache->rho = rho;
    cache->C1 = cache->Quu_inv;
    cache->C2 = cache->AmBKt;
    return 0;
}

int tiny_setup(TinySolver **solverp, tinyMatrix A, tinyMatrix B, tinyMatrix f, tinyMatrix Q, tinyMatrix R, tinytype rho, int nx,
               int nu, int N, int verbose) {
    TinySolver *s = new TinySolver();
    s->solution = new TinySolution();
    s->cache = new TinyCache();
    s->settings = new TinySettings();
    s->work = new TinyWorkspace();
    *solverp = s;
    s->solution->iter = 0;
    s->solution->solved = 0;
    s->solution->x = tinyMatrix::Zero(nx, N);
    s->solution->u = tinyMatrix::Zero(nu, N - 1);
    tiny_set_default_settings(s->settings);
    TinyWorkspace *w = s->work;
    w->nx = nx; w->nu = nu; w->N = N;
    int status = 0;
    status |= check_dim("State transition matrix (A)", "rows", A.rows(), nx);
    status |= check_dim("State transition matrix (A)", "columns", A.cols(), nx);
    status |= check_dim("Input matrix (B)", "rows", B.rows(), nx);
    status |= check_dim("Input matrix (B)", "columns", B.cols(), nu);
    status |= check_dim("Affine vector (f)", "rows", f.rows(), nx);
    status |= check_dim("Affine vector (f)", "columns", f.cols(), 1);
    status |= check_dim("State stage cost (Q)", "rows", Q.rows(), nx);
    status |= check_dim("State stage cost (Q)", "columns", Q.cols(), nx);
    status |= check_dim("State input cost (R)", "rows", R.rows(), nu);
    status |= check_dim("State input cost (R)", "columns", R.cols(), nu);
    if (status) return status;
    for (tinyMatrix *m : {&w->x, &w->q, &w->p, &w->v, &w->vnew, &w->g, &w->vc, &w->vcnew, &w->gc, &w->vl, &w->vlnew, &w->gl,
                          &w->vl_tv, &w->vlnew_tv, &w->gl_tv, &w->Xref})
        *m = tinyMatrix::Zero(nx, N);
    for (tinyMatrix *m : {&w->u, &w->r, &w->d, &w->z, &w->znew, &w->y, &w->zc, &w->zcnew, &w->yc, &w->zl, &w->zlnew, &w->yl,
                          &w->zl_tv, &w->zlnew_tv, &w->yl_tv, &w->Uref})
        *m = tinyMatrix::Zero(nu, N - 1);
    w->numStateCones = w->numInputCones = 0;
    w->numStateLinear = w->numInputLinear = 0;
    w->numtvStateLinear = w->numtvInputLinear = 0;
    w->Q = (Q + rho * tinyMatrix::Identity(nx, nx)).diagonal();
    w->R = (R + rho * tinyMatrix::Identity(nu, nu)).diagonal();
    w->Adyn = A;
    w->Bdyn = B;
    w->fdyn = f;
    w->Qu = tinyVector::Zero(nu);
    w->primal_residual_state = w->primal_residual_input = w->dual_residual_state = w->dual_residual_input = 0;
    w->status = 0;
    w->iter = 0;
    tinyMatrix Qm = w->Q.asDiagonal(), Rm = w->R.asDiagonal();
    return tiny_precompute_and_set_cache(s->cache, A, B, f, Qm, Rm, nx, nu, rho, verbose);
}

int tiny_set_bound_constraints(TinySolver *s, tinyMatrix x_min, tinyMatrix x_max, tinyMatrix u_min, tinyMatrix u_max) {
    if (!s) {
        std::cout << "Error in tiny_set_bound_constraints: solver is nullptr" << std::endl;
        return 1;
    }
    const TinyWorkspace *w = s->work;
    check_dim("Lower state bounds (x_min)", "rows", x_min.rows(), w->nx);
    check_dim("Lower state bounds (x_min)", "cols", x_min.cols(), w->N);
    check_dim("Lower state bounds (x_max)", "rows", x_max.rows(), w->nx);
    check_dim("Lower state bounds (x_max)", "cols", x_max.cols(), w->N);
    check_dim("Lower input bounds (u_min)", "rows", u_min.rows(), w->nu);
    check_dim("Lower input bounds (u_min)", "cols", u_min.cols(), w->N - 1);
    check_dim("Lower input bounds (u_max)", "rows", u_max.rows(), w->nu);
    check_dim("Lower input bounds (u_max)", "cols", u_max.cols(), w->N - 1);
    s->work->x_min = x_min; s->work->x_max = x_max; s->work->u_min = u_min; s->work->u_max = u_max;
    return 0;  // the reference returns 0 even on a mismatch (tiny_api.cpp:173)
}

int tiny_set_cone_constraints(TinySolver *s, VectorXi Acx, VectorXi qcx, tinyVector cx, VectorXi Acu, VectorXi qcu, tinyVector cu) {
    // parameter names here follow the reference DEFINITION: whatever the caller passes first goes to the state cones
    if (!s) {
        std::cout << "Error in tiny_set_cone_constraints: solver is nullptr" << std::endl;
        return 1;
    }
    const int ns = Acx.rows(), ni = Acu.rows();
    int status = 0;
    status |= check_dim("Cone state size (qcx)", "rows", qcx.rows(), ns);
    status |= check_dim("Cone mu value for state (cx)", "rows", cx.rows(), ns);
    status |= check_dim("Cone input size (qcu)", "rows", qcu.rows(), ni);
    status |= check_dim("Cone mu value for input (cu)", "rows", cu.rows(), ni);
    if (status) return status;
    TinyWorkspace *w = s->work;
    w->numStateCones = ns; w->numInputCones = ni;
    w->Acx = Acx; w->qcx = qcx; w->cx = cx; w->Acu = Acu; w->qcu = qcu; w->cu = cu;
    return 0;
}

int tiny_set_linear_constraints(TinySolver *s, tinyMatrix Alin_x, tinyVector blin_x, tinyMatrix Alin_u, tinyVector blin_u) {
    if (!s) {
        std::cout << "Error in tiny_set_linear_constraints: solver is nullptr" << std::endl;
        return 1;
    }
    TinyWorkspace *w = s->work;
    const int nsx = Alin_x.rows(), nsu = Alin_u.rows();
    int status = 0;
    if (nsx > 0) {
        status |= check_dim("State linear constraint matrix (Alin_x)", "columns", Alin_x.cols(), w->nx);
        status |= check_dim("State linear constraint vector (blin_x)", "rows", blin_x.rows(), nsx);
    }
    if (nsu > 0) {
        status |= check_dim("Input linear constraint matrix (Alin_u)", "columns", Alin_u.cols(), w->nu);
        status |= check_dim("Input linear constraint vector (blin_u)", "rows", blin_u.rows(), nsu);
    }
    if (status) return status;
    w->numStateLinear = nsx; w->numInputLinear = nsu;
    w->Alin_x = Alin_x; w->blin_x = blin_x; w->Alin_u = Alin_u; w->blin_u = blin_u;
    return 0;
}

int tiny_set_tv_linear_constraints(TinySolver *s, tinyMatrix tvAx, tinyMatrix tvbx, tinyMatrix tvAu, tinyMatrix tvbu) {
    if (!s) {
        std::cout << "Error in tiny_set_linear_constraints: solver is nullptr" << std::endl;
        return 1;
    }
    TinyWorkspace *w = s->work;
    const int nsx = tvAx.rows() / w->N, nsu = tvAu.rows() / (w->N - 1);
    int status = 0;
    if (nsx > 0) {
        status |= check_dim("State time-varying linear constraint matrix (tv_Alin_x)", "rows", tvAx.rows(), nsx * w->N);
        status |= check_dim("State time-varying linear constraint matrix (tv_Alin_x)", "columns", tvAx.cols(), w->nx);
        status |= check_dim("State time-varying linear constraint vector (tv_blin_x)", "rows", tvbx.rows(), nsx);
        status |= check_dim("State time-varying linear constraint vector (tv_blin_x)", "columns", tvbx.cols(), w->N);
    }
    if (nsu > 0) {
        status |= check_dim("Input time-varying linear constraint matrix (tv_Alin_u)", "rows", tvAu.rows(), nsu * (w->N - 1));
        status |= check_dim("Input time-varying linear constraint matrix (tv_Alin_u)", "columns", tvAu.cols(), w->nu);
        status |= check_dim("Input time-varying linear constraint vector (tv_blin_u)", "rows", tvbu.rows(), nsu);
        status |= check_dim("Input time-varying linear constraint vector (tv_blin_u)", "columns", tvbu.cols(), w->N - 1);
    }
    if (status) return status;
    w->numtvStateLinear = nsx; w->numtvInputLinear = nsu;
    w->tv_Alin_x = tvAx; w->tv_blin_x = tvbx; w->tv_Alin_u = tvAu; w->tv_blin_u = tvbu;
    return 0;
}

int tiny_set_x0(TinySolver *s, tinyVector x0) {
    if (!s) {
        std::cout << "Error in tiny_set_x0: solver is nullptr" << std::endl;
        return 1;
    }
    if (x0.rows() != s->work->nx) perror("Error in tiny_set_x0: x0 is not the correct length");
    s->work->x.col(0) = x0;
    return 0;
}
int tiny_set_x_ref(TinySolver *s, tinyMatrix x_ref) {
    if (!s) {
        std::cout << "Error in tiny_set_x_ref: solver is nullptr" << std::endl;
        return 1;
    }
    check_dim("State reference trajectory (x_ref)", "rows", x_ref.rows(), s->work->nx);
    check_dim("State reference trajectory (x_ref)", "columns", x_ref.cols(), s->work->N);
    s->work->Xref = x_ref;
    return 0;
}
int tiny_set_u_ref(TinySolver *s, tinyMatrix u_ref) {
    if (!s) {
        std::cout << "Error in tiny_set_u_ref: solver is nullptr" << std::endl;
        return 1;
    }
    check_dim("Control/input reference trajectory (u_ref)", "rows", u_ref.rows(), s->work->nu);
    check_dim("Control/input reference trajectory (u_ref)", "columns", u_ref.cols(), s->work->N - 1);
    s->work->Uref = u_ref;
    return 0;
}

// admm.hpp:9 — the ADMM driver itself (admm.cpp:331-455); tiny_solve is the reference's trampoline onto it
int solve(TinySolver *s) {
    TinyWorkspace *w = s->work;
    if (s->settings->adaptive_rho) {  // the reference adds these tables to Kinf / Pinf (rho_benchmark.cpp:204-205)
        const TinyCache *c = s->cache;
        const long nx = w->nx, nu = w->nu;
        if (c->dKinf_drho.rows() != nu || c->dKinf_drho.cols() != nx || c->dPinf_drho.rows() != nx || c->dPinf_drho.cols() != nx) {
            std::cout << "tinympc_b200 shim: settings->adaptive_rho needs cache->dKinf_drho (" << nu << " x " << nx
                      << ") and cache->dPinf_drho (" << nx << " x " << nx << "), got " << c->dKinf_drho.rows() << " x "
                      << c->dKinf_drho.cols() << " and " << c->dPinf_drho.rows() << " x " << c->dPinf_drho.cols()
                      << " (tiny_initialize_sensitivity_matrices fills 4 x 12 / 12 x 12 tables)" << std::endl;
            return 1;
        }
    }
    Impl &im = impl_of(s);
    if (check_counts(s) || ensure_handle(s, im) || push_settings(s, im)) return 1;  // nothing in the tree has changed yet
    const long nx = w->nx, nu = w->nu, N = w->N;
    tinympc_batch_t io;
    std::memset(&io, 0, sizeof(io));
    io.B = 1;
    tinyVector x0 = w->x.col(0);  // tiny_set_x0 wrote it there
    io.x0 = x0.data();
    io.Xref = w->Xref.data(); io.xref_per_instance = 0;
    io.Uref = w->Uref.data(); io.uref_per_instance = 0;
    io.cold_start = 0;  // the struct tree IS the warm-start state
    tinympc_state_t &st = io.state;
    st.x = mptr(w->x, nx, N); st.u = mptr(w->u, nu, N - 1); st.v = mptr(w->v, nx, N); st.z = mptr(w->z, nu, N - 1);
    st.vnew = mptr(w->vnew, nx, N); st.znew = mptr(w->znew, nu, N - 1); st.g = mptr(w->g, nx, N); st.y = mptr(w->y, nu, N - 1);
    st.vcnew = mptr(w->vcnew, nx, N); st.zcnew = mptr(w->zcnew, nu, N - 1); st.gc = mptr(w->gc, nx, N); st.yc = mptr(w->yc, nu, N - 1);
    st.vlnew = mptr(w->vlnew, nx, N); st.zlnew = mptr(w->zlnew, nu, N - 1); st.gl = mptr(w->gl, nx, N); st.yl = mptr(w->yl, nu, N - 1);
    st.vlnew_tv = mptr(w->vlnew_tv, nx, N); st.zlnew_tv = mptr(w->zlnew_tv, nu, N - 1);
    st.gl_tv = mptr(w->gl_tv, nx, N); st.yl_tv = mptr(w->yl_tv, nu, N - 1);
    io.sol_x = mptr(s->solution->x, nx, N);
    io.sol_u = mptr(s->solution->u, nu, N - 1);
    int32_t iter = 0, solved = 0;
    tinytype res[4] = {0, 0, 0, 0};
    io.iter = &iter; io.solved = &solved; io.residuals = res;
    int rc;
    if (s->settings->adaptive_rho) {
        // admm.cpp:397-423 with a value-initialised RhoAdapter (the reference's is uninitialised, admm.cpp:340): one instance
        // whose model blob carries this solver's cache in and the adapted rho / Kinf / Pinf out
        TinyCache *c = s->cache;
        std::vector<tinytype> blob((size_t)tinympc_b200_model_blob_elems((int)nx, (int)nu));
        tinytype *o = blob.data();
        auto put = [&o](const tinytype *p, long n) {
            std::memcpy(o, p, sizeof(tinytype) * n);
            o += n;
        };
        put(w->Adyn.data(), nx * nx); put(w->Bdyn.data(), nx * nu); put(w->fdyn.data(), nx); put(w->Q.data(), nx);
        put(w->R.data(), nu);
        tinytype *oK = o;
        put(c->Kinf.data(), nu * nx);
        tinytype *oP = o;
        put(c->Pinf.data(), nx * nx);
        put(c->Quu_inv.data(), nu * nu); put(c->AmBKt.data(), nx * nx); put(c->APf.data(), nx); put(c->BPf.data(), nu);
        *o = c->rho;
        tinympc_adaptive_rho_t ar;
        std::memset(&ar, 0, sizeof(ar));
        ar.rho_min = s->settings->adaptive_rho_min;
        ar.rho_max = s->settings->adaptive_rho_max;
        ar.enable_clipping = s->settings->adaptive_rho_enable_clipping;
        ar.dKinf_drho = c->dKinf_drho.data();
        ar.dPinf_drho = c->dPinf_drho.data();
        ar.models = blob.data();
        rc = tinympc_b200_solve_adaptive_host(im.h, &io, &ar);
        if (!rc) {  // the adapted cache persists in the TinySolver, as in the reference
            std::memcpy(c->Kinf.data(), oK, sizeof(tinytype) * nu * nx);
            std::memcpy(c->Pinf.data(), oP, sizeof(tinytype) * nx * nx);
            c->rho = *o;
        }
    } else {
        rc = tinympc_b200_solve_host(im.h, &io);
    }
    if (rc) {
        std::cout << "tinympc_b200 shim: " << tinympc_b200_last_error() << std::endl;
        return 1;
    }
    s->solution->iter = iter;
    s->solution->solved = solved;
    w->iter = iter;
    w->status = solved ? 1 : 11;
    if (iter >= s->settings->check_termination) {  // the reference writes the residuals only when a termination check runs
        w->primal_residual_state = res[0]; w->dual_residual_state = res[1];
        w->primal_residual_input = res[2]; w->dual_residual_input = res[3];
    }
    if (solved) std::cout << "Solver converged in " << iter << " iterations" << std::endl;  // admm.cpp:439
    return solved ? 0 : 1;
}

int tiny_solve(TinySolver *s) { return solve(s); }  // tiny_api.cpp:384-386

// admm.hpp:12-17 — the six stage functions exist as symbols so that programs referencing them link; on this backend the
// stages only exist fused inside the solve kernel, so calling one is a loud error, never a silent CPU computation.
void update_linear_cost(TinySolver *) { fused_stage("update_linear_cost"); }
void backward_pass_grad(TinySolver *) { fused_stage("backward_pass_grad"); }
void forward_pass(TinySolver *) { fused_stage("forward_pass"); }
void update_slack(TinySolver *) { fused_stage("update_slack"); }
void update_dual(TinySolver *) { fused_stage("update_dual"); }
bool termination_condition(TinySolver *) { fused_stage("termination_condition"); }

// tiny_api.hpp:54 / tiny_api.cpp:479-540: fills the four sensitivity matrices of the cache with the reference's hard-coded
// (quadrotor-sized: 4x12, 12x12, 4x4, 12x12) tables, whatever the solver's dimensions - as the reference does.  solve() uses
// dKinf_drho / dPinf_drho when settings->adaptive_rho is set, and refuses tables of another shape.
void tiny_initialize_sensitivity_matrices(TinySolver *s) {
    if (!s || !s->cache) return;
    s->cache->dKinf_drho = Map<const Matrix<double, 4, 12>>(k_dKinf_drho);
    s->cache->dPinf_drho = Map<const Matrix<double, 12, 12>>(k_dPinf_drho);
    s->cache->dC1_drho = Map<const Matrix<double, 4, 4>>(k_dC1_drho);
    s->cache->dC2_drho = Map<const Matrix<double, 12, 12>>(k_dC2_drho);
}

// plain-C view of the above for bindings / tests: copies the four matrices (column-major, 48 + 144 + 16 + 144 doubles)
int tinympc_shim_sensitivity_tables(double *dKinf, double *dPinf, double *dC1, double *dC2) {
    TinySolver s;
    TinyCache c;
    s.cache = &c;
    s.work = nullptr; s.settings = nullptr; s.solution = nullptr;
    tiny_initialize_sensitivity_matrices(&s);
    std::memcpy(dKinf, c.dKinf_drho.data(), sizeof(double) * 48);
    std::memcpy(dPinf, c.dPinf_drho.data(), sizeof(double) * 144);
    std::memcpy(dC1, c.dC1_drho.data(), sizeof(double) * 16);
    std::memcpy(dC2, c.dC2_drho.data(), sizeof(double) * 144);
    return 0;
}

int tiny_destroy(TinySolver *s) {
    if (!s) return 0;
    {
        std::lock_guard<std::mutex> lk(table_mutex());
        auto it = table().find(s);
        if (it != table().end()) {
            if (it->second.h) tinympc_b200_destroy(it->second.h);
            table().erase(it);
        }
    }
    delete s->solution; delete s->cache; delete s->settings; delete s->work; delete s;
    return 0;
}

int tiny_solve_batch(TinySolver *s, const tinyMatrix &x0, const tinyMatrix &Xref, tinyMatrix &u0, VectorXi &iter, VectorXi &solved) {
    TinyWorkspace *w = s->work;
    Impl &im = impl_of(s);
    if (check_counts(s) || ensure_handle(s, im) || push_settings(s, im)) return 1;
    const long nx = w->nx, nu = w->nu, N = w->N, B = x0.cols();
    if (x0.rows() != nx || Xref.rows() != nx * N || Xref.cols() != B) return 1;
    std::vector<tinytype> sx((size_t)B * nx * N), su((size_t)B * nu * (N - 1)), ur((size_t)B * nu * (N - 1));
    iter = VectorXi::Zero(B);
    solved = VectorXi::Zero(B);
    tinympc_batch_t io;
    std::memset(&io, 0, sizeof(io));
    io.B = B;
    io.x0 = x0.data();
    io.Xref = Xref.data(); io.xref_per_instance = 1;
    io.Uref = w->Uref.data(); io.uref_per_instance = 0;
    io.cold_start = 1;
    io.state.u = ur.data();
    io.sol_x = sx.data(); io.sol_u = su.data();
    io.iter = iter.data(); io.solved = solved.data();
    if (tinympc_b200_solve_host(im.h, &io)) {
        std::cout << "tinympc_b200 shim: " << tinympc_b200_last_error() << std::endl;
        return 1;
    }
    u0.resize(nu, B);
    for (long b = 0; b < B; ++b)
        for (long j = 0; j < nu; ++j) u0(j, b) = ur[(size_t)b * nu * (N - 1) + j];
    return 0;
}

}  // extern "C"
