// tests/shim/shim_script.cpp — TEST PROGRAM.  A scripted driver of the reference interface (<tinympc/tiny_api.hpp>): it
// applies a binary op stream to one or more TinySolvers and dumps the struct tree after every solve.  The same source is
// built twice:
//   oracle/_ref/shim_tests/script_ref   with the unmodified reference sources, pinned flags (oracle/Makefile)
//   oracle/_ref/shim_tests/script_shim  with tinympc_shim.cpp over libtinympc_b200.so (tinympc_b200/shim/Makefile, defines
//                                       TINYMPC_SCRIPT_SHIM)
// tests/test_gpu_shim_parity.py runs both on the same streams and compares the dumps bit for bit and stdout op by op;
// tests/test_shim_script_oracle.py pins the reference build to the batch oracle.  The only arithmetic done here is the plant
// step, written as scalar loops so that both builds (-ffp-contract=off) produce the same bits.
//
//   shim_script IN OUT                       run one op stream
//   shim_script --threads IN1 OUT1 IN2 OUT2 ...  run several streams at once, one thread (and its own solvers) per stream;
//                                            no op markers are printed in this mode
//
// IN (raw little-endian): a sequence of ops, each `int32 op, int32 solver` followed by the op's payload.  A matrix is
// `int32 rows, int32 cols` and rows*cols float64 in column-major order; an int vector is `int32 n` and n int32.
// OUT: one record per SETUP / PRECOMPUTE (cache), SOLVE / DUMP (tree) and BATCH op: `int32 kind, op index, solver, rc,
// nmat` then nmat matrices in the format above (scalars as 1 x 1).  tests/shim_common.py writes IN and parses OUT.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include <tinympc/tiny_api.hpp>

namespace {

enum Op {
    OP_SETUP = 1, OP_SET_CACHE, OP_BOUNDS, OP_CONES, OP_LINEAR, OP_TV_LINEAR, OP_X0, OP_XREF, OP_UREF, OP_UPDATE_SETTINGS,
    OP_POKE_SETTINGS, OP_POKE_WORK, OP_POKE_COUNTS, OP_PRECOMPUTE, OP_SOLVE, OP_PLANT, OP_BATCH, OP_DUMP
};
const char *kOpNames[] = {"", "setup", "set_cache", "bounds", "cones", "linear", "tv_linear", "x0", "xref", "uref",
                          "update_settings", "poke_settings", "poke_work", "poke_counts", "precompute", "solve", "plant",
                          "batch", "dump"};
enum Kind { K_CACHE = 1, K_TREE = 2, K_BATCH = 3 };
const int kMaxSolvers = 4;

struct Reader {
    FILE *f;
    bool eof() {
        int c = std::fgetc(f);
        if (c == EOF) return true;
        std::ungetc(c, f);
        return false;
    }
    int32_t i() {
        int32_t v;
        if (std::fread(&v, sizeof v, 1, f) != 1) throw 1;
        return v;
    }
    double d() {
        double v;
        if (std::fread(&v, sizeof v, 1, f) != 1) throw 2;
        return v;
    }
    tinyMatrix m() {
        const int r = i(), c = i();
        tinyMatrix out(r, c);
        if ((size_t)r * c && std::fread(out.data(), sizeof(double), (size_t)r * c, f) != (size_t)r * c) throw 3;
        return out;
    }
    VectorXi iv() {
        const int n = i();
        VectorXi out(n);
        for (int k = 0; k < n; ++k) out(k) = i();
        return out;
    }
};

struct Writer {
    FILE *f;
    void head(int kind, int op, int solver, int rc, int nmat) {
        const int32_t h[5] = {kind, op, solver, rc, nmat};
        std::fwrite(h, sizeof(int32_t), 5, f);
    }
    void m(const tinyMatrix &a) {
        const int32_t rc[2] = {(int32_t)a.rows(), (int32_t)a.cols()};
        std::fwrite(rc, sizeof(int32_t), 2, f);
        std::fwrite(a.data(), sizeof(double), a.size(), f);
    }
    void s(double v) { m(tinyMatrix::Constant(1, 1, v)); }
};

void dump_cache(Writer &w, int op, int si, int rc, const TinyCache *c) {
    w.head(K_CACHE, op, si, rc, 7);
    w.s(c->rho); w.m(c->Kinf); w.m(c->Pinf); w.m(c->Quu_inv); w.m(c->AmBKt); w.m(c->APf); w.m(c->BPf);
}

// the whole tree a solve writes back.  work->{q, r, p, d} are left out: they are per-iteration scratch that every iteration
// overwrites before it reads them, and the shim never writes them.
void dump_tree(Writer &o, int op, int si, int rc, const TinySolver *s) {
    const TinyWorkspace *w = s->work;
    const tinyMatrix *m[] = {&s->solution->x, &s->solution->u, &w->x, &w->u, &w->v, &w->vnew, &w->z, &w->znew, &w->g, &w->y,
                             &w->vcnew, &w->zcnew, &w->gc, &w->yc, &w->vlnew, &w->zlnew, &w->gl, &w->yl, &w->vlnew_tv,
                             &w->zlnew_tv, &w->gl_tv, &w->yl_tv, &w->vc, &w->zc, &w->vl, &w->zl, &w->vl_tv, &w->zl_tv,
                             &s->cache->Kinf, &s->cache->Pinf};
    const int nm = sizeof(m) / sizeof(m[0]);
    o.head(K_TREE, op, si, rc, 2 + nm + 7);
    o.s(s->solution->iter); o.s(s->solution->solved);
    for (int k = 0; k < nm; ++k) o.m(*m[k]);
    o.s(w->primal_residual_state); o.s(w->dual_residual_state); o.s(w->primal_residual_input); o.s(w->dual_residual_input);
    o.s(w->status); o.s(w->iter); o.s(s->cache->rho);
}

// the work matrices POKE_WORK can overwrite, by index (tests/shim_common.py: POKE_FIELDS)
tinyMatrix *work_field(TinyWorkspace *w, int k) {
    tinyMatrix *f[] = {&w->Xref, &w->Uref, &w->x_min, &w->x_max, &w->u_min, &w->u_max, &w->x, &w->u, &w->v, &w->z,
                       &w->vnew, &w->znew, &w->g, &w->y, &w->gc, &w->yc, &w->gl, &w->yl, &w->gl_tv, &w->yl_tv};
    if (k < 0 || k >= (int)(sizeof(f) / sizeof(f[0]))) throw 4;
    return f[k];
}

void read_settings(Reader &in, TinySettings *t, bool through_api) {
    const double pri = in.d(), dua = in.d();
    int v[10];
    for (int &x : v) x = in.i();
    if (through_api) {
        tiny_update_settings(t, pri, dua, v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7], v[8], v[9]);
        return;
    }
    t->abs_pri_tol = pri; t->abs_dua_tol = dua; t->max_iter = v[0]; t->check_termination = v[1];
    t->en_state_bound = v[2]; t->en_input_bound = v[3]; t->en_state_soc = v[4]; t->en_input_soc = v[5];
    t->en_state_linear = v[6]; t->en_input_linear = v[7]; t->en_tv_state_linear = v[8]; t->en_tv_input_linear = v[9];
}

// x0 <- A x0 + B u0 + f with u0 = work->u.col(0), ascending index, separate multiply and add
void plant(TinySolver *s) {
    const TinyWorkspace *w = s->work;
    const int nx = w->nx, nu = w->nu;
    tinyVector x0 = w->x.col(0), nxt(nx);
    for (int i = 0; i < nx; ++i) {
        double ax = w->Adyn(i, 0) * x0(0);
        for (int k = 1; k < nx; ++k) ax = ax + w->Adyn(i, k) * x0(k);
        double bu = w->Bdyn(i, 0) * w->u(0, 0);
        for (int j = 1; j < nu; ++j) bu = bu + w->Bdyn(i, j) * w->u(j, 0);
        nxt(i) = (ax + bu) + w->fdyn(i);
    }
    tiny_set_x0(s, nxt);
}

#ifdef TINYMPC_SCRIPT_SHIM
int solve_batch(TinySolver *s, const tinyMatrix &x0, const tinyMatrix &Xref, tinyMatrix &u0, VectorXi &iter, VectorXi &solved) {
    return tiny_solve_batch(s, x0, Xref, u0, iter, solved);
}
#else
// tiny_solve_batch restated on the reference: one cold tiny_solve per column on a saved and restored tree, with the
// "Solver converged" lines kept off stdout (tiny_solve_batch prints none)
int solve_batch(TinySolver *s, const tinyMatrix &x0, const tinyMatrix &Xref, tinyMatrix &u0, VectorXi &iter, VectorXi &solved) {
    TinyWorkspace *w = s->work;
    const int nx = w->nx, nu = w->nu, N = w->N, B = (int)x0.cols();
    const TinyWorkspace saved_w = *w;
    const TinySolution saved_sol = *s->solution;
    u0.resize(nu, B);
    iter.resize(B);
    solved.resize(B);
    std::cout.setstate(std::ios::failbit);
    for (int b = 0; b < B; ++b) {
        for (tinyMatrix *m : {&w->x, &w->v, &w->vnew, &w->g, &w->vcnew, &w->gc, &w->vlnew, &w->gl, &w->vlnew_tv, &w->gl_tv})
            *m = tinyMatrix::Zero(nx, N);
        for (tinyMatrix *m : {&w->u, &w->z, &w->znew, &w->y, &w->zcnew, &w->yc, &w->zlnew, &w->yl, &w->zlnew_tv, &w->yl_tv})
            *m = tinyMatrix::Zero(nu, N - 1);
        w->Xref = Map<const tinyMatrix>(Xref.col(b).data(), nx, N);
        tiny_set_x0(s, x0.col(b));
        tiny_solve(s);
        u0.col(b) = w->u.col(0);
        iter(b) = s->solution->iter;
        solved(b) = s->solution->solved;
    }
    std::cout.clear();
    *w = saved_w;
    *s->solution = saved_sol;
    return 0;
}
#endif

int run(FILE *fin, FILE *fout, bool markers) {
    Reader in{fin};
    Writer out{fout};
    TinySolver *sv[kMaxSolvers] = {};
    int op_index = 0;
    try {
        for (; !in.eof(); ++op_index) {
            const int op = in.i(), si = in.i();
            if (op < OP_SETUP || op > OP_DUMP || si < 0 || si >= kMaxSolvers) throw 5;
            if (markers) std::cout << "## op " << op_index << " " << kOpNames[op] << " solver " << si << std::endl;
            TinySolver *s = sv[si];
            if (op != OP_SETUP && !s) throw 6;
            switch (op) {
            case OP_SETUP: {
                const int nx = in.i(), nu = in.i(), N = in.i();
                const double rho = in.d();
                const tinyMatrix A = in.m(), B = in.m(), f = in.m(), Q = in.m(), R = in.m();
#ifdef TINYMPC_SCRIPT_SHIM
                tiny_destroy(sv[si]);  // a stream may set a slot up again (the reference has no destroy: its old solver leaks)
#endif
                const int rc = tiny_setup(&sv[si], A, B, f, Q, R, rho, nx, nu, N, 0);
                dump_cache(out, op_index, si, rc, sv[si]->cache);
                break;
            }
            case OP_SET_CACHE: {
                TinyCache *c = s->cache;
                c->rho = in.d();
                c->Kinf = in.m(); c->Pinf = in.m(); c->Quu_inv = in.m(); c->AmBKt = in.m(); c->APf = in.m(); c->BPf = in.m();
                c->C1 = c->Quu_inv;
                c->C2 = c->AmBKt;
                break;
            }
            case OP_BOUNDS: {
                const tinyMatrix a = in.m(), b = in.m(), c = in.m(), d = in.m();
                tiny_set_bound_constraints(s, a, b, c, d);
                break;
            }
            case OP_CONES: {
                const VectorXi Acx = in.iv(), qcx = in.iv();
                const tinyVector cx = in.m();
                const VectorXi Acu = in.iv(), qcu = in.iv();
                const tinyVector cu = in.m();
                tiny_set_cone_constraints(s, Acx, qcx, cx, Acu, qcu, cu);  // first triple: state cones (both builds)
                break;
            }
            case OP_LINEAR: {
                const tinyMatrix a = in.m(), b = in.m(), c = in.m(), d = in.m();
                tiny_set_linear_constraints(s, a, b, c, d);
                break;
            }
            case OP_TV_LINEAR: {
                const tinyMatrix a = in.m(), b = in.m(), c = in.m(), d = in.m();
                tiny_set_tv_linear_constraints(s, a, b, c, d);
                break;
            }
            case OP_X0: tiny_set_x0(s, in.m()); break;
            case OP_XREF: tiny_set_x_ref(s, in.m()); break;
            case OP_UREF: tiny_set_u_ref(s, in.m()); break;
            case OP_UPDATE_SETTINGS: read_settings(in, s->settings, true); break;
            case OP_POKE_SETTINGS: read_settings(in, s->settings, false); break;
            case OP_POKE_WORK: {
                const int k = in.i();
                *work_field(s->work, k) = in.m();
                break;
            }
            case OP_POKE_COUNTS: {
                TinyWorkspace *w = s->work;
                w->numStateCones = in.i(); w->numInputCones = in.i(); w->numStateLinear = in.i();
                w->numInputLinear = in.i(); w->numtvStateLinear = in.i(); w->numtvInputLinear = in.i();
                break;
            }
            case OP_PRECOMPUTE: {  // a new rho, as a program re-tuning it would call it (the user's Q, R without rho)
                const double rho = in.d();
                const tinyMatrix Q = in.m(), R = in.m();
                const TinyWorkspace *w = s->work;
                const int rc = tiny_precompute_and_set_cache(s->cache, w->Adyn, w->Bdyn, w->fdyn, Q, R, w->nx, w->nu, rho, 0);
                dump_cache(out, op_index, si, rc, s->cache);
                break;
            }
            case OP_SOLVE: {
                const int rc = tiny_solve(s);
                dump_tree(out, op_index, si, rc, s);
                break;
            }
            case OP_PLANT: plant(s); break;
            case OP_BATCH: {
                const tinyMatrix x0 = in.m(), Xref = in.m();
                tinyMatrix u0;
                VectorXi iter, solved;
                const int rc = solve_batch(s, x0, Xref, u0, iter, solved);
                out.head(K_BATCH, op_index, si, rc, 3);
                out.m(u0); out.m(iter.cast<double>()); out.m(solved.cast<double>());
                break;
            }
            case OP_DUMP: dump_tree(out, op_index, si, -1, s); break;
            }
        }
    } catch (int e) {
        std::fprintf(stderr, "shim_script: bad op stream at op %d (error %d)\n", op_index, e);
        return 10 + e;
    }
#ifdef TINYMPC_SCRIPT_SHIM
    for (TinySolver *s : sv) tiny_destroy(s);
#endif
    return 0;
}

int run_files(const char *pin, const char *pout, bool markers) {
    FILE *in = std::fopen(pin, "rb");
    FILE *out = std::fopen(pout, "wb");
    if (!in || !out) return 2;
    const int rc = run(in, out, markers);
    std::fclose(in);
    std::fclose(out);
    return rc;
}

}  // namespace

int main(int argc, char **argv) {
    if (argc >= 2 && std::string(argv[1]) == "--threads") {
        const int n = (argc - 2) / 2;
        if (n < 1 || argc != 2 + 2 * n) return 3;
        std::vector<int> rcs(n, 0);
        std::vector<std::thread> ts;
        for (int t = 0; t < n; ++t)
            ts.emplace_back([&, t] { rcs[t] = run_files(argv[2 + 2 * t], argv[3 + 2 * t], false); });
        for (auto &t : ts) t.join();
        for (int rc : rcs)
            if (rc) return rc;
        return 0;
    }
    if (argc != 3) return 3;
    return run_files(argv[1], argv[2], true);
}
