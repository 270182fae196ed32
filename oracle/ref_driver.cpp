// oracle/ref_driver.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// A raw-pointer batched driver around the UNMODIFIED reference (TinyMPC/TinyMPC).  It is compiled
// together with the reference's own sources where they lie in a TinyMPC checkout
// (src/tinympc/{admm,tiny_api,rho_benchmark}.cpp + the vendored Eigen) by oracle/Makefile, with outputs
// only into oracle/_ref/ (git-ignored).  Nothing from the reference is copied into this repository.
//
// It exposes the same stateless batch call as the product's C ABI (include/tinympc_b200.h) so that the
// parity tests can feed identical buffers to the reference, to the C restatement (oracle/tinympc_oracle.c)
// and to the CUDA path.  Per instance it pokes the TinyWorkspace exactly the way the reference's examples
// do (examples/quadrotor_tracking.cpp:86-97) and calls the reference's tiny_solve()
// (src/tinympc/tiny_api.cpp:384-386 -> solve(), src/tinympc/admm.cpp:331-455).
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may load this.

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <mutex>
#include <thread>
#include <vector>

#include "tiny_api.hpp"  // the reference's header (resolved through -I by oracle/Makefile)

#include "tinympc_b200.h"  // POD structs shared with the product ABI (structs only)

namespace {

typedef tinytype T;

inline tinyMatrix map_mat(const void *p, int rows, int cols) {
    return Map<const tinyMatrix>(static_cast<const T *>(p), rows, cols);
}
inline tinyVector map_vec(const void *p, int n) { return Map<const tinyVector>(static_cast<const T *>(p), n); }

inline void load(tinyMatrix &dst, const void *base, int64_t b, int rows, int cols) {
    if (base) {
        dst = Map<const tinyMatrix>(static_cast<const T *>(base) + b * (int64_t)rows * cols, rows, cols);
    } else {
        dst = tinyMatrix::Zero(rows, cols);
    }
}
inline void store(void *base, int64_t b, const tinyMatrix &src) {
    if (base) {
        std::memcpy(static_cast<T *>(base) + b * (int64_t)src.size(), src.data(), sizeof(T) * src.size());
    }
}

// Build one TinySolver for `prob` through the reference's own setup path, then overwrite the cache and
// the cost vectors with the caller's values (struct pokes — the struct tree IS the reference's API).
TinySolver *make_solver(const tinympc_problem_t *pr, const tinympc_settings_t *st) {
    const int nx = pr->nx, nu = pr->nu, N = pr->N;
    TinySolver *solver = nullptr;
    tinyMatrix A = map_mat(pr->Adyn, nx, nx), B = map_mat(pr->Bdyn, nx, nu);
    tinyVector f = map_vec(pr->fdyn, nx);
    tinyVector Qw = map_vec(pr->Q, nx), Rw = map_vec(pr->R, nu);
    T rho = (T)pr->rho;
    // tiny_setup wants the user's Q,R (without rho); anything SPD works because every derived quantity
    // is overwritten below.
    tinyVector Qu = Qw.array() - rho, Ru = Rw.array() - rho;
    tinyMatrix Qm = Qu.asDiagonal(), Rm = Ru.asDiagonal();
    int status = tiny_setup(&solver, A, B, f, Qm, Rm, rho, nx, nu, N, 0);
    if (status || !solver) return nullptr;
    solver->work->Q = Qw;
    solver->work->R = Rw;
    solver->cache->rho = rho;
    solver->cache->Kinf = map_mat(pr->Kinf, nu, nx);
    solver->cache->Pinf = map_mat(pr->Pinf, nx, nx);
    solver->cache->Quu_inv = map_mat(pr->Quu_inv, nu, nu);
    solver->cache->AmBKt = map_mat(pr->AmBKt, nx, nx);
    solver->cache->APf = map_vec(pr->APf, nx);
    solver->cache->BPf = map_vec(pr->BPf, nu);
    solver->cache->C1 = solver->cache->Quu_inv;
    solver->cache->C2 = solver->cache->AmBKt;
    if (pr->x_min && pr->x_max && pr->u_min && pr->u_max) {
        tiny_set_bound_constraints(solver, map_mat(pr->x_min, nx, N), map_mat(pr->x_max, nx, N),
                                   map_mat(pr->u_min, nu, N - 1), map_mat(pr->u_max, nu, N - 1));
    }
    if (pr->num_state_cones > 0 || pr->num_input_cones > 0) {
        VectorXi Acx = Map<const VectorXi>(pr->Acx, pr->num_state_cones);
        VectorXi qcx = Map<const VectorXi>(pr->qcx, pr->num_state_cones);
        VectorXi Acu = Map<const VectorXi>(pr->Acu, pr->num_input_cones);
        VectorXi qcu = Map<const VectorXi>(pr->qcu, pr->num_input_cones);
        // positional order of the reference DEFINITION (tiny_api.cpp:176-178): state triple first
        tiny_set_cone_constraints(solver, Acx, qcx, map_vec(pr->cx, pr->num_state_cones), Acu, qcu,
                                  map_vec(pr->cu, pr->num_input_cones));
    }
    if (pr->num_state_linear > 0 || pr->num_input_linear > 0) {
        tiny_set_linear_constraints(solver, map_mat(pr->Alin_x, pr->num_state_linear, nx),
                                    map_vec(pr->blin_x, pr->num_state_linear),
                                    map_mat(pr->Alin_u, pr->num_input_linear, nu),
                                    map_vec(pr->blin_u, pr->num_input_linear));
    }
    if (pr->num_tv_state_linear > 0 || pr->num_tv_input_linear > 0) {
        tiny_set_tv_linear_constraints(solver, map_mat(pr->tv_Alin_x, pr->num_tv_state_linear * N, nx),
                                       map_mat(pr->tv_blin_x, pr->num_tv_state_linear, N),
                                       map_mat(pr->tv_Alin_u, pr->num_tv_input_linear * (N - 1), nu),
                                       map_mat(pr->tv_blin_u, pr->num_tv_input_linear, N - 1));
    }
    tiny_update_settings(solver->settings, (T)st->abs_pri_tol, (T)st->abs_dua_tol, st->max_iter,
                         st->check_termination, st->en_state_bound, st->en_input_bound, st->en_state_soc,
                         st->en_input_soc, st->en_state_linear, st->en_input_linear, st->en_tv_state_linear,
                         st->en_tv_input_linear);
    return solver;
}

void free_solver(TinySolver *s) {  // the reference has no destroy function (SURVEY §8b)
    if (!s) return;
    delete s->solution;
    delete s->cache;
    delete s->settings;
    delete s->work;
    delete s;
}

// One tiny_solve of instance b of `io` on solver `s` (pokes per examples/quadrotor_tracking.cpp:86-97).
void solve_instance(TinySolver *s, const tinympc_problem_t *pr, const tinympc_batch_t *io, int64_t b) {
    const int nx = pr->nx, nu = pr->nu, N = pr->N;
    TinyWorkspace *w = s->work;
    const tinympc_state_t &S = io->state;
    const bool cold = io->cold_start != 0;
    load(w->x, cold ? nullptr : S.x, b, nx, N);
    load(w->u, cold ? nullptr : S.u, b, nu, N - 1);
    load(w->v, cold ? nullptr : S.v, b, nx, N);
    load(w->z, cold ? nullptr : S.z, b, nu, N - 1);
    load(w->vnew, cold ? nullptr : S.vnew, b, nx, N);
    load(w->znew, cold ? nullptr : S.znew, b, nu, N - 1);
    load(w->g, cold ? nullptr : S.g, b, nx, N);
    load(w->y, cold ? nullptr : S.y, b, nu, N - 1);
    load(w->vcnew, cold ? nullptr : S.vcnew, b, nx, N);
    load(w->zcnew, cold ? nullptr : S.zcnew, b, nu, N - 1);
    load(w->gc, cold ? nullptr : S.gc, b, nx, N);
    load(w->yc, cold ? nullptr : S.yc, b, nu, N - 1);
    load(w->vlnew, cold ? nullptr : S.vlnew, b, nx, N);
    load(w->zlnew, cold ? nullptr : S.zlnew, b, nu, N - 1);
    load(w->gl, cold ? nullptr : S.gl, b, nx, N);
    load(w->yl, cold ? nullptr : S.yl, b, nu, N - 1);
    load(w->vlnew_tv, cold ? nullptr : S.vlnew_tv, b, nx, N);
    load(w->zlnew_tv, cold ? nullptr : S.zlnew_tv, b, nu, N - 1);
    load(w->gl_tv, cold ? nullptr : S.gl_tv, b, nx, N);
    load(w->yl_tv, cold ? nullptr : S.yl_tv, b, nu, N - 1);
    load(w->Xref, io->Xref, io->xref_per_instance ? b : 0, nx, N);
    load(w->Uref, io->Uref, io->uref_per_instance ? b : 0, nu, N - 1);
    w->primal_residual_state = 0;
    w->dual_residual_state = 0;
    w->primal_residual_input = 0;
    w->dual_residual_input = 0;
    tiny_set_x0(s, map_vec(static_cast<const T *>(io->x0) + b * nx, nx));

    tiny_solve(s);

    store(io->sol_x, b, s->solution->x);
    store(io->sol_u, b, s->solution->u);
    if (io->iter) io->iter[b] = s->solution->iter;
    if (io->solved) io->solved[b] = s->solution->solved;
    if (io->residuals) {
        T *r = static_cast<T *>(io->residuals) + 4 * b;
        r[0] = w->primal_residual_state;
        r[1] = w->dual_residual_state;
        r[2] = w->primal_residual_input;
        r[3] = w->dual_residual_input;
    }
    store(S.x, b, w->x);
    store(S.u, b, w->u);
    store(S.v, b, w->v);
    store(S.z, b, w->z);
    store(S.vnew, b, w->vnew);
    store(S.znew, b, w->znew);
    store(S.g, b, w->g);
    store(S.y, b, w->y);
    store(S.vcnew, b, w->vcnew);
    store(S.zcnew, b, w->zcnew);
    store(S.gc, b, w->gc);
    store(S.yc, b, w->yc);
    store(S.vlnew, b, w->vlnew);
    store(S.zlnew, b, w->zlnew);
    store(S.gl, b, w->gl);
    store(S.yl, b, w->yl);
    store(S.vlnew_tv, b, w->vlnew_tv);
    store(S.zlnew_tv, b, w->zlnew_tv);
    store(S.gl_tv, b, w->gl_tv);
    store(S.yl_tv, b, w->yl_tv);
}

void run_range(const tinympc_problem_t *pr, const tinympc_settings_t *st, const tinympc_batch_t *io, int64_t b0,
               int64_t b1, int *rc) {
    TinySolver *s = make_solver(pr, st);
    if (!s) {
        *rc = -1;
        return;
    }
    for (int64_t b = b0; b < b1; ++b) solve_instance(s, pr, io, b);
    free_solver(s);
    *rc = 0;
}

// Persistent worker pool for the timing arm (bench.py --impl reference / cpu_baseline): `nthreads` std::threads, each with
// ONE TinySolver built once through the reference's own tiny_setup (BASELINE.md §3.2), parked on a condition variable
// between batches; a batch is handed out in chunks from an atomic counter so that a descheduled thread does not hold
// the others back.
struct Pool {
    tinympc_problem_t pr;  // dims / counts only are read after construction
    std::vector<std::thread> threads;
    std::vector<TinySolver *> solvers;
    std::mutex m;
    std::condition_variable cv_work, cv_done;
    const tinympc_batch_t *job = nullptr;
    std::atomic<int64_t> next{0};
    int64_t chunk = 16;
    uint64_t generation = 0;
    int running = 0, ready = 0;
    bool stop = false, failed = false;

    void worker(int t, const tinympc_problem_t *pr0, const tinympc_settings_t *st0) {
        TinySolver *s = make_solver(pr0, st0);
        {
            std::lock_guard<std::mutex> lk(m);
            solvers[t] = s;
            failed |= (s == nullptr);
            ++ready;
        }
        cv_done.notify_all();
        uint64_t seen = 0;
        for (;;) {
            const tinympc_batch_t *io;
            {
                std::unique_lock<std::mutex> lk(m);
                cv_work.wait(lk, [&] { return stop || generation != seen; });
                if (stop) break;
                seen = generation;
                io = job;
            }
            if (s) {
                for (;;) {
                    int64_t b0 = next.fetch_add(chunk);
                    if (b0 >= io->B) break;
                    int64_t b1 = std::min<int64_t>(io->B, b0 + chunk);
                    for (int64_t b = b0; b < b1; ++b) solve_instance(s, &pr, io, b);
                }
            }
            {
                std::lock_guard<std::mutex> lk(m);
                --running;
            }
            cv_done.notify_all();
        }
        free_solver(s);
    }
};

}  // namespace

extern "C" {

int tinympc_ref_dtype(void) { return sizeof(T) == 8 ? TINYMPC_F64 : TINYMPC_F32; }

// Runs the reference's tiny_setup (tiny_api.cpp:21-147) for user-level Q,R diagonals and returns what it
// derives: work->Q, work->R (diag + rho) and the cache (tiny_precompute_and_set_cache, :307-381).
int tinympc_ref_setup_cache(int32_t nx, int32_t nu, int32_t N, double rho, const void *A, const void *B,
                            const void *f, const void *Qdiag_user, const void *Rdiag_user, void *Q_out,
                            void *R_out, void *Kinf, void *Pinf, void *Quu_inv, void *AmBKt, void *APf,
                            void *BPf) {
    std::ios_base::iostate old = std::cout.rdstate();
    std::cout.setstate(std::ios_base::failbit);
    TinySolver *s = nullptr;
    tinyVector Qd = map_vec(Qdiag_user, nx), Rd = map_vec(Rdiag_user, nu);
    tinyMatrix Qm = Qd.asDiagonal(), Rm = Rd.asDiagonal();
    int status = tiny_setup(&s, map_mat(A, nx, nx), map_mat(B, nx, nu), map_vec(f, nx), Qm, Rm, (T)rho, nx, nu,
                            N, 0);
    std::cout.clear(old);
    if (status || !s) return -1;
    std::memcpy(Q_out, s->work->Q.data(), sizeof(T) * nx);
    std::memcpy(R_out, s->work->R.data(), sizeof(T) * nu);
    std::memcpy(Kinf, s->cache->Kinf.data(), sizeof(T) * nu * nx);
    std::memcpy(Pinf, s->cache->Pinf.data(), sizeof(T) * nx * nx);
    std::memcpy(Quu_inv, s->cache->Quu_inv.data(), sizeof(T) * nu * nu);
    std::memcpy(AmBKt, s->cache->AmBKt.data(), sizeof(T) * nx * nx);
    std::memcpy(APf, s->cache->APf.data(), sizeof(T) * nx);
    std::memcpy(BPf, s->cache->BPf.data(), sizeof(T) * nu);
    free_solver(s);
    return 0;
}

// Batched tiny_solve on host buffers with `nthreads` std::threads, one TinySolver per thread (the
// library has no shared mutable state except std::cout, which is silenced: admm.cpp:439 prints on every
// converged solve).
int tinympc_ref_solve_batch(const tinympc_problem_t *pr, const tinympc_settings_t *st, const tinympc_batch_t *io,
                            int32_t nthreads) {
    if (!pr || !st || !io || !io->x0 || !io->Xref) return -1;
    if (pr->dtype != tinympc_ref_dtype()) return -2;
    std::ios_base::iostate old = std::cout.rdstate();
    std::cout.setstate(std::ios_base::failbit);
    if (nthreads < 1) nthreads = 1;
    if ((int64_t)nthreads > io->B) nthreads = (int)(io->B > 0 ? io->B : 1);
    std::vector<int> rcs(nthreads, 0);
    if (nthreads == 1) {
        run_range(pr, st, io, 0, io->B, &rcs[0]);
    } else {
        std::vector<std::thread> th;
        int64_t per = (io->B + nthreads - 1) / nthreads;
        for (int t = 0; t < nthreads; ++t) {
            int64_t b0 = t * per, b1 = std::min<int64_t>(io->B, b0 + per);
            if (b0 >= b1) break;
            th.emplace_back(run_range, pr, st, io, b0, b1, &rcs[t]);
        }
        for (auto &t : th) t.join();
    }
    std::cout.clear(old);
    for (int r : rcs)
        if (r) return r;
    return 0;
}

// The reference's tiny_initialize_sensitivity_matrices (tiny_api.cpp:479-540; quadrotor-sized hard-coded tables) run on a
// freshly set-up 12 x 4 solver; the four d*_drho matrices are copied out column-major (4x12, 12x12, 4x4, 12x12).  Source of
// the shim's table data (tools/extract_sensitivity_tables.py) and of the test that pins it.
int tinympc_ref_sensitivity_tables(void *dKinf, void *dPinf, void *dC1, void *dC2) {
    const int nx = 12, nu = 4, N = 3;
    std::ios_base::iostate old = std::cout.rdstate();
    std::cout.setstate(std::ios_base::failbit);
    TinySolver *s = nullptr;
    tinyMatrix A = tinyMatrix::Identity(nx, nx), B = tinyMatrix::Zero(nx, nu), Q = tinyMatrix::Identity(nx, nx),
               R = tinyMatrix::Identity(nu, nu);
    for (int j = 0; j < nu; ++j) B(j, j) = 1;
    tinyVector f = tinyVector::Zero(nx);
    int status = tiny_setup(&s, A, B, f, Q, R, (T)1, nx, nu, N, 0);
    if (status || !s) {
        std::cout.clear(old);
        return -1;
    }
    tiny_initialize_sensitivity_matrices(s);
    std::cout.clear(old);
    std::memcpy(dKinf, s->cache->dKinf_drho.data(), sizeof(T) * nu * nx);
    std::memcpy(dPinf, s->cache->dPinf_drho.data(), sizeof(T) * nx * nx);
    std::memcpy(dC1, s->cache->dC1_drho.data(), sizeof(T) * nu * nu);
    std::memcpy(dC2, s->cache->dC2_drho.data(), sizeof(T) * nx * nx);
    free_solver(s);
    return 0;
}

// ---- persistent pool (timing arm) ----
void *tinympc_ref_pool_create(const tinympc_problem_t *pr, const tinympc_settings_t *st, int32_t nthreads) {
    if (!pr || !st || pr->dtype != tinympc_ref_dtype()) return nullptr;
    if (nthreads < 1) nthreads = 1;
    std::ios_base::iostate old = std::cout.rdstate();
    std::cout.setstate(std::ios_base::failbit);
    Pool *p = new Pool;
    p->pr = *pr;
    p->solvers.assign(nthreads, nullptr);
    for (int t = 0; t < nthreads; ++t) p->threads.emplace_back(&Pool::worker, p, t, pr, st);
    {
        std::unique_lock<std::mutex> lk(p->m);
        p->cv_done.wait(lk, [&] { return p->ready == nthreads; });
    }
    std::cout.clear(old);
    return p;
}

// One batched tiny_solve on the pool; `chunk` instances are handed to a thread at a time.  Returns seconds of wall time
// (steady_clock around hand-out .. last thread done) through *seconds.
int tinympc_ref_pool_solve(void *pool, const tinympc_batch_t *io, int32_t chunk, double *seconds) {
    Pool *p = static_cast<Pool *>(pool);
    if (!p || !io || !io->x0 || !io->Xref || p->failed) return -1;
    std::ios_base::iostate old = std::cout.rdstate();
    std::cout.setstate(std::ios_base::failbit);
    auto t0 = std::chrono::steady_clock::now();
    {
        std::lock_guard<std::mutex> lk(p->m);
        p->job = io;
        p->chunk = chunk > 0 ? chunk : 16;
        p->next.store(0);
        p->running = (int)p->threads.size();
        ++p->generation;
    }
    p->cv_work.notify_all();
    {
        std::unique_lock<std::mutex> lk(p->m);
        p->cv_done.wait(lk, [&] { return p->running == 0; });
    }
    auto t1 = std::chrono::steady_clock::now();
    std::cout.clear(old);
    if (seconds) *seconds = std::chrono::duration<double>(t1 - t0).count();
    return 0;
}

void tinympc_ref_pool_destroy(void *pool) {
    Pool *p = static_cast<Pool *>(pool);
    if (!p) return;
    {
        std::lock_guard<std::mutex> lk(p->m);
        p->stop = true;
    }
    p->cv_work.notify_all();
    for (auto &t : p->threads) t.join();
    delete p;
}

}  // extern "C"
