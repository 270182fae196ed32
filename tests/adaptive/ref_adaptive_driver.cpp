// tests/adaptive/ref_adaptive_driver.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// Runs the UNMODIFIED reference's adaptive-rho solve, batched over instances.  It is compiled together with the
// reference's own sources (src/tinympc/{admm,tiny_api,rho_benchmark}.cpp and the vendored Eigen) with the pinned parity
// flags by tests/golden/make_golden_adaptive.py, into a temporary directory; only the fixtures it writes are kept.
//
// The reference's solve() (admm.cpp:331-455) cannot be called for this: its RhoAdapter is declared uninitialised
// (admm.cpp:340) and format_matrices reads adapter->matrices_initialized (rho_benchmark.cpp:56), so an adaptive solve
// is undefined behaviour (a crash with the pinned build).  This driver repeats solve()'s loop control with
// `RhoAdapter adapter{}` and calls the reference's compiled stage functions for every step: update_linear_cost,
// backward_pass_grad, forward_pass, update_slack, update_dual, benchmark_rho_adaptation,
// update_matrices_with_derivatives and termination_condition.
//
// Per instance the solver's model, cache and rho come from the instance's model blob (tinympc_b200/csrc/model_blob.h
// layout) and the adapted rho / Kinf / Pinf are written back to it, so no cache leaks from one instance to the next.
#include <cstdint>
#include <cstring>
#include <iostream>

#include "admm.hpp"
#include "rho_benchmark.hpp"
#include "tiny_api.hpp"

#include "tinympc_b200.h"

namespace {

typedef tinytype T;

void load(tinyMatrix &dst, const void *base, int64_t b, int rows, int cols) {
    if (base)
        dst = Map<const tinyMatrix>(static_cast<const T *>(base) + b * (int64_t)rows * cols, rows, cols);
    else
        dst = tinyMatrix::Zero(rows, cols);
}
void store(void *base, int64_t b, const tinyMatrix &src) {
    if (base) std::memcpy(static_cast<T *>(base) + b * (int64_t)src.size(), src.data(), sizeof(T) * src.size());
}

// admm.cpp:331-455 loop control with a value-initialised RhoAdapter; adaptive_rho is on
void solve_adaptive(TinySolver *solver) {
    solver->solution->solved = 0;
    solver->solution->iter = 0;
    solver->work->status = 11;
    solver->work->iter = 0;
    RhoAdapter adapter{};
    adapter.rho_min = solver->settings->adaptive_rho_min;
    adapter.rho_max = solver->settings->adaptive_rho_max;
    adapter.clip = solver->settings->adaptive_rho_enable_clipping;
    RhoBenchmarkResult rho_result{};
    for (int i = 0; i < solver->settings->max_iter; i++) {
        update_linear_cost(solver);
        backward_pass_grad(solver);
        forward_pass(solver);
        update_slack(solver);
        update_dual(solver);
        solver->work->iter += 1;
        if (i > 0 && i % 5 == 0) {
            benchmark_rho_adaptation(&adapter, solver->work->x, solver->work->u, solver->work->vnew, solver->work->znew,
                                     solver->work->g, solver->work->y, solver->cache, solver->work, solver->work->N,
                                     &rho_result);
            update_matrices_with_derivatives(solver->cache, rho_result.final_rho);
        }
        if (termination_condition(solver)) {
            solver->work->status = 1;
            solver->solution->iter = solver->work->iter;
            solver->solution->solved = 1;
            solver->solution->x = solver->work->vnew;
            solver->solution->u = solver->work->znew;
            return;
        }
        solver->work->v = solver->work->vnew;
        solver->work->z = solver->work->znew;
    }
    solver->solution->iter = solver->work->iter;
    solver->solution->solved = 0;
    solver->solution->x = solver->work->vnew;
    solver->solution->u = solver->work->znew;
}

}  // namespace

extern "C" int tinympc_ref_adaptive_dtype(void) { return sizeof(T) == 8 ? TINYMPC_F64 : TINYMPC_F32; }

// Batched adaptive solve on host buffers: box constraints (pr's bounds), state fields x, u, v, z, vnew, znew, g, y.
extern "C" int tinympc_ref_solve_adaptive(const tinympc_problem_t *pr, const tinympc_settings_t *st, const tinympc_batch_t *io,
                                          const tinympc_adaptive_rho_t *ar) {
    if (!pr || !st || !io || !ar || !ar->models || pr->dtype != tinympc_ref_adaptive_dtype()) return -1;
    const int nx = pr->nx, nu = pr->nu, N = pr->N;
    const int64_t oA = 0, oB = oA + nx * nx, of = oB + nx * nu, oQ = of + nx, oR = oQ + nx, oK = oR + nu, oP = oK + nu * nx;
    const int64_t oQuu = oP + nx * nx, oAm = oQuu + nu * nu, oAPf = oAm + nx * nx, oBPf = oAPf + nx, orho = oBPf + nu;
    const int64_t blob = orho + 1;
    std::ios_base::iostate old = std::cout.rdstate();
    std::cout.setstate(std::ios_base::failbit);
    int rc = 0;
    for (int64_t b = 0; b < io->B && !rc; ++b) {
        T *mb = static_cast<T *>(ar->models) + b * blob;
        auto mat = [&](int64_t off, int r, int c) { return tinyMatrix(Map<const tinyMatrix>(mb + off, r, c)); };
        const T rho = mb[orho];
        // tiny_setup wants the user's Q, R (without rho); every derived quantity is overwritten below
        tinyVector Qu = mat(oQ, nx, 1).array() - rho, Ru = mat(oR, nu, 1).array() - rho;
        tinyMatrix Qm = Qu.asDiagonal(), Rm = Ru.asDiagonal();
        TinySolver *s = nullptr;
        if (tiny_setup(&s, mat(oA, nx, nx), mat(oB, nx, nu), mat(of, nx, 1), Qm, Rm, rho, nx, nu, N, 0) || !s) {
            rc = -2;
            break;
        }
        TinyWorkspace *w = s->work;
        TinyCache *c = s->cache;
        w->Q = mat(oQ, nx, 1);
        w->R = mat(oR, nu, 1);
        c->rho = rho;
        c->Kinf = mat(oK, nu, nx);
        c->Pinf = mat(oP, nx, nx);
        c->Quu_inv = mat(oQuu, nu, nu);
        c->AmBKt = mat(oAm, nx, nx);
        c->APf = mat(oAPf, nx, 1);
        c->BPf = mat(oBPf, nu, 1);
        c->C1 = c->Quu_inv;
        c->C2 = c->AmBKt;
        c->dKinf_drho = Map<const tinyMatrix>(static_cast<const T *>(ar->dKinf_drho), nu, nx);
        c->dPinf_drho = Map<const tinyMatrix>(static_cast<const T *>(ar->dPinf_drho), nx, nx);
        c->dC1_drho = tinyMatrix::Zero(nu, nu);
        c->dC2_drho = tinyMatrix::Zero(nx, nx);
        tiny_set_bound_constraints(s, Map<const tinyMatrix>(static_cast<const T *>(pr->x_min), nx, N),
                                   Map<const tinyMatrix>(static_cast<const T *>(pr->x_max), nx, N),
                                   Map<const tinyMatrix>(static_cast<const T *>(pr->u_min), nu, N - 1),
                                   Map<const tinyMatrix>(static_cast<const T *>(pr->u_max), nu, N - 1));
        tiny_update_settings(s->settings, (T)st->abs_pri_tol, (T)st->abs_dua_tol, st->max_iter, st->check_termination,
                             st->en_state_bound, st->en_input_bound, 0, 0, 0, 0, 0, 0);
        s->settings->adaptive_rho = 1;
        s->settings->adaptive_rho_min = (T)ar->rho_min;
        s->settings->adaptive_rho_max = (T)ar->rho_max;
        s->settings->adaptive_rho_enable_clipping = ar->enable_clipping;

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
        load(w->Xref, io->Xref, io->xref_per_instance ? b : 0, nx, N);
        load(w->Uref, io->Uref, io->uref_per_instance ? b : 0, nu, N - 1);
        w->primal_residual_state = w->dual_residual_state = w->primal_residual_input = w->dual_residual_input = 0;
        tiny_set_x0(s, Map<const tinyVector>(static_cast<const T *>(io->x0) + b * nx, nx));

        solve_adaptive(s);

        std::memcpy(mb + oK, c->Kinf.data(), sizeof(T) * nu * nx);
        std::memcpy(mb + oP, c->Pinf.data(), sizeof(T) * nx * nx);
        mb[orho] = c->rho;
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
        if (io->u0) std::memcpy(static_cast<T *>(io->u0) + b * nu, w->u.data(), sizeof(T) * nu);
        store(S.x, b, w->x);
        store(S.u, b, w->u);
        store(S.v, b, w->v);
        store(S.z, b, w->z);
        store(S.vnew, b, w->vnew);
        store(S.znew, b, w->znew);
        store(S.g, b, w->g);
        store(S.y, b, w->y);
        delete s->solution;
        delete s->cache;
        delete s->settings;
        delete s->work;
        delete s;
    }
    std::cout.clear(old);
    return rc;
}
