// tests/adaptive/shim_adaptive_loop.cpp — TEST PROGRAM.  A one-robot closed loop written against the reference interface
// (tiny_setup, tiny_initialize_sensitivity_matrices, settings->adaptive_rho = 1, tiny_set_x0, tiny_solve) and compiled with
// the C++ shim by tinympc_b200/shim/Makefile; tests/test_gpu_adaptive.py compares what it writes with the C restatement.
//
//   shim_adaptive_loop IN OUT        run the loop described by IN, write every step's results to OUT
//   shim_adaptive_loop --bad-tables  adaptive rho with sensitivity tables of the wrong shape: tiny_solve must return 1
//
// IN (raw little-endian): int32 nx, nu, N, steps, max_iter, check_termination, enable_clipping;
// float64 abs_pri_tol, abs_dua_tol, rho_min, rho_max; then float64 arrays, column-major: the model blob
// (A | B | f | Q | R | Kinf | Pinf | Quu_inv | AmBKt | APf | BPf | rho, Q / R with rho added), dKinf_drho, dPinf_drho, x_min, x_max,
// u_min, u_max (nx x N, nu x N-1), Xref (nx x N), x0 of every step (steps x nx).
// OUT per step: float64 vnew, znew, x, u, v, z, g, y, iter, solved, residuals[4], rho, Kinf, Pinf; int32 tiny_solve's return.
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include <tinympc/tiny_api.hpp>

namespace {

template <class T>
T get(FILE *f) {
    T v;
    if (fread(&v, sizeof(T), 1, f) != 1) throw 1;
    return v;
}
tinyMatrix getm(FILE *f, int r, int c) {
    tinyMatrix m(r, c);
    if (fread(m.data(), sizeof(double), (size_t)r * c, f) != (size_t)r * c) throw 2;
    return m;
}
void putm(FILE *f, const tinyMatrix &m) { fwrite(m.data(), sizeof(double), m.size(), f); }
void putd(FILE *f, double v) { fwrite(&v, sizeof(double), 1, f); }

int bad_tables() {
    const int nx = 4, nu = 2, N = 10;
    tinyMatrix A = tinyMatrix::Identity(nx, nx), B = tinyMatrix::Zero(nx, nu), Q = tinyMatrix::Identity(nx, nx),
               R = tinyMatrix::Identity(nu, nu);
    B(0, 0) = B(1, 1) = 0.1;
    tinyMatrix f = tinyMatrix::Zero(nx, 1);
    TinySolver *s = nullptr;
    if (tiny_setup(&s, A, B, f, Q, R, 1.0, nx, nu, N, 0)) return 3;
    tiny_initialize_sensitivity_matrices(s);  // the reference's 4 x 12 / 12 x 12 tables: wrong for a 4 / 2 solver
    s->settings->adaptive_rho = 1;
    tinyVector x0 = tinyVector::Ones(nx);
    tiny_set_x0(s, x0);
    const int rc = tiny_solve(s);
    std::printf("tiny_solve returned %d\n", rc);
    return rc == 1 ? 0 : 4;
}

}  // namespace

int main(int argc, char **argv) {
    if (argc == 2 && std::string(argv[1]) == "--bad-tables") return bad_tables();
    if (argc != 3) return 5;
    FILE *in = std::fopen(argv[1], "rb");
    FILE *out = std::fopen(argv[2], "wb");
    if (!in || !out) return 6;
    try {
        const int nx = get<int32_t>(in), nu = get<int32_t>(in), N = get<int32_t>(in), steps = get<int32_t>(in);
        const int max_iter = get<int32_t>(in), check = get<int32_t>(in), clip = get<int32_t>(in);
        const double pri = get<double>(in), dua = get<double>(in), rmin = get<double>(in), rmax = get<double>(in);
        const tinyMatrix A = getm(in, nx, nx), Bm = getm(in, nx, nu), f = getm(in, nx, 1), Qw = getm(in, nx, 1), Rw = getm(in, nu, 1);
        const tinyMatrix K = getm(in, nu, nx), P = getm(in, nx, nx), Quu = getm(in, nu, nu), AmBKt = getm(in, nx, nx);
        const tinyMatrix APf = getm(in, nx, 1), BPf = getm(in, nu, 1);
        const double rho = get<double>(in);
        const tinyMatrix dK = getm(in, nu, nx), dP = getm(in, nx, nx);
        const tinyMatrix xmin = getm(in, nx, N), xmax = getm(in, nx, N), umin = getm(in, nu, N - 1), umax = getm(in, nu, N - 1);
        const tinyMatrix Xref = getm(in, nx, N), x0s = getm(in, nx, steps);
        // tiny_setup takes the user's Q, R (without rho); the cache and work->Q / R are then set to the given ones
        tinyVector Qu = Qw.array() - rho, Ru = Rw.array() - rho;
        tinyMatrix Qm = Qu.asDiagonal(), Rm = Ru.asDiagonal();
        TinySolver *s = nullptr;
        if (tiny_setup(&s, A, Bm, f, Qm, Rm, rho, nx, nu, N, 0)) return 7;
        s->work->Q = Qw;
        s->work->R = Rw;
        s->cache->rho = rho;
        s->cache->Kinf = K; s->cache->Pinf = P; s->cache->Quu_inv = Quu; s->cache->AmBKt = AmBKt;
        s->cache->APf = APf; s->cache->BPf = BPf;
        s->cache->dKinf_drho = dK;
        s->cache->dPinf_drho = dP;
        tiny_set_bound_constraints(s, xmin, xmax, umin, umax);
        tiny_update_settings(s->settings, pri, dua, max_iter, check, 1, 1, 0, 0, 0, 0, 0, 0);
        s->settings->adaptive_rho = 1;
        s->settings->adaptive_rho_min = rmin;
        s->settings->adaptive_rho_max = rmax;
        s->settings->adaptive_rho_enable_clipping = clip;
        tiny_set_x_ref(s, Xref);
        for (int k = 0; k < steps; ++k) {
            tinyVector x0 = x0s.col(k);
            tiny_set_x0(s, x0);
            const int32_t rc = tiny_solve(s);
            TinyWorkspace *w = s->work;
            putm(out, w->vnew); putm(out, w->znew); putm(out, w->x); putm(out, w->u); putm(out, w->v); putm(out, w->z);
            putm(out, w->g); putm(out, w->y);
            putd(out, s->solution->iter); putd(out, s->solution->solved);
            putd(out, w->primal_residual_state); putd(out, w->dual_residual_state);
            putd(out, w->primal_residual_input); putd(out, w->dual_residual_input);
            putd(out, s->cache->rho); putm(out, s->cache->Kinf); putm(out, s->cache->Pinf);
            fwrite(&rc, sizeof(rc), 1, out);
        }
    } catch (int e) {
        return 10 + e;
    }
    std::fclose(out);
    std::fclose(in);
    return 0;
}
