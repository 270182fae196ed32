// tpi_kernel.cuh — thread-per-instance (TPI) batched ADMM solve.
//
// One CUDA thread runs one whole MPC instance: tiny_solve() -> solve()
// (TinyMPC src/tinympc/admm.cpp:331-455), i.e. per iteration
//   update_linear_cost (admm.cpp:262-304) fused into backward_pass_grad (:13-20),
//   forward_pass (:25-32) fused with update_slack (:81-213), update_dual (:219-256) and the residuals of
//   termination_condition (:310-328).
// The 32 lanes of a warp are 32 different instances, so every matrix entry is warp-uniform: the cache
// matrices live in the kernel parameter block (constant bank) and are folded into the FMA/FMUL
// instructions as constant operands — no loads, no shuffles for the mat-vecs.  The p / x recursions live
// in registers.  The N-indexed per-instance state (vnew, g, znew, y, d [+ cone / hyperplane twins]) does
// not fit on chip for 32 instances per warp, so it streams through a structure-of-arrays workspace in
// HBM/L2 as 16-byte vectors: element (k, vec j) of instance b at [(k*NV + j)*Bpad + b] -> every warp
// access is one fully coalesced 512-byte transaction.  The kernel is therefore HBM-bound
// (DESIGN.md §5 gives the byte count per iteration).
#pragma once
#include "common.cuh"

namespace tmpc {

template <typename T, int NE>
struct SoA {
    using V = typename Vec16<T>::type;
    static constexpr int E = Vec16<T>::E;
    static constexpr int NV = (NE + E - 1) / E;

    __device__ __forceinline__ static void load(const void *base, int k, int64_t S, int64_t b, T (&out)[NE]) {
        const V *p = reinterpret_cast<const V *>(base) + ((int64_t)k * NV) * S + b;
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            V v = p[(int64_t)j * S];
            const T *e = reinterpret_cast<const T *>(&v);
#pragma unroll
            for (int t = 0; t < E; ++t)
                if (j * E + t < NE) out[j * E + t] = e[t];
        }
    }
    __device__ __forceinline__ static void store(void *base, int k, int64_t S, int64_t b, const T (&in)[NE]) {
        V *p = reinterpret_cast<V *>(base) + ((int64_t)k * NV) * S + b;
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            V v;
            T *e = reinterpret_cast<T *>(&v);
#pragma unroll
            for (int t = 0; t < E; ++t) e[t] = (j * E + t < NE) ? in[j * E + t] : T(0);
            p[(int64_t)j * S] = v;
        }
    }
};

// contiguous per-instance column in user layout (instance-major); vectorised when 16-byte aligned
template <typename T, int NE>
__device__ __forceinline__ void load_col(const T *p, T (&out)[NE]) {
    constexpr int E = Vec16<T>::E;
    if constexpr ((NE % E) == 0) {
        if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) {
            using V = typename Vec16<T>::type;
#pragma unroll
            for (int j = 0; j < NE / E; ++j) {
                V v = __ldg(reinterpret_cast<const V *>(p) + j);
                const T *e = reinterpret_cast<const T *>(&v);
#pragma unroll
                for (int t = 0; t < E; ++t) out[j * E + t] = e[t];
            }
            return;
        }
    }
#pragma unroll
    for (int i = 0; i < NE; ++i) out[i] = __ldg(p + i);
}
template <typename T, int NE>
__device__ __forceinline__ void store_col(T *p, const T (&in)[NE]) {
    constexpr int E = Vec16<T>::E;
    if constexpr ((NE % E) == 0) {
        if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) {
            using V = typename Vec16<T>::type;
#pragma unroll
            for (int j = 0; j < NE / E; ++j) {
                V v;
                T *e = reinterpret_cast<T *>(&v);
#pragma unroll
                for (int t = 0; t < E; ++t) e[t] = in[j * E + t];
                reinterpret_cast<V *>(p)[j] = v;
            }
            return;
        }
    }
#pragma unroll
    for (int i = 0; i < NE; ++i) p[i] = in[i];
}

template <typename T, int NE>
__device__ __forceinline__ void zero(T (&a)[NE]) {
#pragma unroll
    for (int i = 0; i < NE; ++i) a[i] = T(0);
}

template <typename T, int NE>
__device__ __forceinline__ void soc_cols(T (&v)[NE], int ncones, const int *start, const T *mu) {
    for (int c = 0; c < ncones; ++c) {
        const int s = start[c];
        T s0 = T(0), s1 = T(0), s2 = T(0);
#pragma unroll
        for (int i = 0; i < NE; ++i) {
            if (i == s) s0 = v[i];
            if (i == s + 1) s1 = v[i];
            if (i == s + 2) s2 = v[i];
        }
        project_soc3(s0, s1, s2, mu[c]);
#pragma unroll
        for (int i = 0; i < NE; ++i) {
            if (i == s) v[i] = s0;
            if (i == s + 1) v[i] = s1;
            if (i == s + 2) v[i] = s2;
        }
    }
}

constexpr int TPI_THREADS = 128;

template <typename T, int NX, int NU, bool FAST, bool EXT>
__global__ void __launch_bounds__(TPI_THREADS, (sizeof(T) == 4 && !EXT) ? 4 : 2) tpi_solve_kernel(const __grid_constant__ KParams<T, NX, NU> P) {
    using SX = SoA<T, NX>;
    using SU = SoA<T, NU>;
    const int N = P.N;
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= P.B) return;
    const int64_t S = P.Bpad;
    const T rho = P.rho;

    const T *x0p = P.x0 + b * NX;
    const T *xrefp = P.Xref + (P.xref_pi ? b * (int64_t)N * NX : 0);
    const T *urefp = P.Uref ? P.Uref + (P.uref_pi ? b * (int64_t)(N - 1) * NU : 0) : nullptr;
    const int64_t offx = b * (int64_t)N * NX, offu = b * (int64_t)(N - 1) * NU;
    const bool cold = P.cold != 0;

    T x0[NX];
    load_col<T, NX>(x0p, x0);

    // ---------------- prologue: warm-start state -> workspace ----------------
    if (!cold) {
        for (int k = 0; k < N; ++k) {
            T a[NX];
            if (P.s_vnew) load_col<T, NX>(P.s_vnew + offx + (int64_t)k * NX, a); else zero(a);
            SX::store(P.w_v[0], k, S, b, a);
            if (P.s_v) load_col<T, NX>(P.s_v + offx + (int64_t)k * NX, a); else zero(a);
            SX::store(P.w_v[1], k, S, b, a);
            if (P.s_g) load_col<T, NX>(P.s_g + offx + (int64_t)k * NX, a); else zero(a);
            SX::store(P.w_g, k, S, b, a);
        }
        for (int k = 0; k < N - 1; ++k) {
            T a[NU];
            if (P.s_znew) load_col<T, NU>(P.s_znew + offu + (int64_t)k * NU, a); else zero(a);
            SU::store(P.w_z[0], k, S, b, a);
            if (P.s_z) load_col<T, NU>(P.s_z + offu + (int64_t)k * NU, a); else zero(a);
            SU::store(P.w_z[1], k, S, b, a);
            if (P.s_y) load_col<T, NU>(P.s_y + offu + (int64_t)k * NU, a); else zero(a);
            SU::store(P.w_y, k, S, b, a);
        }
    }
    if constexpr (EXT) {
        // admm.cpp:352-376: cone / hyperplane slacks start from the previous rollout x,u (x[:,0] = x0);
        // their duals persist.
        for (int k = 0; k < N; ++k) {
            T xin[NX], a[NX];
            if (k == 0) {
#pragma unroll
                for (int i = 0; i < NX; ++i) xin[i] = x0[i];
            } else if (!cold && P.s_x) {
                load_col<T, NX>(P.s_x + offx + (int64_t)k * NX, xin);
            } else {
                zero(xin);
            }
            if (P.soc_x) {
                SX::store(P.w_vc, k, S, b, xin);
                if (!cold && P.s_gc) load_col<T, NX>(P.s_gc + offx + (int64_t)k * NX, a); else zero(a);
                SX::store(P.w_gc, k, S, b, a);
            }
            if (P.lin_x) {
                SX::store(P.w_vl, k, S, b, xin);
                if (!cold && P.s_gl) load_col<T, NX>(P.s_gl + offx + (int64_t)k * NX, a); else zero(a);
                SX::store(P.w_gl, k, S, b, a);
            }
            if (P.tvl_x) {
                SX::store(P.w_vlt, k, S, b, xin);
                if (!cold && P.s_gl_tv) load_col<T, NX>(P.s_gl_tv + offx + (int64_t)k * NX, a); else zero(a);
                SX::store(P.w_glt, k, S, b, a);
            }
        }
        for (int k = 0; k < N - 1; ++k) {
            T uin[NU], a[NU];
            if (!cold && P.s_u) load_col<T, NU>(P.s_u + offu + (int64_t)k * NU, uin); else zero(uin);
            if (P.soc_u) {
                SU::store(P.w_zc, k, S, b, uin);
                if (!cold && P.s_yc) load_col<T, NU>(P.s_yc + offu + (int64_t)k * NU, a); else zero(a);
                SU::store(P.w_yc, k, S, b, a);
            }
            if (P.lin_u) {
                SU::store(P.w_zl, k, S, b, uin);
                if (!cold && P.s_yl) load_col<T, NU>(P.s_yl + offu + (int64_t)k * NU, a); else zero(a);
                SU::store(P.w_yl, k, S, b, a);
            }
            if (P.tvl_u) {
                SU::store(P.w_zlt, k, S, b, uin);
                if (!cold && P.s_yl_tv) load_col<T, NU>(P.s_yl_tv + offu + (int64_t)k * NU, a); else zero(a);
                SU::store(P.w_ylt, k, S, b, a);
            }
        }
    }

    // ---------------- ADMM iterations ----------------
    int it_done = 0, solved = 0, last_dst = 0;
    bool conv_first = false;  // converged at the first iteration: work->v keeps its input value
    T res_px = T(0), res_dx = T(0), res_pu = T(0), res_du = T(0);

    for (int it = 0; it < P.max_iter; ++it) {
        const int c = it & 1, dst = c ^ 1;
        const bool zin = cold && it == 0;  // vnew, g, znew, y (and v, z) are all zero on entry
        const int vs = (it == 0) ? 1 : c;  // where work->v / work->z live for the dual residual

        // ---- update_linear_cost (terminal) : p_{N-1} = -(Pinf^T xref_{N-1}) - rho (vnew - g) [...] ----
        T p[NX];
        {
            T xr[NX], vn[NX], g[NX];
            load_col<T, NX>(xrefp + (int64_t)(N - 1) * NX, xr);
            if (zin) { zero(vn); zero(g); } else { SX::load(P.w_v[c], N - 1, S, b, vn); SX::load(P.w_g, N - 1, S, b, g); }
            T pt[NX];
            dots_f<FAST, NX, NX>([&](int j, int i) { return P.Pinf[i + NX * j]; }, xr, pt);  // (Pinf^T xref)(j), i ascending
#pragma unroll
            for (int j = 0; j < NX; ++j) p[j] = nmac<FAST>(-pt[j], rho, vn[j] - g[j]);
            if constexpr (EXT) {
                if (P.soc_x) {
                    SX::load(P.w_vc, N - 1, S, b, vn); SX::load(P.w_gc, N - 1, S, b, g);
#pragma unroll
                    for (int j = 0; j < NX; ++j) p[j] = nmac<FAST>(p[j], rho, vn[j] - g[j]);
                }
                if (P.lin_x) {
                    SX::load(P.w_vl, N - 1, S, b, vn); SX::load(P.w_gl, N - 1, S, b, g);
#pragma unroll
                    for (int j = 0; j < NX; ++j) p[j] = nmac<FAST>(p[j], rho, vn[j] - g[j]);
                }
                if (P.tvl_x) {
                    SX::load(P.w_vlt, N - 1, S, b, vn); SX::load(P.w_glt, N - 1, S, b, g);
#pragma unroll
                    for (int j = 0; j < NX; ++j) p[j] = nmac<FAST>(p[j], rho, vn[j] - g[j]);
                }
            }
        }

        // ---- backward_pass_grad fused with update_linear_cost ----
        for (int k = N - 2; k >= 0; --k) {
            T q[NX], r[NU], tb[NU], pa_[NX];
            {
                // every global load of this step is issued before the first use (a thread has no other way to overlap
                // them: one dependent load round costs ~1 us and the EXT path used to have five per step)
                T xr[NX], vn[NX], g[NX], ur[NU], zn[NU], y[NU];
                T ev[EXT ? 3 : 1][NX], eg[EXT ? 3 : 1][NX], ez[EXT ? 3 : 1][NU], ey[EXT ? 3 : 1][NU];
                load_col<T, NX>(xrefp + (int64_t)k * NX, xr);
                if (urefp) load_col<T, NU>(urefp + (int64_t)k * NU, ur); else zero(ur);
                if (zin) { zero(vn); zero(g); zero(zn); zero(y); } else {
                    SX::load(P.w_v[c], k, S, b, vn); SX::load(P.w_g, k, S, b, g);
                    SU::load(P.w_z[c], k, S, b, zn); SU::load(P.w_y, k, S, b, y);
                }
                if constexpr (EXT) {
                    if (P.soc_x) { SX::load(P.w_vc, k, S, b, ev[0]); SX::load(P.w_gc, k, S, b, eg[0]); }
                    if (P.lin_x) { SX::load(P.w_vl, k, S, b, ev[1]); SX::load(P.w_gl, k, S, b, eg[1]); }
                    if (P.tvl_x) { SX::load(P.w_vlt, k, S, b, ev[2]); SX::load(P.w_glt, k, S, b, eg[2]); }
                    if (P.soc_u) { SU::load(P.w_zc, k, S, b, ez[0]); SU::load(P.w_yc, k, S, b, ey[0]); }
                    if (P.lin_u) { SU::load(P.w_zl, k, S, b, ez[1]); SU::load(P.w_yl, k, S, b, ey[1]); }
                    if (P.tvl_u) { SU::load(P.w_zlt, k, S, b, ez[2]); SU::load(P.w_ylt, k, S, b, ey[2]); }
                }
                // the two products that only need p_{k+1} run while those loads are in flight
                dots_f<FAST, NU, NX>([&](int j, int i) { return P.Bm[i + NX * j]; }, p, tb);  // B^T p
                dots_f<FAST, NX, NX>([&](int i, int m) { return P.AmBKt[i + NX * m]; }, p, pa_);
#pragma unroll
                for (int i = 0; i < NX; ++i) q[i] = nmac<FAST>(-(xr[i] * P.Qd[i]), rho, vn[i] - g[i]);
#pragma unroll
                for (int j = 0; j < NU; ++j) r[j] = nmac<FAST>(-(ur[j] * P.Rd[j]), rho, zn[j] - y[j]);
                if constexpr (EXT) {
                    const bool fx[3] = {P.soc_x != 0, P.lin_x != 0, P.tvl_x != 0}, fu[3] = {P.soc_u != 0, P.lin_u != 0, P.tvl_u != 0};
#pragma unroll
                    for (int t = 0; t < 3; ++t) {  // admm.cpp:268-276 / :281-289, in the reference's order
                        if (fx[t]) {
#pragma unroll
                            for (int i = 0; i < NX; ++i) q[i] = nmac<FAST>(q[i], rho, ev[t][i] - eg[t][i]);
                        }
                        if (fu[t]) {
#pragma unroll
                            for (int j = 0; j < NU; ++j) r[j] = nmac<FAST>(r[j], rho, ez[t][j] - ey[t][j]);
                        }
                    }
                }
            }
            // d_k = Quu_inv * ((B^T p_{k+1} + r_k) + BPf)                                (admm.cpp:17)
            T s[NU], d[NU];
#pragma unroll
            for (int j = 0; j < NU; ++j) s[j] = (tb[j] + r[j]) + P.BPf[j];
            dots_f<FAST, NU, NU>([&](int j, int m) { return P.Quu[j + NU * m]; }, s, d);
            SU::store(P.w_d, k, S, b, d);
            // p_k = ((q_k + AmBKt p_{k+1}) - Kinf^T r_k) + APf                             (admm.cpp:18)
            T kr[NX];
            dots_f<FAST, NX, NU>([&](int i, int j) { return P.Kinf[j + NU * i]; }, r, kr);
#pragma unroll
            for (int i = 0; i < NX; ++i) p[i] = ((q[i] + pa_[i]) - kr[i]) + P.APf[i];
        }

        // ---- forward_pass fused with update_slack, update_dual, residuals ----
        T x[NX];
#pragma unroll
        for (int i = 0; i < NX; ++i) x[i] = x0[i];
        T rpx = T(0), rdx = T(0), rpu = T(0), rdu = T(0);
        for (int k = 0; k < N; ++k) {
            // all global loads of the column first (state part, then — if the column has inputs — the input part)
            T g[NX], vo[NX], vn[NX], d[NU], y[NU], zo[NU];
            T egx[EXT ? 3 : 1][NX], eyu[EXT ? 3 : 1][NU];
            const bool hasu = k < N - 1;
            if (zin) { zero(g); zero(vo); zero(y); zero(zo); } else {
                SX::load(P.w_g, k, S, b, g); SX::load(P.w_v[vs], k, S, b, vo);
                if (hasu) { SU::load(P.w_y, k, S, b, y); SU::load(P.w_z[vs], k, S, b, zo); }
            }
            if (hasu) SU::load(P.w_d, k, S, b, d);
            if constexpr (EXT) {
                if (P.soc_x) SX::load(P.w_gc, k, S, b, egx[0]);
                if (P.lin_x) SX::load(P.w_gl, k, S, b, egx[1]);
                if (P.tvl_x) SX::load(P.w_glt, k, S, b, egx[2]);
                if (hasu) {
                    if (P.soc_u) SU::load(P.w_yc, k, S, b, eyu[0]);
                    if (P.lin_u) SU::load(P.w_yl, k, S, b, eyu[1]);
                    if (P.tvl_u) SU::load(P.w_ylt, k, S, b, eyu[2]);
                }
            }
            // Kinf x_k and A x_k only need x_k: computed while the loads above are in flight
            T kx[NU], ax[NX];
            if (hasu) {
                dots_f<FAST, NU, NX>([&](int j, int m) { return P.Kinf[j + NU * m]; }, x, kx);
                dots_f<FAST, NX, NX>([&](int i, int m) { return P.A[i + NX * m]; }, x, ax);
            }
            {   // state column k
                auto upd_x = [&](auto lo, auto hi) {  // vnew = clamp(x + g); g += x - vnew; residual maxima
#pragma unroll
                    for (int i = 0; i < NX; ++i) {
                        const T v = FAST ? fmin(fmax(x[i] + g[i], lo(i)), hi(i)) : clamp_ref(x[i] + g[i], lo(i), hi(i));
                        vn[i] = v;
                        g[i] = (g[i] + x[i]) - v;
                        rpx = fmax(rpx, tabs(x[i] - v));  // == (|d| > m) ? |d| : m  (m is never NaN)
                        rdx = fmax(rdx, tabs(vo[i] - v));
                    }
                };
                if (P.bounds_tv && P.en_state_bound)
                    upd_x([&](int i) { return __ldg(P.x_min + (int64_t)k * NX + i); }, [&](int i) { return __ldg(P.x_max + (int64_t)k * NX + i); });
                else
                    upd_x([&](int i) { return P.xlo[i]; }, [&](int i) { return P.xhi[i]; });  // constant-bank operands; (-inf,+inf) if disabled
                SX::store(P.w_v[dst], k, S, b, vn);
                SX::store(P.w_g, k, S, b, g);
                if constexpr (EXT) {
                    if (P.soc_x) {
                        T(&gc)[NX] = egx[0];
                        T vc[NX];
#pragma unroll
                        for (int i = 0; i < NX; ++i) vc[i] = x[i] + gc[i];
                        soc_cols<T, NX>(vc, P.ncx, P.cone_x_start, P.cone_x_mu);
#pragma unroll
                        for (int i = 0; i < NX; ++i) gc[i] = (gc[i] + x[i]) - vc[i];
                        SX::store(P.w_vc, k, S, b, vc);
                        SX::store(P.w_gc, k, S, b, gc);
                    }
                    if (P.lin_x) {
                        T(&gl)[NX] = egx[1];
                        T vl[NX];
#pragma unroll
                        for (int i = 0; i < NX; ++i) vl[i] = x[i] + gl[i];
                        project_rows<FAST, T, NX>(vl, P.Alin_x, P.nlx, 0, P.nlx, P.blin_x);
#pragma unroll
                        for (int i = 0; i < NX; ++i) gl[i] = (gl[i] + x[i]) - vl[i];
                        SX::store(P.w_vl, k, S, b, vl);
                        SX::store(P.w_gl, k, S, b, gl);
                    }
                    if (P.tvl_x) {
                        T(&gl)[NX] = egx[2];
                        T vl[NX];
#pragma unroll
                        for (int i = 0; i < NX; ++i) vl[i] = x[i] + gl[i];
                        project_rows<FAST, T, NX>(vl, P.tv_Alin_x, P.ntvx * N, P.ntvx * k, P.ntvx, P.tv_blin_x + (int64_t)k * P.ntvx);
#pragma unroll
                        for (int i = 0; i < NX; ++i) gl[i] = (gl[i] + x[i]) - vl[i];
                        SX::store(P.w_vlt, k, S, b, vl);
                        SX::store(P.w_glt, k, S, b, gl);
                    }
                }
            }
            if (hasu) {  // input column k and the rollout step
                T u[NU], zn[NU];
#pragma unroll
                for (int j = 0; j < NU; ++j) u[j] = (-kx[j]) - d[j];  // u_k = -(Kinf x_k) - d_k    (admm.cpp:29)
                auto upd_u = [&](auto lo, auto hi) {
#pragma unroll
                    for (int j = 0; j < NU; ++j) {
                        const T z = FAST ? fmin(fmax(u[j] + y[j], lo(j)), hi(j)) : clamp_ref(u[j] + y[j], lo(j), hi(j));
                        zn[j] = z;
                        y[j] = (y[j] + u[j]) - z;
                        rpu = fmax(rpu, tabs(u[j] - z));
                        rdu = fmax(rdu, tabs(zo[j] - z));
                    }
                };
                if (P.bounds_tv && P.en_input_bound)
                    upd_u([&](int j) { return __ldg(P.u_min + (int64_t)k * NU + j); }, [&](int j) { return __ldg(P.u_max + (int64_t)k * NU + j); });
                else
                    upd_u([&](int j) { return P.ulo[j]; }, [&](int j) { return P.uhi[j]; });
                SU::store(P.w_z[dst], k, S, b, zn);
                SU::store(P.w_y, k, S, b, y);
                if constexpr (EXT) {
                    if (P.soc_u) {
                        T(&yc)[NU] = eyu[0];
                        T zc[NU];
#pragma unroll
                        for (int j = 0; j < NU; ++j) zc[j] = u[j] + yc[j];
                        soc_cols<T, NU>(zc, P.ncu, P.cone_u_start, P.cone_u_mu);
#pragma unroll
                        for (int j = 0; j < NU; ++j) yc[j] = (yc[j] + u[j]) - zc[j];
                        SU::store(P.w_zc, k, S, b, zc);
                        SU::store(P.w_yc, k, S, b, yc);
                    }
                    if (P.lin_u) {
                        T(&yl)[NU] = eyu[1];
                        T zl[NU];
#pragma unroll
                        for (int j = 0; j < NU; ++j) zl[j] = u[j] + yl[j];
                        project_rows<FAST, T, NU>(zl, P.Alin_u, P.nlu, 0, P.nlu, P.blin_u);
#pragma unroll
                        for (int j = 0; j < NU; ++j) yl[j] = (yl[j] + u[j]) - zl[j];
                        SU::store(P.w_zl, k, S, b, zl);
                        SU::store(P.w_yl, k, S, b, yl);
                    }
                    if (P.tvl_u) {
                        T(&yl)[NU] = eyu[2];
                        T zl[NU];
#pragma unroll
                        for (int j = 0; j < NU; ++j) zl[j] = u[j] + yl[j];
                        project_rows<FAST, T, NU>(zl, P.tv_Alin_u, P.ntvu * (N - 1), P.ntvu * k, P.ntvu, P.tv_blin_u + (int64_t)k * P.ntvu);
#pragma unroll
                        for (int j = 0; j < NU; ++j) yl[j] = (yl[j] + u[j]) - zl[j];
                        SU::store(P.w_zlt, k, S, b, zl);
                        SU::store(P.w_ylt, k, S, b, yl);
                    }
                }
                // x_{k+1} = (A x_k + B u_k) + f                                            (admm.cpp:30)
                T bu[NX];
                dots_f<FAST, NX, NU>([&](int i, int j) { return P.Bm[i + NX * j]; }, u, bu);
#pragma unroll
                for (int i = 0; i < NX; ++i) x[i] = (ax[i] + bu[i]) + P.f[i];
            }
        }
        it_done = it + 1;
        last_dst = dst;
        // termination_condition (admm.cpp:310-328)
        if (it_done % P.check_termination == 0) {
            res_px = rpx;
            res_dx = rdx * rho;
            res_pu = rpu;
            res_du = rdu * rho;
            if (res_px < P.pri_tol && res_pu < P.pri_tol && res_dx < P.dua_tol && res_du < P.dua_tol) {
                solved = 1;
                conv_first = (it == 0);
                break;
            }
        }
    }

    // ---------------- epilogue ----------------
    if (P.iter) P.iter[b] = it_done;
    if (P.solved) P.solved[b] = solved;
    if (P.residuals) {
        T *r = P.residuals + 4 * b;
        r[0] = res_px; r[1] = res_dx; r[2] = res_pu; r[3] = res_du;
    }
    const bool ran = it_done > 0;
    // solution->x = vnew, solution->u = znew (admm.cpp:436-437, 452-453); work->v = previous vnew when the
    // solve converged (return at :441 precedes :445), else = vnew.
    const int vfin = ran ? last_dst : 0;
    const int vprev = solved ? (1 - last_dst) : vfin;
    for (int k = 0; k < N; ++k) {
        T a[NX];
        if (ran || !cold) SX::load(P.w_v[vfin], k, S, b, a); else zero(a);
        if (P.sol_x) store_col<T, NX>(P.sol_x + offx + (int64_t)k * NX, a);
        if (P.s_vnew) store_col<T, NX>(P.s_vnew + offx + (int64_t)k * NX, a);
        if (P.s_v && ran && !conv_first) {
            SX::load(P.w_v[vprev], k, S, b, a);
            store_col<T, NX>(P.s_v + offx + (int64_t)k * NX, a);
        } else if (P.s_v && cold) {
            zero(a);
            store_col<T, NX>(P.s_v + offx + (int64_t)k * NX, a);
        }
        if (P.s_g) {
            if (ran || !cold) SX::load(P.w_g, k, S, b, a); else zero(a);
            store_col<T, NX>(P.s_g + offx + (int64_t)k * NX, a);
        }
        if constexpr (EXT) {
            if (P.soc_x && P.s_vcnew) { SX::load(P.w_vc, k, S, b, a); store_col<T, NX>(P.s_vcnew + offx + (int64_t)k * NX, a); }
            if (P.soc_x && P.s_gc) { SX::load(P.w_gc, k, S, b, a); store_col<T, NX>(P.s_gc + offx + (int64_t)k * NX, a); }
            if (P.lin_x && P.s_vlnew) { SX::load(P.w_vl, k, S, b, a); store_col<T, NX>(P.s_vlnew + offx + (int64_t)k * NX, a); }
            if (P.lin_x && P.s_gl) { SX::load(P.w_gl, k, S, b, a); store_col<T, NX>(P.s_gl + offx + (int64_t)k * NX, a); }
            if (P.tvl_x && P.s_vlnew_tv) { SX::load(P.w_vlt, k, S, b, a); store_col<T, NX>(P.s_vlnew_tv + offx + (int64_t)k * NX, a); }
            if (P.tvl_x && P.s_gl_tv) { SX::load(P.w_glt, k, S, b, a); store_col<T, NX>(P.s_gl_tv + offx + (int64_t)k * NX, a); }
        }
    }
    for (int k = 0; k < N - 1; ++k) {
        T a[NU];
        if (ran || !cold) SU::load(P.w_z[vfin], k, S, b, a); else zero(a);
        if (P.sol_u) store_col<T, NU>(P.sol_u + offu + (int64_t)k * NU, a);
        if (P.s_znew) store_col<T, NU>(P.s_znew + offu + (int64_t)k * NU, a);
        if (P.s_z && ran && !conv_first) {
            SU::load(P.w_z[vprev], k, S, b, a);
            store_col<T, NU>(P.s_z + offu + (int64_t)k * NU, a);
        } else if (P.s_z && cold) {
            zero(a);
            store_col<T, NU>(P.s_z + offu + (int64_t)k * NU, a);
        }
        if (P.s_y) {
            if (ran || !cold) SU::load(P.w_y, k, S, b, a); else zero(a);
            store_col<T, NU>(P.s_y + offu + (int64_t)k * NU, a);
        }
        if constexpr (EXT) {
            if (P.soc_u && P.s_zcnew) { SU::load(P.w_zc, k, S, b, a); store_col<T, NU>(P.s_zcnew + offu + (int64_t)k * NU, a); }
            if (P.soc_u && P.s_yc) { SU::load(P.w_yc, k, S, b, a); store_col<T, NU>(P.s_yc + offu + (int64_t)k * NU, a); }
            if (P.lin_u && P.s_zlnew) { SU::load(P.w_zl, k, S, b, a); store_col<T, NU>(P.s_zlnew + offu + (int64_t)k * NU, a); }
            if (P.lin_u && P.s_yl) { SU::load(P.w_yl, k, S, b, a); store_col<T, NU>(P.s_yl + offu + (int64_t)k * NU, a); }
            if (P.tvl_u && P.s_zlnew_tv) { SU::load(P.w_zlt, k, S, b, a); store_col<T, NU>(P.s_zlnew_tv + offu + (int64_t)k * NU, a); }
            if (P.tvl_u && P.s_yl_tv) { SU::load(P.w_ylt, k, S, b, a); store_col<T, NU>(P.s_yl_tv + offu + (int64_t)k * NU, a); }
        }
    }
    // work->u.col(0): the control every example applies (quadrotor_hovering.cpp:92) — one rollout step from d_0
    if (P.u0) {
        T u[NU];
        zero(u);
        if (ran) {
            T d[NU], kx[NU];
            SU::load(P.w_d, 0, S, b, d);
            dots_f<FAST, NU, NX>([&](int j, int m) { return P.Kinf[j + NU * m]; }, x0, kx);
#pragma unroll
            for (int j = 0; j < NU; ++j) u[j] = (-kx[j]) - d[j];
        } else if (!cold && P.s_u) {
            load_col<T, NU>(P.s_u + offu, u);
        }
        store_col<T, NU>(P.u0 + b * NU, u);
    }
    // work->x / work->u (the rollout every example applies, e.g. quadrotor_hovering.cpp:92): recomputed
    // from d and x0 with the same arithmetic as the last forward pass — bit-identical to it.
    if (P.s_x || P.s_u) {
        T x[NX];
#pragma unroll
        for (int i = 0; i < NX; ++i) x[i] = x0[i];
        for (int k = 0; k < N; ++k) {
            if (P.s_x) {
                if (ran || k == 0) {
                    store_col<T, NX>(P.s_x + offx + (int64_t)k * NX, x);
                } else if (cold) {  // no iteration ran: x[:,1:] keeps its (zero) input
                    T a[NX];
                    zero(a);
                    store_col<T, NX>(P.s_x + offx + (int64_t)k * NX, a);
                }
            }
            if (k < N - 1 && ran) {
                T d[NU], u[NU];
                SU::load(P.w_d, k, S, b, d);
                T kx[NU], ax[NX], bu[NX];
                dots_f<FAST, NU, NX>([&](int j, int m) { return P.Kinf[j + NU * m]; }, x, kx);
#pragma unroll
                for (int j = 0; j < NU; ++j) u[j] = (-kx[j]) - d[j];
                if (P.s_u) store_col<T, NU>(P.s_u + offu + (int64_t)k * NU, u);
                dots_f<FAST, NX, NX>([&](int i, int m) { return P.A[i + NX * m]; }, x, ax);
                dots_f<FAST, NX, NU>([&](int i, int j) { return P.Bm[i + NX * j]; }, u, bu);
#pragma unroll
                for (int i = 0; i < NX; ++i) x[i] = (ax[i] + bu[i]) + P.f[i];
            } else if (k < N - 1 && P.s_u && cold) {
                T a[NU];
                zero(a);
                store_col<T, NU>(P.s_u + offu + (int64_t)k * NU, a);
            }
        }
    }
}

}  // namespace tmpc
