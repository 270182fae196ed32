// common.cuh — arithmetic policy, vector helpers and the kernel parameter block shared by the TPI, GPI and GPS kernels.
//
// Arithmetic contract (DESIGN.md §4; SURVEY.md Appendix A/B.2):
//   every translation unit is compiled with -fmad=false, so plain `a*b + c` is NEVER contracted;
//   STRICT mode uses plain operators only  -> bit-identical to the pinned reference build
//   FAST   mode calls fma()/fmaf() explicitly in dot products and axpy-like updates (same order of terms).
// Division and square root are IEEE (no --use_fast_math).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tmpc {

template <bool FAST, typename T>
__device__ __forceinline__ T mac(T acc, T a, T b) {  // acc + a*b
    if constexpr (FAST) {
        return fma(a, b, acc);
    } else {
        return acc + a * b;
    }
}
template <bool FAST, typename T>
__device__ __forceinline__ T nmac(T acc, T a, T b) {  // acc - a*b
    if constexpr (FAST) {
        return fma(-a, b, acc);
    } else {
        return acc - a * b;
    }
}
// ---- several ascending-k dot products against the same vector -------------------------------------------------
// out[r] = M[r][0]*v[0]; out[r] = out[r] + M[r][k]*v[k]   (k ascending; STRICT: separate multiply and add, never
// contracted under -fmad=false; FAST: fma with the same order of terms).
// element-wise o = a + b / o = a - b on short vectors
template <typename T, int NV>
__device__ __forceinline__ void vadd(const T (&a)[NV], const T (&b)[NV], T (&o)[NV]) {
#pragma unroll
    for (int e = 0; e < NV; ++e) o[e] = a[e] + b[e];
}
template <typename T, int NV>
__device__ __forceinline__ void vsub(const T (&a)[NV], const T (&b)[NV], T (&o)[NV]) {
#pragma unroll
    for (int e = 0; e < NV; ++e) o[e] = a[e] - b[e];
}

template <bool FAST, int NR, int NE, typename T>
__device__ __forceinline__ void dots(const T (&M)[NR][NE], const T (&v)[NE], T (&out)[NR]) {
#pragma unroll
    for (int r = 0; r < NR; ++r) {
        T s = M[r][0] * v[0];
#pragma unroll
        for (int k = 1; k < NE; ++k) s = mac<FAST>(s, M[r][k], v[k]);
        out[r] = s;
    }
}

// same, with the coefficients supplied by a callable coef(r, k) (e.g. constant-bank matrix entries in the TPI kernel)
template <bool FAST, int NR, int NE, typename F, typename T>
__device__ __forceinline__ void dots_f(F coef, const T (&v)[NE], T (&out)[NR]) {
#pragma unroll
    for (int r = 0; r < NR; ++r) {
        T s = coef(r, 0) * v[0];
#pragma unroll
        for (int k = 1; k < NE; ++k) s = mac<FAST>(s, coef(r, k), v[k]);
        out[r] = s;
    }
}

template <typename T>
__device__ __forceinline__ T tabs(T a) {
    return a < T(0) ? -a : a;
}
__device__ __forceinline__ float tabs(float a) { return fabsf(a); }
__device__ __forceinline__ double tabs(double a) { return fabs(a); }
__device__ __forceinline__ float tsqrt(float a) { return sqrtf(a); }
__device__ __forceinline__ double tsqrt(double a) { return sqrt(a); }

// Eigen's x_max.cwiseMin(x_min.cwiseMax(v)) as executed (SURVEY A.2): m = (lo<v)?v:lo ; r = (m<hi)?m:hi
template <typename T>
__device__ __forceinline__ T clamp_ref(T v, T lo, T hi) {
    T m = (lo < v) ? v : lo;
    return (m < hi) ? m : hi;
}

// project_soc for a 3-vector exactly as the reference executes it (admm.cpp:39-60, SURVEY A.4):
// mu and the norm are narrowed to float even when T = double.
template <typename T>
__device__ __forceinline__ void project_soc3(T &s0, T &s1, T &s2, T mu_T) {
    const float mu = (float)mu_T;
    const T u0 = s2 * (T)mu;
    T sq = s0 * s0;
    sq = sq + s1 * s1;
    const float a = (float)tsqrt(sq);
    if ((T)a <= -u0) {
        s0 = T(0);
        s1 = T(0);
        s2 = T(0);
    } else if ((T)a <= u0) {
        // inside the cone: unchanged
    } else {
        const T third = (T)(a / mu);  // float division (admm.cpp:54)
        const T c = T(0.5) * (T(1) + u0 / (T)a);
        s0 = c * s0;
        s1 = c * s1;
        s2 = c * third;
    }
}

// branch-free twin of project_soc3 (same operations, same results): every lane of a warp projects a different cone, so
// the three cases are computed and selected instead of branched on
template <typename T>
__device__ __forceinline__ void project_soc3_sel(T &s0, T &s1, T &s2, T mu_T) {
    const float mu = (float)mu_T;
    const T u0 = s2 * (T)mu;
    T sq = s0 * s0;
    sq = sq + s1 * s1;
    const float a = (float)tsqrt(sq);
    const T ad = (T)a;
    const bool below = ad <= -u0, inside = ad <= u0;
    const T third = (T)(a / mu);
    const T c = T(0.5) * (T(1) + u0 / ad);
    const T r0 = c * s0, r1 = c * s1, r2 = c * third;
    s0 = below ? T(0) : (inside ? s0 : r0);
    s1 = below ? T(0) : (inside ? s1 : r1);
    s2 = below ? T(0) : (inside ? s2 : r2);
}

// sequential hyperplane projections on one column (admm.cpp:148-157 / :186-195, SURVEY A.5).
// A is (ld x NE) column-major in global memory; rows row0 .. row0+n-1; b[k] at bvec[k].
template <bool FAST, typename T, int NE>
__device__ __forceinline__ void project_rows(T (&z)[NE], const T *A, int ld, int row0, int n, const T *bvec) {
    for (int r = 0; r < n; ++r) {
        T a[NE];
#pragma unroll
        for (int j = 0; j < NE; ++j) a[j] = __ldg(A + row0 + r + (int64_t)j * ld);
        const T bb = __ldg(bvec + r);
        T cv = a[0] * z[0];
#pragma unroll
        for (int j = 1; j < NE; ++j) cv = mac<FAST>(cv, a[j], z[j]);
        if (cv > bb) {
            T nn = a[0] * a[0];
#pragma unroll
            for (int j = 1; j < NE; ++j) nn = mac<FAST>(nn, a[j], a[j]);
            const T dist = (cv - bb) / nn;  // a.dot(z) is recomputed by the reference; same value
#pragma unroll
            for (int j = 0; j < NE; ++j) z[j] = nmac<FAST>(z[j], dist, a[j]);
        }
    }
}

// the 16-byte vector type of T and its element count
template <typename T> struct Vec16;
template <> struct Vec16<float> { using type = float4; static constexpr int E = 4; };
template <> struct Vec16<double> { using type = double2; static constexpr int E = 2; };

constexpr int MAX_CONES = 4;  // cones per knot point and per side held in the parameter block

// Run-time part of the streamed lane-group kernel's workspace description (gps_kernel.cuh); the record layout itself is a
// compile-time function of the shape and of the compiled-in constraint families (GpsRec).
struct GpsLayout {
    int has_b;  // the optional-output region (previous box slacks, family slacks) is allocated and maintained
};

// Kernel parameter block.  Passed by value (__grid_constant__): it lives in the constant bank, so with
// compile-time indices the matrix entries become immediate constant operands of the FMA instructions.
// All matrices are column-major copies of the reference's cache / workspace (types.hpp:43-51,186-190).
template <typename T, int NX, int NU>
struct KParams {
    T A[NX * NX];
    T Bm[NX * NU];
    T f[NX];
    T Qd[NX];
    T Rd[NU];
    T Kinf[NU * NX];
    T Pinf[NX * NX];
    T Quu[NU * NU];
    T AmBKt[NX * NX];
    T APf[NX];
    T BPf[NU];
    T rho, pri_tol, dua_tol;
    int N, max_iter, check_termination;
    int en_state_bound, en_input_bound;
    int soc_x, soc_u;    // en_*_soc && num cones > 0  (admm.cpp:102,107)
    int ncx, ncu;        // cone loops run under en_*_soc alone (admm.cpp:112,125)
    int lin_x, lin_u, nlx, nlu;
    int tvl_x, tvl_u, ntvx, ntvu;
    int cone_x_start[MAX_CONES], cone_u_start[MAX_CONES];
    T cone_x_mu[MAX_CONES], cone_u_mu[MAX_CONES];
    int64_t B;     // instances in this launch
    int64_t Bpad;  // workspace stride (instances, multiple of 32)
    int cold;
    int bounds_tv;      // bounds vary along the horizon (else row 0 is used for every k)
    T xlo[NX], xhi[NX], ulo[NU], uhi[NU];  // time-invariant bounds (column 0); (-inf, +inf) when the bound is disabled
    const T *Pinf_g;    // Pinf in global memory (column-major), GPI terminal cost
    int xref_pi, uref_pi;
    // inputs (user layout, instance-major)
    const T *x0, *Xref, *Uref;
    // bounds (device, column-major nx x N etc.)
    const T *x_min, *x_max, *u_min, *u_max;
    // hyperplanes (device)
    const T *Alin_x, *blin_x, *Alin_u, *blin_u;
    const T *tv_Alin_x, *tv_blin_x, *tv_Alin_u, *tv_blin_u;
    // warm-start state in/out (user layout), any may be null
    T *s_x, *s_u, *s_v, *s_z, *s_vnew, *s_znew, *s_g, *s_y;
    T *s_vcnew, *s_zcnew, *s_gc, *s_yc, *s_vlnew, *s_zlnew, *s_gl, *s_yl;
    T *s_vlnew_tv, *s_zlnew_tv, *s_gl_tv, *s_yl_tv;
    // outputs
    T *sol_x, *sol_u;  // may be null
    int32_t *iter, *solved;
    T *residuals;
    T *u0;  // [B][nu] first rollout input, may be null
    const T *models;  // GPI: per-instance cache blobs [B][blob+1] (A,B,f,Qd,Rd,Kinf,Pinf,Quu,AmBKt,APf,BPf,rho) or null
    T *gpi_vscratch;  // GPI: [B][N][L][PVP] copy of the previous primal pack (work->v / work->z) while v,z are persisted
    T *gps_ws;        // GPS: [resident warps][N][gps.rec] streamed state records
    GpsLayout gps;
    // TPI workspace (structure-of-arrays, 16-byte vectors, [k][vec][Bpad]).  The streamed kernel's GPS_CONES variants find the
    // per-instance cone coefficients in w_vc (state cones) and w_zc (input cones).
    void *w_v[2], *w_z[2], *w_g, *w_y, *w_d;
    void *w_vc, *w_zc, *w_gc, *w_yc, *w_vl, *w_zl, *w_gl, *w_yl, *w_vlt, *w_zlt, *w_glt, *w_ylt;
};

}  // namespace tmpc
