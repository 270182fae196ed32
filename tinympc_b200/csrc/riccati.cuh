// riccati.cuh — the one-time Riccati precompute and its rho-sensitivity, written once for the host and the device.
//
// Restates tiny_precompute_and_set_cache (TinyMPC src/tinympc/tiny_api.cpp:307-381):
//   Q1 = diag(Qw) + rho I, R1 = diag(Rw) + rho I           (:317-318; Qw = Qdiag + rho, Rw = Rdiag + rho already: the "double rho")
//   P <- rho I, K_prev <- 0                                (:330-333)
//   repeat <= 1000:  K = (R1 + B'PB)^-1 B'PA ;  Pn = Q1 + A'P(A - BK) ; stop if max|K - K_prev| < 1e-5   (:335-349)
//   Quu_inv = (R1 + B'Pinf B)^-1 ; AmBKt = (A - B Kinf)' ; APf = AmBKt Pinf f ; BPf = B' Pinf f   (:352-357)
// With TANGENT, the forward-mode derivative with respect to rho is carried beside the primal and ended by the primal's own
// stop test (the tables dKinf/drho, dPinf/drho of adaptive rho; the role rho_benchmark.cpp:215-229's tables play for the
// reference's one hard-coded quadrotor):
//   dQ1 = dR1 = 2 I (rho enters Q1, R1 twice), dP = I (P starts at rho I)
//   per sweep, S = R1 + B'PB:  dS = dR1 + B'dP B ;  dK = S^-1 (B'dP A - dS K) ;  dPn = (dQ1 + A'dP (A - BK)) - A'P (B dK)
//
// Arithmetic contract: every element is produced by one fixed operation sequence — products accumulated from 0 in ascending
// inner index with separate multiply and add (the Makefile compiles without contraction), Gauss-Jordan with partial pivoting
// and IEEE division — whichever lanes share the work.  The host runs it with one lane (tinympc_b200_precompute_cache and the
// batched host calls), the device with the 32 lanes of a warp (riccati_kernel), so their blobs and tables are bit-identical.
// The result agrees with Eigen's to rounding (different summation order / LU), not bit for bit; the solve kernels accept ANY
// cache through the C ABI, so parity of the solve path never depends on this routine.
#pragma once
#include <algorithm>
#include <cmath>

#include "launch.h"
#include "model_blob.h"

namespace tmpc {

// dimensions: run-time values on the host (any nx, nu > 0), compile-time constants in the kernels
struct DynDims {
    int nx, nu;
};
template <int NX, int NU>
struct FixDims {
    static constexpr int nx = NX, nu = NU;
};

// the lanes that share the elements of every operation: lane `lane` takes every n-th element, sync() orders their
// shared-memory traffic, max() reduces a value over the lanes
struct HostLanes {
    static constexpr int n = 1;
    int lane = 0;
    __host__ __device__ void sync() const {}
    template <typename T>
    __host__ __device__ T max(T v) const { return v; }
};
struct WarpLanes {
    static constexpr int n = 32;
    int lane;
    __host__ __device__ void sync() const {
#ifdef __CUDA_ARCH__
        __syncwarp();
#endif
    }
    template <typename T>
    __host__ __device__ T max(T v) const {
#ifdef __CUDA_ARCH__
#pragma unroll
        for (int m = 16; m >= 1; m >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, m));
#endif
        return v;
    }
};

// element offsets of one instance's scratch, every matrix column-major; the T* pieces exist only with the tangent
struct RiccatiScratch {
    int A, B, At, Bt, P, Pn, BtP, BtPA, K, Kp, S, Si, AmBK, AtP, Pf, Q1, R1, mult;
    int Qw, Rw, dP, dPn, dAtP, BdK, dBtP, T1, T2, dK, dS;
    int total;
};
__host__ __device__ constexpr RiccatiScratch riccati_scratch(int nx, int nu, bool tangent) {
    const int xx = nx * nx, xu = nx * nu, uu = nu * nu, t = tangent ? 1 : 0;
    RiccatiScratch s{};
    s.A = 0, s.B = s.A + xx, s.At = s.B + xu, s.Bt = s.At + xx, s.P = s.Bt + xu, s.Pn = s.P + xx, s.BtP = s.Pn + xx, s.BtPA = s.BtP + xu, s.K = s.BtPA + xu;
    s.Kp = s.K + xu, s.S = s.Kp + xu, s.Si = s.S + uu, s.AmBK = s.Si + uu, s.AtP = s.AmBK + xx, s.Pf = s.AtP + xx, s.Q1 = s.Pf + nx;
    s.R1 = s.Q1 + nx, s.mult = s.R1 + nu, s.Qw = s.mult + nu;
    s.Rw = s.Qw + t * nx, s.dP = s.Rw + t * nu, s.dPn = s.dP + t * xx, s.dAtP = s.dPn + t * xx, s.BdK = s.dAtP + t * xx;
    s.dBtP = s.BdK + t * xx, s.T1 = s.dBtP + t * xu, s.T2 = s.T1 + t * xu, s.dK = s.T2 + t * xu, s.dS = s.dK + t * xu;
    s.total = s.dS + t * uu;
    return s;
}

// f(i, j, e) for every element (i, j) of an R x C matrix, e = i + j R, dealt to the lanes (one lane: no index division)
template <class Lanes, class F>
__host__ __device__ __forceinline__ void ric_each(Lanes L, int R, int C, F f) {
    if constexpr (Lanes::n == 1) {
        for (int j = 0; j < C; ++j)
            for (int i = 0; i < R; ++i) f(i, j, i + j * R);
    } else {
        for (int e = L.lane; e < R * C; e += L.n) f(e % R, e / R, e);
    }
}

// a column-major matrix operand: element (i, l) at p[i + l * sl]
template <typename T>
struct RicView {
    const T *p;
    int sl;
    __host__ __device__ T operator()(int i, int l) const { return p[i + l * sl]; }
};

// z = X(:, l0 .. l0+3) y(l0 .. l0+3) added to z term by term in ascending l: four steps of a column's sums on one lane, so that
// z is loaded and stored once per four; X contiguous down its columns (column stride sl), z and X never overlap
template <typename T>
__host__ __device__ inline void ric_axpy4(T *__restrict__ z, const T *__restrict__ x, int sl, const T *v, int R) {
    const T *x0 = x, *x1 = x + sl, *x2 = x + 2 * sl, *x3 = x + 3 * sl;
    for (int i = 0; i < R; ++i) z[i] = (((z[i] + x0[i] * v[0]) + x1[i] * v[1]) + x2[i] * v[2]) + x3[i] * v[3];
}
template <typename T>
__host__ __device__ inline void ric_axpy(T *__restrict__ z, const T *__restrict__ x, T v, int R) {
    for (int i = 0; i < R; ++i) z[i] = z[i] + x[i] * v;
}

// Z (R x C) = X (R x KK) Y (KK x C): element (i, j) accumulated from 0 over l ascending.  One lane runs a column's sums
// side by side (l outside i), so that they are not one long dependency chain each; the sequence per element is the same.
template <typename T, class Lanes>
__host__ __device__ __forceinline__ void ric_mul(Lanes L, T *Z, int R, int C, int KK, RicView<T> x, RicView<T> y) {
    if constexpr (Lanes::n == 1) {
        for (int j = 0; j < C; ++j) {
            T *z = Z + j * R;
            for (int i = 0; i < R; ++i) z[i] = T(0);
            int l = 0;
            for (; l + 4 <= KK; l += 4) {
                const T v[4] = {y(l, j), y(l + 1, j), y(l + 2, j), y(l + 3, j)};
                ric_axpy4(z, x.p + l * x.sl, x.sl, v, R);
            }
            for (; l < KK; ++l) ric_axpy(z, x.p + l * x.sl, y(l, j), R);
        }
    } else {
        ric_each(L, R, C, [&](int i, int j, int e) {
            T acc = T(0);
#ifdef __CUDA_ARCH__
#pragma unroll 4
#endif
            for (int l = 0; l < KK; ++l) acc = acc + x(i, l) * y(l, j);
            Z[e] = acc;
        });
    }
    L.sync();
}

// Gauss-Jordan with partial pivoting on the n x n matrix X (destroyed) -> inv; mult: n elements of scratch for the column's
// multipliers, saved before the elimination so that it can update X in place.  Returns false when a pivot is exactly zero.
template <typename T, class Lanes>
__host__ __device__ __forceinline__ bool ric_invert(Lanes L, T *X, T *inv, T *mult, int n) {
    ric_each(L, n, n, [&](int i, int j, int e) { inv[e] = i == j ? T(1) : T(0); });
    L.sync();
    for (int c = 0; c < n; ++c) {
        int piv = c;
        for (int i = c + 1; i < n; ++i)
            if (fabs(X[i + c * n]) > fabs(X[piv + c * n])) piv = i;
        if (X[piv + c * n] == T(0)) return false;
        L.sync();
        if (piv != c) {
            for (int j = L.lane; j < 2 * n; j += L.n) {
                T *M = j < n ? X : inv;
                const int jj = j < n ? j : j - n;
                const T a = M[c + jj * n], b = M[piv + jj * n];
                M[c + jj * n] = b;
                M[piv + jj * n] = a;
            }
            L.sync();
        }
        const T d = T(1) / X[c + c * n];
        for (int i = L.lane; i < n; i += L.n) mult[i] = X[i + c * n];
        L.sync();
        for (int j = L.lane; j < 2 * n; j += L.n) {
            T *M = j < n ? X : inv;
            const int jj = j < n ? j : j - n;
            M[c + jj * n] = M[c + jj * n] * d;
        }
        L.sync();
        // eliminate column c from every other row: M(i, j) - m_i M(c, j) for X (columns j < n) and inv (the next n)
        ric_each(L, n, 2 * n, [&](int i, int jj, int) {
            T *M = jj < n ? X : inv;
            const int j = jj < n ? jj : jj - n;
            const T m = mult[i];
            if (i != c && m != T(0)) M[i + j * n] = M[i + j * n] - m * M[c + j * n];
        });
        L.sync();
    }
    return true;
}

// The outputs the caller picks: without the tangent the cache pieces (Kinf .. BPf, f their input), with it the tables dK
// (nu x nx) and dP (nx x nx)
template <typename T>
struct RiccatiOut {
    const T *f;
    T *Kinf, *Pinf, *Quu, *AmBKt, *APf, *BPf;
    T *dK, *dP;
};

// One model's recursion on the scratch w (riccati_scratch(nx, nu, TANGENT).total elements).  A, B, Qw, Rw as in the cache
// blob (Qw, Rw with rho added once).  Returns the sweeps used, or -1 when R1 + B'PB is singular (outputs then unwritten).
template <typename T, bool TANGENT, class Dims, class Lanes>
__host__ __device__ __forceinline__ int riccati(Dims D, Lanes L, T *w, const T *Ain, const T *Bin, const T *Qw, const T *Rw, T rho,
                                                const RiccatiOut<T> &out) {
    const int nx = D.nx, nu = D.nu, xx = nx * nx, xu = nx * nu, uu = nu * nu;
    const RiccatiScratch s = riccati_scratch(nx, nu, TANGENT);
    T *A = w + s.A, *Bm = w + s.B, *At = w + s.At, *Bt = w + s.Bt, *P = w + s.P, *Pn = w + s.Pn, *BtP = w + s.BtP, *BtPA = w + s.BtPA, *K = w + s.K, *Kp = w + s.Kp,
      *S = w + s.S, *Si = w + s.Si, *AmBK = w + s.AmBK, *AtP = w + s.AtP, *Pf = w + s.Pf, *Q1 = w + s.Q1, *R1 = w + s.R1,
      *mult = w + s.mult;
    T *dP = w + s.dP, *dPn = w + s.dPn, *dAtP = w + s.dAtP, *BdK = w + s.BdK, *dBtP = w + s.dBtP, *T1 = w + s.T1, *T2 = w + s.T2,
      *dK = w + s.dK, *dS = w + s.dS;
    ric_each(L, nx, nx, [&](int i, int j, int e) {
        A[e] = Ain[e];
        At[j + i * nx] = Ain[e];
        P[e] = i == j ? rho : T(0);  // P <- rho I
        if constexpr (TANGENT) dP[e] = i == j ? T(1) : T(0);  // dP <- I
    });
    ric_each(L, nx, nu, [&](int i, int j, int e) {
        Bm[e] = Bin[e];
        Bt[j + i * nu] = Bin[e];
        Kp[e] = T(0);
    });
    for (int e = L.lane; e < nx; e += L.n) Q1[e] = Qw[e] + rho;  // tiny_api.cpp:317
    for (int e = L.lane; e < nu; e += L.n) R1[e] = Rw[e] + rho;  // :318
    L.sync();
    auto mat = [](const T *M, int rows) { return RicView<T>{M, rows}; };
    const RicView<T> a_ = mat(A, nx), at_ = mat(At, nx), b_ = mat(Bm, nx), bt_ = mat(Bt, nu);
    // Z = diag(d) + (BtX) B: off-diagonal entries are 0 + product
    auto form_S = [&](T *Z, const T *BtX, auto d) {
        ric_mul(L, Z, nu, nu, nx, mat(BtX, nu), b_);
        ric_each(L, nu, nu, [&](int i, int j, int e) { Z[e] = (i == j ? d(i) : T(0)) + Z[e]; });
        L.sync();
    };
    auto r1_ = [&](int j) { return R1[j]; };
    int sweeps = 0;
    for (int it = 0; it < 1000; ++it) {
        ric_mul(L, BtP, nu, nx, nx, bt_, mat(P, nx));
        form_S(S, BtP, r1_);
        if (!ric_invert(L, S, Si, mult, nu)) return -1;
        ric_mul(L, BtPA, nu, nx, nx, mat(BtP, nu), a_);
        ric_mul(L, K, nu, nx, nu, mat(Si, nu), mat(BtPA, nu));
        if constexpr (TANGENT) {  // dK = S^-1 (B'dP A - dS K), dS = 2 I + B'dP B
            ric_mul(L, dBtP, nu, nx, nx, bt_, mat(dP, nx));
            ric_mul(L, T1, nu, nx, nx, mat(dBtP, nu), a_);
            form_S(dS, dBtP, [](int) { return T(2); });
            ric_mul(L, T2, nu, nx, nu, mat(dS, nu), mat(K, nu));
            for (int e = L.lane; e < xu; e += L.n) T1[e] = T1[e] - T2[e];
            L.sync();
            ric_mul(L, dK, nu, nx, nu, mat(Si, nu), mat(T1, nu));
        }
        // AmBK = A - B K ; Pn = Q1 + A'P AmBK
        ric_mul(L, AmBK, nx, nx, nu, b_, mat(K, nu));
        for (int e = L.lane; e < xx; e += L.n) AmBK[e] = A[e] - AmBK[e];
        L.sync();
        ric_mul(L, AtP, nx, nx, nx, at_, mat(P, nx));
        ric_mul(L, Pn, nx, nx, nx, mat(AtP, nx), mat(AmBK, nx));
        ric_each(L, nx, nx, [&](int i, int j, int e) { Pn[e] = (i == j ? Q1[i] : T(0)) + Pn[e]; });
        if constexpr (TANGENT) {  // dPn = (2 I + A'dP AmBK) - A'P (B dK)
            ric_mul(L, dAtP, nx, nx, nx, at_, mat(dP, nx));
            ric_mul(L, dPn, nx, nx, nx, mat(dAtP, nx), mat(AmBK, nx));
            ric_mul(L, BdK, nx, nx, nu, b_, mat(dK, nu));
            ric_mul(L, dAtP, nx, nx, nx, mat(AtP, nx), mat(BdK, nx));  // dAtP is free again: A'P (B dK)
            ric_each(L, nx, nx, [&](int i, int j, int e) { dPn[e] = (i == j ? T(2) + dPn[e] : dPn[e]) - dAtP[e]; });
        }
        L.sync();
        sweeps = it + 1;
        T md = T(0);  // a NaN never raises md
        for (int e = L.lane; e < xu; e += L.n) {
            const T d = fabs(K[e] - Kp[e]);
            md = d > md ? d : md;
        }
        if (L.max(md) < (T)1e-5) break;
        for (int e = L.lane; e < xu; e += L.n) Kp[e] = K[e];
        for (int e = L.lane; e < xx; e += L.n) {
            P[e] = Pn[e];
            if constexpr (TANGENT) dP[e] = dPn[e];
        }
        L.sync();
    }
    // Quu_inv = (R1 + B' Pinf B)^-1, which the tables' models must have too
    ric_mul(L, BtP, nu, nx, nx, bt_, mat(Pn, nx));
    form_S(S, BtP, r1_);
    if (!ric_invert(L, S, Si, mult, nu)) return -1;
    if constexpr (TANGENT) {
        for (int e = L.lane; e < xu; e += L.n) out.dK[e] = dK[e];
        for (int e = L.lane; e < xx; e += L.n) out.dP[e] = dPn[e];
    } else {  // AmBK still holds A - B Kinf from the last sweep
        ric_mul(L, Pf, nx, 1, nx, mat(Pn, nx), mat(out.f, nx));
        for (int e = L.lane; e < xu; e += L.n) out.Kinf[e] = K[e];
        ric_each(L, nx, nx, [&](int i, int j, int e) {
            out.Pinf[e] = Pn[e];
            out.AmBKt[e] = AmBK[j + i * nx];  // (A - B K)'
        });
        L.sync();
        for (int e = L.lane; e < uu; e += L.n) out.Quu[e] = Si[e];
        // APf = AmBKt Pf, BPf = B' Pf
        ric_mul(L, out.APf, nx, 1, nx, mat(out.AmBKt, nx), mat(Pf, nx));
        ric_mul(L, out.BPf, nu, 1, nx, bt_, mat(Pf, nx));
    }
    return sweeps;
}

// Instance b of a batch (launch.h: RiccatiBatch).  Without the tangent the instance's model blob gets
// A | B | f | Qw | Rw | cache | rho, with it the tables; Qw, Rw = diagonals + rho (tiny_api.cpp:117-118).
template <typename T, bool TANGENT, class Dims, class Lanes>
__host__ __device__ __forceinline__ int riccati_instance(Dims D, Lanes L, T *w, const RiccatiBatch<T> &a, int64_t b) {
    const int nx = D.nx, nu = D.nu;
    const T *Ab = a.A + b * nx * nx, *Bb = a.B + b * nx * nu, *Qd = a.Qd + b * nx, *Rd = a.Rd + b * nu;
    const T rho = a.rho[b];
    T *Qw, *Rw;
    RiccatiOut<T> out{};
    if constexpr (TANGENT) {
        const RiccatiScratch s = riccati_scratch(nx, nu, true);
        Qw = w + s.Qw, Rw = w + s.Rw;
        out.dK = a.dK + b * nx * nu, out.dP = a.dP + b * nx * nx;
    } else {
        const ModelBlobT<int64_t> mb = model_blob<int64_t>(nx, nu);
        T *o = a.models + b * mb.model;
        const T *fb = a.f + b * nx;
        for (int e = L.lane; e < nx * nx; e += L.n) o[mb.A + e] = Ab[e];
        for (int e = L.lane; e < nx * nu; e += L.n) o[mb.B + e] = Bb[e];
        for (int e = L.lane; e < nx; e += L.n) o[mb.f + e] = fb[e];
        if (L.lane == 0) o[mb.rho] = rho;
        Qw = o + mb.Qd, Rw = o + mb.Rd;
        out = {fb, o + mb.Kinf, o + mb.Pinf, o + mb.Quu, o + mb.AmBKt, o + mb.APf, o + mb.BPf, nullptr, nullptr};
    }
    for (int e = L.lane; e < nx; e += L.n) Qw[e] = Qd[e] + rho;  // tiny_api.cpp:117
    for (int e = L.lane; e < nu; e += L.n) Rw[e] = Rd[e] + rho;  // :118
    L.sync();
    return riccati<T, TANGENT>(D, L, w, Ab, Bb, Qw, Rw, rho, out);
}

// The batch on the device: one warp per instance, its scratch in shared memory; sweeps (may be null) gets each instance's
// sweep count, or -1 when it is singular
constexpr int RIC_WARPS = 4;

template <typename T, int NX, int NU, bool TANGENT>
__global__ void __launch_bounds__(RIC_WARPS * 32) riccati_kernel(int64_t Bn, RiccatiBatch<T> a, int32_t *__restrict__ sweeps) {
    extern __shared__ __align__(16) unsigned char ric_smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T *w = reinterpret_cast<T *>(ric_smem_raw) + (size_t)warp * riccati_scratch(NX, NU, TANGENT).total;
    for (int64_t b = (int64_t)blockIdx.x * RIC_WARPS + warp; b < Bn; b += (int64_t)gridDim.x * RIC_WARPS) {
        const int rc = riccati_instance<T, TANGENT>(FixDims<NX, NU>(), WarpLanes{lane}, w, a, b);
        if (lane == 0 && sweeps) sweeps[b] = rc;
        __syncwarp();
    }
}

template <typename T, int NX, int NU, bool TANGENT>
int launch_riccati(int64_t Bn, const RiccatiBatch<T> &a, int32_t *sweeps, int sm_count, cudaStream_t stream) {
    auto kern = riccati_kernel<T, NX, NU, TANGENT>;
    const size_t smem = (size_t)RIC_WARPS * riccati_scratch(NX, NU, TANGENT).total * sizeof(T);
    if (!set_dynamic_smem(kern, smem)) return TINYMPC_ERR_CUDA;
    const int64_t want = (Bn + RIC_WARPS - 1) / RIC_WARPS;
    const int ctas = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)sm_count * 8, want));
    kern<<<ctas, RIC_WARPS * 32, smem, stream>>>(Bn, a, sweeps);
    return cudaGetLastError() == cudaSuccess ? TINYMPC_OK : TINYMPC_ERR_CUDA;
}

}  // namespace tmpc
