// precompute_kernel.cuh — batched cache precompute ON THE DEVICE for heterogeneous batches (SURVEY §8f-2).
//
// One warp per instance computes what tiny_setup + tiny_precompute_and_set_cache compute for one model
// (TinyMPC src/tinympc/tiny_api.cpp:117-118, 307-381):
//   Qw = Qdiag + rho, Rw = Rdiag + rho                     (:117-118)
//   Q1 = diag(Qw) + rho I, R1 = diag(Rw) + rho I           (:317-318, the "double rho")
//   P <- rho I, K_prev <- 0                                (:330-333)
//   repeat <= 1000:  K = (R1 + B'PB)^-1 B'PA ;  Pn = Q1 + A'P(A - BK) ; stop if max|K - K_prev| < 1e-5   (:335-349)
//   Quu_inv = (R1 + B'Pinf B)^-1 ; AmBKt = (A - B Kinf)' ; APf = AmBKt Pinf f ; BPf = B' Pinf f          (:352-357)
// and writes the instance's model blob  A | B | f | Qw | Rw | Kinf | Pinf | Quu_inv | AmBKt | APf | BPf | rho
// (tinympc_batch_t.models) straight into device memory.
//
// Arithmetic contract: every output element is produced by exactly the operation sequence of the host routine
// (host_precompute.h: products accumulated from 0 in ascending inner index with separate multiply and add,
// Gauss-Jordan inverse with partial pivoting, IEEE division), so the blobs are BIT-IDENTICAL to
// tinympc_b200_precompute_cache_batch's (tests/test_gpu_parity.py).  The 32 lanes split the output elements of
// each product; the matrices live in shared memory (≈ 6 nx² + 6 nx·nu + 3 nu² elements per warp).
#pragma once
#include "common.cuh"
#include "model_blob.h"

namespace tmpc {

constexpr int PC_WARPS = 4;

template <int NX, int NU>
struct PcLayout {
    static constexpr int XX = NX * NX, XU = NX * NU, UU = NU * NU;
    // offsets (elements) inside one warp's scratch
    static constexpr int A = 0, B = A + XX, P = B + XU, PN = P + XX, BTP = PN + XX, BTPA = BTP + XU, K = BTPA + XU, KP = K + XU,
                         S = KP + XU, SI = S + UU, AMBK = SI + UU, ATP = AMBK + XX, F = ATP + XX, PF = F + NX, Q1 = PF + NX, R1 = Q1 + NX,
                         TOTAL = R1 + NU;
};

// Z(i,j) = sum_l x(i,l) * y(l,j), l ascending, accumulated from 0 (host_precompute.h: mul); Z is R x C column-major
template <typename T, int R, int C, int KK, class FX, class FY>
__device__ __forceinline__ void pc_mul(T *Z, FX x, FY y, int lane) {
    for (int e = lane; e < R * C; e += 32) {
        const int i = e % R, j = e / R;
        T acc = T(0);
#pragma unroll 4
        for (int l = 0; l < KK; ++l) acc = acc + x(i, l) * y(l, j);
        Z[e] = acc;
    }
    __syncwarp();
}

// Gauss-Jordan with partial pivoting on the n x n matrix X (destroyed) -> inv; same element operations as
// host_precompute.h: invert.  Returns false when a pivot is exactly zero.
template <typename T, int n>
__device__ __forceinline__ bool pc_invert(T *X, T *inv, int lane) {
    for (int e = lane; e < n * n; e += 32) inv[e] = (e % n == e / n) ? T(1) : T(0);
    __syncwarp();
    for (int c = 0; c < n; ++c) {
        int piv = c;
        for (int i = c + 1; i < n; ++i)
            if (fabs(X[i + c * n]) > fabs(X[piv + c * n])) piv = i;
        if (X[piv + c * n] == T(0)) return false;
        __syncwarp();
        if (piv != c) {
            for (int j = lane; j < 2 * n; j += 32) {
                T *M = j < n ? X : inv;
                const int jj = j < n ? j : j - n;
                const T a = M[c + jj * n], b = M[piv + jj * n];
                M[c + jj * n] = b;
                M[piv + jj * n] = a;
            }
            __syncwarp();
        }
        const T d = T(1) / X[c + c * n];
        __syncwarp();
        for (int j = lane; j < 2 * n; j += 32) {
            T *M = j < n ? X : inv;
            const int jj = j < n ? j : j - n;
            M[c + jj * n] = M[c + jj * n] * d;
        }
        __syncwarp();
        // eliminate column c from every other row: element (i, j) of X and of inv, all independent once the
        // multipliers m_i = X(i,c) and the scaled pivot row are fixed
        T upd[(2 * n * n + 31) / 32];
        int cnt = 0;
        for (int e = lane; e < 2 * n * n; e += 32, ++cnt) {
            const int half = e / (n * n), r = e - half * n * n;
            const int i = r % n, j = r / n;
            T *M = half ? inv : X;
            const T m = X[i + c * n];
            T v = M[i + j * n];
            if (i != c && m != T(0)) v = v - m * M[c + j * n];
            upd[cnt] = v;
        }
        __syncwarp();
        cnt = 0;
        for (int e = lane; e < 2 * n * n; e += 32, ++cnt) {
            const int half = e / (n * n), r = e - half * n * n;
            (half ? inv : X)[r] = upd[cnt];
        }
        __syncwarp();
    }
    return true;
}

template <typename T, int NX, int NU>
__global__ void __launch_bounds__(PC_WARPS * 32)
    precompute_cache_kernel(int64_t Bn, const T *__restrict__ Ag, const T *__restrict__ Bg, const T *__restrict__ fg,
                            const T *__restrict__ Qg, const T *__restrict__ Rg, const T *__restrict__ rhog, T *__restrict__ out,
                            int32_t *__restrict__ sweeps_out) {
    using Lo = PcLayout<NX, NU>;
    extern __shared__ __align__(16) unsigned char pc_smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T *w = reinterpret_cast<T *>(pc_smem_raw) + (size_t)warp * Lo::TOTAL;
    T *A = w + Lo::A, *Bm = w + Lo::B, *P = w + Lo::P, *Pn = w + Lo::PN, *BtP = w + Lo::BTP, *BtPA = w + Lo::BTPA, *K = w + Lo::K,
      *Kp = w + Lo::KP, *S = w + Lo::S, *Si = w + Lo::SI, *AmBK = w + Lo::AMBK, *AtP = w + Lo::ATP, *f = w + Lo::F, *Pf = w + Lo::PF,
      *Q1 = w + Lo::Q1, *R1 = w + Lo::R1;
    constexpr ModelBlob MB = model_blob(NX, NU);

    for (int64_t b = (int64_t)blockIdx.x * PC_WARPS + warp; b < Bn; b += (int64_t)gridDim.x * PC_WARPS) {
        T *o = out + b * (int64_t)MB.model;
        T *oA = o + MB.A, *oB = o + MB.B, *oF = o + MB.f, *oQ = o + MB.Qd, *oR = o + MB.Rd, *oK = o + MB.Kinf, *oP = o + MB.Pinf,
          *oQuu = o + MB.Quu, *oAm = o + MB.AmBKt, *oAPf = o + MB.APf, *oBPf = o + MB.BPf;
        const T rho = rhog[b];
        for (int e = lane; e < Lo::XX; e += 32) {
            const T a = Ag[b * Lo::XX + e];
            A[e] = a;
            oA[e] = a;
            P[e] = (e % NX == e / NX) ? rho : T(0);  // P <- rho I
            Pn[e] = T(0);
        }
        for (int e = lane; e < Lo::XU; e += 32) {
            const T v = Bg[b * Lo::XU + e];
            Bm[e] = v;
            oB[e] = v;
            Kp[e] = T(0);
            K[e] = T(0);
        }
        for (int e = lane; e < NX; e += 32) {
            const T fv = fg[b * NX + e], qw = Qg[b * NX + e] + rho;  // tiny_api.cpp:117
            f[e] = fv;
            oF[e] = fv;
            oQ[e] = qw;
            Q1[e] = qw + rho;  // :317
        }
        for (int e = lane; e < NU; e += 32) {
            const T rw = Rg[b * NU + e] + rho;  // :118
            oR[e] = rw;
            R1[e] = rw + rho;  // :318
        }
        __syncwarp();
        auto a_ = [&](int i, int j) { return A[i + j * NX]; };
        auto at_ = [&](int i, int j) { return A[j + i * NX]; };
        auto b_ = [&](int i, int j) { return Bm[i + j * NX]; };
        auto bt_ = [&](int i, int j) { return Bm[j + i * NX]; };
        auto mat = [](const T *M, int rows) { return [M, rows](int i, int j) { return M[i + j * rows]; }; };
        // S = R1 + (BtX) B   (R1 diagonal: off-diagonal entries are 0 + product, as in add(R1, mul(..)))
        auto form_S = [&](const T *BtX) {
            pc_mul<T, NU, NU, NX>(S, mat(BtX, NU), b_, lane);
            for (int e = lane; e < Lo::UU; e += 32) S[e] = ((e % NU == e / NU) ? R1[e % NU] : T(0)) + S[e];
            __syncwarp();
        };
        // AmBK = A - B K
        auto form_AmBK = [&]() {
            pc_mul<T, NX, NX, NU>(AmBK, b_, mat(K, NU), lane);
            for (int e = lane; e < Lo::XX; e += 32) AmBK[e] = A[e] - AmBK[e];
            __syncwarp();
        };
        int sweeps = 0;
        bool ok = true;
        for (int it = 0; it < 1000; ++it) {
            pc_mul<T, NU, NX, NX>(BtP, bt_, mat(P, NX), lane);
            form_S(BtP);
            if (!pc_invert<T, NU>(S, Si, lane)) {
                ok = false;
                break;
            }
            pc_mul<T, NU, NX, NX>(BtPA, mat(BtP, NU), a_, lane);
            pc_mul<T, NU, NX, NU>(K, mat(Si, NU), mat(BtPA, NU), lane);
            form_AmBK();
            pc_mul<T, NX, NX, NX>(AtP, at_, mat(P, NX), lane);
            pc_mul<T, NX, NX, NX>(Pn, mat(AtP, NX), mat(AmBK, NX), lane);
            for (int e = lane; e < Lo::XX; e += 32) Pn[e] = ((e % NX == e / NX) ? Q1[e % NX] : T(0)) + Pn[e];
            __syncwarp();
            sweeps = it + 1;
            T md = T(0);
            for (int e = lane; e < Lo::XU; e += 32) md = fmax(md, fabs(K[e] - Kp[e]));
#pragma unroll
            for (int m = 16; m >= 1; m >>= 1) md = fmax(md, __shfl_xor_sync(0xffffffffu, md, m));
            if (md < (T)1e-5) break;
            for (int e = lane; e < Lo::XU; e += 32) Kp[e] = K[e];
            for (int e = lane; e < Lo::XX; e += 32) P[e] = Pn[e];
            __syncwarp();
        }
        if (ok) {
            pc_mul<T, NU, NX, NX>(BtP, bt_, mat(Pn, NX), lane);  // B' Pinf
            form_S(BtP);
            ok = pc_invert<T, NU>(S, Si, lane);
        }
        if (ok) {
            form_AmBK();
            pc_mul<T, NX, 1, NX>(Pf, mat(Pn, NX), mat(f, NX), lane);
            for (int e = lane; e < Lo::XU; e += 32) oK[e] = K[e];
            for (int e = lane; e < Lo::XX; e += 32) {
                oP[e] = Pn[e];
                oAm[e] = AmBK[(e / NX) + (e % NX) * NX];  // (A - B K)'
            }
            for (int e = lane; e < Lo::UU; e += 32) oQuu[e] = Si[e];
            // APf = AmBKt Pf, BPf = B' Pf
            for (int i = lane; i < NX; i += 32) {
                T acc = T(0);
                for (int l = 0; l < NX; ++l) acc = acc + AmBK[l + i * NX] * Pf[l];
                oAPf[i] = acc;
            }
            for (int j = lane; j < NU; j += 32) {
                T acc = T(0);
                for (int l = 0; l < NX; ++l) acc = acc + Bm[l + j * NX] * Pf[l];
                oBPf[j] = acc;
            }
        }
        if (lane == 0) {
            o[MB.rho] = rho;
            if (sweeps_out) sweeps_out[b] = ok ? sweeps : -1;
        }
        __syncwarp();
    }
}

template <typename T, int NX, int NU>
int launch_precompute_T(int64_t Bn, const void *A, const void *Bm, const void *f, const void *Q, const void *R, const void *rho, void *out,
                        int32_t *sweeps, int sm_count, cudaStream_t stream) {
    using Lo = PcLayout<NX, NU>;
    auto kern = precompute_cache_kernel<T, NX, NU>;
    const size_t smem = (size_t)PC_WARPS * Lo::TOTAL * sizeof(T);
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return TINYMPC_ERR_CUDA;
    const int64_t want = (Bn + PC_WARPS - 1) / PC_WARPS;
    const int ctas = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)sm_count * 8, want));
    kern<<<ctas, PC_WARPS * 32, smem, stream>>>(Bn, (const T *)A, (const T *)Bm, (const T *)f, (const T *)Q, (const T *)R, (const T *)rho,
                                                (T *)out, sweeps);
    return cudaGetLastError() == cudaSuccess ? TINYMPC_OK : TINYMPC_ERR_CUDA;
}

// ---- sensitivity tables dKinf/drho, dPinf/drho (host_precompute.h: precompute_sensitivity) ----
// The same primal recursion with its tangent carried alongside, one warp per instance, every element by the host routine's
// operation sequence: the tables are BIT-IDENTICAL to tinympc_b200_precompute_sensitivity_batch's.  A singular S is found by
// the same pc_invert calls as in precompute_cache_kernel, so sweeps_out is -1 for exactly the same models.
template <int NX, int NU>
struct PsLayout : PcLayout<NX, NU> {
    using Pc = PcLayout<NX, NU>;
    // the tangent's scratch behind the primal's
    static constexpr int DP = Pc::TOTAL, DPN = DP + Pc::XX, DATP = DPN + Pc::XX, BDK = DATP + Pc::XX, DBTP = BDK + Pc::XX, T1 = DBTP + Pc::XU,
                         T2 = T1 + Pc::XU, DK = T2 + Pc::XU, DS = DK + Pc::XU, TOTAL = DS + Pc::UU;
};

template <typename T, int NX, int NU>
__global__ void __launch_bounds__(PC_WARPS * 32)
    precompute_sensitivity_kernel(int64_t Bn, const T *__restrict__ Ag, const T *__restrict__ Bg, const T *__restrict__ Qg,
                                  const T *__restrict__ Rg, const T *__restrict__ rhog, T *__restrict__ dK_out, T *__restrict__ dP_out,
                                  int32_t *__restrict__ sweeps_out) {
    using Lo = PsLayout<NX, NU>;
    extern __shared__ __align__(16) unsigned char pc_smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T *w = reinterpret_cast<T *>(pc_smem_raw) + (size_t)warp * Lo::TOTAL;
    T *A = w + Lo::A, *Bm = w + Lo::B, *P = w + Lo::P, *Pn = w + Lo::PN, *BtP = w + Lo::BTP, *BtPA = w + Lo::BTPA, *K = w + Lo::K,
      *Kp = w + Lo::KP, *S = w + Lo::S, *Si = w + Lo::SI, *AmBK = w + Lo::AMBK, *AtP = w + Lo::ATP, *Q1 = w + Lo::Q1, *R1 = w + Lo::R1;
    T *dP = w + Lo::DP, *dPn = w + Lo::DPN, *dAtP = w + Lo::DATP, *BdK = w + Lo::BDK, *dBtP = w + Lo::DBTP, *T1 = w + Lo::T1,
      *T2 = w + Lo::T2, *dK = w + Lo::DK, *dS = w + Lo::DS;

    for (int64_t b = (int64_t)blockIdx.x * PC_WARPS + warp; b < Bn; b += (int64_t)gridDim.x * PC_WARPS) {
        const T rho = rhog[b];
        for (int e = lane; e < Lo::XX; e += 32) {
            const bool diag = e % NX == e / NX;
            A[e] = Ag[b * Lo::XX + e];
            P[e] = diag ? rho : T(0);    // P <- rho I
            dP[e] = diag ? T(1) : T(0);  // dP <- I
        }
        for (int e = lane; e < Lo::XU; e += 32) {
            Bm[e] = Bg[b * Lo::XU + e];
            Kp[e] = T(0);
        }
        for (int e = lane; e < NX; e += 32) Q1[e] = (Qg[b * NX + e] + rho) + rho;  // tiny_api.cpp:117, :317
        for (int e = lane; e < NU; e += 32) R1[e] = (Rg[b * NU + e] + rho) + rho;  // :118, :318
        __syncwarp();
        auto a_ = [&](int i, int j) { return A[i + j * NX]; };
        auto at_ = [&](int i, int j) { return A[j + i * NX]; };
        auto b_ = [&](int i, int j) { return Bm[i + j * NX]; };
        auto bt_ = [&](int i, int j) { return Bm[j + i * NX]; };
        auto mat = [](const T *M, int rows) { return [M, rows](int i, int j) { return M[i + j * rows]; }; };
        // Z = diag(d) + (BtX) B, as add(diagonal matrix, mul(..)): off-diagonal entries are 0 + product
        auto form_S = [&](T *Z, const T *BtX, auto d) {
            pc_mul<T, NU, NU, NX>(Z, mat(BtX, NU), b_, lane);
            for (int e = lane; e < Lo::UU; e += 32) Z[e] = ((e % NU == e / NU) ? d(e % NU) : T(0)) + Z[e];
            __syncwarp();
        };
        auto r1_ = [&](int j) { return R1[j]; };
        int sweeps = 0;
        bool ok = true;
        for (int it = 0; it < 1000; ++it) {
            pc_mul<T, NU, NX, NX>(BtP, bt_, mat(P, NX), lane);
            pc_mul<T, NU, NX, NX>(dBtP, bt_, mat(dP, NX), lane);
            form_S(S, BtP, r1_);
            if (!pc_invert<T, NU>(S, Si, lane)) {
                ok = false;
                break;
            }
            pc_mul<T, NU, NX, NX>(BtPA, mat(BtP, NU), a_, lane);
            pc_mul<T, NU, NX, NU>(K, mat(Si, NU), mat(BtPA, NU), lane);
            // dK = S^-1 (B'dP A - dS K), dS = 2 I + B'dP B
            pc_mul<T, NU, NX, NX>(T1, mat(dBtP, NU), a_, lane);
            form_S(dS, dBtP, [](int) { return T(2); });
            pc_mul<T, NU, NX, NU>(T2, mat(dS, NU), mat(K, NU), lane);
            for (int e = lane; e < Lo::XU; e += 32) T1[e] = T1[e] - T2[e];
            __syncwarp();
            pc_mul<T, NU, NX, NU>(dK, mat(Si, NU), mat(T1, NU), lane);
            // AmBK = A - B K ; Pn = Q1 + A'P AmBK
            pc_mul<T, NX, NX, NU>(AmBK, b_, mat(K, NU), lane);
            for (int e = lane; e < Lo::XX; e += 32) AmBK[e] = A[e] - AmBK[e];
            __syncwarp();
            pc_mul<T, NX, NX, NX>(AtP, at_, mat(P, NX), lane);
            pc_mul<T, NX, NX, NX>(Pn, mat(AtP, NX), mat(AmBK, NX), lane);
            for (int e = lane; e < Lo::XX; e += 32) Pn[e] = ((e % NX == e / NX) ? Q1[e % NX] : T(0)) + Pn[e];
            // dPn = (2 I + A'dP AmBK) - A'P (B dK)
            pc_mul<T, NX, NX, NX>(dAtP, at_, mat(dP, NX), lane);
            pc_mul<T, NX, NX, NX>(dPn, mat(dAtP, NX), mat(AmBK, NX), lane);
            pc_mul<T, NX, NX, NU>(BdK, b_, mat(dK, NU), lane);
            pc_mul<T, NX, NX, NX>(dAtP, mat(AtP, NX), mat(BdK, NX), lane);  // dAtP is free again: A'P (B dK)
            for (int e = lane; e < Lo::XX; e += 32) {
                const T v = (e % NX == e / NX) ? T(2) + dPn[e] : dPn[e];
                dPn[e] = v - dAtP[e];
            }
            __syncwarp();
            sweeps = it + 1;
            T md = T(0);
            for (int e = lane; e < Lo::XU; e += 32) md = fmax(md, fabs(K[e] - Kp[e]));
#pragma unroll
            for (int m = 16; m >= 1; m >>= 1) md = fmax(md, __shfl_xor_sync(0xffffffffu, md, m));
            if (md < (T)1e-5) break;
            for (int e = lane; e < Lo::XU; e += 32) Kp[e] = K[e];
            for (int e = lane; e < Lo::XX; e += 32) {
                P[e] = Pn[e];
                dP[e] = dPn[e];
            }
            __syncwarp();
        }
        if (ok) {  // the cache's Quu_inv = (R1 + B' Pinf B)^-1 must exist too
            pc_mul<T, NU, NX, NX>(BtP, bt_, mat(Pn, NX), lane);
            form_S(S, BtP, r1_);
            ok = pc_invert<T, NU>(S, Si, lane);
        }
        if (ok) {
            for (int e = lane; e < Lo::XU; e += 32) dK_out[b * Lo::XU + e] = dK[e];
            for (int e = lane; e < Lo::XX; e += 32) dP_out[b * Lo::XX + e] = dPn[e];
        }
        if (lane == 0 && sweeps_out) sweeps_out[b] = ok ? sweeps : -1;
        __syncwarp();
    }
}

template <typename T, int NX, int NU>
int launch_sensitivity_T(int64_t Bn, const void *A, const void *Bm, const void *Q, const void *R, const void *rho, void *dK, void *dP,
                         int32_t *sweeps, int sm_count, cudaStream_t stream) {
    using Lo = PsLayout<NX, NU>;
    auto kern = precompute_sensitivity_kernel<T, NX, NU>;
    const size_t smem = (size_t)PC_WARPS * Lo::TOTAL * sizeof(T);
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return TINYMPC_ERR_CUDA;
    const int64_t want = (Bn + PC_WARPS - 1) / PC_WARPS;
    const int ctas = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)sm_count * 8, want));
    kern<<<ctas, PC_WARPS * 32, smem, stream>>>(Bn, (const T *)A, (const T *)Bm, (const T *)Q, (const T *)R, (const T *)rho, (T *)dK,
                                                (T *)dP, sweeps);
    return cudaGetLastError() == cudaSuccess ? TINYMPC_OK : TINYMPC_ERR_CUDA;
}

}  // namespace tmpc
