// lanegroup.cuh — what the on-chip (gpi_kernel.cuh) and the streamed (gps_kernel.cuh) lane-group kernels share.
// Lane mapping: L lanes form a group that owns one instance (GPS: NI instances); lane l of the group owns the state rows
// [l*RX, (l+1)*RX) and the input rows [l*RU, (l+1)*RU) of every vector (RX = ceil(nx/L), RU = ceil(nu/L)).  A row past
// nx / nu is a padding row: it computes zeros.
#pragma once
#include "common.cuh"
#include "launch.h"
#include "model_blob.h"

namespace tmpc {

template <int NX, int NU, int L, int ES>
struct LaneGeom {
    static constexpr int RX = (NX + L - 1) / L;  // state rows per lane
    static constexpr int RU = (NU + L - 1) / L;  // input rows per lane
    static constexpr int IPW = 32 / L;           // lane groups per warp
    static constexpr int W = 16 / ES;            // elements per 16-byte shared-memory vector
    static constexpr int NXP = (L * RX + W - 1) / W * W;  // gather buffer width (state vectors)
    static constexpr int NUP = (L * RU + W - 1) / W * W;  // gather buffer width (input vectors)
};

template <bool B> struct BoolTag { static constexpr bool value = B; };
template <int J> struct IntTag { static constexpr int value = J; };

// ---- shared-memory accessors on 32-bit shared-window addresses (no generic->shared conversion, no 64-bit address
// arithmetic in the hot loops).  16-byte vector forms move a whole 16-byte piece per instruction ----
__device__ __forceinline__ float lds(unsigned a, float) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ double lds(unsigned a, double) {
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ void sts(unsigned a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
__device__ __forceinline__ void sts(unsigned a, double v) { asm volatile("st.shared.f64 [%0], %1;" ::"r"(a), "d"(v) : "memory"); }
__device__ __forceinline__ void ldsv(unsigned a, float (&v)[4]) {
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]) : "r"(a));
}
__device__ __forceinline__ void ldsv(unsigned a, double (&v)[2]) {
    asm volatile("ld.shared.v2.f64 {%0,%1}, [%2];" : "=d"(v[0]), "=d"(v[1]) : "r"(a));
}
__device__ __forceinline__ void stsv(unsigned a, const float (&v)[4]) {
    asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(a), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory");
}
__device__ __forceinline__ void stsv(unsigned a, const double (&v)[2]) {
    asm volatile("st.shared.v2.f64 [%0], {%1,%2};" ::"r"(a), "d"(v[0]), "d"(v[1]) : "memory");
}

// chunked piece moves between registers and shared memory: a piece of R elements in chunks of CB bytes
__device__ __forceinline__ void lds_chunk(unsigned a, float (&v)[1]) { v[0] = lds(a, 0.f); }
__device__ __forceinline__ void lds_chunk(unsigned a, float (&v)[2]) {
    asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(v[0]), "=f"(v[1]) : "r"(a));
}
__device__ __forceinline__ void lds_chunk(unsigned a, float (&v)[4]) { ldsv(a, v); }
__device__ __forceinline__ void lds_chunk(unsigned a, double (&v)[1]) { v[0] = lds(a, 0.0); }
__device__ __forceinline__ void lds_chunk(unsigned a, double (&v)[2]) { ldsv(a, v); }
__device__ __forceinline__ void sts_chunk(unsigned a, const float (&v)[1]) { sts(a, v[0]); }
__device__ __forceinline__ void sts_chunk(unsigned a, const float (&v)[2]) {
    asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(a), "f"(v[0]), "f"(v[1]) : "memory");
}
__device__ __forceinline__ void sts_chunk(unsigned a, const float (&v)[4]) { stsv(a, v); }
__device__ __forceinline__ void sts_chunk(unsigned a, const double (&v)[1]) { sts(a, v[0]); }
__device__ __forceinline__ void sts_chunk(unsigned a, const double (&v)[2]) { stsv(a, v); }

template <typename T, int R, int CB>
__device__ __forceinline__ void lds_piece(unsigned a, T (&v)[R]) {
    constexpr int E = CB / (int)sizeof(T);
#pragma unroll
    for (int c = 0; c < R / E; ++c) {
        T t[E];
        lds_chunk(a + (unsigned)(c * CB), t);
#pragma unroll
        for (int e = 0; e < E; ++e) v[c * E + e] = t[e];
    }
}
template <typename T, int R, int CB>
__device__ __forceinline__ void sts_piece(unsigned a, const T (&v)[R]) {
    constexpr int E = CB / (int)sizeof(T);
#pragma unroll
    for (int c = 0; c < R / E; ++c) {
        T t[E];
#pragma unroll
        for (int e = 0; e < E; ++e) t[e] = v[c * E + e];
        sts_chunk(a + (unsigned)(c * CB), t);
    }
}

// ---- mbarrier + bulk copy (cp.async.bulk, TMA) primitives; `mb` is the shared-window address of a 64-bit mbarrier ----
__device__ __forceinline__ void mbar_init(unsigned mb) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mb)); }
// makes the initialisations above visible to the async proxy
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// one bulk copy of `bytes` (a multiple of 16) from global `src` to shared `dst`; completion is counted on barrier mb
__device__ __forceinline__ void bulk_g2s(unsigned dst, const void *src, unsigned bytes, unsigned mb) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mb), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
                 "r"(bytes), "r"(mb)
                 : "memory");
}
// spin until the phase with parity `par` of barrier mb has completed
__device__ __forceinline__ void mbar_wait(unsigned mb, unsigned par) {
    unsigned done = 0;
    while (!done) {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
                     : "=r"(done)
                     : "r"(mb), "r"(par)
                     : "memory");
    }
}
// orders this thread's generic-proxy global stores before its later async-proxy operations (bulk copies reading them back)
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// CTA prologue: thread 0 copies the cache blob (`bytes`, see cache_stage_bytes) from global memory to `stage` in shared
// memory with one bulk copy on barrier `mbar`; every thread returns once it has landed
__device__ __forceinline__ void stage_blob(void *stage, const void *gmat, unsigned bytes, unsigned long long *mbar) {
    if (threadIdx.x == 0) {
        const unsigned mb = (unsigned)__cvta_generic_to_shared(mbar);
        mbar_init(mb);
        mbar_init_fence();
        bulk_g2s((unsigned)__cvta_generic_to_shared(stage), gmat, bytes, mb);
    }
    __syncthreads();
    mbar_wait((unsigned)__cvta_generic_to_shared(mbar), 0u);
}

// ---- lane rows of the cache matrices.  rd(e) reads element e of a blob in the model_blob.h layout (GPI: a generic
// pointer to the staged or the instance's own blob; GPS: the staged copy through a shared-window address).  `ok` = false
// (a padding row) gives zeros; the caller passes a clamped row index for it, so that every read stays inside the blob.
// Row i of the column-major matrix with leading dimension LD at blob offset off: o[m] = M(i, m)
template <int LD, int NC, typename T, typename RD>
__device__ __forceinline__ void blob_row(RD rd, int off, int i, bool ok, T (&o)[NC]) {
#pragma unroll
    for (int m = 0; m < NC; ++m) o[m] = ok ? rd(off + i + LD * m) : T(0);
}
// column i of it (row i of the transpose): o[m] = M(m, i)
template <int LD, int NR, typename T, typename RD>
__device__ __forceinline__ void blob_col(RD rd, int off, int i, bool ok, T (&o)[NR]) {
#pragma unroll
    for (int m = 0; m < NR; ++m) o[m] = ok ? rd(off + m + LD * i) : T(0);
}

// the iteration-invariant part of the terminal cost, -(Pinf^T xref_{N-1}), of state row i: m ascending, xr(m) = xref_{N-1}(m)
template <bool FAST, int NX, typename T, typename XR>
__device__ __forceinline__ T terminal_cost(XR xr, const T *pinf, int i) {
    T sacc = xr(0) * __ldg(pinf + NX * i);
    for (int m = 1; m < NX; ++m) sacc = mac<FAST>(sacc, xr(m), __ldg(pinf + m + NX * i));
    return -sacc;
}

// ---- box bounds of this lane's rows.  enx / enu: the state / input bounds are enabled; xv(a) / uv(b): row a / b of the
// lane is a real row.  A disabled bound or a padding row is (-inf, +inf): the clamp is then the identity on every non-NaN
// value, so it can stay unconditional in the hot loop.  INIT: column 0; else column k of time-varying bounds, the input side
// only when the column has inputs (HASU), a disabled bound keeping its value ----
template <bool INIT, typename T, int NX, int NU, int RX, int RU, typename XV, typename UV>
__device__ __forceinline__ void box_bounds(const KParams<T, NX, NU> &P, int l, int k, const bool HASU, const bool enx, const bool enu,
                                           XV xv, UV uv, T (&loX)[RX], T (&hiX)[RX], T (&loU)[RU], T (&hiU)[RU]) {
    const T kInf = (T)INFINITY;
    if constexpr (INIT) {
#pragma unroll
        for (int a = 0; a < RX; ++a) {
            loX[a] = (enx && xv(a)) ? __ldg(P.x_min + l * RX + a) : -kInf;
            hiX[a] = (enx && xv(a)) ? __ldg(P.x_max + l * RX + a) : kInf;
        }
#pragma unroll
        for (int b = 0; b < RU; ++b) {
            loU[b] = (enu && uv(b)) ? __ldg(P.u_min + l * RU + b) : -kInf;
            hiU[b] = (enu && uv(b)) ? __ldg(P.u_max + l * RU + b) : kInf;
        }
    } else {
#pragma unroll
        for (int a = 0; a < RX; ++a) {
            loX[a] = (enx && xv(a)) ? __ldg(P.x_min + (int64_t)k * NX + l * RX + a) : loX[a];
            hiX[a] = (enx && xv(a)) ? __ldg(P.x_max + (int64_t)k * NX + l * RX + a) : hiX[a];
        }
        if (HASU) {
#pragma unroll
            for (int b = 0; b < RU; ++b) {
                loU[b] = (enu && uv(b)) ? __ldg(P.u_min + (int64_t)k * NU + l * RU + b) : loU[b];
                hiU[b] = (enu && uv(b)) ? __ldg(P.u_max + (int64_t)k * NU + l * RU + b) : hiU[b];
            }
        }
    }
}
// the same for per-instance bounds (tinympc_batch_t.bounds_per_instance): column k of the instance whose columns start at
// element ox of the state bounds and ou of the input bounds (k = 0 for INIT)
template <bool INIT, typename T, int NX, int NU, int RX, int RU, typename XV, typename UV>
__device__ __forceinline__ void box_bounds_at(const KParams<T, NX, NU> &P, int64_t ox, int64_t ou, int l, int k, const bool HASU,
                                              const bool enx, const bool enu, XV xv, UV uv, T (&loX)[RX], T (&hiX)[RX], T (&loU)[RU],
                                              T (&hiU)[RU]) {
    const T kInf = (T)INFINITY;
    const int64_t bx = ox + (int64_t)k * NX + l * RX, bu = ou + (int64_t)k * NU + l * RU;
#pragma unroll
    for (int a = 0; a < RX; ++a) {
        loX[a] = (enx && xv(a)) ? __ldg(P.x_min + bx + a) : (INIT ? -kInf : loX[a]);
        hiX[a] = (enx && xv(a)) ? __ldg(P.x_max + bx + a) : (INIT ? kInf : hiX[a]);
    }
    if (INIT || HASU) {
#pragma unroll
        for (int b = 0; b < RU; ++b) {
            loU[b] = (enu && uv(b)) ? __ldg(P.u_min + bu + b) : (INIT ? -kInf : loU[b]);
            hiU[b] = (enu && uv(b)) ? __ldg(P.u_max + bu + b) : (INIT ? kInf : hiU[b]);
        }
    }
}

template <typename T, int L>
__device__ __forceinline__ T group_max(T v) {
#pragma unroll
    for (int m = L / 2; m >= 1; m >>= 1) {
        T o = __shfl_xor_sync(0xffffffffu, v, m, L);
        v = (o > v) ? o : v;
    }
    return v;
}

// Box clamp.  STRICT keeps Eigen's compare-select form (differs from fmax/fmin only in the sign of a zero
// result when a bound is a signed zero); FAST uses the single-instruction min/max.
template <bool FAST, typename T>
__device__ __forceinline__ T clamp_box(T v, T lo, T hi) {
    if constexpr (FAST) {
        return fmin(fmax(v, lo), hi);
    } else {
        return clamp_ref(v, lo, hi);
    }
}
// max(m, |d|): identical to the oracle's (|d| > m) ? |d| : m  because m is never NaN and |d| >= +0
__device__ __forceinline__ float absmax(float m, float d) { return fmaxf(m, fabsf(d)); }
// fp64: the oracle's compare-select itself.  fmax(double) has no single instruction: DSETP.MAX + SEL + FSEL + a NaN-quieting
// LOP3 + register moves, 7 instructions per use and 9 % of the streamed fp64 kernel's instruction count (ncu source view).
__device__ __forceinline__ double absmax(double m, double d) {
    const double a = fabs(d);
    return (a > m) ? a : m;
}

// own rows of a vector every lane of the group holds in full: out[a] = full[l*R + a] without dynamic register indexing
template <typename T, int NE, int R, int L>
__device__ __forceinline__ void extract_own(const T (&full)[NE], int l, T (&out)[R]) {
#pragma unroll
    for (int a = 0; a < R; ++a) {
        T v = T(0);
#pragma unroll
        for (int g = 0; g < L; ++g)
            if (g * R + a < NE) v = (l == g) ? full[g * R + a] : v;
        out[a] = v;
    }
}

}  // namespace tmpc
