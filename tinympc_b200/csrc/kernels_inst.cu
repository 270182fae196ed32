// kernels_inst.cu — compiled three times per supported (nx, nu) with -DTM_NX=.. -DTM_NU=.. -DTM_PART=0|1|2 (see Makefile):
//   part 0: thread-per-instance kernels (tpi_kernel.cuh), device precompute, and the type-erased DimEntry
//   part 1: on-chip lane-group kernels (gpi_kernel.cuh)
//   part 2: streamed lane-group kernels (gps_kernel.cuh)
// Three objects per dimension pair keep `make -j` busy and an edit of one kernel family from recompiling the others.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <limits>

#include "kparams_fill.h"
#include "launch.h"

#if !defined(TM_NX) || !defined(TM_NU) || !defined(TM_PART)
#error "compile with -DTM_NX=<nx> -DTM_NU=<nu> -DTM_PART=<0|1|2>"
#endif

#define TM_CAT3(a, b, c) a##b##_##c
#define TM_CAT(a, b, c) TM_CAT3(a, b, c)
#define TM_SYM(prefix) TM_CAT(prefix, TM_NX, TM_NU)

// cross-part entry points of this dimension pair
extern "C" int TM_SYM(tm_gpi_launch_)(tmpc::LaunchDesc *d);
extern "C" tmpc::GpiPlan TM_SYM(tm_gpi_plan_)(int dtype, int N, int max_smem_optin);
extern "C" int TM_SYM(tm_gps_launch_)(tmpc::LaunchDesc *d);
extern "C" int TM_SYM(tm_gps_lanes_)(int dtype);
extern "C" int TM_SYM(tm_gps_het_slots_)(const tmpc::LaunchDesc *d);

#if TM_PART == 0
// =========================================================================================================
#include "precompute_kernel.cuh"
#include "tpi_kernel.cuh"

namespace tmpc {
namespace {

template <typename T, bool FAST, bool EXT>
int launch_tpi(LaunchDesc *d) {
    KParams<T, TM_NX, TM_NU> P;
    fill_params<T, TM_NX, TM_NU>(P, *d);
    const int threads = TPI_THREADS;
    const int64_t blocks = (d->io.B + threads - 1) / threads;
    if (blocks <= 0) return TINYMPC_OK;
    tpi_solve_kernel<T, TM_NX, TM_NU, FAST, EXT><<<(unsigned)blocks, threads, 0, d->stream>>>(P);
    return launch_done(d, threads, (int)blocks, 0, 1, threads);
}

template <typename T>
int launch_T(LaunchDesc *d) {
    if (d->io.models) return TINYMPC_ERR_UNSUPPORTED;  // per-instance models: the lane-group kernels only
    if (d->ext) return d->fast ? launch_tpi<T, true, true>(d) : launch_tpi<T, false, true>(d);
    return d->fast ? launch_tpi<T, true, false>(d) : launch_tpi<T, false, false>(d);
}

int launch(LaunchDesc *d) {
    if (d->family == TINYMPC_KERNEL_GPI) return TM_SYM(tm_gpi_launch_)(d);
    if (d->family == TINYMPC_KERNEL_GPS) return TM_SYM(tm_gps_launch_)(d);
    if (d->dtype == TINYMPC_F32) return launch_T<float>(d);
    if (d->dtype == TINYMPC_F64) return launch_T<double>(d);
    return TINYMPC_ERR_ARG;
}

int precompute_batch(int dtype, int64_t B, const void *A, const void *Bm, const void *f, const void *Qdiag, const void *Rdiag,
                     const void *rho, void *models_out, int32_t *sweeps_out, int sm_count, cudaStream_t stream) {
    if (dtype == TINYMPC_F32)
        return launch_precompute_T<float, TM_NX, TM_NU>(B, A, Bm, f, Qdiag, Rdiag, rho, models_out, sweeps_out, sm_count, stream);
    if (dtype == TINYMPC_F64)
        return launch_precompute_T<double, TM_NX, TM_NU>(B, A, Bm, f, Qdiag, Rdiag, rho, models_out, sweeps_out, sm_count, stream);
    return TINYMPC_ERR_ARG;
}

}  // namespace
}  // namespace tmpc

extern "C" const tmpc::DimEntry *TM_SYM(tm_dim_entry_)() {
    static const tmpc::DimEntry e = {TM_NX,
                                     TM_NU,
                                     &tmpc::launch,
                                     &TM_SYM(tm_gpi_plan_),
                                     &tmpc::precompute_batch,
                                     &TM_SYM(tm_gps_lanes_),
                                     &TM_SYM(tm_gps_het_slots_)};
    return &e;
}

#elif TM_PART == 1
// =========================================================================================================
#include "gpi_kernel.cuh"

namespace tmpc {
namespace {

template <typename T, int NX, int NU, bool FAST>
int launch_gpi(LaunchDesc *d) {
    const GpiPlan plan = gpi_plan<T, NX, NU>(d->N, d->max_smem_optin - 64);
    if (plan.L == 0 || !d->gmat || !d->work_queue) return TINYMPC_ERR_UNSUPPORTED;
    KParams<T, NX, NU> P;
    fill_params<T, NX, NU>(P, *d);
    const T *gmat = (const T *)d->gmat;
    const bool het = d->io.models != nullptr;  // heterogeneous batch: per-instance model blobs
    // STRICT fp32, shared model (the headline path): min / max clamp when no bound is a signed zero
#define TM_GPI_CASE(LL, HH)                                                                                              \
    if (plan.L == LL && het == HH) {                                                                                     \
        if constexpr (!FAST && !HH && sizeof(T) == 4) {                                                                  \
            if (d->bounds_zero_free) return launch_gpi_L<T, NX, NU, LL, FAST, HH, true>(d, plan, P, gmat);               \
        }                                                                                                                \
        return launch_gpi_L<T, NX, NU, LL, FAST, HH>(d, plan, P, gmat);                                                  \
    }
#define TM_GPI_L(LL) TM_GPI_CASE(LL, false) TM_GPI_CASE(LL, true)
    TM_GPI_L(4)
    TM_GPI_L(8)
#ifdef TM_GPI_L16
    TM_GPI_L(16)
#else
    if constexpr (sizeof(T) == 8) {  // fp64 may need L = 16 for the widest states (see gpi_plan)
        TM_GPI_L(16)
    }
#endif
#undef TM_GPI_L
#undef TM_GPI_CASE
    return TINYMPC_ERR_UNSUPPORTED;
}

// adaptive rho: heterogeneous STRICT batches; the tables take gpi_adapt_bytes of shared memory per CTA
template <typename T, int NX, int NU>
int launch_gpi_adapt(LaunchDesc *d) {
    const int extra = (int)gpi_adapt_bytes(NX, NU, sizeof(T));
    GpiPlan plan = gpi_plan<T, NX, NU>(d->N, d->max_smem_optin - 64 - extra);
    if (plan.L == 0 || d->fast || !d->gmat || !d->work_queue || !d->io.models) return TINYMPC_ERR_UNSUPPORTED;
    plan.smem += extra;
    KParams<T, NX, NU> P;
    fill_params<T, NX, NU>(P, *d);
    if (!d->adapt_args) return TINYMPC_ERR_UNSUPPORTED;
    set_gpi_adapt_args<T>(P, d->adapt_args);  // GpiAdapt<T> + tables, uploaded by the caller (capi.cu: upload_adaptive)
    const T *gmat = (const T *)d->gmat;
    if (plan.L == 4) return launch_gpi_adapt_L<T, NX, NU, 4>(d, plan, P, gmat);
    if (plan.L == 8) return launch_gpi_adapt_L<T, NX, NU, 8>(d, plan, P, gmat);
#ifndef TM_GPI_L16
    if constexpr (sizeof(T) == 8)
#endif
        if (plan.L == 16) return launch_gpi_adapt_L<T, NX, NU, 16>(d, plan, P, gmat);
    return TINYMPC_ERR_UNSUPPORTED;
}

template <typename T>
int launch_T(LaunchDesc *d) {
    if (d->ext) return TINYMPC_ERR_UNSUPPORTED;  // the on-chip kernel covers box constraints; the rest streams (gps)
    if (d->adapt) return launch_gpi_adapt<T, TM_NX, TM_NU>(d);
    return d->fast ? launch_gpi<T, TM_NX, TM_NU, true>(d) : launch_gpi<T, TM_NX, TM_NU, false>(d);
}

}  // namespace
}  // namespace tmpc

extern "C" int TM_SYM(tm_gpi_launch_)(tmpc::LaunchDesc *d) {
    if (d->dtype == TINYMPC_F32) return tmpc::launch_T<float>(d);
    if (d->dtype == TINYMPC_F64) return tmpc::launch_T<double>(d);
    return TINYMPC_ERR_ARG;
}
extern "C" tmpc::GpiPlan TM_SYM(tm_gpi_plan_)(int dtype, int N, int max_smem_optin) {
    if (dtype == TINYMPC_F32) return tmpc::gpi_plan<float, TM_NX, TM_NU>(N, max_smem_optin - 64);
    if (dtype == TINYMPC_F64) return tmpc::gpi_plan<double, TM_NX, TM_NU>(N, max_smem_optin - 64);
    return tmpc::GpiPlan{};
}

#else
// =========================================================================================================
#include "gps_kernel.cuh"

namespace tmpc {
namespace {

// io.models set: the per-instance-model variant (launch_gps)
template <typename T>
int launch_T(LaunchDesc *d) {
    KParams<T, TM_NX, TM_NU> P;
    fill_params<T, TM_NX, TM_NU>(P, *d);
    return d->fast ? launch_gps<T, TM_NX, TM_NU, true>(d, P) : launch_gps<T, TM_NX, TM_NU, false>(d, P);
}

}  // namespace
}  // namespace tmpc

extern "C" int TM_SYM(tm_gps_launch_)(tmpc::LaunchDesc *d) {
    if (d->dtype == TINYMPC_F32) return tmpc::launch_T<float>(d);
    if (d->dtype == TINYMPC_F64) return tmpc::launch_T<double>(d);
    return TINYMPC_ERR_ARG;
}
// lanes per instance of the streamed lane-group kernel for this shape (0 = not available)
extern "C" int TM_SYM(tm_gps_lanes_)(int dtype) {
    // lanes per instance in bits 0-7, instances per lane group (1 or 2) in bits 8-15
    auto lanes = [](auto t) {
        using T = decltype(t);
        constexpr int L = tmpc::gps_pick_L<T, TM_NX, TM_NU>();
        if constexpr (L == 0) return 0;
        else return L | (tmpc::gps_pick_NI<T, TM_NX, TM_NU, L>() << 8);
    };
    return dtype == TINYMPC_F32 ? lanes(0.f) : (dtype == TINYMPC_F64 ? lanes(0.0) : 0);
}
extern "C" int TM_SYM(tm_gps_het_slots_)(const tmpc::LaunchDesc *d) {
    if (d->dtype == TINYMPC_F32) return tmpc::gps_het_slots<float, TM_NX, TM_NU>(*d);
    if (d->dtype == TINYMPC_F64) return tmpc::gps_het_slots<double, TM_NX, TM_NU>(*d);
    return 0;
}
#endif
