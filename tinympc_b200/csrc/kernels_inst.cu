// kernels_inst.cu — compiled four times per supported (nx, nu) with -DTM_NX=.. -DTM_NU=.. -DTM_PART=0|1|2|3 (see Makefile):
//   part 0: thread-per-instance kernels (tpi_kernel.cuh), device precompute, and the type-erased DimEntry
//   part 1: on-chip lane-group kernels (gpi_kernel.cuh), all but the GPI_PLANT variants
//   part 2: streamed lane-group kernels (gps_kernel.cuh)
//   part 3: the on-chip GPI_PLANT variants (rollouts against plants of their own), reached through part 1's launcher
// Four objects per dimension pair keep `make -j` busy and an edit of one kernel family from recompiling the others; the
// plant variants have an object of their own so that the on-chip objects, the longest compiles, take no longer than without them.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <limits>

#include "kparams_fill.h"
#include "launch.h"

#if !defined(TM_NX) || !defined(TM_NU) || !defined(TM_PART)
#error "compile with -DTM_NX=<nx> -DTM_NU=<nu> -DTM_PART=<0|1|2|3>"
#endif

#define TM_CAT3(a, b, c) a##b##_##c
#define TM_CAT(a, b, c) TM_CAT3(a, b, c)
#define TM_SYM(prefix) TM_CAT(prefix, TM_NX, TM_NU)

// cross-part entry points of this dimension pair
extern "C" int TM_SYM(tm_gpi_launch_)(tmpc::LaunchDesc *d);
extern "C" int TM_SYM(tm_gpi_plant_launch_)(tmpc::LaunchDesc *d);
extern "C" tmpc::GpiPlan TM_SYM(tm_gpi_plan_)(int dtype, int N, int max_smem_optin);
extern "C" int TM_SYM(tm_gps_launch_)(tmpc::LaunchDesc *d);
extern "C" int TM_SYM(tm_gps_lanes_)(int dtype);
extern "C" int TM_SYM(tm_gps_het_slots_)(int dtype, bool soc, bool lin, bool cones, int max_smem_optin);

#if TM_PART == 0
// =========================================================================================================
#include "riccati.cuh"
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
    if (d->pi.any()) return TINYMPC_ERR_UNSUPPORTED;  // per-instance data: the lane-group kernels only
    if (d->ft.ext) return d->fast ? launch_tpi<T, true, true>(d) : launch_tpi<T, false, true>(d);
    return d->fast ? launch_tpi<T, true, false>(d) : launch_tpi<T, false, false>(d);
}

int launch(LaunchDesc *d) {
    if (d->family == TINYMPC_KERNEL_GPI) return TM_SYM(tm_gpi_launch_)(d);
    if (d->family == TINYMPC_KERNEL_GPS) return TM_SYM(tm_gps_launch_)(d);
    if (d->pd->dtype == TINYMPC_F32) return launch_T<float>(d);
    if (d->pd->dtype == TINYMPC_F64) return launch_T<double>(d);
    return TINYMPC_ERR_ARG;
}

int riccati_batch(int dtype, bool tangent, int64_t B, const RiccatiBatch<void> &a, int32_t *sweeps_out, int sm_count,
                  cudaStream_t stream) {
    auto go = [&](auto t) {
        using T = decltype(t);
        return tangent ? launch_riccati<T, TM_NX, TM_NU, true>(B, a.as<T>(), sweeps_out, sm_count, stream)
                       : launch_riccati<T, TM_NX, TM_NU, false>(B, a.as<T>(), sweeps_out, sm_count, stream);
    };
    if (dtype == TINYMPC_F32) return go(0.f);
    if (dtype == TINYMPC_F64) return go(0.0);
    return TINYMPC_ERR_ARG;
}

}  // namespace
}  // namespace tmpc

extern "C" const tmpc::DimEntry *TM_SYM(tm_dim_entry_)() {
    static const tmpc::DimEntry e = {TM_NX,
                                     TM_NU,
                                     &tmpc::launch,
                                     &TM_SYM(tm_gpi_plan_),
                                     &tmpc::riccati_batch,
                                     &TM_SYM(tm_gps_lanes_),
                                     &TM_SYM(tm_gps_het_slots_)};
    return &e;
}

#elif TM_PART == 1 || TM_PART == 3
// =========================================================================================================
#include "gpi_kernel.cuh"

namespace tmpc {
namespace {

// the on-chip kernel of the solve's variant (launch.h: gpi_variant, gpi_compiled) with the plan d->gpi, which comes from the
// caller (capi.cu: plan_solve, through the DimEntry's gpi_plan); a variant that is not compiled is TINYMPC_ERR_UNSUPPORTED.
// Part 1 instantiates the variants without GPI_PLANT, part 3 those with it.
template <typename T, int NX, int NU, bool FAST>
int launch_gpi(LaunchDesc *d) {
    if (d->gpi.L == 0 || !d->work_queue || (d->adapt && !d->adapt_args) || (d->rollout && !d->roll_args)) return TINYMPC_ERR_UNSUPPORTED;
    KParams<T, NX, NU> P;
    fill_params<T, NX, NU>(P, *d);
    if (d->adapt) set_gpi_adapt_args<T>(P, d->adapt_args);  // GpiAdapt<T> + tables, uploaded by the caller (capi.cu: upload_adaptive)
    if (d->rollout) set_gpi_roll_args<T>(P, d->roll_args);  // GpiRoll<T>, uploaded by the caller (capi.cu: upload_rollout)
    const GpiVariant v = gpi_variant(*d);
    int rc = TINYMPC_ERR_UNSUPPORTED;
    walk_cases([&](auto i) {  // case i: L = 4, 8, 16; variant bits; het; mm
        constexpr int I = decltype(i)::value, LL = 4 << (I / 128), BB = I / 4 % 32 * GPI_ADAPT;
        constexpr bool HH = I / 2 % 2, MM = I % 2;
        if constexpr (gpi_compiled(LL, BB, HH, MM, FAST, sizeof(T) == 8) && ((BB & GPI_PLANT) != 0) == (TM_PART == 3))
            if (d->gpi.L == LL && v.bits == BB && v.het == HH && v.mm == MM)
                rc = launch_gpi_L<T, NX, NU, LL + BB, FAST, HH, MM>(d, P, (const T *)d->pd->blob);
    }, std::make_integer_sequence<int, 3 * 128>());
    return rc;
}

template <typename T>
int launch_T(LaunchDesc *d) {
    if (d->ft.ext) return TINYMPC_ERR_UNSUPPORTED;  // the on-chip kernel covers box constraints; the rest streams (gps)
    return d->fast ? launch_gpi<T, TM_NX, TM_NU, true>(d) : launch_gpi<T, TM_NX, TM_NU, false>(d);
}

}  // namespace
}  // namespace tmpc

#if TM_PART == 1
extern "C" int TM_SYM(tm_gpi_launch_)(tmpc::LaunchDesc *d) {
    if (tmpc::gpi_variant(*d).bits & tmpc::GPI_PLANT) return TM_SYM(tm_gpi_plant_launch_)(d);
    if (d->pd->dtype == TINYMPC_F32) return tmpc::launch_T<float>(d);
    if (d->pd->dtype == TINYMPC_F64) return tmpc::launch_T<double>(d);
    return TINYMPC_ERR_ARG;
}
// the on-chip kernel's launch plan; 64 bytes of the opt-in shared memory stay back for the kernel's static shared memory (its mbarrier)
extern "C" tmpc::GpiPlan TM_SYM(tm_gpi_plan_)(int dtype, int N, int max_smem_optin) {
    auto plan = [&](auto t) { return tmpc::gpi_plan<decltype(t), TM_NX, TM_NU>(N, max_smem_optin - 64); };
    return dtype == TINYMPC_F32 ? plan(0.f) : (dtype == TINYMPC_F64 ? plan(0.0) : tmpc::GpiPlan{});
}
#else
extern "C" int TM_SYM(tm_gpi_plant_launch_)(tmpc::LaunchDesc *d) {
    if (d->pd->dtype == TINYMPC_F32) return tmpc::launch_T<float>(d);
    if (d->pd->dtype == TINYMPC_F64) return tmpc::launch_T<double>(d);
    return TINYMPC_ERR_ARG;
}
#endif

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
    if (d->pd->dtype == TINYMPC_F32) return tmpc::launch_T<float>(d);
    if (d->pd->dtype == TINYMPC_F64) return tmpc::launch_T<double>(d);
    return TINYMPC_ERR_ARG;
}
// lanes per instance of the streamed lane-group kernel for this shape (0 = not available)
extern "C" int TM_SYM(tm_gps_lanes_)(int dtype) {
    if (dtype == TINYMPC_F32) return tmpc::gps_pick_L<float, TM_NX, TM_NU>();
    if (dtype == TINYMPC_F64) return tmpc::gps_pick_L<double, TM_NX, TM_NU>();
    return 0;
}
extern "C" int TM_SYM(tm_gps_het_slots_)(int dtype, bool soc, bool lin, bool cones, int max_smem_optin) {
    const int fam = tmpc::gps_family_mask(soc, lin);
    if (dtype == TINYMPC_F32) return tmpc::gps_het_slots<float, TM_NX, TM_NU>(fam, cones && soc, max_smem_optin);
    if (dtype == TINYMPC_F64) return tmpc::gps_het_slots<double, TM_NX, TM_NU>(fam, cones && soc, max_smem_optin);
    return 0;
}
#endif
