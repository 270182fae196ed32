// launch.h — type-erased problem and launch descriptors between the C-ABI layer (capi.cu) and the per-(nx,nu)
// kernel translation units (kernels_inst.cu compiled once per supported dimension pair).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/tinympc_b200.h"

namespace tmpc {

// launch plan of the on-chip lane-group kernel (gpi_kernel.cuh: gpi_plan) for one (dtype, N); L == 0: not available
struct GpiPlan {
    int L = 0, warps = 0;              // lanes per instance, warps per CTA
    size_t smem = 0;                   // dynamic shared memory per CTA (bytes)
    int instances_per_cta = 0;         // instances resident per CTA (warps * 32 / L)
    size_t vscratch_per_instance = 0;  // bytes of work->v / work->z scratch per instance (launch.h: gpi_vscratch)
};

// The problem a handle solves, described once by tinympc_b200_create.  Arrays are in the native dtype.
struct ProblemDesc {
    int nx = 0, nu = 0, N = 0, dtype = 0;  // dtype: TINYMPC_F32 / F64
    double rho = 0;
    std::vector<char> h_blob;                      // host copy of the cache blob (model_blob.h), the bytes at `blob`
    std::vector<char> h_xlo, h_xhi, h_ulo, h_uhi;  // column 0 of the bounds; empty when the bounds were not given
    int bounds_tv = 0;         // the bounds vary along the horizon
    int bounds_zero_free = 1;  // no element of the box bounds is +-0 (lets STRICT kernels clamp with min / max instructions)
    int ncx = 0, ncu = 0, nlx = 0, nlu = 0, ntvx = 0, ntvu = 0;  // cones, hyperplanes, time-varying hyperplanes per side
    int cone_x_start[4] = {}, cone_u_start[4] = {};
    double cone_x_mu[4] = {}, cone_u_mu[4] = {};  // already rounded to the native dtype
    // device arrays: pieces of one allocation, the cache blob at offset 0 and every piece 256-byte aligned; null when not given
    const void *blob = nullptr;
    const void *x_min = nullptr, *x_max = nullptr, *u_min = nullptr, *u_max = nullptr;
    const void *Alin_x = nullptr, *blin_x = nullptr, *Alin_u = nullptr, *blin_u = nullptr;
    const void *tv_Alin_x = nullptr, *tv_blin_x = nullptr, *tv_Alin_u = nullptr, *tv_blin_u = nullptr;
};

// the constraint families a solve runs with (the problem's cones and hyperplanes under the current settings)
struct Features {
    int soc_x, soc_u, lin_x, lin_u, tvl_x, tvl_u, ext;  // ext: any of them
};

// The kinds of per-instance data a batch can bring besides models, each with arrays in place of the handle's (capi.cu: KINDS)
enum InstKind { KIND_BOUNDS, KIND_CONES, KIND_PLANES, NKINDS };

// What a solve's batch brings per instance (given) and what its kernel reads (read).  given[k] is the batch's mode field
// (bounds: 1 one column, 2 a horizon per instance).  Bounds are read whenever given; cones and hyperplanes only when a loop
// of theirs runs, else the solve is the one without them.
struct PerInstance {
    bool models = false;  // io.models: per-instance models, or the blobs adaptive rho adapts
    int given[NKINDS] = {}, read[NKINDS] = {};
    bool any() const {  // does the kernel read any per-instance data?
        for (int k = 0; k < NKINDS; ++k)
            if (read[k]) return true;
        return models;
    }
};

// Variant bits of the streamed kernel (gps_kernel.cuh), added to its constraint-family mask (0 box only, 1 cones, 6
// hyperplanes, 7 both): per-instance models, box bounds, cone coefficients and static hyperplanes
constexpr int GPS_HET = 8, GPS_BOUNDS = 16, GPS_CONES = 32, GPS_PLANES = 64;
constexpr int GPS_VARIANTS = GPS_HET | GPS_BOUNDS | GPS_CONES | GPS_PLANES;  // the family-mask bits that are not constraint families

// Which streamed kernels are compiled, for a family mask, variant bits and mode.  FAST: the shared and the per-instance-model
// solves only.  Per-instance cones with a cone family (1, 7), hyperplanes with a static hyperplane family (6, 7), never
// with bounds or cones.
__host__ __device__ constexpr bool gps_compiled(int fam, int var, bool fast) {
    if (fast && var != 0 && var != GPS_HET) return false;
    if ((var & GPS_CONES) && fam != 1 && fam != 7) return false;
    if ((var & GPS_PLANES) && (fam < 6 || (var & (GPS_BOUNDS | GPS_CONES)))) return false;
    return true;
}
// instances per lane group of a compiled variant: the shared solve's (ni) unless per-instance models or bounds hold a lane
// group's registers
__host__ __device__ constexpr int gps_variant_ni(int var, int ni) { return (var & (GPS_HET | GPS_BOUNDS)) ? 1 : ni; }
// the variant bits of per-instance data (kinds: PerInstance::given or read)
inline int gps_variant(bool models, const int (&kinds)[NKINDS]) {
    return (models ? GPS_HET : 0) | (kinds[KIND_BOUNDS] ? GPS_BOUNDS : 0) | (kinds[KIND_CONES] ? GPS_CONES : 0) |
           (kinds[KIND_PLANES] ? GPS_PLANES : 0);
}

// Variant bits of the on-chip kernel (gpi_kernel.cuh), added to its lane count L (its lane parameter LA; L = LA % GPI_ADAPT):
// a separate template parameter or kernel argument would rename the existing kernels, a shared __device__ body or a larger
// KParams changes their machine code.  GPI_ADAPT: adaptive rho (tinympc_b200_solve_adaptive), GpiAdapt arguments (adapt.h);
// GPI_ADAPT_TABLES on top: its per-instance sensitivity tables, a variant of its own because a run-time choice between staged
// and per-instance tables cost the shared-table kernel 2-3 % (DESIGN.md §5.5).  GPI_ROLLOUT: closed-loop rollouts
// (tinympc_b200_rollout), GpiRoll arguments (rollout.h).  GPI_BOUNDS: per-instance box bounds (bounds_per_instance), P.x_min ...
// u_max at the batch's columns or horizons (P.bounds_tv), each slot's column 0 loaded at its refill.  GPI_PLANT on top of
// GPI_ROLLOUT: a rollout against a plant of each instance's own and / or with measurement noise (GpiRoll's plant fields).
constexpr int GPI_ADAPT = 64, GPI_ADAPT_TABLES = 128, GPI_ROLLOUT = 256, GPI_BOUNDS = 512, GPI_PLANT = 1024;

// Which on-chip kernels are compiled, for a lane count, variant bits, per-instance models (het), the min / max clamp (mm),
// mode and dtype.  FAST: the plain solves only.  MM: fp32 with a shared model, plain or rollout (with or without a plant).
// Adaptive rho (with or without its tables): per-instance models only.  Rollouts and bounds: never with each other or with
// adaptive rho.  A plant: rollouts only.  L = 16: fp64 only.
__host__ __device__ constexpr bool gpi_compiled(int L, int bits, bool het, bool mm, bool fast, bool fp64) {
    if (L != 4 && L != 8 && !(L == 16 && fp64)) return false;
    if (bits & ~(GPI_ADAPT | GPI_ADAPT_TABLES | GPI_ROLLOUT | GPI_BOUNDS | GPI_PLANT)) return false;
    if (fast && (bits != 0 || mm)) return false;
    if (mm && (fp64 || het || (bits != 0 && (bits & ~GPI_PLANT) != GPI_ROLLOUT))) return false;
    if ((bits & GPI_PLANT) && !(bits & GPI_ROLLOUT)) return false;
    if ((bits & GPI_ADAPT) && !het) return false;
    if ((bits & GPI_ADAPT_TABLES) && !(bits & GPI_ADAPT)) return false;
    return !!(bits & GPI_ADAPT) + !!(bits & GPI_ROLLOUT) + !!(bits & GPI_BOUNDS) <= 1;
}

// the walks over kernel variants: f(std::integral_constant<int, i>()) for every case i, which f decodes and checks against
// gps_compiled or gpi_compiled with if constexpr, so that only compiled variants are instantiated
template <typename F, int... I>
inline void walk_cases(F &&f, std::integer_sequence<int, I...>) {
    (f(std::integral_constant<int, I>()), ...);
}

struct LaunchDesc {
    const ProblemDesc *pd;
    tinympc_settings_t st;
    Features ft;
    int fast;    // TINYMPC_MODE_FAST ?
    int family;  // TINYMPC_KERNEL_TPI / GPI / GPS (resolved, never AUTO)

    tinympc_batch_t io;  // device pointers
    int64_t Bpad;
    void *tpi_ws;      // TPI: the workspace (kparams_fill.h: tpi_workspace)
    void *work_queue;  // GPI: device int64 counter (zeroed by the caller)
    GpiPlan gpi;       // GPI: the launch plan (for adaptive rho the adaptive kernel's, its tables' shared memory included)
    void *gpi_vscratch;  // GPI: scratch for work->v / work->z persistence (allocated by the caller when state.v/z given)
    void *gps_ws;        // GPS: streamed state records of the resident slots (allocated by the caller, see out_ws_need)
    size_t gps_ws_bytes;

    // adaptive rho (tinympc_b200_solve_adaptive): io.models is then the in/out blob array; adapt_args = device copy of
    // GpiAdapt<T> (adapt.h) followed by dKinf_drho and dPinf_drho
    int adapt;  // 0: no; 1: one shared table pair; 2: per-instance tables
    const void *adapt_args;
    // closed-loop rollout (tinympc_b200_rollout): io.Xref / io.Uref are then the reference trajectories, roll_args = device copy
    // of GpiRoll<T> (rollout.h); 1: against the controller's model, 2: against plants of their own or with measurement noise
    int rollout;
    const void *roll_args;
    // per-instance data: the lane-group kernels' GPI_BOUNDS and GPS_HET / BOUNDS / CONES / PLANES variants read io's arrays
    PerInstance pi;

    cudaStream_t stream;
    int sm_count;
    int max_smem_optin;

    // filled by the launcher
    int out_threads, out_ctas, out_smem, out_lanes_per_instance, out_instances_per_cta;
    size_t out_ws_need;  // GPS: workspace bytes this launch needs (set when the launcher returns TM_ERR_WORKSPACE)
};

// The on-chip kernel a launch wants (launch_gpi runs it when gpi_compiled admits it): variant bits, per-instance models and
// the min / max clamp, which fp32 STRICT solves with a shared model use when no bound of the problem is a signed zero (the
// host cannot scan per-instance bounds, so they rule it out)
struct GpiVariant { int bits; bool het, mm; };
inline GpiVariant gpi_variant(const LaunchDesc &d) {
    const bool bounds = d.pi.read[KIND_BOUNDS] != 0;
    const int bits = (d.adapt ? GPI_ADAPT : 0) | (d.adapt == 2 ? GPI_ADAPT_TABLES : 0) | (d.rollout ? GPI_ROLLOUT : 0) |
                     (d.rollout == 2 ? GPI_PLANT : 0) | (bounds ? GPI_BOUNDS : 0);
    return {bits, d.pi.models, !d.fast && d.pd->dtype == TINYMPC_F32 && !d.pi.models && !bounds && d.pd->bounds_zero_free};
}

// launch epilogue of every kernel family: record the launch geometry in the descriptor, return the launch status
inline int launch_done(LaunchDesc *d, int threads, int ctas, size_t smem, int lanes, int instances_per_cta) {
    d->out_threads = threads;
    d->out_ctas = ctas;
    d->out_smem = (int)smem;
    d->out_lanes_per_instance = lanes;
    d->out_instances_per_cta = instances_per_cta;
    return cudaGetLastError() == cudaSuccess ? TINYMPC_OK : TINYMPC_ERR_CUDA;
}
template <typename K>
inline bool set_dynamic_smem(K kern, size_t smem) {
    return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) == cudaSuccess;
}

// internal: the launcher needs a larger gps_ws (size in out_ws_need); never leaves the library
constexpr int TM_ERR_WORKSPACE = -100;

// A batch of the Riccati precompute (riccati.cuh), host or device pointers, instance after instance and column-major:
// A [B][nx*nx], B [B][nx*nu], f [B][nx], the user's diagonals Qd [B][nx] and Rd [B][nu], rho [B].  Without the tangent the
// results are one model blob per instance (models, model_blob.h), with it the tables dK [B][nu*nx] and dP [B][nx*nx].
template <typename T>
struct RiccatiBatch {
    const T *A, *B, *f, *Qd, *Rd, *rho;
    T *models, *dK, *dP;
    template <typename U>
    RiccatiBatch<U> as() const {
        return {(const U *)A, (const U *)B, (const U *)f, (const U *)Qd, (const U *)Rd, (const U *)rho, (U *)models, (U *)dK, (U *)dP};
    }
};

// per-(nx,nu) entry: returns 0 on success, TINYMPC_ERR_UNSUPPORTED when (dtype,family,...) is not compiled
typedef int (*launch_fn)(LaunchDesc *);

struct DimEntry {
    int nx, nu;
    launch_fn launch;
    // GPI capability query: the on-chip kernel's launch plan for (dtype, N)
    GpiPlan (*gpi_plan)(int dtype, int N, int max_smem_optin);
    // batched Riccati precompute on the device (riccati.cuh: riccati_kernel), the cache or with the tangent the tables
    int (*riccati_batch)(int dtype, bool tangent, int64_t B, const RiccatiBatch<void> &a, int32_t *sweeps_out, int sm_count,
                         cudaStream_t stream);
    // streamed lane-group kernel (gps_kernel.cuh): lanes per instance; 0 = shape not available
    int (*gps_lanes)(int dtype);
    // its per-instance-model variant (io.models): instances per CTA when the batch fills every SM, for the shape and the
    // constraint families (cones, hyperplanes), with or without per-instance cone coefficients; 0 = not available
    int (*gps_het_slots)(int dtype, bool soc, bool lin, bool cones, int max_smem_optin);
};

}  // namespace tmpc

// the list of compiled dimension pairs: X(nx, nu)
#define TM_DIMS(X) \
    X(4, 1)        \
    X(6, 3)        \
    X(12, 4)       \
    X(4, 2)        \
    X(4, 4)        \
    X(4, 8)        \
    X(8, 2)        \
    X(8, 4)        \
    X(8, 8)        \
    X(12, 2)       \
    X(12, 8)       \
    X(16, 2)       \
    X(16, 4)       \
    X(16, 8)
