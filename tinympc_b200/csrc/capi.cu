// capi.cu — implementation of the C ABI declared in include/tinympc_b200.h.
//
// Host glue only: handle management, problem upload, workspace sizing, kernel-family selection,
// launch + CUDA-event timing, and the host-pointer convenience path (pinned staging, chunked so that
// H2D copies, the solve kernel and D2H copies of consecutive chunks overlap on three streams).
// No CPU fallback exists: every solve goes through a CUDA kernel of this library or returns an error.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "adapt.h"
#include "kparams_fill.h"
#include "model_blob.h"
#include "riccati.cuh"
#include "rollout.h"

#define TM_DECL(nx, nu) extern "C" const tmpc::DimEntry *tm_dim_entry_##nx##_##nu();
TM_DIMS(TM_DECL)
#undef TM_DECL

namespace {

// x0[b] <- (A x0[b] + B u[b][:,0]) + f ; one thread per (instance, row); matrices column-major in the blob of instance b,
// blob + b * bstride (bstride 0: one blob for every instance)
template <typename T>
__global__ void advance_kernel(int nx, int nu, int64_t ustride, int64_t B, const T *__restrict__ blob, int64_t bstride, T *x0,
                               const T *__restrict__ u) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = t < B * nx;
    T r = T(0);
    if (valid) {
        const int64_t b = t / nx;
        const int i = (int)(t - b * nx);
        const tmpc::ModelBlob mb = tmpc::model_blob(nx, nu);
        const T *mdl = blob + b * bstride;
        const T *A = mdl + mb.A, *Bm = mdl + mb.B, *f = mdl + mb.f;
        const T *xb = x0 + b * nx, *ub = u + b * ustride;
        T ax = A[i] * xb[0];
        for (int m = 1; m < nx; ++m) ax = ax + A[i + nx * m] * xb[m];
        T bu = Bm[i] * ub[0];
        for (int j = 1; j < nu; ++j) bu = bu + Bm[i + nx * j] * ub[j];
        r = (ax + bu) + f[i];
    }
    __syncthreads();  // blockDim is a multiple of nx: all rows of an instance have read x0 before any row writes it
    if (valid) x0[t] = r;
}

thread_local std::string g_err;
int fail(int code, const std::string &msg) {
    g_err = msg;
    return code;
}
#define CUDA_TRY(expr)                                                                             \
    do {                                                                                           \
        cudaError_t e_ = (expr);                                                                   \
        if (e_ != cudaSuccess)                                                                     \
            return fail(TINYMPC_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));     \
    } while (0)

const tmpc::DimEntry *find_dim(int nx, int nu) {
#define TM_FIND(a, b) \
    if (nx == a && nu == b) return tm_dim_entry_##a##_##b();
    TM_DIMS(TM_FIND)
#undef TM_FIND
    return nullptr;
}

size_t esize(int dtype) { return dtype == TINYMPC_F64 ? 8 : 4; }

// a growable buffer of device memory or of page-locked host memory, released with the handle
template <bool PINNED>
struct Buf {
    void *p = nullptr;
    size_t bytes = 0;
    Buf() = default;
    Buf(const Buf &) = delete;
    Buf &operator=(const Buf &) = delete;
    ~Buf() { release(); }
    int ensure(size_t n) {
        if (n <= bytes) return 0;
        release();
        if ((PINNED ? cudaMallocHost(&p, n) : cudaMalloc(&p, n)) != cudaSuccess) {
            p = nullptr;
            return -1;
        }
        bytes = n;
        return 0;
    }
    void release() {
        if (p) PINNED ? cudaFreeHost(p) : cudaFree(p);
        p = nullptr;
        bytes = 0;
    }
};
using DevBuf = Buf<false>;
using PinBuf = Buf<true>;

}  // namespace

struct tinympc_b200_solver {
    int device = 0;
    int sm_count = 0;
    int max_smem_optin = 0;
    int l2_bytes = 0;
    const tmpc::DimEntry *dim = nullptr;
    tmpc::ProblemDesc pd;
    DevBuf problem;  // the device arrays of pd
    tinympc_settings_t settings;
    int mode = TINYMPC_MODE_STRICT;
    int family = TINYMPC_KERNEL_AUTO;
    // workspace (one solve at a time per handle: enqueue() serialises launches issued on different streams)
    DevBuf ws;
    DevBuf queue;
    DevBuf vscratch;
    DevBuf xtrue;  // rollout with measurement noise: the true plant states [B][nx] (GpiRoll::xtrue)
    DevBuf gps_ws;
    DevBuf shared_ref;  // host path: references shared by the whole batch
    DevBuf d_args;      // adaptive rho: GpiAdapt arguments + the shared dKinf_drho + dPinf_drho (adapt.h); rollout: GpiRoll (rollout.h)
    // page-locked staging of d_args's contents, a ring so that the copy stays asynchronous: slot i is rewritten only once
    // the copy three solves back (ev_args[i]) has read it
    PinBuf args_pin[3];
    cudaEvent_t ev_args[3] = {};
    bool args_used[3] = {false, false, false};
    int args_next = 0;
    cudaEvent_t ev_last = nullptr;  // recorded after the last enqueue
    cudaStream_t last_stream = nullptr;
    bool have_last = false;
    // host-path staging (per pipeline slot)
    static constexpr int SLOTS = 3;
    DevBuf dio[SLOTS];
    PinBuf pin_in[SLOTS], pin_out[SLOTS];
    cudaStream_t st_h2d = nullptr, st_k = nullptr, st_d2h = nullptr;
    cudaEvent_t ev_in[SLOTS] = {}, ev_k[SLOTS] = {}, ev_out[SLOTS] = {};
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool timed = false;
    tinympc_b200_stats_t stats;
};

namespace {

tmpc::Features features(const tinympc_b200_solver *s) {
    tmpc::Features f;
    const tinympc_settings_t &st = s->settings;
    f.soc_x = st.en_state_soc && s->pd.ncx > 0;
    f.soc_u = st.en_input_soc && s->pd.ncu > 0;
    f.lin_x = st.en_state_linear != 0;
    f.lin_u = st.en_input_linear != 0;
    f.tvl_x = st.en_tv_state_linear != 0;
    f.tvl_u = st.en_tv_input_linear != 0;
    f.ext = f.soc_x || f.soc_u || f.lin_x || f.lin_u || f.tvl_x || f.tvl_u;
    return f;
}

// The per-instance kinds of a batch besides models (tmpc::InstKind order): the mode field and its reserved neighbour, the
// arrays with their side and elements per instance, when a side's loop runs and reads them, and the words of the errors.
// check_solve, plan_solve, enqueue and the host path all work from this table.
using BatchArray = const void *tinympc_batch_t::*;
using BatchInt = int32_t tinympc_batch_t::*;
struct KindArray {
    BatchArray member;
    int side;                                              // 0: state, 1: input
    size_t (*elems)(const tmpc::ProblemDesc &, int mode);  // elements per instance
};
struct KindDesc {
    BatchInt mode, reserved;
    int max_mode;
    KindArray arrays[4];
    bool (*runs)(const tinympc_b200_solver *s, int side);  // the side's loop runs and reads its arrays
    bool gps_only;      // served by the streamed kernel only; read only while a loop runs (else routed by the flag)
    const char *mode_msg;
    const char *pairs_msg;  // a side's arrays come together, whether its loop runs or not; null: no such rule
    int missing_code;   // a side whose loop runs lacks an array
    const char *missing_msg;
    const char *handles, *noun, *field, *exclusive;  // "the handle's <handles>", "per-instance <noun>", the mode field, kinds it does not combine with
};

const KindDesc KINDS[tmpc::NKINDS] = {
    {&tinympc_batch_t::bounds_per_instance, &tinympc_batch_t::reserved2, 2,
     {{&tinympc_batch_t::x_min, 0, [](const tmpc::ProblemDesc &pd, int m) { return (size_t)pd.nx * (m == 2 ? pd.N : 1); }},
      {&tinympc_batch_t::x_max, 0, [](const tmpc::ProblemDesc &pd, int m) { return (size_t)pd.nx * (m == 2 ? pd.N : 1); }},
      {&tinympc_batch_t::u_min, 1, [](const tmpc::ProblemDesc &pd, int m) { return (size_t)pd.nu * (m == 2 ? pd.N - 1 : 1); }},
      {&tinympc_batch_t::u_max, 1, [](const tmpc::ProblemDesc &pd, int m) { return (size_t)pd.nu * (m == 2 ? pd.N - 1 : 1); }}},
     [](const tinympc_b200_solver *s, int side) { return (side ? s->settings.en_input_bound : s->settings.en_state_bound) != 0; },
     false,
     "bounds_per_instance must be 0 (the handle's bounds), 1 (one column per instance) or 2 (a horizon per instance), and "
     "reserved2 must be 0",
     "per-instance bounds: x_min / x_max and u_min / u_max are given in pairs",
     TINYMPC_ERR_NO_BOUNDS,
     "per-instance bounds: en_state_bound/en_input_bound set but the batch has no x_min/x_max or u_min/u_max",
     "bounds", "bounds", "bounds_per_instance", "hyperplanes"},
    {&tinympc_batch_t::cones_per_instance, &tinympc_batch_t::reserved3, 1,
     {{&tinympc_batch_t::cone_x_mu, 0, [](const tmpc::ProblemDesc &pd, int) { return (size_t)pd.ncx; }},
      {&tinympc_batch_t::cone_u_mu, 1, [](const tmpc::ProblemDesc &pd, int) { return (size_t)pd.ncu; }}},
     [](const tinympc_b200_solver *s, int side) { return (bool)(side ? features(s).soc_u : features(s).soc_x); },
     true,
     "cones_per_instance must be 0 (the handle's cone coefficients) or 1 (cone_x_mu / cone_u_mu per instance), and reserved3 "
     "must be 0",
     nullptr,
     TINYMPC_ERR_ARG,
     "per-instance cones: en_state_soc / en_input_soc set on a side with cones but the batch has no cone_x_mu / cone_u_mu for it",
     "cone coefficients", "cones", "cones_per_instance", "hyperplanes"},
    {&tinympc_batch_t::planes_per_instance, &tinympc_batch_t::reserved4, 1,
     {{&tinympc_batch_t::Alin_x, 0, [](const tmpc::ProblemDesc &pd, int) { return (size_t)pd.nx * pd.nlx; }},
      {&tinympc_batch_t::blin_x, 0, [](const tmpc::ProblemDesc &pd, int) { return (size_t)pd.nlx; }},
      {&tinympc_batch_t::Alin_u, 1, [](const tmpc::ProblemDesc &pd, int) { return (size_t)pd.nu * pd.nlu; }},
      {&tinympc_batch_t::blin_u, 1, [](const tmpc::ProblemDesc &pd, int) { return (size_t)pd.nlu; }}},
     [](const tinympc_b200_solver *s, int side) { return side ? features(s).lin_u && s->pd.nlu > 0 : features(s).lin_x && s->pd.nlx > 0; },
     true,
     "planes_per_instance must be 0 (the handle's hyperplanes) or 1 (Alin_x / blin_x / Alin_u / blin_u per instance), and "
     "reserved4 must be 0",
     nullptr,
     TINYMPC_ERR_ARG,
     "per-instance hyperplanes: en_state_linear / en_input_linear set on a side with rows but the batch has no Alin_x / blin_x "
     "or Alin_u / blin_u for it",
     "hyperplanes", "hyperplanes", "planes_per_instance", "bounds or cones"},
};

// what a batch brings per instance and what its solve's kernel reads (tmpc::PerInstance)
tmpc::PerInstance per_instance(const tinympc_b200_solver *s, const tinympc_batch_t *io) {
    tmpc::PerInstance pi;
    pi.models = io->models != nullptr;
    for (int k = 0; k < tmpc::NKINDS; ++k) {
        const KindDesc &kd = KINDS[k];
        pi.given[k] = io->*kd.mode;
        pi.read[k] = pi.given[k] && (!kd.gps_only || kd.runs(s, 0) || kd.runs(s, 1)) ? pi.given[k] : 0;
    }
    return pi;
}

// The checks of a solve before it is planned: the handle's state, then the arguments (ar: adaptive rho, or null).  Their
// order decides which error a caller sees.
int check_solve(const tinympc_b200_solver *s, const tinympc_batch_t *io, const tinympc_adaptive_rho_t *ar) {
    const tinympc_settings_t &st = s->settings;
    for (const KindDesc &kd : KINDS) {
        const int mode = io->*kd.mode;
        if (mode < 0 || mode > kd.max_mode || io->*kd.reserved != 0) return fail(TINYMPC_ERR_ARG, kd.mode_msg);
        if (mode == 0) {  // the handle's arrays: only bounds can be missing from a handle
            if (&kd == &KINDS[tmpc::KIND_BOUNDS] && ((st.en_state_bound && !s->pd.x_min) || (st.en_input_bound && !s->pd.u_min)))
                return fail(TINYMPC_ERR_NO_BOUNDS, "en_state_bound/en_input_bound set but bounds were never provided");
            continue;
        }
        // the batch's arrays replace the handle's; a side whose loop does not run is never read
        int n[2] = {}, have[2] = {};  // arrays per side, and those of them the batch gives
        for (const KindArray &a : kd.arrays)
            if (a.member) {
                ++n[a.side];
                have[a.side] += io->*a.member != nullptr;
            }
        if (kd.pairs_msg && ((have[0] && have[0] != n[0]) || (have[1] && have[1] != n[1]))) return fail(TINYMPC_ERR_ARG, kd.pairs_msg);
        if ((kd.runs(s, 0) && have[0] < n[0]) || (kd.runs(s, 1) && have[1] < n[1])) return fail(kd.missing_code, kd.missing_msg);
    }
    if (st.check_termination <= 0) return fail(TINYMPC_ERR_ARG, "check_termination must be >= 1");
    if (!io->x0 || !io->Xref) return fail(TINYMPC_ERR_ARG, "x0 and Xref are required");
    if (ar && io->models) return fail(TINYMPC_ERR_ARG, "adaptive rho: the model blobs go in tinympc_adaptive_rho_t.models (in/out); io->models must be NULL");
    if (ar && (!ar->models || !ar->dKinf_drho || !ar->dPinf_drho || ar->reserved != 0))
        return fail(TINYMPC_ERR_ARG, "adaptive rho: models, dKinf_drho and dPinf_drho are required and reserved must be 0");
    if (ar && ar->tables_per_instance != 0 && ar->tables_per_instance != 1)
        return fail(TINYMPC_ERR_ARG, "adaptive rho: tables_per_instance must be 0 (one table pair for the batch) or 1 (one pair per instance)");
    return 0;
}

// How a solve runs: the kernel family, the on-chip kernel's launch plan, and the instances one CTA holds when the batch fills
// every SM (the host path rounds its chunks to whole waves of these).
struct SolvePlan {
    int family = -1;
    tmpc::GpiPlan gpi;    // L == 0: no on-chip plan
    int64_t per_cta = 0;  // 0: chunks are not rounded
};

// shared memory the adaptive kernel adds per CTA for its tables
size_t adapt_smem(const tinympc_b200_solver *s) { return tmpc::gpi_adapt_bytes(s->pd.nx, s->pd.nu, esize(s->pd.dtype)); }

// The entry points only an on-chip kernel variant serves (rollouts, adaptive rho): the variant bits, and plan_solve's
// refusals in the order it checks them (mode, constraint families, kernel family, horizon)
struct OnChipOnly {
    int bits;
    const char *strict, *box, *family, *fit;
} const ONCHIP_ONLY[2] = {
    {tmpc::GPI_ROLLOUT, "rollouts are available in STRICT mode only", "rollouts cover box constraints only (no cones or hyperplanes)",
     "rollouts run on the on-chip (GPI) kernel family only", "rollout: the horizon does not fit the on-chip kernel"},
    {tmpc::GPI_ADAPT, "adaptive rho is available in STRICT mode only", "adaptive rho covers box constraints only (no cones or hyperplanes)",
     "adaptive rho runs on the on-chip (GPI) kernel family only", "adaptive rho: the horizon does not fit the on-chip kernel"}};

// The plan of a solve of B instances (pi: its per-instance data; adapt: adaptive rho).  GPI = lane groups, state on chip (box
// constraints, horizon fits in shared memory); GPS = lane groups, state streamed (everything else the lane mapping covers);
// TPI = one thread per instance.  Fails when an explicit request or a feature cannot be served.
int plan_solve(const tinympc_b200_solver *s, const tmpc::PerInstance &pi, bool adapt, int64_t B, SolvePlan *p, bool rollout = false) {
    const tmpc::Features ft = features(s);
    // per-instance kinds have STRICT solve variants only; the refusals look at the flags, planes first, then cones, then bounds
    for (int k = tmpc::NKINDS - 1; k >= 0; --k) {
        if (!pi.given[k]) continue;
        const KindDesc &kd = KINDS[k];
        if (rollout) return fail(TINYMPC_ERR_UNSUPPORTED, std::string("rollouts run with the handle's ") + kd.handles + " (" + kd.field + " must be 0)");
        if (adapt) return fail(TINYMPC_ERR_UNSUPPORTED, std::string("adaptive rho runs with the handle's ") + kd.handles + " (" + kd.field + " must be 0)");
        if (s->mode == TINYMPC_MODE_FAST)
            return fail(TINYMPC_ERR_UNSUPPORTED, std::string("per-instance ") + kd.noun + " are available in STRICT mode only");
        if (kd.gps_only && s->family == TINYMPC_KERNEL_TPI)
            return fail(TINYMPC_ERR_UNSUPPORTED, std::string("per-instance ") + kd.noun +
                                                     " run on the streamed lane-group kernel (GPS), not on one thread per instance");
        bool compiled = false;  // some streamed kernel serves the kinds the batch gives together
        for (int fam : {0, 1, 6, 7}) compiled |= tmpc::gps_compiled(fam, tmpc::gps_variant(pi.models, pi.given), false);
        if (!compiled)
            return fail(TINYMPC_ERR_UNSUPPORTED, std::string("per-instance ") + kd.noun + " do not combine with per-instance " +
                                                     kd.exclusive + " in one batch");
    }
    if (rollout || adapt) {  // the on-chip kernel's variant, with the on-chip plan a solve would use less the adaptive tables
        const OnChipOnly &oc = ONCHIP_ONLY[rollout ? 0 : 1];
        bool compiled = false;  // some on-chip kernel serves the variant in this mode (adaptive rho adapts per-instance blobs)
        for (int L : {4, 8, 16})
            compiled |= tmpc::gpi_compiled(L, oc.bits, adapt || pi.models, false, s->mode == TINYMPC_MODE_FAST, s->pd.dtype == TINYMPC_F64);
        if (!compiled) return fail(TINYMPC_ERR_UNSUPPORTED, oc.strict);
        if (ft.ext) return fail(TINYMPC_ERR_UNSUPPORTED, oc.box);
        if (s->family == TINYMPC_KERNEL_TPI || s->family == TINYMPC_KERNEL_GPS) return fail(TINYMPC_ERR_UNSUPPORTED, oc.family);
        const size_t tables = oc.bits == tmpc::GPI_ADAPT ? adapt_smem(s) : 0;
        p->gpi = s->dim->gpi_plan(s->pd.dtype, s->pd.N, s->max_smem_optin - (int)tables);
        if (p->gpi.smem <= 0) return fail(TINYMPC_ERR_UNSUPPORTED, oc.fit);
        p->gpi.smem += tables;
        p->family = TINYMPC_KERNEL_GPI;
        p->per_cta = p->gpi.instances_per_cta;
        return 0;
    }
    if (!ft.ext) p->gpi = s->dim->gpi_plan(s->pd.dtype, s->pd.N, s->max_smem_optin);
    const bool gpi_ok = p->gpi.smem > 0;
    const bool gps_ok = s->dim->gps_lanes(s->pd.dtype) > 0;
    if (s->family == TINYMPC_KERNEL_GPI) {
        p->family = gpi_ok ? TINYMPC_KERNEL_GPI : (gps_ok ? TINYMPC_KERNEL_GPS : -1);
    } else if (s->family == TINYMPC_KERNEL_GPS) {
        p->family = gps_ok ? TINYMPC_KERNEL_GPS : -1;
    } else if (s->family == TINYMPC_KERNEL_TPI) {
        p->family = TINYMPC_KERNEL_TPI;
    } else if (ft.ext) {  // AUTO (measured rules; evidence: tools/auto_rule_sweep.py, DESIGN.md §5).  Cones / hyperplanes: streamed lane groups
        p->family = gps_ok ? TINYMPC_KERNEL_GPS : TINYMPC_KERNEL_TPI;
    } else {
        const bool big_batch = B >= (int64_t)s->sm_count * 384;  // one thread per instance fills the GPU
        // box constraints, streamed alternative when the state does not stay on chip: one thread per instance for big batches
        // (it beats the streamed lane groups on every measured shape, fp64 (6,3,100) included: 60.0 vs 63.9 ms); small batches
        // cannot fill the GPU with one thread per instance
        const int streamed = (gps_ok && !big_batch) ? TINYMPC_KERNEL_GPS : TINYMPC_KERNEL_TPI;
        // Big batches leave the chip when shared memory holds too few instances per SM, except for (16,8), where the
        // thread-per-instance register footprint costs more than the low on-chip occupancy.  Measured on H100 (B = 131 072 fp32 /
        // 65 536 fp64, 50 iterations): fp32 on chip wins from 16 instances per SM on ((12,8,50): 45 vs 69 ms thread per instance;
        // (12,4,100): 85 vs 94 ms) and loses at 8 ((4,8,100): 128 vs 78 ms); fp64 (rows re-read per sweep) on chip wins with three
        // warps per SM ((4,2,50): 13 vs 19 ms; (16,8,50): 80 vs 197 ms) unless they hold only 6 instances ((12,4,50): 73 vs 60 ms),
        // and loses badly with one warp ((6,3,100): 143 vs 60 ms thread per instance).
        const int ipc = p->gpi.instances_per_cta;
        const bool tpi_heavy = s->pd.nx >= 16 && s->pd.nu >= 8;
        const bool few = s->pd.dtype == TINYMPC_F64 ? (p->gpi.warps < 2 || ipc < 8) : ipc < 16;
        p->family = (!gpi_ok || (ipc > 0 && few && !tpi_heavy && big_batch)) ? streamed : TINYMPC_KERNEL_GPI;
    }
    if (p->family == TINYMPC_KERNEL_GPI) p->per_cta = p->gpi.instances_per_cta;
    // Per-instance data (models, bounds or both): the on-chip kernel, exactly as without them, when the family is AUTO or GPI
    // and the problem has box constraints only and an on-chip plan (per_cta is left as the rules above set it: the host path
    // rounds such chunks by the family a shared model would get).  Otherwise the streamed kernel's one-instance-per-lane-group
    // variant: explicit GPS, cones or hyperplanes, or a horizon that does not fit on chip.  One thread per instance has no
    // such variant.
    if (pi.models || pi.given[tmpc::KIND_BOUNDS]) {
        if (s->family == TINYMPC_KERNEL_TPI)
            return fail(TINYMPC_ERR_UNSUPPORTED, "per-instance models and bounds run on the lane-group kernel families (GPI, GPS), not on one thread per instance");
        if (s->family != TINYMPC_KERNEL_GPS && !ft.ext && gpi_ok) {
            p->family = TINYMPC_KERNEL_GPI;
        } else {
            if (!gps_ok) return fail(TINYMPC_ERR_UNSUPPORTED, "per-instance models / bounds: this problem needs the streamed lane-group kernel, which does not cover this shape");
            p->family = TINYMPC_KERNEL_GPS;
            p->per_cta = s->dim->gps_het_slots(s->pd.dtype, ft.soc_x || ft.soc_u, ft.lin_x || ft.lin_u || ft.tvl_x || ft.tvl_u,
                                               pi.read[tmpc::KIND_CONES], s->max_smem_optin);
        }
    }
    // A cone or static hyperplane loop routes the solve to the streamed kernel when it covers the shape; its GPS_CONES /
    // GPS_PLANES variants keep the plan the rules above chose (alone: the shared solve's, whose chunks are not rounded; with
    // models or bounds: gps_het_slots)
    for (int k = 0; k < tmpc::NKINDS; ++k)
        if (KINDS[k].gps_only && pi.read[k] && p->family != TINYMPC_KERNEL_GPS)
            return fail(TINYMPC_ERR_UNSUPPORTED, std::string("per-instance ") + KINDS[k].noun +
                                                     ": this problem needs the streamed lane-group kernel, which does not cover this shape");
    if (p->family < 0) return fail(TINYMPC_ERR_UNSUPPORTED, "the requested lane-group kernel does not cover this problem shape");
    return 0;
}

// `bytes` of launch arguments of an on-chip kernel variant, written by fill(host staging), into s->d_args, ordered on `stream`:
// an asynchronous copy from a page-locked staging slot (the host returns without waiting for earlier work on the stream).
// `what` names the variant in error messages.
template <typename F>
int upload_args(tinympc_b200_solver *s, size_t bytes, cudaStream_t stream, const char *what, F &&fill) {
    if (s->d_args.bytes < bytes) {
        if (s->have_last) CUDA_TRY(cudaEventSynchronize(s->ev_last));  // a previous solve may still read the old buffer
        if (s->d_args.ensure(bytes)) return fail(TINYMPC_ERR_CUDA, std::string(what) + " argument allocation failed");
    }
    const int slot = s->args_next;
    s->args_next = (slot + 1) % 3;
    if (!s->ev_args[slot]) CUDA_TRY(cudaEventCreateWithFlags(&s->ev_args[slot], cudaEventDisableTiming));
    if (s->args_used[slot]) CUDA_TRY(cudaEventSynchronize(s->ev_args[slot]));  // its previous copy has been read
    if (s->args_pin[slot].ensure(bytes)) return fail(TINYMPC_ERR_CUDA, std::string(what) + " staging allocation failed");
    char *h = (char *)s->args_pin[slot].p;
    std::memset(h, 0, bytes);
    fill(h);
    CUDA_TRY(cudaMemcpyAsync(s->d_args.p, h, bytes, cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaEventRecord(s->ev_args[slot], stream));
    s->args_used[slot] = true;
    return 0;
}

// the adaptive kernel's arguments (GpiAdapt<T>, then the shared tables).  Per-instance tables are device arrays already: the
// arguments point at them and nothing follows the header.
template <typename T>
int upload_adaptive(tinympc_b200_solver *s, const tinympc_adaptive_rho_t *ar, const void *models, cudaStream_t stream) {
    const size_t nk = (size_t)s->pd.nu * s->pd.nx, np = (size_t)s->pd.nx * s->pd.nx;
    const bool per = ar->tables_per_instance != 0;
    const size_t bytes = tmpc::GPI_ADAPT_HDR + (per ? 0 : (nk + np) * sizeof(T));
    return upload_args(s, bytes, stream, "adaptive-rho", [&](char *h) {
        tmpc::GpiAdapt<T> a{};
        a.models = (T *)models;
        if (per) {  // [B][nu*nx], [B][nx*nx] device arrays, read by the GPI_ADAPT_TABLES kernel variant
            a.dK = (const T *)ar->dKinf_drho;
            a.dP = (const T *)ar->dPinf_drho;
        } else {
            T *tab = (T *)(h + tmpc::GPI_ADAPT_HDR);
            std::memcpy(tab, ar->dKinf_drho, nk * sizeof(T));
            std::memcpy(tab + nk, ar->dPinf_drho, np * sizeof(T));
            a.dK = (const T *)((char *)s->d_args.p + tmpc::GPI_ADAPT_HDR);
            a.dP = a.dK + nk;
        }
        a.rho_min = (T)ar->rho_min;
        a.rho_max = (T)ar->rho_max;
        a.clip = ar->enable_clipping != 0;
        const long cols = (long)s->pd.nx * s->pd.N + (long)s->pd.nu * (s->pd.N - 1);
        a.maskA = tmpc::gemv_block_mask((long)(s->pd.nx + s->pd.nu) * (s->pd.N - 1), cols, sizeof(T));
        a.maskP = tmpc::gemv_block_mask(cols, cols, sizeof(T));
        static_assert(sizeof(a) <= tmpc::GPI_ADAPT_HDR, "GpiAdapt must fit its header");
        std::memcpy(h, &a, sizeof(a));
    });
}

// elements of a plant record (A | B | f): the first three pieces of a model blob
int64_t plant_elems(const tinympc_b200_solver *s) { return tmpc::model_blob<int64_t>(s->pd.nx, s->pd.nu).Qd; }

// does a rollout need the GPI_PLANT variant (a plant of its own or measurement noise)?
bool rollout_plant(const tinympc_rollout_t *ro) { return ro->plant || ro->noise; }

// the rollout kernel's arguments (GpiRoll<T>).  Without a plant of their own, the instances' plant is the controller's model:
// the handle's blob or the batch's model blobs, whose first pieces are a plant record.
template <typename T>
int upload_rollout(tinympc_b200_solver *s, const tinympc_batch_t *io, const tinympc_rollout_t *ro, cudaStream_t stream) {
    return upload_args(s, sizeof(tmpc::GpiRoll<T>), stream, "rollout", [&](char *h) {
        tmpc::GpiRoll<T> r{};
        r.steps = ro->T;
        r.reset_duals = ro->reset_duals;
        r.w = (const T *)ro->w;
        r.x_traj = (T *)ro->x_traj;
        r.u_traj = (T *)ro->u_traj;
        r.res_traj = (T *)ro->residuals_traj;
        r.iter_traj = ro->iter_traj;
        r.solved_traj = ro->solved_traj;
        if (rollout_plant(ro)) {
            if (ro->plant) {
                r.plant = (const T *)ro->plant;
                r.plant_stride = ro->plant_per_instance ? plant_elems(s) : 0;
            } else if (io->models) {
                r.plant = (const T *)io->models;
                r.plant_stride = tinympc_b200_model_blob_elems(s->pd.nx, s->pd.nu);
            } else {
                r.plant = (const T *)s->pd.blob;
            }
            r.noise = (const T *)ro->noise;
            r.xtrue = ro->noise ? (T *)s->xtrue.p : nullptr;
        }
        std::memcpy(h, &r, sizeof(r));
    });
}

// enqueue one batched solve on `stream` (device pointers, checked by check_solve); fills stats.  io->models: the model blobs
// the kernel reads, the per-instance models or, with ar (adaptive rho, else null), the blobs it adapts in place
int enqueue(tinympc_b200_solver *s, const tinympc_batch_t *io, cudaStream_t stream, bool timed,
            const tinympc_adaptive_rho_t *ar = nullptr, const tinympc_rollout_t *ro = nullptr) {
    const tmpc::PerInstance pi = per_instance(s, io);
    SolvePlan plan;
    if (ar || ro || io->B > 0)  // an adaptive solve or a rollout is checked whole even when the batch is empty
        if (int rc = plan_solve(s, pi, ar != nullptr, io->B, &plan, ro != nullptr))
            return rc;
    if (io->B <= 0 || (ro && ro->T == 0)) return TINYMPC_OK;
    const int family = plan.family;
    // The launch scratch of a handle (work queue, workspaces, timing events) is single-buffered: a solve enqueued on a
    // different stream than the previous one first waits for it.
    if (s->have_last && s->last_stream != stream) CUDA_TRY(cudaStreamWaitEvent(stream, s->ev_last, 0));
    size_t ws_bytes = 0;
    tmpc::LaunchDesc d{};
    d.pd = &s->pd;
    d.st = s->settings;
    d.ft = features(s);
    d.fast = s->mode == TINYMPC_MODE_FAST;
    d.sm_count = s->sm_count;
    d.max_smem_optin = s->max_smem_optin;
    d.pi = pi;
    if (ar) {
        if (int rc = s->pd.dtype == TINYMPC_F64 ? upload_adaptive<double>(s, ar, io->models, stream)
                                                : upload_adaptive<float>(s, ar, io->models, stream))
            return rc;
        d.adapt = ar->tables_per_instance ? 2 : 1;
        d.adapt_args = s->d_args.p;
    }
    if (ro) {
        if (ro->noise && s->xtrue.ensure((size_t)io->B * s->pd.nx * esize(s->pd.dtype) + 256))
            return fail(TINYMPC_ERR_CUDA, "rollout true-state allocation failed");
        if (int rc = s->pd.dtype == TINYMPC_F64 ? upload_rollout<double>(s, io, ro, stream) : upload_rollout<float>(s, io, ro, stream))
            return rc;
        d.rollout = rollout_plant(ro) ? 2 : 1;
        d.roll_args = s->d_args.p;
    }
    if (timed) CUDA_TRY(cudaEventRecord(s->ev0, stream));
    d.family = family;
    d.stream = stream;
    d.io = *io;
    d.Bpad = (io->B + 31) / 32 * 32;
    if (family == TINYMPC_KERNEL_TPI) {
        const tmpc::ProblemDesc &pd = s->pd;
        if (s->ws.ensure(tmpc::tpi_workspace(pd.nx, pd.nu, pd.N, pd.dtype, d.Bpad, d.ft) + 256)) return fail(TINYMPC_ERR_CUDA, "workspace allocation failed");
        d.tpi_ws = s->ws.p;
        ws_bytes = s->ws.bytes;
    } else {
        if (s->queue.ensure(256)) return fail(TINYMPC_ERR_CUDA, "queue allocation failed");
        CUDA_TRY(cudaMemsetAsync(s->queue.p, 0, 256, stream));
        d.work_queue = s->queue.p;
        d.gpi = plan.gpi;
        // previous-iteration slacks are staged in pack layout, one 16-byte store per knot point; a rollout carries them there from
        // one step to the next
        if (family == TINYMPC_KERNEL_GPI && (ro ? ro->carry_v != 0 : (io->state.v || io->state.z))) {
            if (s->vscratch.ensure((size_t)io->B * plan.gpi.vscratch_per_instance + 256)) return fail(TINYMPC_ERR_CUDA, "GPI v-scratch allocation failed");
            d.gpi_vscratch = s->vscratch.p;
        }
        d.gps_ws = s->gps_ws.p;
        d.gps_ws_bytes = s->gps_ws.bytes;
    }
    int rc = s->dim->launch(&d);
    if (rc == tmpc::TM_ERR_WORKSPACE) {  // the streamed kernel sizes its workspace by resident slots: grow and retry
        if (s->have_last) CUDA_TRY(cudaEventSynchronize(s->ev_last));  // a previous solve may still use the old buffer
        if (s->gps_ws.ensure(d.out_ws_need + 256)) return fail(TINYMPC_ERR_CUDA, "GPS workspace allocation failed");
        d.gps_ws = s->gps_ws.p;
        d.gps_ws_bytes = s->gps_ws.bytes;
        rc = s->dim->launch(&d);
    }
    if (rc == TINYMPC_ERR_CUDA) return fail(rc, std::string("kernel launch failed: ") + cudaGetErrorString(cudaGetLastError()));
    if (rc) return fail(TINYMPC_ERR_UNSUPPORTED, "no compiled kernel for this (dtype, mode, family) combination");
    if (family == TINYMPC_KERNEL_GPS) ws_bytes = d.out_ws_need;
    s->stats.lanes_per_instance = d.out_lanes_per_instance;
    s->stats.instances_per_cta = d.out_instances_per_cta;
    s->stats.smem_bytes_per_cta = d.out_smem;
    s->stats.threads_per_cta = d.out_threads;
    if (timed) CUDA_TRY(cudaEventRecord(s->ev1, stream));
    CUDA_TRY(cudaEventRecord(s->ev_last, stream));
    s->last_stream = stream;
    s->have_last = true;
    s->timed = timed;
    s->stats.instances = io->B;
    s->stats.kernel_launches = 1;
    s->stats.kernel_family = family;
    s->stats.ctas = d.out_ctas;
    s->stats.gpi_instances = family == TINYMPC_KERNEL_TPI ? 0 : io->B;
    s->stats.workspace_bytes = (int64_t)ws_bytes;
    return TINYMPC_OK;
}

}  // namespace

namespace {
// The batched host precompute: the instances dealt to nthreads threads, each with a scratch of its own; the first singular
// instance, if any, is reported
template <typename T, bool TANGENT>
int riccati_batch_T(int nx, int nu, int64_t B, const tmpc::RiccatiBatch<T> &a, int nthreads) {
    nthreads = (int)std::max<int64_t>(1, std::min<int64_t>(nthreads, B));
    std::vector<int64_t> bad(nthreads, 0);
    auto work = [&](int t) {
        std::vector<T> w(tmpc::riccati_scratch(nx, nu, TANGENT).total);
        for (int64_t b = t; b < B; b += nthreads)
            if (tmpc::riccati_instance<T, TANGENT>(tmpc::DynDims{nx, nu}, tmpc::HostLanes{}, w.data(), a, b) < 0 && bad[t] == 0) bad[t] = b + 1;
    };
    std::vector<std::thread> th;
    for (int t = 1; t < nthreads; ++t) th.emplace_back(work, t);
    work(0);
    for (auto &x : th) x.join();
    int64_t first = 0;
    for (int64_t v : bad)
        if (v && (!first || v < first)) first = v;
    if (first) return fail(TINYMPC_ERR_SINGULAR, "singular R + B'PB in the Riccati recursion of instance " + std::to_string(first - 1));
    return 0;
}

int riccati_batch_host(int32_t dtype, bool tangent, int nx, int nu, int64_t B, const tmpc::RiccatiBatch<void> &a, int nthreads) {
    if (dtype == TINYMPC_F64)
        return tangent ? riccati_batch_T<double, true>(nx, nu, B, a.as<double>(), nthreads)
                       : riccati_batch_T<double, false>(nx, nu, B, a.as<double>(), nthreads);
    if (dtype == TINYMPC_F32)
        return tangent ? riccati_batch_T<float, true>(nx, nu, B, a.as<float>(), nthreads)
                       : riccati_batch_T<float, false>(nx, nu, B, a.as<float>(), nthreads);
    return fail(TINYMPC_ERR_ARG, "bad dtype");
}

int riccati_batch_device(tinympc_b200_solver_t *s, bool tangent, int64_t B, const tmpc::RiccatiBatch<void> &a, int32_t *sweeps_out,
                         void *stream) {
    if (!s) return fail(TINYMPC_ERR_ARG, "null handle");
    if (!a.A || !a.B || !a.Qd || !a.Rd || !a.rho || (tangent ? !a.dK || !a.dP : !a.f || !a.models) || B < 0)
        return fail(TINYMPC_ERR_ARG, "null pointer or bad size");
    if (B == 0) return TINYMPC_OK;
    CUDA_TRY(cudaSetDevice(s->device));
    const int rc = s->dim->riccati_batch(s->pd.dtype, tangent, B, a, sweeps_out, s->sm_count, (cudaStream_t)stream);
    const std::string what = tangent ? "sensitivity" : "precompute";
    if (rc == TINYMPC_ERR_CUDA) return fail(rc, what + " kernel launch failed: " + cudaGetErrorString(cudaGetLastError()));
    if (rc) return fail(rc, what + " kernel unavailable for this dtype");
    return TINYMPC_OK;
}
}  // namespace

extern "C" {

const char *tinympc_b200_last_error(void) { return g_err.c_str(); }
const char *tinympc_b200_version(void) { return "tinympc_b200 0.1 (sm_90a)"; }

int tinympc_b200_supported(int32_t dtype, int32_t nx, int32_t nu) {
    return (dtype == TINYMPC_F32 || dtype == TINYMPC_F64) && find_dim(nx, nu) != nullptr;
}

int tinympc_b200_default_settings(tinympc_settings_t *s) {
    if (!s) return fail(TINYMPC_ERR_ARG, "settings is null");
    s->abs_pri_tol = 1e-3;  // tiny_api_constants.hpp:5-16
    s->abs_dua_tol = 1e-3;
    s->max_iter = 1000;
    s->check_termination = 1;
    s->en_state_bound = 1;
    s->en_input_bound = 1;
    s->en_state_soc = 0;
    s->en_input_soc = 0;
    s->en_state_linear = 0;
    s->en_input_linear = 0;
    s->en_tv_state_linear = 0;
    s->en_tv_input_linear = 0;
    return TINYMPC_OK;
}

int tinympc_b200_precompute_cache(int32_t dtype, int32_t nx, int32_t nu, double rho, const void *A, const void *B,
                                  const void *f, const void *Q, const void *R, void *Kinf, void *Pinf, void *Quu_inv,
                                  void *AmBKt, void *APf, void *BPf) {
    if (!A || !B || !f || !Q || !R || !Kinf || !Pinf || !Quu_inv || !AmBKt || !APf || !BPf || nx <= 0 || nu <= 0)
        return fail(TINYMPC_ERR_ARG, "null pointer or bad size");
    auto one = [&](auto t) {
        using T = decltype(t);
        std::vector<T> w(tmpc::riccati_scratch(nx, nu, false).total);
        const tmpc::RiccatiOut<T> out{(const T *)f, (T *)Kinf, (T *)Pinf, (T *)Quu_inv, (T *)AmBKt, (T *)APf, (T *)BPf, nullptr, nullptr};
        return tmpc::riccati<T, false>(tmpc::DynDims{nx, nu}, tmpc::HostLanes{}, w.data(), (const T *)A, (const T *)B, (const T *)Q,
                                       (const T *)R, (T)rho, out);
    };
    int rc;
    if (dtype == TINYMPC_F64)
        rc = one(0.0);
    else if (dtype == TINYMPC_F32)
        rc = one(0.f);
    else
        return fail(TINYMPC_ERR_ARG, "bad dtype");
    if (rc < 0) return fail(TINYMPC_ERR_ARG, "singular R + B'PB in the Riccati recursion");
    return rc;
}

int64_t tinympc_b200_model_blob_elems(int32_t nx, int32_t nu) {
    return tmpc::model_blob<int64_t>(nx, nu).model;
}

int tinympc_b200_precompute_cache_batch(int32_t dtype, int32_t nx, int32_t nu, int64_t B, const void *A, const void *Bm,
                                        const void *f, const void *Qdiag, const void *Rdiag, const void *rho,
                                        void *models_out, int32_t nthreads) {
    if (!A || !Bm || !f || !Qdiag || !Rdiag || !rho || !models_out || nx <= 0 || nu <= 0 || B < 0)
        return fail(TINYMPC_ERR_ARG, "null pointer or bad size");
    return riccati_batch_host(dtype, false, nx, nu, B, {A, Bm, f, Qdiag, Rdiag, rho, models_out, nullptr, nullptr}, nthreads);
}

int tinympc_b200_precompute_cache_batch_device(tinympc_b200_solver_t *s, int64_t B, const void *A, const void *Bm, const void *f,
                                               const void *Qdiag, const void *Rdiag, const void *rho, void *models_out,
                                               int32_t *sweeps_out, void *stream) {
    return riccati_batch_device(s, false, B, {A, Bm, f, Qdiag, Rdiag, rho, models_out, nullptr, nullptr}, sweeps_out, stream);
}

int tinympc_b200_precompute_sensitivity_batch(int32_t dtype, int32_t nx, int32_t nu, int64_t B, const void *A, const void *Bm,
                                              const void *f, const void *Qdiag, const void *Rdiag, const void *rho, void *dK_out,
                                              void *dP_out, int32_t nthreads) {
    if (!A || !Bm || !Qdiag || !Rdiag || !rho || !dK_out || !dP_out || nx <= 0 || nu <= 0 || B < 0)
        return fail(TINYMPC_ERR_ARG, "null pointer or bad size");
    // the affine term f does not enter Kinf / Pinf
    return riccati_batch_host(dtype, true, nx, nu, B, {A, Bm, f, Qdiag, Rdiag, rho, nullptr, dK_out, dP_out}, nthreads);
}

int tinympc_b200_precompute_sensitivity_batch_device(tinympc_b200_solver_t *s, int64_t B, const void *A, const void *Bm, const void *f,
                                                     const void *Qdiag, const void *Rdiag, const void *rho, void *dK_out, void *dP_out,
                                                     int32_t *sweeps_out, void *stream) {
    return riccati_batch_device(s, true, B, {A, Bm, f, Qdiag, Rdiag, rho, nullptr, dK_out, dP_out}, sweeps_out, stream);
}

int tinympc_b200_create(const tinympc_problem_t *p, int32_t device, tinympc_b200_solver_t **out) {
    if (!p || !out) return fail(TINYMPC_ERR_ARG, "null argument");
    *out = nullptr;
    if (p->nx <= 0 || p->nu <= 0 || p->N < 2) return fail(TINYMPC_ERR_ARG, "need nx>0, nu>0, N>=2");
    if (p->dtype != TINYMPC_F32 && p->dtype != TINYMPC_F64) return fail(TINYMPC_ERR_ARG, "bad dtype");
    if (!p->Adyn || !p->Bdyn || !p->fdyn || !p->Q || !p->R || !p->Kinf || !p->Pinf || !p->Quu_inv || !p->AmBKt ||
        !p->APf || !p->BPf)
        return fail(TINYMPC_ERR_ARG, "model / cache pointer is null");
    const tmpc::DimEntry *dim = find_dim(p->nx, p->nu);
    if (!dim) return fail(TINYMPC_ERR_UNSUPPORTED, "no kernel compiled for this (nx, nu); add it to TM_DIMS in csrc/launch.h");
    if (p->num_state_cones > 4 || p->num_input_cones > 4) return fail(TINYMPC_ERR_UNSUPPORTED, "at most 4 cones per side");
    for (int c = 0; c < p->num_state_cones && p->Acx && p->qcx; ++c)
        if (p->qcx[c] != 3 || p->Acx[c] < 0 || p->Acx[c] + 3 > p->nx) return fail(TINYMPC_ERR_CONE_DIM, "state cone must be 3-dimensional and inside the state");
    for (int c = 0; c < p->num_input_cones && p->Acu && p->qcu; ++c)
        if (p->qcu[c] != 3 || p->Acu[c] < 0 || p->Acu[c] + 3 > p->nu) return fail(TINYMPC_ERR_CONE_DIM, "input cone must be 3-dimensional and inside the input");

    if (p->num_state_linear < 0 || p->num_input_linear < 0 || p->num_tv_state_linear < 0 || p->num_tv_input_linear < 0)
        return fail(TINYMPC_ERR_ARG, "negative constraint count");
    if ((p->num_state_linear > 0 && (!p->Alin_x || !p->blin_x)) || (p->num_input_linear > 0 && (!p->Alin_u || !p->blin_u)) ||
        (p->num_tv_state_linear > 0 && (!p->tv_Alin_x || !p->tv_blin_x)) ||
        (p->num_tv_input_linear > 0 && (!p->tv_Alin_u || !p->tv_blin_u)))
        return fail(TINYMPC_ERR_ARG, "hyperplane count > 0 with a NULL normal matrix or offset vector");
    if ((p->num_state_cones > 0 && (!p->Acx || !p->qcx || !p->cx)) || (p->num_input_cones > 0 && (!p->Acu || !p->qcu || !p->cu)))
        return fail(TINYMPC_ERR_ARG, "cone count > 0 with a NULL index / mu vector");

    int ndev = 0;
    CUDA_TRY(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(TINYMPC_ERR_ARG, "bad device index");
    CUDA_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return fail(TINYMPC_ERR_UNSUPPORTED, "this library is built for sm_90a (H100) only");

    tinympc_b200_solver *s = new tinympc_b200_solver();
    s->device = device;
    s->sm_count = prop.multiProcessorCount;
    s->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
    s->l2_bytes = prop.l2CacheSize;
    s->dim = dim;
    const size_t es = esize(p->dtype), nx = p->nx, nu = p->nu, N = p->N;
    tinympc_b200_default_settings(&s->settings);
    tmpc::ProblemDesc &pd = s->pd;
    pd.nx = p->nx; pd.nu = p->nu; pd.N = p->N; pd.dtype = p->dtype; pd.rho = p->rho;
    {   // the cache blob (model_blob.h): the kernel parameters are filled from it, the lane-group kernels stage it into shared memory
        const tmpc::ModelBlob mb = tmpc::model_blob(p->nx, p->nu);
        pd.h_blob.assign(((size_t)mb.cache * es + 63) / 64 * 64, 0);
        auto put = [&](int off, const void *v, size_t elems) { std::memcpy(pd.h_blob.data() + (size_t)off * es, v, elems * es); };
        put(mb.A, p->Adyn, nx * nx); put(mb.B, p->Bdyn, nx * nu); put(mb.f, p->fdyn, nx); put(mb.Qd, p->Q, nx); put(mb.Rd, p->R, nu);
        put(mb.Kinf, p->Kinf, nu * nx); put(mb.Pinf, p->Pinf, nx * nx); put(mb.Quu, p->Quu_inv, nu * nu); put(mb.AmBKt, p->AmBKt, nx * nx);
        put(mb.APf, p->APf, nx); put(mb.BPf, p->BPf, nu);
    }
    auto varies = [&](const void *m, size_t rows, size_t cols) {  // does a (rows x cols) column-major matrix vary along columns?
        if (!m) return false;
        const char *c = (const char *)m;
        for (size_t k = 1; k < cols; ++k)
            if (std::memcmp(c, c + k * rows * es, rows * es) != 0) return true;
        return false;
    };
    auto has_zero = [&](const void *m, size_t n) {  // any element == +-0 ?
        if (!m) return false;
        for (size_t i = 0; i < n; ++i)
            if ((es == 8 ? ((const double *)m)[i] : (double)((const float *)m)[i]) == 0.0) return true;
        return false;
    };
    pd.bounds_zero_free = !(has_zero(p->x_min, (size_t)nx * N) || has_zero(p->x_max, (size_t)nx * N) ||
                            has_zero(p->u_min, (size_t)nu * (N - 1)) || has_zero(p->u_max, (size_t)nu * (N - 1)));
    pd.bounds_tv = varies(p->x_min, nx, N) || varies(p->x_max, nx, N) || varies(p->u_min, nu, N - 1) || varies(p->u_max, nu, N - 1);
    const bool xb = p->x_min && p->x_max, ub = p->u_min && p->u_max;
    auto col0 = [&](std::vector<char> &h, const void *m, size_t rows) { h.assign((const char *)m, (const char *)m + rows * es); };
    if (xb) { col0(pd.h_xlo, p->x_min, nx); col0(pd.h_xhi, p->x_max, nx); }
    if (ub) { col0(pd.h_ulo, p->u_min, nu); col0(pd.h_uhi, p->u_max, nu); }
    auto rd = [&](const void *base, int i) { return p->dtype == TINYMPC_F64 ? ((const double *)base)[i] : (double)((const float *)base)[i]; };
    pd.ncx = p->num_state_cones; pd.ncu = p->num_input_cones;
    for (int c = 0; c < pd.ncx; ++c) { pd.cone_x_start[c] = p->Acx[c]; pd.cone_x_mu[c] = rd(p->cx, c); }
    for (int c = 0; c < pd.ncu; ++c) { pd.cone_u_start[c] = p->Acu[c]; pd.cone_u_mu[c] = rd(p->cu, c); }
    pd.nlx = p->num_state_linear; pd.nlu = p->num_input_linear;
    pd.ntvx = p->num_tv_state_linear; pd.ntvu = p->num_tv_input_linear;
    // the device arrays, in one allocation: the cache blob at offset 0 (cudaMalloc's alignment for its bulk copy), then each
    // array 256-byte aligned; an array that is not given stays null
    const struct { const void *src; size_t bytes; const void **dev; } arrays[] = {
        {pd.h_blob.data(), pd.h_blob.size(), &pd.blob},
        {xb ? p->x_min : nullptr, es * nx * N, &pd.x_min}, {xb ? p->x_max : nullptr, es * nx * N, &pd.x_max},
        {ub ? p->u_min : nullptr, es * nu * (N - 1), &pd.u_min}, {ub ? p->u_max : nullptr, es * nu * (N - 1), &pd.u_max},
        {p->Alin_x, es * pd.nlx * nx, &pd.Alin_x}, {p->blin_x, es * pd.nlx, &pd.blin_x},
        {p->Alin_u, es * pd.nlu * nu, &pd.Alin_u}, {p->blin_u, es * pd.nlu, &pd.blin_u},
        {p->tv_Alin_x, es * pd.ntvx * N * nx, &pd.tv_Alin_x}, {p->tv_blin_x, es * pd.ntvx * N, &pd.tv_blin_x},
        {p->tv_Alin_u, es * pd.ntvu * (N - 1) * nu, &pd.tv_Alin_u}, {p->tv_blin_u, es * pd.ntvu * (N - 1), &pd.tv_blin_u},
    };
    auto aligned = [](size_t n) { return (n + 255) / 256 * 256; };
    size_t bytes = 0;
    for (const auto &a : arrays)
        if (a.src && a.bytes) bytes += aligned(a.bytes);
    bool ok = !s->problem.ensure(bytes);
    size_t off = 0;
    for (const auto &a : arrays) {
        if (!ok || !a.src || !a.bytes) continue;
        *a.dev = (char *)s->problem.p + off;
        ok &= cudaMemcpy((char *)s->problem.p + off, a.src, a.bytes, cudaMemcpyHostToDevice) == cudaSuccess;
        off += aligned(a.bytes);
    }
    ok &= cudaEventCreate(&s->ev0) == cudaSuccess && cudaEventCreate(&s->ev1) == cudaSuccess &&
          cudaEventCreateWithFlags(&s->ev_last, cudaEventDisableTiming) == cudaSuccess;
    if (!ok) {
        tinympc_b200_destroy(s);
        return fail(TINYMPC_ERR_CUDA, std::string("problem upload failed: ") + cudaGetErrorString(cudaGetLastError()));
    }
    std::memset(&s->stats, 0, sizeof(s->stats));
    *out = s;
    return TINYMPC_OK;
}

int tinympc_b200_destroy(tinympc_b200_solver_t *s) {
    if (!s) return TINYMPC_OK;
    cudaSetDevice(s->device);
    for (int i = 0; i < 3; ++i)
        if (s->ev_args[i]) cudaEventDestroy(s->ev_args[i]);
    for (int i = 0; i < tinympc_b200_solver::SLOTS; ++i) {
        if (s->ev_in[i]) cudaEventDestroy(s->ev_in[i]);
        if (s->ev_k[i]) cudaEventDestroy(s->ev_k[i]);
        if (s->ev_out[i]) cudaEventDestroy(s->ev_out[i]);
    }
    if (s->st_h2d) cudaStreamDestroy(s->st_h2d);
    if (s->st_k) cudaStreamDestroy(s->st_k);
    if (s->st_d2h) cudaStreamDestroy(s->st_d2h);
    if (s->ev_last) cudaEventDestroy(s->ev_last);
    if (s->ev0) cudaEventDestroy(s->ev0);
    if (s->ev1) cudaEventDestroy(s->ev1);
    delete s;  // the buffers free their memory
    return TINYMPC_OK;
}

int tinympc_b200_update_settings(tinympc_b200_solver_t *s, const tinympc_settings_t *st) {
    if (!s || !st) return fail(TINYMPC_ERR_ARG, "null argument");
    if (st->check_termination <= 0) return fail(TINYMPC_ERR_ARG, "check_termination must be >= 1");
    s->settings = *st;
    return TINYMPC_OK;
}

int tinympc_b200_get_settings(const tinympc_b200_solver_t *s, tinympc_settings_t *st) {
    if (!s || !st) return fail(TINYMPC_ERR_ARG, "null argument");
    *st = s->settings;
    return TINYMPC_OK;
}

int tinympc_b200_set_mode(tinympc_b200_solver_t *s, int32_t mode, int32_t family) {
    if (!s) return fail(TINYMPC_ERR_ARG, "null solver");
    if (mode != TINYMPC_MODE_STRICT && mode != TINYMPC_MODE_FAST) return fail(TINYMPC_ERR_ARG, "bad mode");
    if (family != TINYMPC_KERNEL_AUTO && family != TINYMPC_KERNEL_TPI && family != TINYMPC_KERNEL_GPI && family != TINYMPC_KERNEL_GPS)
        return fail(TINYMPC_ERR_ARG, "bad kernel family");
    s->mode = mode;
    s->family = family;
    return TINYMPC_OK;
}

int tinympc_b200_solve(tinympc_b200_solver_t *s, const tinympc_batch_t *io, void *cuda_stream) {
    if (!s || !io) return fail(TINYMPC_ERR_ARG, "null argument");
    CUDA_TRY(cudaSetDevice(s->device));
    if (int rc = check_solve(s, io, nullptr)) return rc;
    return enqueue(s, io, (cudaStream_t)cuda_stream, true);
}

int tinympc_b200_solve_adaptive(tinympc_b200_solver_t *s, const tinympc_batch_t *io, const tinympc_adaptive_rho_t *ar,
                                void *cuda_stream) {
    if (!s || !io || !ar) return fail(TINYMPC_ERR_ARG, "null argument");
    CUDA_TRY(cudaSetDevice(s->device));
    if (int rc = check_solve(s, io, ar)) return rc;
    tinympc_batch_t adapted = *io;
    adapted.models = ar->models;  // the blobs the kernel adapts in place
    return enqueue(s, &adapted, (cudaStream_t)cuda_stream, true, ar);
}

int tinympc_b200_rollout(tinympc_b200_solver_t *s, const tinympc_batch_t *io, const tinympc_rollout_t *ro, void *cuda_stream) {
    if (!s || !io || !ro) return fail(TINYMPC_ERR_ARG, "null argument");
    if (io->Xref || io->Uref || io->iter || io->solved || io->residuals || io->u0)
        return fail(TINYMPC_ERR_ARG, "rollout: io->Xref, Uref, iter, solved, residuals and u0 must be NULL (the references and "
                                     "per-step outputs are trajectories in tinympc_rollout_t)");
    if (io->state.x || io->state.u) return fail(TINYMPC_ERR_ARG, "rollout: io->state.x and state.u must be NULL");
    if (ro->T < 0 || !ro->Xref) return fail(TINYMPC_ERR_ARG, "rollout: T must be >= 0 and Xref is required");
    if ((ro->reset_duals != 0 && ro->reset_duals != 1) || (ro->carry_v != 0 && ro->carry_v != 1))
        return fail(TINYMPC_ERR_ARG, "rollout: reset_duals and carry_v must be 0 or 1");
    if (ro->reserved != 0 || ro->reserved1[0] != 0 || ro->reserved1[1] != 0) return fail(TINYMPC_ERR_ARG, "rollout: reserved fields must be 0");
    if (!ro->carry_v && (io->state.v || io->state.z))
        return fail(TINYMPC_ERR_ARG, "rollout: io->state.v / state.z need carry_v = 1 (without it work->v / work->z read as zeros)");
    if ((ro->plant_per_instance != 0 && ro->plant_per_instance != 1) || ro->reserved2 != 0)
        return fail(TINYMPC_ERR_ARG, "rollout: plant_per_instance must be 0 or 1 and reserved2 must be 0");
    if (ro->plant_per_instance && !ro->plant) return fail(TINYMPC_ERR_ARG, "rollout: plant_per_instance = 1 needs a plant");
    CUDA_TRY(cudaSetDevice(s->device));
    tinympc_batch_t b = *io;  // the first step's window is the trajectory's start: the kernel reads the trajectories in its place
    b.Xref = ro->Xref;
    b.xref_per_instance = ro->xref_per_instance;
    b.Uref = ro->Uref;
    b.uref_per_instance = ro->uref_per_instance;
    if (int rc = check_solve(s, &b, nullptr)) return rc;
    return enqueue(s, &b, (cudaStream_t)cuda_stream, true, nullptr, ro);
}

namespace {
// tinympc_b200_advance[_models]: x0[b] <- (A_b x0[b] + B_b u_b) + f_b with the model of blob + b * bstride
int advance_impl(tinympc_b200_solver_t *s, int64_t B, void *x0, const void *u, int64_t u_stride, const void *blob, int64_t bstride,
                 void *cuda_stream) {
    if (B <= 0) return TINYMPC_OK;
    CUDA_TRY(cudaSetDevice(s->device));
    // threads per block = a multiple of nx so that all rows of an instance read x0 before any row writes it
    const int per = std::max(1, 256 / s->pd.nx) * s->pd.nx;
    const int64_t total = B * s->pd.nx;
    const unsigned blocks = (unsigned)((total + per - 1) / per);
    cudaStream_t st = (cudaStream_t)cuda_stream;
    if (s->pd.dtype == TINYMPC_F32)
        advance_kernel<float><<<blocks, per, 0, st>>>(s->pd.nx, s->pd.nu, u_stride, B, (const float *)blob, bstride, (float *)x0, (const float *)u);
    else
        advance_kernel<double><<<blocks, per, 0, st>>>(s->pd.nx, s->pd.nu, u_stride, B, (const double *)blob, bstride, (double *)x0, (const double *)u);
    CUDA_TRY(cudaGetLastError());
    return TINYMPC_OK;
}
}  // namespace

int tinympc_b200_advance(tinympc_b200_solver_t *s, int64_t B, void *x0, const void *u, int64_t u_stride, void *cuda_stream) {
    if (!s || !x0 || !u) return fail(TINYMPC_ERR_ARG, "null argument");
    return advance_impl(s, B, x0, u, u_stride, s->pd.blob, 0, cuda_stream);
}

int tinympc_b200_advance_models(tinympc_b200_solver_t *s, int64_t B, void *x0, const void *u, int64_t u_stride, const void *models,
                                void *cuda_stream) {
    if (!s || !x0 || !u || !models) return fail(TINYMPC_ERR_ARG, "null argument");
    return advance_impl(s, B, x0, u, u_stride, models, tinympc_b200_model_blob_elems(s->pd.nx, s->pd.nu), cuda_stream);
}

int tinympc_b200_advance_plant(tinympc_b200_solver_t *s, int64_t B, void *x0, const void *u, int64_t u_stride, const void *plant,
                               int32_t plant_per_instance, void *cuda_stream) {
    if (!s || !x0 || !u || !plant) return fail(TINYMPC_ERR_ARG, "null argument");
    if (plant_per_instance != 0 && plant_per_instance != 1) return fail(TINYMPC_ERR_ARG, "advance_plant: plant_per_instance must be 0 or 1");
    return advance_impl(s, B, x0, u, u_stride, plant, plant_per_instance ? plant_elems(s) : 0, cuda_stream);
}

int tinympc_b200_get_stats(const tinympc_b200_solver_t *s, tinympc_b200_stats_t *out) {
    if (!s || !out) return fail(TINYMPC_ERR_ARG, "null argument");
    tinympc_b200_solver *m = const_cast<tinympc_b200_solver *>(s);
    if (m->timed) {
        CUDA_TRY(cudaSetDevice(s->device));
        CUDA_TRY(cudaEventSynchronize(m->ev1));
        float ms = 0.f;
        CUDA_TRY(cudaEventElapsedTime(&ms, m->ev0, m->ev1));
        m->stats.kernel_ms = ms;
        m->timed = false;
    }
    *out = m->stats;
    return TINYMPC_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Host-pointer path.  The batch is cut into chunks; chunk c uses slot c % SLOTS (its own pinned in/out
// buffers and device io buffers).  Three streams: H2D, kernels, D2H, chained by events, so that the copy
// of chunk c+1 overlaps the solve of chunk c and the read-back of chunk c-1.
// ---------------------------------------------------------------------------------------------------------
namespace {

struct Field {
    const void *src;   // host input (may be null)
    void *dst;         // host output (may be null)
    size_t per_inst;   // bytes per instance
    bool is_in, is_out;
    void **dev_slot;   // where the device pointer goes in the device-side descriptors
    bool pinned = false;  // the caller's buffer is page-locked: DMA straight from/to it, no staging copy
};

bool is_pinned(const void *p) {
    if (!p) return false;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeHost;
}

}  // namespace

namespace {
// tinympc_b200_solve_host; with `ar` (host model blobs, in/out) the adaptive-rho solve
int solve_host_impl(tinympc_b200_solver_t *s, const tinympc_batch_t *io, const tinympc_adaptive_rho_t *ar) {
    if (!io->x0 || !io->Xref) return fail(TINYMPC_ERR_ARG, "x0 and Xref are required");
    CUDA_TRY(cudaSetDevice(s->device));
    if (int rc = check_solve(s, io, ar)) return rc;
    const int64_t B = io->B;
    // chunking: big enough to fill the GPU several times over, small enough to pipeline
    int64_t chunk = B;
    if (B > 16384) chunk = std::max<int64_t>(8192, (B + 7) / 8);
    chunk = (chunk + 31) / 32 * 32;
    SolvePlan plan;  // of a chunk
    if (ar || B > 0)  // an adaptive solve is checked whole even when the batch is empty
        if (int rc = plan_solve(s, per_instance(s, io), ar != nullptr, chunk, &plan))
            return rc;
    if (B <= 0) return TINYMPC_OK;
    const size_t es = esize(s->pd.dtype);
    const size_t bx = es * s->pd.nx * s->pd.N, bu = es * s->pd.nu * (s->pd.N - 1);
    constexpr int SLOTS = tinympc_b200_solver::SLOTS;
    if (!s->st_h2d) {
        CUDA_TRY(cudaStreamCreateWithFlags(&s->st_h2d, cudaStreamNonBlocking));
        CUDA_TRY(cudaStreamCreateWithFlags(&s->st_k, cudaStreamNonBlocking));
        CUDA_TRY(cudaStreamCreateWithFlags(&s->st_d2h, cudaStreamNonBlocking));
        for (int i = 0; i < SLOTS; ++i) {
            CUDA_TRY(cudaEventCreateWithFlags(&s->ev_in[i], cudaEventDisableTiming));
            CUDA_TRY(cudaEventCreateWithFlags(&s->ev_k[i], cudaEventDisableTiming));
            CUDA_TRY(cudaEventCreateWithFlags(&s->ev_out[i], cudaEventDisableTiming));
        }
    }

    // shared (not per-instance) references are uploaded once, into a buffer the handle keeps
    DevBuf &shared_ref = s->shared_ref;
    // template for the device-side descriptors: the batch, and the adaptive-rho arguments whose per-instance tables are staged
    struct {
        tinympc_batch_t io;
        tinympc_adaptive_rho_t ar;
    } args{*io, ar ? *ar : tinympc_adaptive_rho_t{}};
    tinympc_batch_t &dev = args.io;
    const bool cold = io->cold_start != 0;
    std::vector<Field> fields;
    fields.push_back({io->x0, nullptr, es * s->pd.nx, true, false, (void **)&dev.x0});
    if (io->xref_per_instance) fields.push_back({io->Xref, nullptr, bx, true, false, (void **)&dev.Xref});
    if (io->Uref && io->uref_per_instance) fields.push_back({io->Uref, nullptr, bu, true, false, (void **)&dev.Uref});
    if (io->models) fields.push_back({io->models, nullptr, es * (size_t)tinympc_b200_model_blob_elems(s->pd.nx, s->pd.nu), true, false, (void **)&dev.models});
    // adaptive rho: the model blobs are in/out; they travel in dev.models (io->models is NULL), where the kernel adapts them
    if (ar) fields.push_back({ar->models, ar->models, es * (size_t)tinympc_b200_model_blob_elems(s->pd.nx, s->pd.nu), true, true, (void **)&dev.models});
    for (const KindDesc &kd : KINDS) {  // sliced per chunk like the models; a side whose loop does not run is never read
        const int mode = io->*kd.mode;
        if (!mode) continue;
        for (const KindArray &a : kd.arrays) {
            if (!a.member) continue;
            if (kd.runs(s, a.side)) fields.push_back({io->*a.member, nullptr, es * a.elems(s->pd, mode), true, false, (void **)&(dev.*a.member)});
            else dev.*a.member = nullptr;
        }
    }
    if (ar && ar->tables_per_instance) {  // sliced per chunk like the models
        fields.push_back({ar->dKinf_drho, nullptr, es * s->pd.nu * s->pd.nx, true, false, (void **)&args.ar.dKinf_drho});
        fields.push_back({ar->dPinf_drho, nullptr, es * s->pd.nx * s->pd.nx, true, false, (void **)&args.ar.dPinf_drho});
    }
    {
        size_t need = (io->xref_per_instance ? 0 : bx) + ((io->Uref && !io->uref_per_instance) ? bu : 0);
        if (need) {
            if (need + 256 > shared_ref.bytes && s->have_last) CUDA_TRY(cudaEventSynchronize(s->ev_last));  // about to reallocate
            if (shared_ref.ensure(need + 256)) return fail(TINYMPC_ERR_CUDA, "shared reference allocation failed");
            char *c = (char *)shared_ref.p;
            if (!io->xref_per_instance) {
                CUDA_TRY(cudaMemcpyAsync(c, io->Xref, bx, cudaMemcpyHostToDevice, s->st_h2d));
                dev.Xref = c;
                c += (bx + 255) / 256 * 256;
            }
            if (io->Uref && !io->uref_per_instance) {
                CUDA_TRY(cudaMemcpyAsync(c, io->Uref, bu, cudaMemcpyHostToDevice, s->st_h2d));
                dev.Uref = c;
            }
        }
    }
    {
        void *const *sp = (void *const *)&io->state;
        void **dp = (void **)&dev.state;
        const int nfields = sizeof(tinympc_state_t) / sizeof(void *);
        for (int i = 0; i < nfields; ++i) {
            if (!sp[i]) continue;
            const bool is_x = (i % 2) == 0;  // x,v,vnew,g,... alternate with u,z,znew,y,...
            fields.push_back({cold ? nullptr : sp[i], sp[i], is_x ? bx : bu, !cold, true, &dp[i]});
        }
    }
    if (io->sol_x) fields.push_back({nullptr, io->sol_x, bx, false, true, (void **)&dev.sol_x});
    if (io->sol_u) fields.push_back({nullptr, io->sol_u, bu, false, true, (void **)&dev.sol_u});
    if (io->u0) fields.push_back({nullptr, io->u0, es * s->pd.nu, false, true, (void **)&dev.u0});
    if (io->iter) fields.push_back({nullptr, io->iter, sizeof(int32_t), false, true, (void **)&dev.iter});
    if (io->solved) fields.push_back({nullptr, io->solved, sizeof(int32_t), false, true, (void **)&dev.solved});
    if (io->residuals) fields.push_back({nullptr, io->residuals, 4 * es, false, true, (void **)&dev.residuals});

    for (Field &f : fields) f.pinned = is_pinned(f.is_out ? f.dst : f.src) && (!f.is_in || !f.src || is_pinned(f.src));
    // the persistent lane-group kernels hold sm_count * per_cta instances at a time: make a chunk a whole number of such waves
    // so that no chunk ends on a mostly empty wave
    const int64_t wave = (int64_t)s->sm_count * plan.per_cta;
    if (B > 16384 && wave > 0 && wave < B) chunk = std::max<int64_t>(1, (chunk + wave / 2) / wave) * wave;
    if (const char *e = std::getenv("TINYMPC_HOST_CHUNK")) {  // experiment knob
        long long v = std::atoll(e);
        if (v > 0) chunk = std::min<int64_t>(B, (v + 31) / 32 * 32);
    }
    const int64_t nchunks = (B + chunk - 1) / chunk;
    const size_t align = 256;
    auto padded = [&](size_t n) { return (n + align - 1) / align * align; };
    size_t dev_bytes = 0, in_bytes = 0, out_bytes = 0;
    for (const Field &f : fields) {
        dev_bytes += padded(f.per_inst * chunk);
        if (f.is_in) in_bytes += padded(f.per_inst * chunk);
        if (f.is_out) out_bytes += padded(f.per_inst * chunk);
    }
    const int used_slots = (int)std::min<int64_t>(SLOTS, nchunks);
    for (int i = 0; i < used_slots; ++i) {
        if (s->dio[i].ensure(dev_bytes) || s->pin_in[i].ensure(in_bytes + align) || s->pin_out[i].ensure(out_bytes + align))
            return fail(TINYMPC_ERR_CUDA, "staging allocation failed");
    }
    int64_t launches = 0;
    struct Pending { int64_t b0, nb; bool active; };
    Pending pend[SLOTS] = {};
    auto drain = [&](int slot) -> int {  // copy the pinned outputs of a finished chunk to the user's buffers
        if (!pend[slot].active) return 0;
        if (cudaEventSynchronize(s->ev_out[slot]) != cudaSuccess) return -1;
        char *po = (char *)s->pin_out[slot].p;
        for (const Field &f : fields) {
            if (!f.is_out) continue;
            if (!f.pinned) std::memcpy((char *)f.dst + f.per_inst * pend[slot].b0, po, f.per_inst * pend[slot].nb);
            po += padded(f.per_inst * chunk);
        }
        pend[slot].active = false;
        return 0;
    };
    for (int64_t c = 0; c < nchunks; ++c) {
        const int slot = (int)(c % SLOTS);
        const int64_t b0 = c * chunk, nb = std::min<int64_t>(chunk, B - b0);
        if (drain(slot)) return fail(TINYMPC_ERR_CUDA, "event sync failed");
        // stage inputs into pinned memory, then one async copy per field
        char *pi = (char *)s->pin_in[slot].p, *pd = (char *)s->dio[slot].p;
        auto da = args;
        tinympc_batch_t &d = da.io;
        d.B = nb;
        // device layout
        {
            char *cur = pd;
            const char *base = (const char *)&args;
            for (const Field &f : fields) {
                size_t off = (const char *)f.dev_slot - base;
                *(void **)((char *)&da + off) = cur;
                cur += padded(f.per_inst * chunk);
            }
        }
        {
            char *cur = pd;
            for (const Field &f : fields) {
                if (f.is_in && f.src) {
                    const char *hsrc = (const char *)f.src + f.per_inst * b0;
                    if (!f.pinned) {
                        std::memcpy(pi, hsrc, f.per_inst * nb);
                        hsrc = pi;
                    }
                    CUDA_TRY(cudaMemcpyAsync(cur, hsrc, f.per_inst * nb, cudaMemcpyHostToDevice, s->st_h2d));
                    pi += padded(f.per_inst * chunk);
                }
                cur += padded(f.per_inst * chunk);
            }
        }
        CUDA_TRY(cudaEventRecord(s->ev_in[slot], s->st_h2d));
        CUDA_TRY(cudaStreamWaitEvent(s->st_k, s->ev_in[slot], 0));
        if (int rc = enqueue(s, &d, s->st_k, false, ar ? &da.ar : nullptr)) return rc;
        launches += s->stats.kernel_launches;
        CUDA_TRY(cudaEventRecord(s->ev_k[slot], s->st_k));
        CUDA_TRY(cudaStreamWaitEvent(s->st_d2h, s->ev_k[slot], 0));
        {
            char *cur = pd, *po = (char *)s->pin_out[slot].p;
            for (const Field &f : fields) {
                if (f.is_out) {
                    char *hdst = f.pinned ? (char *)f.dst + f.per_inst * b0 : po;
                    CUDA_TRY(cudaMemcpyAsync(hdst, cur, f.per_inst * nb, cudaMemcpyDeviceToHost, s->st_d2h));
                    po += padded(f.per_inst * chunk);
                }
                cur += padded(f.per_inst * chunk);
            }
        }
        CUDA_TRY(cudaEventRecord(s->ev_out[slot], s->st_d2h));
        // the next use of this slot's pinned input buffer must wait for its H2D copy: ev_in is synchronised
        // implicitly because drain() waits for ev_out, which is ordered after ev_in.
        pend[slot] = {b0, nb, true};
    }
    for (int i = 0; i < SLOTS; ++i)
        if (drain(i)) return fail(TINYMPC_ERR_CUDA, "event sync failed");
    CUDA_TRY(cudaStreamSynchronize(s->st_h2d));
    s->stats.instances = B;
    s->stats.kernel_launches = launches;
    s->timed = false;
    s->stats.kernel_ms = 0.f;
    return TINYMPC_OK;
}
}  // namespace

int tinympc_b200_solve_host(tinympc_b200_solver_t *s, const tinympc_batch_t *io) {
    if (!s || !io) return fail(TINYMPC_ERR_ARG, "null argument");
    return solve_host_impl(s, io, nullptr);
}

int tinympc_b200_solve_adaptive_host(tinympc_b200_solver_t *s, const tinympc_batch_t *io, const tinympc_adaptive_rho_t *ar) {
    if (!s || !io || !ar) return fail(TINYMPC_ERR_ARG, "null argument");
    return solve_host_impl(s, io, ar);
}

}  // extern "C"
