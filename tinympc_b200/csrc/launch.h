// launch.h — type-erased launch descriptor between the C-ABI layer (capi.cu) and the per-(nx,nu)
// kernel translation units (kernels_inst.cu compiled once per supported dimension pair).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/tinympc_b200.h"

namespace tmpc {

struct LaunchDesc {
    int dtype;   // TINYMPC_F32 / F64
    int fast;    // TINYMPC_MODE_FAST ?
    int family;  // TINYMPC_KERNEL_TPI / GPI / GPS (resolved, never AUTO)
    int ext;     // any of soc / linear / tv-linear enabled

    // host copies of the model + cache in the native dtype (column-major)
    const void *A, *Bm, *f, *Qd, *Rd, *Kinf, *Pinf, *Quu, *AmBKt, *APf, *BPf;
    double rho, pri_tol, dua_tol;
    int N, max_iter, check_termination;
    int en_state_bound, en_input_bound;
    int soc_x, soc_u, ncx, ncu;
    int lin_x, lin_u, nlx, nlu;
    int tvl_x, tvl_u, ntvx, ntvu;
    int cone_x_start[4], cone_u_start[4];
    double cone_x_mu[4], cone_u_mu[4];  // already rounded to the native dtype

    // device pointers
    const void *x_min, *x_max, *u_min, *u_max;
    const void *Alin_x, *blin_x, *Alin_u, *blin_u, *tv_Alin_x, *tv_blin_x, *tv_Alin_u, *tv_blin_u;
    tinympc_batch_t io;  // device pointers
    int64_t Bpad;
    void *w_v[2], *w_z[2], *w_g, *w_y, *w_d;
    void *w_vc, *w_zc, *w_gc, *w_yc, *w_vl, *w_zl, *w_gl, *w_yl, *w_vlt, *w_zlt, *w_glt, *w_ylt;
    const void *gmat;  // device blob: A,B,f,Qd,Rd,Kinf,Pinf,Quu,AmBKt,APf,BPf packed (native dtype)
    int bounds_tv;
    int bounds_zero_free;  // no element of the box bounds is +-0 (lets STRICT kernels clamp with min / max instructions)
    const void *h_xlo, *h_xhi, *h_ulo, *h_uhi;  // host copies of column 0 of the bounds (native dtype), may be null
    void *work_queue;  // GPI: device int64 counter (zeroed by the caller)
    void *gpi_vscratch;  // GPI: scratch for work->v / work->z persistence (allocated by the caller when state.v/z given)
    void *gps_ws;        // GPS: streamed state records of the resident slots (allocated by the caller, see out_ws_need)
    size_t gps_ws_bytes;

    // adaptive rho (tinympc_b200_solve_adaptive): io.models is then the in/out blob array; adapt_args = device copy of
    // GpiAdapt<T> (adapt.h) followed by dKinf_drho and dPinf_drho
    int adapt;
    const void *adapt_args;

    cudaStream_t stream;
    int sm_count;
    int max_smem_optin;

    // filled by the launcher
    int out_threads, out_ctas, out_smem, out_lanes_per_instance, out_instances_per_cta;
    size_t out_ws_need;  // GPS: workspace bytes this launch needs (set when the launcher returns TM_ERR_WORKSPACE)
};

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

// per-(nx,nu) entry: returns 0 on success, TINYMPC_ERR_UNSUPPORTED when (dtype,family,...) is not compiled
typedef int (*launch_fn)(LaunchDesc *);

// launch plan of the on-chip lane-group kernel (gpi_kernel.cuh: gpi_plan) for one (dtype, N); L == 0: not available
struct GpiPlan {
    int L = 0, warps = 0;              // lanes per instance, warps per CTA
    size_t smem = 0;                   // dynamic shared memory per CTA (bytes)
    int instances_per_cta = 0;         // instances resident per CTA (warps * 32 / L)
    size_t vscratch_per_instance = 0;  // bytes of work->v / work->z scratch per instance (launch.h: gpi_vscratch)
};

struct DimEntry {
    int nx, nu;
    launch_fn launch;
    // GPI capability query: the on-chip kernel's launch plan for (dtype, N)
    GpiPlan (*gpi_plan)(int dtype, int N, int max_smem_optin);
    // batched cache precompute on the device (precompute_kernel.cuh): device pointers, one model blob per instance
    int (*precompute_batch)(int dtype, int64_t B, const void *A, const void *Bm, const void *f, const void *Qdiag, const void *Rdiag,
                            const void *rho, void *models_out, int32_t *sweeps_out, int sm_count, cudaStream_t stream);
    // streamed lane-group kernel (gps_kernel.cuh): lanes per instance (bits 0-7) | instances per lane group << 8; 0 = shape not available
    int (*gps_lanes)(int dtype);
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
