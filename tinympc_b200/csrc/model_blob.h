// model_blob.h — the one definition of the cache / model blob layout (host and device).
//
// A cache blob is the problem's model and cached Riccati terms packed back to back, each column-major in the native dtype:
//   A | B | f | Qd | Rd | Kinf | Pinf | Quu_inv | AmBKt | APf | BPf
// A model blob (tinympc_batch_t.models, one per instance) is a cache blob with rho appended.  The handle keeps one cache
// blob on the device (the lane-group kernels stage it into shared memory with one TMA bulk copy); the batch precompute
// (host and device) writes model blobs.
#pragma once
#include <stddef.h>

#if defined(__CUDACC__)
#define TM_BLOB_HD __host__ __device__
#else
#define TM_BLOB_HD
#endif

namespace tmpc {

// element offsets of the pieces, and element counts (I = the index type of the caller's arithmetic)
template <typename I>
struct ModelBlobT {
    I A, B, f, Qd, Rd, Kinf, Pinf, Quu, AmBKt, APf, BPf;
    I cache;  // elements of a cache blob (A .. BPf)
    I rho;    // offset of rho in a model blob
    I model;  // elements of a model blob (cache blob + rho)
};
using ModelBlob = ModelBlobT<int>;

template <typename I = int>
TM_BLOB_HD constexpr ModelBlobT<I> model_blob(I nx, I nu) {
    ModelBlobT<I> m{};
    m.A = 0, m.B = m.A + nx * nx, m.f = m.B + nx * nu, m.Qd = m.f + nx, m.Rd = m.Qd + nx, m.Kinf = m.Rd + nu;
    m.Pinf = m.Kinf + nu * nx, m.Quu = m.Pinf + nx * nx, m.AmBKt = m.Quu + nu * nu, m.APf = m.AmBKt + nx * nx, m.BPf = m.APf + nx;
    m.cache = m.BPf + nu, m.rho = m.cache, m.model = m.cache + 1;
    return m;
}

// bytes of the staged cache blob: one bulk copy moves a multiple of 16 bytes
TM_BLOB_HD constexpr size_t cache_stage_bytes(int nx, int nu, size_t es) {
    return ((size_t)model_blob(nx, nu).cache * es + 15) / 16 * 16;
}

// shared memory the lane-group planners set aside for the staged blob: one nx-vector more than the cache, rounded to 16
// bytes.  The kernels use only cache_stage_bytes of it; the launch plans were measured with this reserve.
TM_BLOB_HD constexpr size_t cache_reserve_bytes(int nx, int nu, size_t es) {
    return ((size_t)(model_blob(nx, nu).cache + nx) * es + 15) / 16 * 16;
}

}  // namespace tmpc

#undef TM_BLOB_HD
