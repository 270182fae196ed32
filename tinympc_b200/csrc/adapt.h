// adapt.h — launch arguments of the adaptive-rho variant of the on-chip kernel (gpi_kernel.cuh), shared with the host
// (capi.cu), and the sizes both sides derive from them.
#pragma once
#include <stddef.h>

namespace tmpc {

// Adaptive rho (tinympc_b200_solve_adaptive, on-chip kernel only): the adaptive kernel reads this struct from device memory
// at KParams::gps_ws (a field only the streamed kernel uses otherwise), the tables follow it there.  The per-instance model
// blobs (KParams::models) are in/out: the adapted rho / Kinf / Pinf of an instance are written back into its blob.
template <typename T>
struct GpiAdapt {
    T *models;           // = KParams::models, writable
    const T *dK, *dP;    // dKinf_drho (nu x nx), dPinf_drho (nx x nx), column-major, device memory
    T rho_min, rho_max;  // clip bounds (settings->adaptive_rho_min / max)
    int clip;
    int maskA, maskP;    // column-block width - 1 of Eigen's GEMV for A_matrix / P_matrix (15 or 3), 127: a single block
};
constexpr size_t GPI_ADAPT_HDR = 64;  // bytes reserved for GpiAdapt in front of the tables
// shared memory the adaptive kernel adds behind the state regions for the staged tables
__host__ __device__ constexpr size_t gpi_adapt_bytes(int nx, int nu, size_t es) { return ((size_t)(nu * nx + nx * nx) * es + 15) / 16 * 16; }
// where the arguments travel: KParams::gps_ws (the streamed kernel's workspace pointer, which the on-chip kernel never reads)
template <typename T, typename KP>
__host__ __device__ inline const GpiAdapt<T> *gpi_adapt_args(const KP &P) {
    return reinterpret_cast<const GpiAdapt<T> *>(P.gps_ws);
}
template <typename T, typename KP>
inline void set_gpi_adapt_args(KP &P, const void *args) {  // args: device memory, GpiAdapt<T> then the tables
    P.gps_ws = static_cast<T *>(const_cast<void *>(args));
}
// Eigen's column-block width (GeneralMatrixVector.h:149) for a rows x cols column-major operand, as a mask (block - 1)
inline int gemv_block_mask(long rows, long cols, size_t es) {
    if (cols < 128) return 127;  // one block: every column index is below 128
    return rows * (long)es < 32000 ? 15 : 3;
}

}  // namespace tmpc
