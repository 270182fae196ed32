// rollout.h — launch arguments of the closed-loop rollout variant of the on-chip kernel (gpi_kernel.cuh), shared with the host
// (capi.cu: tinympc_b200_rollout).
#pragma once
#include <stdint.h>

namespace tmpc {

// A rollout (tinympc_b200_rollout, on-chip kernel only) runs `steps` warm-started MPC steps per instance in one launch.  The
// kernel reads this struct from device memory at KParams::gps_ws (a field only the streamed kernel uses otherwise; adaptive rho,
// the other user of that field, never combines with a rollout).  The reference trajectories travel in KParams::Xref / Uref
// ([B][steps+N-1][nx] / [B][steps+N-2][nu], or one shared trajectory), the carried work->v / work->z in KParams::gpi_vscratch
// (null: they read as zeros at every step).  The GPI_PLANT variant advances a plant of each instance's own from its true
// state and solves from a measurement of it.
template <typename T>
struct GpiRoll {
    int steps;        // T >= 1
    int reset_duals;  // g, y zeroed before every step after the first
    const T *w;       // [B][steps][nx] disturbance added to the plant state after each step, or null
    T *x_traj;        // [B][steps+1][nx] plant states, or null
    T *u_traj;        // [B][steps][nu] applied inputs, or null
    T *res_traj;      // [B][steps][4] residuals, or null
    int32_t *iter_traj, *solved_traj;  // [B][steps], or null
    // GPI_PLANT (launch.h) only, appended so that the fields above keep their offsets.  The plant record of instance b (A | B | f,
    // the first pieces of a model blob: its own plant, one shared plant, or the controller's model) is at plant + b * plant_stride.
    const T *plant;
    int64_t plant_stride;  // 0: one plant for the batch
    const T *noise;        // [B][steps][nx] measurement noise added to the state the solve starts from, or null
    T *xtrue;              // [B][nx] the true plant state while the slot's x0 holds the measured one (noise given)
};
template <typename T, typename KP>
__host__ __device__ inline const GpiRoll<T> *gpi_roll_args(const KP &P) {
    return reinterpret_cast<const GpiRoll<T> *>(P.gps_ws);
}
template <typename T, typename KP>
inline void set_gpi_roll_args(KP &P, const void *args) {
    P.gps_ws = static_cast<T *>(const_cast<void *>(args));
}

}  // namespace tmpc
