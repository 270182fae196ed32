// kparams_fill.h — LaunchDesc (type-erased, host) -> KParams<T,NX,NU> (the kernels' parameter block), and the layout of the
// thread-per-instance workspace.
#pragma once
#include <cstddef>
#include <cstring>
#include <limits>

#include "common.cuh"
#include "launch.h"
#include "model_blob.h"

namespace tmpc {

// The thread-per-instance workspace (tpi_kernel.cuh) for Bpad instances: structure-of-arrays slabs of 16-byte vectors,
// [k][vec][Bpad], back to back.  Slab i backs the i-th of KParams' w_* pointers: v[0] v[1] z[0] z[1] g y d, then vc zc gc yc,
// vl zl gl yl and vlt zlt glt ylt, each pair of a constraint family present only when the family is enabled.  Returns the
// bytes; with `w` given, also points w[i] at slab i in `base` (null for an absent slab).
constexpr int TPI_SLABS = 19;
inline size_t tpi_workspace(int nx, int nu, int N, int dtype, int64_t Bpad, const Features &ft, char *base = nullptr,
                            void **w = nullptr) {
    const int E = dtype == TINYMPC_F64 ? 2 : 4;
    const size_t szx = (size_t)N * ((nx + E - 1) / E) * 16 * Bpad, szu = (size_t)(N - 1) * ((nu + E - 1) / E) * 16 * Bpad;
    const bool state[TPI_SLABS] = {1, 1, 0, 0, 1, 0, 0, 1, 0, 1, 0, 1, 0, 1, 0, 1, 0, 1, 0};
    const bool on[TPI_SLABS] = {1, 1, 1, 1, 1, 1, 1,
                                (bool)ft.soc_x, (bool)ft.soc_u, (bool)ft.soc_x, (bool)ft.soc_u,
                                (bool)ft.lin_x, (bool)ft.lin_u, (bool)ft.lin_x, (bool)ft.lin_u,
                                (bool)ft.tvl_x, (bool)ft.tvl_u, (bool)ft.tvl_x, (bool)ft.tvl_u};
    size_t bytes = 0;
    for (int i = 0; i < TPI_SLABS; ++i) {
        if (w) w[i] = on[i] ? base + bytes : nullptr;
        if (on[i]) bytes += state[i] ? szx : szu;
    }
    return bytes;
}

template <typename T, int NX, int NU>
inline void fill_params(KParams<T, NX, NU> &P, const LaunchDesc &d) {
    using KP = KParams<T, NX, NU>;
    std::memset(&P, 0, sizeof(P));
    const ProblemDesc &pd = *d.pd;
    const tinympc_settings_t &st = d.st;
    const Features &ft = d.ft;
    const ModelBlob mb = model_blob(NX, NU);
    const T *blob = (const T *)pd.h_blob.data();
    std::memcpy(P.A, blob + mb.A, sizeof(P.A));
    std::memcpy(P.Bm, blob + mb.B, sizeof(P.Bm));
    std::memcpy(P.f, blob + mb.f, sizeof(P.f));
    std::memcpy(P.Qd, blob + mb.Qd, sizeof(P.Qd));
    std::memcpy(P.Rd, blob + mb.Rd, sizeof(P.Rd));
    std::memcpy(P.Kinf, blob + mb.Kinf, sizeof(P.Kinf));
    std::memcpy(P.Pinf, blob + mb.Pinf, sizeof(P.Pinf));
    std::memcpy(P.Quu, blob + mb.Quu, sizeof(P.Quu));
    std::memcpy(P.AmBKt, blob + mb.AmBKt, sizeof(P.AmBKt));
    std::memcpy(P.APf, blob + mb.APf, sizeof(P.APf));
    std::memcpy(P.BPf, blob + mb.BPf, sizeof(P.BPf));
    P.rho = (T)pd.rho;
    P.pri_tol = (T)st.abs_pri_tol;
    P.dua_tol = (T)st.abs_dua_tol;
    P.N = pd.N;
    P.max_iter = st.max_iter;
    P.check_termination = st.check_termination;
    P.en_state_bound = st.en_state_bound;
    P.en_input_bound = st.en_input_bound;
    P.soc_x = ft.soc_x; P.soc_u = ft.soc_u; P.ncx = st.en_state_soc ? pd.ncx : 0; P.ncu = st.en_input_soc ? pd.ncu : 0;
    P.lin_x = ft.lin_x; P.lin_u = ft.lin_u; P.nlx = pd.nlx; P.nlu = pd.nlu;
    P.tvl_x = ft.tvl_x; P.tvl_u = ft.tvl_u; P.ntvx = pd.ntvx; P.ntvu = pd.ntvu;
    for (int c = 0; c < MAX_CONES; ++c) {
        P.cone_x_start[c] = pd.cone_x_start[c];
        P.cone_u_start[c] = pd.cone_u_start[c];
        P.cone_x_mu[c] = (T)pd.cone_x_mu[c];
        P.cone_u_mu[c] = (T)pd.cone_u_mu[c];
    }
    const tinympc_batch_t &io = d.io;
    P.B = io.B;
    P.Bpad = d.Bpad;
    P.cold = io.cold_start;
    P.bounds_tv = pd.bounds_tv;
    {
        const T inf = std::numeric_limits<T>::infinity();
        auto col0 = [&](const std::vector<char> &h, int i, bool en, T dflt) { return en && !h.empty() ? ((const T *)h.data())[i] : dflt; };
        for (int i = 0; i < NX; ++i) {
            P.xlo[i] = col0(pd.h_xlo, i, st.en_state_bound, -inf);
            P.xhi[i] = col0(pd.h_xhi, i, st.en_state_bound, inf);
        }
        for (int j = 0; j < NU; ++j) {
            P.ulo[j] = col0(pd.h_ulo, j, st.en_input_bound, -inf);
            P.uhi[j] = col0(pd.h_uhi, j, st.en_input_bound, inf);
        }
    }
    P.Pinf_g = (const T *)pd.blob + mb.Pinf;
    P.xref_pi = io.xref_per_instance;
    P.uref_pi = io.uref_per_instance;
    P.x0 = (const T *)io.x0; P.Xref = (const T *)io.Xref; P.Uref = (const T *)io.Uref;
    P.x_min = (const T *)pd.x_min; P.x_max = (const T *)pd.x_max; P.u_min = (const T *)pd.u_min; P.u_max = (const T *)pd.u_max;
    if (d.pi.read[KIND_BOUNDS]) {  // per-instance bounds replace the problem's; the kernels derive an instance's offset from NX, NU, N and bounds_tv
        P.x_min = (const T *)io.x_min; P.x_max = (const T *)io.x_max; P.u_min = (const T *)io.u_min; P.u_max = (const T *)io.u_max;
        P.bounds_tv = d.pi.read[KIND_BOUNDS] == 2;
    }
    P.Alin_x = (const T *)pd.Alin_x; P.blin_x = (const T *)pd.blin_x; P.Alin_u = (const T *)pd.Alin_u; P.blin_u = (const T *)pd.blin_u;
    P.tv_Alin_x = (const T *)pd.tv_Alin_x; P.tv_blin_x = (const T *)pd.tv_blin_x;
    P.tv_Alin_u = (const T *)pd.tv_Alin_u; P.tv_blin_u = (const T *)pd.tv_blin_u;
    const tinympc_state_t &s = io.state;
    P.s_x = (T *)s.x; P.s_u = (T *)s.u; P.s_v = (T *)s.v; P.s_z = (T *)s.z;
    P.s_vnew = (T *)s.vnew; P.s_znew = (T *)s.znew; P.s_g = (T *)s.g; P.s_y = (T *)s.y;
    P.s_vcnew = (T *)s.vcnew; P.s_zcnew = (T *)s.zcnew; P.s_gc = (T *)s.gc; P.s_yc = (T *)s.yc;
    P.s_vlnew = (T *)s.vlnew; P.s_zlnew = (T *)s.zlnew; P.s_gl = (T *)s.gl; P.s_yl = (T *)s.yl;
    P.s_vlnew_tv = (T *)s.vlnew_tv; P.s_zlnew_tv = (T *)s.zlnew_tv; P.s_gl_tv = (T *)s.gl_tv; P.s_yl_tv = (T *)s.yl_tv;
    P.sol_x = (T *)io.sol_x; P.sol_u = (T *)io.sol_u;
    P.iter = io.iter; P.solved = io.solved; P.residuals = (T *)io.residuals;
    P.u0 = (T *)io.u0;
    P.models = (const T *)io.models;
    P.gpi_vscratch = (T *)d.gpi_vscratch;
    if (d.tpi_ws) {
        static_assert(offsetof(KP, w_ylt) == offsetof(KP, w_v) + (TPI_SLABS - 1) * sizeof(void *), "w_* are the slab pointers in order");
        void *w[TPI_SLABS];
        tpi_workspace(NX, NU, pd.N, pd.dtype, d.Bpad, ft, (char *)d.tpi_ws, w);
        std::memcpy((char *)&P + offsetof(KP, w_v), w, sizeof(w));
    }
    if (d.pi.read[KIND_CONES]) {  // per-instance cone coefficients ride in two workspace pointers the streamed kernel never reads (gps_kernel.cuh: GPS_CONES)
        P.w_vc = const_cast<void *>(d.io.cone_x_mu);
        P.w_zc = const_cast<void *>(d.io.cone_u_mu);
    }
    if (d.pi.read[KIND_PLANES]) {  // per-instance static hyperplanes replace the problem's; the kernel adds the slot's instance offset
        P.Alin_x = (const T *)io.Alin_x; P.blin_x = (const T *)io.blin_x; P.Alin_u = (const T *)io.Alin_u; P.blin_u = (const T *)io.blin_u;
    }
}

}  // namespace tmpc
