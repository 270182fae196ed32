// gpi_kernel.cuh — lane-group-per-instance (GPI) batched ADMM solve with the whole per-instance state
// resident on chip.  This is the kernel BASELINE.json's north_star describes.
//
//   * L lanes (4, 8 or 16) own one MPC instance, 32/L instances per warp; lane l owns the state rows
//     [l*RX, (l+1)*RX) and the input rows [l*RU, (l+1)*RU)  (RX = ceil(nx/L), RU = ceil(nu/L)) of every vector.
//   * the rows of Kinf / Quu_inv / AmBKt / A / B that a lane needs are loaded ONCE into registers (staged
//     through shared memory by a TMA bulk copy, cp.async.bulk), the p / x recursions run in registers, each
//     mat-vec is RX (or RU) independent ascending-k dot products per lane (bit-identical to the pinned
//     oracle in STRICT mode), and the freshly computed vector is all-gathered inside the lane group through
//     a small shared-memory buffer (STS + 16-byte broadcast LDS);
//   * the N-indexed state lives in shared memory for the whole solve: the primal pack (vnew rows, znew rows) and the
//     dual pack (g rows, y rows) as one 16-byte vector per lane and knot point each, and d; only the final
//     trajectories / residuals are written back;
//   * fp64: only the rows of the running sweep are in registers (re-read from the resident blob at every sweep start), so
//     that narrower lane groups fit (gpi_per_sweep_rows);
//   * the kernel is persistent: one CTA per SM; every lane group ("slot") pulls its next instance from a
//     global atomic counter as soon as its current one terminates (per-instance termination, admm.cpp:310-328).
// Reference semantics: tiny_solve -> solve (admm.cpp:331-455); per-iteration order as in SURVEY A.2.
// Scope: box constraints (admm.cpp:85-98).  Cones / hyperplanes run on the streamed lane-group kernel (gps_kernel.cuh).
#pragma once
#include <algorithm>
#include <cstdlib>

#include "adapt.h"
#include "common.cuh"
#include "lanegroup.cuh"
#include "model_blob.h"

namespace tmpc {

template <int NX, int NU, int L, int ES>
struct GpiCfg : LaneGeom<NX, NU, L, ES> {
    using G = LaneGeom<NX, NU, L, ES>;
    static constexpr int RX = G::RX, RU = G::RU, IPW = G::IPW, W = G::W, NXP = G::NXP, NUP = G::NUP;
    static constexpr int PV = RX + RU;      // values a lane owns per knot point (state rows, then input rows)
    static constexpr int PVP = (PV + W - 1) / W * W;
    static constexpr int NPV = PVP / W;     // vectors per pack
    static constexpr int GBUF1 = IPW * (NXP > NUP ? NXP : NUP);  // the gather buffer
    // registers needed for the per-lane matrix rows (in elements of T)
    static constexpr int MAT_REGS = RX * (2 * NX + 2 * NU + 3) + RU * (2 * NX + NU + 2);
    // shared-memory elements per warp for horizon N: primal pack + dual pack per (k, lane), d, gather scratch
    __host__ __device__ static constexpr size_t warp_elems(int N) {
        return (size_t)N * 32 * PVP * 2 + (size_t)(N - 1) * RU * 32 + GBUF1;
    }
    // per-sweep register needs (elements): backward AmBKt / B^T rows, Kinf^T, Quu_inv, APf, BPf, Qd, Rd; forward A / Kinf rows, B, f
    static constexpr int BWD_REGS = (RX + RU) * NX + RX * NU + RU * NU + 2 * RX + 2 * RU;
    static constexpr int FWD_REGS = (RX + RU) * NX + RX * NU + RX;
    static constexpr int SWEEP_REGS = BWD_REGS > FWD_REGS ? BWD_REGS : FWD_REGS;
};

// fp64: only the rows of the RUNNING sweep are in registers (re-read from the staged blob in shared memory - or from the
// instance's own blob in a heterogeneous batch - at every sweep start), which halves the register footprint of the matrices
// and lets fp64 problems use narrower lane groups (nx = 12: L = 8 instead of 16, twice the instances per warp)
template <typename T>
__host__ __device__ constexpr bool gpi_per_sweep_rows() {
    return sizeof(T) == 8;
}
template <typename T, int NX, int NU, int L>
__host__ __device__ constexpr bool gpi_feasible() {
    // keep the matrix rows + working set under the 255-register ceiling
    using Cfg = GpiCfg<NX, NU, L, (int)sizeof(T)>;
    if (gpi_per_sweep_rows<T>()) return Cfg::SWEEP_REGS * 2 <= 112;
    return Cfg::MAT_REGS * (int)(sizeof(T) / 4) <= 150;
}

constexpr int GPI_MAX_WARPS = 8;

// Adaptive rho (tinympc_b200_solve_adaptive): the kernel is instantiated with GPI_ADAPT added to its lane count; it then
// runs heterogeneous STRICT batches and reads its GpiAdapt arguments (adapt.h: gpi_adapt_args).  (A separate template
// parameter or kernel argument would rename the existing kernels, a shared __device__ body or a larger KParams changes their
// machine code.)
constexpr int GPI_ADAPT = 64;

// MM (STRICT only): the box clamp as min / max instructions.  Identical to Eigen's compare-select form for every input
// (NaN included: both return the bound) except when a bound is a signed zero - the host sets MM only when no bound is +-0.
template <typename T, int NX, int NU, int LA, bool FAST, bool HET, bool MM = false>
__global__ void __launch_bounds__(GPI_MAX_WARPS * 32, 1)
    gpi_solve_kernel(const __grid_constant__ KParams<T, NX, NU> P, const T *__restrict__ gmat, unsigned long long *queue) {
    constexpr bool ADAPT = LA >= GPI_ADAPT;  // adaptive rho
    constexpr int L = LA % GPI_ADAPT;
    static_assert(LA < 2 * GPI_ADAPT && L > 0, "lane count: 4, 8 or 16, plus GPI_ADAPT for the adaptive variant");
    static_assert(!ADAPT || (HET && !FAST && !MM), "adaptive rho runs on heterogeneous STRICT batches");
    GpiAdapt<T> AP{};
    if constexpr (ADAPT) AP = *gpi_adapt_args<T>(P);
    using Cfg = GpiCfg<NX, NU, L, (int)sizeof(T)>;
    constexpr int RX = Cfg::RX, RU = Cfg::RU, IPW = Cfg::IPW, W = Cfg::W, PVP = Cfg::PVP, NPV = Cfg::NPV;
    constexpr int NXP = Cfg::NXP, NUP = Cfg::NUP;
    constexpr bool PS = gpi_per_sweep_rows<T>();  // matrix rows re-read at every sweep start (fp64)
    constexpr bool EXACT = (RX * L == NX) && (RU * L == NU);  // no padding rows: predicates vanish
    constexpr unsigned ES = (unsigned)sizeof(T);
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int N = P.N;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int l = lane % L;     // lane inside the instance group
    const int slot = lane / L;  // which of the warp's instances
    // HET = heterogeneous batch (tinympc_batch_t.models): every instance brings its own model / cache blob and rho;
    // the homogeneous kernel keeps rho a launch constant and its matrix rows immutable registers.
    T rho_m = P.rho;
    auto rho_ = [&]() -> T {
        if constexpr (HET) return rho_m;
        else return P.rho;
    };

    // ---- stage the cache blob into shared memory with one TMA bulk copy per CTA, then pull this lane's rows into
    // registers.  The staging area aliases the first warp's state region and is dead before the solve starts.
    constexpr ModelBlob MB = model_blob(NX, NU);
    constexpr unsigned BLOB_BYTES = (unsigned)cache_stage_bytes(NX, NU, sizeof(T));
    T *stage = reinterpret_cast<T *>(smem_raw);
    __shared__ __align__(8) unsigned long long mbar;
    stage_blob(stage, gmat, BLOB_BYTES, &mbar);

    // per-lane matrix rows (registers)
    // stage-1 rows (dot with the gathered nx-vector): backward = [AmBKt rows ; B^T rows], forward = [A rows ; Kinf rows]
    T mS1b[RX + RU][NX], mS1f[RX + RU][NX];
    T mKt[RX][NU], mB[RX][NU], vQd[RX], vAPf[RX], vf[RX];
    T mQuu[RU][NU], vRd[RU], vBPf[RU];
    bool xv[RX], uv[RU];  // row validity (padding rows compute zeros)
#pragma unroll
    for (int a = 0; a < RX; ++a) xv[a] = EXACT || (l * RX + a < NX);
#pragma unroll
    for (int b = 0; b < RU; ++b) uv[b] = EXACT || (l * RU + b < NU);
    // `src` = a cache blob in the layout above (the staged shared-memory copy, or one instance's blob in global memory).
    // Backward-sweep rows (AmBKt, B^T, Kinf^T, Quu_inv, APf, BPf and the cost weights Qd, Rd) and forward-sweep rows (A, Kinf,
    // B, f) load separately: fp64 re-reads the rows of a sweep when it starts (PS), everything else loads both once.
    auto load_bwd_rows = [&](const T *src) {
        auto rd = [src](int e) {
            if constexpr (ADAPT) return __ldcg(src + e);
            else return src[e];
        };
#pragma unroll
        for (int a = 0; a < RX; ++a) {
            const int ii = xv[a] ? l * RX + a : 0;
            blob_row<NX, NX>(rd, MB.AmBKt, ii, xv[a], mS1b[a]);
            blob_col<NU, NU>(rd, MB.Kinf, ii, xv[a], mKt[a]);
            vQd[a] = xv[a] ? rd(MB.Qd + ii) : T(0);
            vAPf[a] = xv[a] ? rd(MB.APf + ii) : T(0);
        }
#pragma unroll
        for (int b = 0; b < RU; ++b) {
            const int jj = uv[b] ? l * RU + b : 0;
            blob_col<NX, NX>(rd, MB.B, jj, uv[b], mS1b[RX + b]);
            blob_row<NU, NU>(rd, MB.Quu, jj, uv[b], mQuu[b]);
            vRd[b] = uv[b] ? rd(MB.Rd + jj) : T(0);
            vBPf[b] = uv[b] ? rd(MB.BPf + jj) : T(0);
        }
    };
    auto load_fwd_rows = [&](const T *src) {
        auto rd = [src](int e) {
            if constexpr (ADAPT) return __ldcg(src + e);
            else return src[e];
        };
#pragma unroll
        for (int a = 0; a < RX; ++a) {
            const int ii = xv[a] ? l * RX + a : 0;
            blob_row<NX, NX>(rd, MB.A, ii, xv[a], mS1f[a]);
            blob_row<NX, NU>(rd, MB.B, ii, xv[a], mB[a]);
            vf[a] = xv[a] ? rd(MB.f + ii) : T(0);
        }
#pragma unroll
        for (int b = 0; b < RU; ++b) {
            const int jj = uv[b] ? l * RU + b : 0;
            blob_row<NU, NX>(rd, MB.Kinf, jj, uv[b], mS1f[RX + b]);
        }
    };
    // both sets at once (everything but fp64), row by row with the backward and forward matrices interleaved: the load
    // order the kernel was tuned with (load_bwd_rows + load_fwd_rows compiles to a different schedule)
    auto load_rows = [&](const T *src) {
        auto rd = [src](int e) {
            if constexpr (ADAPT) return __ldcg(src + e);
            else return src[e];
        };
#pragma unroll
        for (int a = 0; a < RX; ++a) {
            const int ii = xv[a] ? l * RX + a : 0;
#pragma unroll
            for (int m = 0; m < NX; ++m) {
                mS1b[a][m] = xv[a] ? rd(MB.AmBKt + ii + NX * m) : T(0);
                mS1f[a][m] = xv[a] ? rd(MB.A + ii + NX * m) : T(0);
            }
#pragma unroll
            for (int j = 0; j < NU; ++j) {
                mKt[a][j] = xv[a] ? rd(MB.Kinf + j + NU * ii) : T(0);  // Kinf^T(i,j) = Kinf(j,i)
                mB[a][j] = xv[a] ? rd(MB.B + ii + NX * j) : T(0);
            }
            vQd[a] = xv[a] ? rd(MB.Qd + ii) : T(0);
            vAPf[a] = xv[a] ? rd(MB.APf + ii) : T(0);
            vf[a] = xv[a] ? rd(MB.f + ii) : T(0);
        }
#pragma unroll
        for (int b = 0; b < RU; ++b) {
            const int jj = uv[b] ? l * RU + b : 0;
#pragma unroll
            for (int m = 0; m < NX; ++m) {
                mS1b[RX + b][m] = uv[b] ? rd(MB.B + m + NX * jj) : T(0);  // B^T(j,m) = B(m,j)
                mS1f[RX + b][m] = uv[b] ? rd(MB.Kinf + jj + NU * m) : T(0);
            }
            blob_row<NU, NU>(rd, MB.Quu, jj, uv[b], mQuu[b]);
            vRd[b] = uv[b] ? rd(MB.Rd + jj) : T(0);
            vBPf[b] = uv[b] ? rd(MB.BPf + jj) : T(0);
        }
    };
    // where this lane's rows come from at a sweep start (PS): the staged blob, or its slot's own blob (heterogeneous batch)
    // ADAPT reads rows with ld.global.cg (the blobs are rewritten during the launch), so its rows come from a global blob
    // (the first instance's) even for a slot that never gets an instance, never from the staged shared-memory copy
    const T *rowsrc = stage;
    if constexpr (ADAPT) rowsrc = P.models;
    if constexpr (!PS) load_rows(rowsrc);
    __syncthreads();  // staging area is reused as state below

    // ---- shared-memory state of this warp ----
    //   PA[k][lane][PVP] : primal pack  (vnew rows of this lane, then znew rows)      16-byte vectors,
    //   PB[k][lane][PVP] : dual pack    (g rows, then y rows)                          conflict free
    //   D [k][b][lane]   : d
    //   GB[...]          : gather scratch (one vector of one instance per row)
    const int warp_elems = (int)Cfg::warp_elems(N);
    // fp64 (PS): the staged blob stays in shared memory for the whole kernel, the state regions start behind it
    constexpr size_t BLOB_KEEP = PS ? (size_t)BLOB_BYTES : 0;
    T *wbase = reinterpret_cast<T *>(smem_raw + BLOB_KEEP) + (size_t)warp * warp_elems;
    T *gPA = wbase, *gPB = gPA + N * 32 * PVP, *gD = gPB + N * 32 * PVP, *gGB = gD + (N - 1) * RU * 32;
    const unsigned aPA = (unsigned)__cvta_generic_to_shared(gPA) + (unsigned)(lane * PVP) * ES;
    const unsigned aPB = (unsigned)__cvta_generic_to_shared(gPB) + (unsigned)(lane * PVP) * ES;
    const unsigned aD = (unsigned)__cvta_generic_to_shared(gD) + (unsigned)lane * ES;
    const unsigned aGB = (unsigned)__cvta_generic_to_shared(gGB);
    // ADAPT: dKinf_drho / dPinf_drho staged behind the state regions of all warps (and behind the dead blob staging area)
    const T *sdK = nullptr, *sdP = nullptr;
    if constexpr (ADAPT) {
        size_t off = BLOB_KEEP + (size_t)(blockDim.x >> 5) * warp_elems * ES;
        off = ((off > BLOB_BYTES ? off : (size_t)BLOB_BYTES) + 15) / 16 * 16;
        T *t = reinterpret_cast<T *>(smem_raw + off);
        for (int e = threadIdx.x; e < NU * NX + NX * NX; e += blockDim.x) t[e] = AP.dK[e];  // dP follows dK
        __syncthreads();
        sdK = t;
        sdP = t + NU * NX;
    }
    constexpr unsigned KSTR = 32u * PVP * ES;  // bytes per knot point in PA / PB
    constexpr unsigned DSTR = (unsigned)RU * 32u * ES;
    auto load_pack = [&](unsigned base, int k, T (&v)[PVP]) {
#pragma unroll
        for (int c = 0; c < NPV; ++c) {
            T t[W];
            ldsv(base + (unsigned)k * KSTR + (unsigned)(c * W) * ES, t);
#pragma unroll
            for (int e = 0; e < W; ++e) v[c * W + e] = t[e];
        }
    };
    auto store_pack = [&](unsigned base, int k, const T (&v)[PVP]) {
#pragma unroll
        for (int c = 0; c < NPV; ++c) {
            T t[W];
#pragma unroll
            for (int e = 0; e < W; ++e) t[e] = v[c * W + e];
            stsv(base + (unsigned)k * KSTR + (unsigned)(c * W) * ES, t);
        }
    };
    // dual pack / d accessors
    auto load_pb = [&](int k, T (&v)[PVP]) { load_pack(aPB, k, v); };
    auto store_pb = [&](int k, const T (&v)[PVP]) { store_pack(aPB, k, v); };
    auto load_d = [&](int k, T (&d)[RU]) {
#pragma unroll
        for (int b = 0; b < RU; ++b) d[b] = lds(aD + (unsigned)k * DSTR + (unsigned)(b * 32) * ES, T());
    };
    auto store_d = [&](int k, const T (&d)[RU], const bool live) {
#pragma unroll
        for (int b = 0; b < RU; ++b)
            if (live && uv[b]) sts(aD + (unsigned)k * DSTR + (unsigned)(b * 32) * ES, d[b]);
    };
    // all-gather inside the lane group through shared memory: every lane stores its R values, then reads the
    // whole vector with 16-byte broadcast loads (absolute row order -> ascending-k dot products as in the oracle).
    // One buffer: the leading barrier protects the previous gather's readers before it is overwritten.
    auto gather_x = [&](const T (&own)[RX], T (&full)[NX]) {
        __syncwarp();
#pragma unroll
        for (int a = 0; a < RX; ++a) sts(aGB + (unsigned)(slot * NXP + l * RX + a) * ES, own[a]);
        __syncwarp();
#pragma unroll
        for (int c = 0; c < NXP / W; ++c) {
            T t[W];
            ldsv(aGB + (unsigned)(slot * NXP + c * W) * ES, t);
#pragma unroll
            for (int e = 0; e < W; ++e)
                if (c * W + e < NX) full[c * W + e] = t[e];
        }
    };
    auto gather_u = [&](const T (&own)[RU], T (&full)[NU]) {
        __syncwarp();
#pragma unroll
        for (int b = 0; b < RU; ++b) sts(aGB + (unsigned)(slot * NUP + l * RU + b) * ES, own[b]);
        __syncwarp();
#pragma unroll
        for (int c = 0; c < NUP / W; ++c) {
            T t[W];
            ldsv(aGB + (unsigned)(slot * NUP + c * W) * ES, t);
#pragma unroll
            for (int e = 0; e < W; ++e)
                if (c * W + e < NU) full[c * W + e] = t[e];
        }
    };

    const bool cold = P.cold != 0;
    const bool tvb = P.bounds_tv != 0;
    const bool enx = P.en_state_bound != 0, enu = P.en_input_bound != 0;
    auto xok = [&](int a) { return xv[a]; };
    auto uok = [&](int b) { return uv[b]; };
    T loX[RX], hiX[RX], loU[RU], hiU[RU];  // bounds of this lane's rows (reloaded per k only if time-varying)
    box_bounds<true>(P, l, 0, true, enx, enu, xok, uok, loX, hiX, loU, hiU);
    const T kInf = (T)INFINITY;
    const bool keep_v = (P.s_v != nullptr) || (P.s_z != nullptr);
    // where element (k, row i) of instance-slot s lives inside a pack region
    auto idx_x = [&](int s, int k, int i) { return (k * 32 + s * L + i / RX) * PVP + (i % RX); };
    auto idx_u = [&](int s, int k, int j) { return (k * 32 + s * L + j / RU) * PVP + RX + (j % RU); };

    // ---- per-slot bookkeeping (identical in the L lanes of a slot) ----
    int64_t inst = -1;    // instance held by this lane's slot
    bool busy = false;    // the slot holds an unfinished instance
    bool want = true;     // the slot should try to fetch an instance
    int it = 0, solved = 0;
    // ADAPT: an adaptation of this slot's Kinf / Pinf waiting to be applied (at the next iteration start or at retire: the
    // retire-time replay of work->x / work->u must use the Kinf of the last forward pass); the two deltas of
    // update_matrices_with_derivatives (rho_benchmark.cpp:240, admm.cpp:421)
    bool pend = false;
    T adelta = T(0), adelta2 = T(0);
    T res_px = T(0), res_dx = T(0), res_pu = T(0), res_du = T(0);
    T x0o[RX], pterm[RX];
#pragma unroll
    for (int a = 0; a < RX; ++a) x0o[a] = pterm[a] = T(0);
    const T *xrefp = P.Xref + l * RX;
    const bool has_uref = P.Uref != nullptr;  // warp-uniform: keeps the loops free of divergence bookkeeping
    const T *urefp = has_uref ? P.Uref + l * RU : P.Xref;
    int64_t offx = 0, offu = 0;

    // linear cost of column k for this lane's rows (update_linear_cost, admm.cpp:266-280):
    //   q = -(xref*Qd) - rho*(vnew - g),  r = -(uref*Rd) - rho*(znew - y)
    // split in two so that the global (reference) and shared (state) loads of column k-1 are issued at the top of
    // backward step k and consumed only at its end, behind the dot-product chains: with one warp per scheduler a
    // load consumed right after issue is fully exposed (per-instance references come from L2/HBM)
    auto cost_load = [&](int k, const T *xp, const T *up, T (&xr)[RX], T (&ur)[RU], T (&pa)[PVP], T (&pb)[PVP]) {
#pragma unroll
        for (int a = 0; a < RX; ++a) xr[a] = xv[a] ? __ldg(xp + a) : T(0);
#pragma unroll
        for (int b = 0; b < RU; ++b) ur[b] = (has_uref && uv[b]) ? __ldg(up + b) : T(0);
        load_pack(aPA, k, pa);
        load_pb(k, pb);
    };
    auto cost_eval = [&](const T (&xr)[RX], const T (&ur)[RU], const T (&pa)[PVP], const T (&pb)[PVP], T (&q)[RX], T (&r)[RU]) {
        if constexpr (FAST) {
#pragma unroll
            for (int a = 0; a < RX; ++a) q[a] = nmac<FAST>(-(xr[a] * vQd[a]), rho_(), pa[a] - pb[a]);
#pragma unroll
            for (int b = 0; b < RU; ++b) r[b] = nmac<FAST>(-(ur[b] * vRd[b]), rho_(), pa[RX + b] - pb[RX + b]);
        } else {
            // the same operations on the whole pack (state rows, input rows, padding): (-(ref*W)) - rho*(pa - pb), with the
            // subtractions issued as packed pairs (fp32)
            T m[PVP], df[PVP], t[PVP], o[PVP];
#pragma unroll
            for (int e = 0; e < PVP; ++e) m[e] = T(0);
#pragma unroll
            for (int a = 0; a < RX; ++a) m[a] = -(xr[a] * vQd[a]);
#pragma unroll
            for (int b = 0; b < RU; ++b) m[RX + b] = -(ur[b] * vRd[b]);
            vsub<T, PVP>(pa, pb, df);
#pragma unroll
            for (int e = 0; e < PVP; ++e) t[e] = rho_() * df[e];
            vsub<T, PVP>(m, t, o);
#pragma unroll
            for (int a = 0; a < RX; ++a) q[a] = o[a];
#pragma unroll
            for (int b = 0; b < RU; ++b) r[b] = o[RX + b];
        }
    };

    // forward pass fused with slack / dual update / residuals.  SLOW = some slot is in the first iteration of a
    // warm start (work->v / work->z come from the caller) or work->v / work->z are being persisted.
    auto forward = [&](auto tag, const bool vin, T &rpx, T &rdx, T &rpu, T &rdu) {
        constexpr bool SLOW = decltype(tag)::value;
        if constexpr (PS) load_fwd_rows(rowsrc);
        T xo[RX], Xf[NX];
#pragma unroll
        for (int a = 0; a < RX; ++a) xo[a] = x0o[a];
        gather_x(xo, Xf);
        // one column: slack + dual update of this lane's rows, residual maxima; HASU = the column has inputs
        auto column = [&](int k, const bool HASU, const T (&u)[RU], const T (&vprev)[PVP], const T (&pb)[PVP]) {  // always inlined with a literal HASU
            T pa[PVP], na[PVP], nb[PVP];
            load_pack(aPA, k, pa);
#pragma unroll
            for (int e = 0; e < PVP; ++e) {
                na[e] = pa[e];
                nb[e] = pb[e];
            }
            if (tvb) box_bounds<false>(P, l, k, HASU, enx, enu, xok, uok, loX, hiX, loU, hiU);
            if constexpr (FAST) {
    #pragma unroll
                for (int a = 0; a < RX; ++a) {  // vnew = clamp(x + g), g += x - vnew
                    T vo = pa[a];
                    if constexpr (SLOW) {
                        if (vin) vo = vprev[a];
                    }
                    const T v = clamp_box<FAST>(xo[a] + pb[a], loX[a], hiX[a]);
                    na[a] = v;
                    nb[a] = (pb[a] + xo[a]) - v;
                    rpx = absmax(rpx, xo[a] - v);
                    rdx = absmax(rdx, vo - v);
                }
                if (HASU) {
    #pragma unroll
                    for (int b = 0; b < RU; ++b) {
                        T zo = pa[RX + b];
                        if constexpr (SLOW) {
                            if (vin) zo = vprev[RX + b];
                        }
                        const T z = clamp_box<FAST>(u[b] + pb[RX + b], loU[b], hiU[b]);
                        na[RX + b] = z;
                        nb[RX + b] = (pb[RX + b] + u[b]) - z;
                        rpu = absmax(rpu, u[b] - z);
                        rdu = absmax(rdu, zo - z);
                    }
                }
            } else {
                // the same update on the whole pack (state rows, input rows, padding) with the additions / subtractions
                // issued as packed pairs (fp32): vnew = clamp(x + g), g' = (g + x) - vnew, residual differences
                T X[PVP], lo[PVP], hi[PVP], vo[PVP], sum[PVP], v[PVP], dg[PVP], dx[PVP], dv[PVP];
#pragma unroll
                for (int e = 0; e < PVP; ++e) {
                    X[e] = T(0);
                    lo[e] = -kInf;
                    hi[e] = kInf;
                    vo[e] = pa[e];
                    if constexpr (SLOW) {
                        if (vin) vo[e] = vprev[e];
                    }
                }
#pragma unroll
                for (int a = 0; a < RX; ++a) {
                    X[a] = xo[a];
                    lo[a] = loX[a];
                    hi[a] = hiX[a];
                }
#pragma unroll
                for (int b = 0; b < RU; ++b) {
                    X[RX + b] = u[b];
                    lo[RX + b] = loU[b];
                    hi[RX + b] = hiU[b];
                }
                vadd<T, PVP>(X, pb, sum);
#pragma unroll
                for (int e = 0; e < PVP; ++e) v[e] = (e < RX + RU) ? clamp_box<FAST || MM>(sum[e], lo[e], hi[e]) : sum[e];
                vsub<T, PVP>(sum, v, dg);
                vsub<T, PVP>(X, v, dx);
                vsub<T, PVP>(vo, v, dv);
#pragma unroll
                for (int a = 0; a < RX; ++a) {
                    na[a] = v[a];
                    nb[a] = dg[a];
                    rpx = absmax(rpx, dx[a]);
                    rdx = absmax(rdx, dv[a]);
                }
                if (HASU) {
#pragma unroll
                    for (int b = 0; b < RU; ++b) {
                        na[RX + b] = v[RX + b];
                        nb[RX + b] = dg[RX + b];
                        rpu = absmax(rpu, dx[RX + b]);
                        rdu = absmax(rdu, dv[RX + b]);
                    }
                }
            }
            if (busy) {
                store_pack(aPA, k, na);
                store_pb(k, nb);
                if constexpr (SLOW) {
                    // work->v / work->z of this iteration = the primal pack as it was before this column's update
                    // (kept in pack layout in global scratch: one 16-byte store; transposed out only if the solve converges)
                    if (P.gpi_vscratch && !vin) {
                        T *dst = P.gpi_vscratch + ((inst * N + k) * L + l) * PVP;
#pragma unroll
                        for (int c = 0; c < NPV; ++c) {
                            using V16 = typename Vec16<T>::type;
                            V16 v16;
                            T *e16 = reinterpret_cast<T *>(&v16);
#pragma unroll
                            for (int e = 0; e < W; ++e) e16[e] = pa[c * W + e];
                            reinterpret_cast<V16 *>(dst)[c] = v16;
                        }
                    }
                }
            }
        };
        auto load_vprev = [&](int k, T (&vp)[PVP]) {  // caller's work->v / work->z column (first warm iteration only)
#pragma unroll
            for (int e = 0; e < PVP; ++e) vp[e] = T(0);
            if constexpr (SLOW) {
                if (vin && P.gpi_vscratch) {
                    const T *src = P.gpi_vscratch + ((inst * N + k) * L + l) * PVP;
#pragma unroll
                    for (int c = 0; c < NPV; ++c) {
                        using V16 = typename Vec16<T>::type;
                        const V16 v16 = reinterpret_cast<const V16 *>(src)[c];
                        const T *e16 = reinterpret_cast<const T *>(&v16);
#pragma unroll
                        for (int e = 0; e < W; ++e) vp[c * W + e] = e16[e];
                    }
                }
            }
        };
        for (int k = 0; k < N - 1; ++k) {
            T u[RU], Uf[NU], t1[RX + RU], bu[RX], vprev[PVP], pbk[PVP], dk[RU];
            load_vprev(k, vprev);
            load_pb(k, pbk);
            load_d(k, dk);
            dots<FAST>(mS1f, Xf, t1);  // [A x_k ; Kinf x_k]
#pragma unroll
            for (int b = 0; b < RU; ++b) u[b] = (-t1[RX + b]) - dk[b];  // u_k = -(Kinf x_k) - d_k
            gather_u(u, Uf);
            column(k, true, u, vprev, pbk);
            dots<FAST>(mB, Uf, bu);
            {   // x_{k+1} = (A x_k + B u_k) + f
                T ax[RX], tx[RX];
#pragma unroll
                for (int a = 0; a < RX; ++a) ax[a] = t1[a];
                vadd<T, RX>(ax, bu, tx);
                vadd<T, RX>(tx, vf, xo);
            }
            gather_x(xo, Xf);
        }
        {
            T udummy[RU], vprev[PVP], pbk[PVP];
#pragma unroll
            for (int b = 0; b < RU; ++b) udummy[b] = T(0);
            load_vprev(N - 1, vprev);
            load_pb(N - 1, pbk);
            column(N - 1, false, udummy, vprev, pbk);
        }
    };

    // ---- cooperative (all 32 lanes) load of instance `ib` into slot `s`: zero the slot's shared-memory state,
    // read a warm start, and set up the slot's lanes (x0 rows, terminal-cost constant, reference pointers) ----
    auto load_slot = [&](int s, int64_t ib) {
        // the slot owns L consecutive lanes (L*PVP contiguous elements = VPK 16-byte vectors) of every [k][lane][PVP]
        // row of PA and PB; d is always written before it is read and needs no initialisation
        {
            constexpr int VPK = (L * PVP * (int)sizeof(T)) / 16;  // vectors per knot point of one slot
            float4 *a4 = reinterpret_cast<float4 *>(gPA), *b4 = reinterpret_cast<float4 *>(gPB);
            constexpr int ROW4 = (32 * PVP * (int)sizeof(T)) / 16;  // vectors per knot point of the whole warp
            const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int e = lane; e < N * VPK; e += 32) {
                const int k = e / VPK, w = e - k * VPK;
                a4[k * ROW4 + s * VPK + w] = z4;
                b4[k * ROW4 + s * VPK + w] = z4;
            }
        }
        __syncwarp();
        if (!cold) {
            // warm start: the instance's vnew/g/znew/y blocks are contiguous in global memory; loads are batched four
            // deep before the dependent shared-memory stores (one warp cannot hide a load-use pair per iteration)
            const int64_t ox = ib * (int64_t)N * NX, ou = ib * (int64_t)(N - 1) * NU;
            constexpr int UNR = 4;
            for (int e0 = lane; e0 < N * NX; e0 += 32 * UNR) {
                T va[UNR], vb[UNR];
#pragma unroll
                for (int t = 0; t < UNR; ++t) {
                    const int e = e0 + 32 * t;
                    const bool ok = e < N * NX;
                    va[t] = (ok && P.s_vnew) ? P.s_vnew[ox + e] : T(0);
                    vb[t] = (ok && P.s_g) ? P.s_g[ox + e] : T(0);
                }
#pragma unroll
                for (int t = 0; t < UNR; ++t) {
                    const int e = e0 + 32 * t;
                    if (e < N * NX) {
                        const int k = e / NX, i = e - k * NX;
                        const int w = idx_x(s, k, i);
                        gPA[w] = va[t];
                        gPB[w] = vb[t];
                    }
                }
            }
            for (int e0 = lane; e0 < (N - 1) * NU; e0 += 32 * UNR) {
                T va[UNR], vb[UNR];
#pragma unroll
                for (int t = 0; t < UNR; ++t) {
                    const int e = e0 + 32 * t;
                    const bool ok = e < (N - 1) * NU;
                    va[t] = (ok && P.s_znew) ? P.s_znew[ou + e] : T(0);
                    vb[t] = (ok && P.s_y) ? P.s_y[ou + e] : T(0);
                }
#pragma unroll
                for (int t = 0; t < UNR; ++t) {
                    const int e = e0 + 32 * t;
                    if (e < (N - 1) * NU) {
                        const int k = e / NU, j = e - k * NU;
                        const int w = idx_u(s, k, j);
                        gPA[w] = va[t];
                        gPB[w] = vb[t];
                    }
                }
            }
            // work->v / work->z of the caller (only read by the first iteration's dual residual): staged into the global
            // scratch in pack layout, so that the first forward pass fetches them with one 16-byte load per knot point
            if (P.gpi_vscratch) {
                T *sc = P.gpi_vscratch + ib * (int64_t)N * L * PVP;
                for (int e0 = lane; e0 < N * NX; e0 += 32 * UNR) {
                    T va[UNR];
#pragma unroll
                    for (int t = 0; t < UNR; ++t) {
                        const int e = e0 + 32 * t;
                        va[t] = (e < N * NX && P.s_v) ? P.s_v[ox + e] : T(0);
                    }
#pragma unroll
                    for (int t = 0; t < UNR; ++t) {
                        const int e = e0 + 32 * t;
                        if (e < N * NX) {
                            const int k = e / NX, i = e - k * NX;
                            sc[(k * L + i / RX) * PVP + (i % RX)] = va[t];
                        }
                    }
                }
                for (int e0 = lane; e0 < (N - 1) * NU; e0 += 32 * UNR) {
                    T va[UNR];
#pragma unroll
                    for (int t = 0; t < UNR; ++t) {
                        const int e = e0 + 32 * t;
                        va[t] = (e < (N - 1) * NU && P.s_z) ? P.s_z[ou + e] : T(0);
                    }
#pragma unroll
                    for (int t = 0; t < UNR; ++t) {
                        const int e = e0 + 32 * t;
                        if (e < (N - 1) * NU) {
                            const int k = e / NU, j = e - k * NU;
                            sc[(k * L + j / RU) * PVP + RX + (j % RU)] = va[t];
                        }
                    }
                }
            }
            __syncwarp();
        }
        // L2 prefetch, one "generation" of tickets ahead: tickets are handed out in order, so instance ib + PF will be
        // loaded by some warp shortly; touching its per-instance inputs now turns that warp's latency-exposed loads
        // (one warp per scheduler cannot hide them) into L2 hits.  The current instance's references are touched too.
        {
            constexpr int64_t PF = 1024;
            auto touch = [&](const T *base, int64_t elems) {
                const char *pb_ = reinterpret_cast<const char *>(base);
                for (int64_t o = (int64_t)lane * 128; o < elems * (int64_t)sizeof(T); o += 32 * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pb_ + o));
            };
            const int64_t nxN = (int64_t)N * NX, nuN = (int64_t)(N - 1) * NU;
            if (P.xref_pi) touch(P.Xref + ib * nxN, nxN);
            if (has_uref && P.uref_pi) touch(P.Uref + ib * nuN, nuN);
            const int64_t ip = ib + PF;
            if (ip < P.B) {
                if (P.xref_pi) touch(P.Xref + ip * nxN, nxN);
                if (has_uref && P.uref_pi) touch(P.Uref + ip * nuN, nuN);
                if (!cold) {
                    if (P.s_vnew) touch(P.s_vnew + ip * nxN, nxN);
                    if (P.s_g) touch(P.s_g + ip * nxN, nxN);
                    if (P.s_znew) touch(P.s_znew + ip * nuN, nuN);
                    if (P.s_y) touch(P.s_y + ip * nuN, nuN);
                    if (P.s_v && P.gpi_vscratch) touch(P.s_v + ip * nxN, nxN);
                    if (P.s_z && P.gpi_vscratch) touch(P.s_z + ip * nuN, nuN);
                }
            }
        }
        if (slot == s) {
            inst = ib;
            busy = true;
            pend = false;
            it = 0;
            solved = 0;
            res_px = res_dx = res_pu = res_du = T(0);
            offx = ib * (int64_t)N * NX;
            offu = ib * (int64_t)(N - 1) * NU;
            xrefp = P.Xref + (P.xref_pi ? offx : 0) + l * RX;
            urefp = has_uref ? P.Uref + (P.uref_pi ? offu : 0) + l * RU : P.Xref;
            // heterogeneous batch: this instance has its own model / cache blob (same layout as the shared one, rho appended)
            const T *pinf = P.Pinf_g;
            if constexpr (HET) {
                const T *mb = P.models + ib * (int64_t)MB.model;
                if constexpr (PS) rowsrc = mb;
                else load_rows(mb);
                rho_m = mb[MB.rho];
                pinf = mb + MB.Pinf;
            }
            // x0 (own rows) and the iteration-invariant part of the terminal cost
            T xr[NX];
            const T *xl = xrefp - l * RX + (int64_t)(N - 1) * NX;
#pragma unroll
            for (int m = 0; m < NX; ++m) xr[m] = __ldg(xl + m);
#pragma unroll
            for (int a = 0; a < RX; ++a) {
                const int i = l * RX + a, ii = xv[a] ? i : 0;
                x0o[a] = xv[a] ? __ldg(P.x0 + ib * NX + ii) : T(0);
                const T pt = terminal_cost<FAST, NX>([&](int m) { return xr[m]; }, pinf, ii);
                pterm[a] = xv[a] ? pt : T(0);
            }
        }
        __syncwarp();
    };

    // ---- ADAPT: adaptive rho (admm.cpp:397-423 with a value-initialised RhoAdapter) ----
    // Kinf += delta*dK; Kinf += delta2*dK (and Pinf) in this slot's blob for a pending slot, elements split over its L lanes
    auto adapt_blob = [&](const bool on) {
        T *mb = AP.models + (inst < 0 ? 0 : inst) * (int64_t)MB.model;
        for (int e0 = 0; e0 < NU * NX + NX * NX; e0 += L) {
            const int e = e0 + l;
            if (on && e < NU * NX + NX * NX) {
                const int o = e < NU * NX ? MB.Kinf + e : MB.Pinf + (e - NU * NX);
                const T dv = e < NU * NX ? sdK[e] : sdP[e - NU * NX];
                const T v1 = __ldcg(mb + o) + adelta * dv;
                mb[o] = v1 + adelta2 * dv;
            }
        }
    };
    // apply the pending adaptation before an iteration: blob, fp32 register copies of Kinf (mKt and the forward rows, same
    // arithmetic as the blob), terminal-cost constant from the new Pinf
    auto adapt_apply = [&]() {
        adapt_blob(pend);
        __syncwarp();
        if (pend) {
            if constexpr (!PS) {
#pragma unroll
                for (int a = 0; a < RX; ++a) {
                    const int ii = xv[a] ? l * RX + a : 0;
#pragma unroll
                    for (int j = 0; j < NU; ++j) {
                        const T dv = sdK[j + NU * ii];
                        mKt[a][j] = xv[a] ? (mKt[a][j] + adelta * dv) + adelta2 * dv : T(0);
                    }
                }
#pragma unroll
                for (int b = 0; b < RU; ++b) {
                    const int jj = uv[b] ? l * RU + b : 0;
#pragma unroll
                    for (int m = 0; m < NX; ++m) {
                        const T dv = sdK[jj + NU * m];
                        mS1f[RX + b][m] = uv[b] ? (mS1f[RX + b][m] + adelta * dv) + adelta2 * dv : T(0);
                    }
                }
            }
            const T *pinf = AP.models + inst * (int64_t)MB.model + MB.Pinf;
            const T *xl = xrefp - l * RX + (int64_t)(N - 1) * NX;
#pragma unroll
            for (int a = 0; a < RX; ++a) {
                const int ii = xv[a] ? l * RX + a : 0;
                T sacc = __ldg(xl) * __ldcg(pinf + NX * ii);
                for (int m = 1; m < NX; ++m) sacc = mac<false>(sacc, __ldg(xl + m), __ldcg(pinf + m + NX * ii));
                pterm[a] = xv[a] ? -sacc : T(0);
            }
            pend = false;
        }
    };
    // residuals of format_matrices / compute_residuals (rho_benchmark.cpp:47-188) for the slots with `ad`, then predict_rho:
    // the rollout of this iteration is replayed from x0 and d (bit-identical to the forward pass), vnew / znew / g / y are the
    // updated packs.  A x and P x follow Eigen's column-major GEMV (sums of column-block partials), A^T y its row-major one.
    auto adapt_sweep = [&](const bool ad) {
        if constexpr (PS) load_fwd_rows(rowsrc);
        const T *mbp = AP.models + (inst < 0 ? 0 : inst) * (int64_t)MB.model;
        const int S = NX + NU, mA = AP.maskA, mP = AP.maskP;
        T ax_m = T(0), z_m = T(0), rp_m = T(0), px_m = T(0), aty_m = T(0), q_m = T(0), rd_m = T(0);
        auto amax = [](T &m, T v) {
            const T a = fabs(v);
            m = (m < a) ? a : m;
        };
        T xo[RX], Xf[NX];
#pragma unroll
        for (int a = 0; a < RX; ++a) xo[a] = x0o[a];
        gather_x(xo, Xf);
        for (int k = 0; k < N; ++k) {
            const bool more = k < N - 1;  // uniform
            T pa[PVP], pb[PVP], pa1[PVP], Gf[NX], u[RU], Uf[NU], t1[RX + RU], bu[RX], xn[RX];
            load_pack(aPA, k, pa);
            load_pb(k, pb);
#pragma unroll
            for (int b = 0; b < RU; ++b) u[b] = T(0);
#pragma unroll
            for (int a = 0; a < RX; ++a) xn[a] = T(0);
#pragma unroll
            for (int m = 0; m < NX; ++m) Gf[m] = T(0);
#pragma unroll
            for (int e = 0; e < PVP; ++e) pa1[e] = T(0);
            if (more) {
                T dk[RU];
                load_d(k, dk);
                dots<false>(mS1f, Xf, t1);
#pragma unroll
                for (int b = 0; b < RU; ++b) u[b] = (-t1[RX + b]) - dk[b];
                gather_u(u, Uf);
                dots<false>(mB, Uf, bu);
#pragma unroll
                for (int a = 0; a < RX; ++a) xn[a] = (t1[a] + bu[a]) + vf[a];
                T pb1[PVP], gown[RX];
                load_pb(k + 1, pb1);
                load_pack(aPA, k + 1, pa1);
#pragma unroll
                for (int a = 0; a < RX; ++a) gown[a] = pb1[a];
                gather_x(gown, Gf);
            }
            const int c0 = k * S;
#pragma unroll
            for (int a = 0; a < RX; ++a) {
                if (!xv[a]) continue;
                const int i = l * RX + a;
                const T q = __ldg(mbp + MB.Qd + i) * xo[a];
                T px = q;
                if (!more) {  // P x of the terminal block: Pinf row i against x_{N-1}
                    T res = T(0), c = T(0);
                    int blk = c0 & ~mP;
#pragma unroll
                    for (int j = 0; j < NX; ++j) {
                        const int bj = (c0 + j) & ~mP;
                        if (bj != blk) { res = res + c; c = T(0); blk = bj; }
                        c = (__ldcg(mbp + MB.Pinf + i + NX * j) * Xf[j]) + c;
                    }
                    px = res + c;
                }
                T aty = T(0);
                if (k >= 1) aty = (T(-1) * pb[a]) + aty;
                if (more) {
#pragma unroll
                    for (int r = 0; r < NX; ++r) aty = (__ldg(mbp + MB.A + r + NX * i) * Gf[r]) + aty;
                }
                amax(px_m, px);
                amax(q_m, q);
                amax(aty_m, aty);
                amax(rd_m, (px + q) + aty);
                if (more) {  // dynamics row i of step k: A(i,:) x_k + B(i,:) u_k - x_{k+1}(i) against vnew_{k+1}(i)
                    T res = T(0), c = T(0);
                    int blk = c0 & ~mA;
#pragma unroll
                    for (int j = 0; j < NX; ++j) {
                        const int bj = (c0 + j) & ~mA;
                        if (bj != blk) { res = res + c; c = T(0); blk = bj; }
                        c = (mS1f[a][j] * Xf[j]) + c;
                    }
#pragma unroll
                    for (int j = 0; j < NU; ++j) {
                        const int bj = (c0 + NX + j) & ~mA;
                        if (bj != blk) { res = res + c; c = T(0); blk = bj; }
                        c = (mB[a][j] * Uf[j]) + c;
                    }
                    {
                        const int bj = (c0 + S + i) & ~mA;
                        if (bj != blk) { res = res + c; c = T(0); blk = bj; }
                        c = (T(-1) * xn[a]) + c;
                    }
                    const T axv = res + c, z = pa1[a];
                    amax(ax_m, axv);
                    amax(z_m, z);
                    amax(rp_m, axv - z);
                }
            }
            if (more) {
#pragma unroll
                for (int b = 0; b < RU; ++b) {
                    if (!uv[b]) continue;
                    const int j = l * RU + b;
                    const T rj = __ldg(mbp + MB.Rd + j);
                    const T px = rj * u[b], q = rj * u[b];
                    T aty = (T(1) * pb[RX + b]) + T(0);
#pragma unroll
                    for (int r = 0; r < NX; ++r) aty = (__ldg(mbp + MB.B + r + NX * j) * Gf[r]) + aty;
                    amax(px_m, px);
                    amax(q_m, q);
                    amax(aty_m, aty);
                    amax(rd_m, (px + q) + aty);
                    const T z = pa[RX + b];
                    amax(ax_m, u[b]);
                    amax(z_m, z);
                    amax(rp_m, u[b] - z);
                }
#pragma unroll
                for (int a = 0; a < RX; ++a) xo[a] = xn[a];
                gather_x(xo, Xf);
            }
        }
        rp_m = group_max<T, L>(rp_m);
        rd_m = group_max<T, L>(rd_m);
        ax_m = group_max<T, L>(ax_m);
        z_m = group_max<T, L>(z_m);
        px_m = group_max<T, L>(px_m);
        aty_m = group_max<T, L>(aty_m);
        q_m = group_max<T, L>(q_m);
        if (ad) {  // predict_rho (rho_benchmark.cpp:190-213), then update_matrices_with_derivatives twice (deferred)
            const T pn = (ax_m < z_m) ? z_m : ax_m;
            const T dm = (px_m < aty_m) ? aty_m : px_m;
            const T dn = (dm < q_m) ? q_m : dm;
            const T eps = (T)1e-10;
            const T np_ = rp_m / (pn + eps);
            const T nd_ = rd_m / (dn + eps);
            const T ratio = np_ / (nd_ + eps);
            T nr = rho_m * sqrt(ratio);
            if (AP.clip) {
                nr = (nr < AP.rho_min) ? AP.rho_min : nr;
                nr = (AP.rho_max < nr) ? AP.rho_max : nr;
            }
            adelta = nr - rho_m;
            adelta2 = nr - nr;
            rho_m = nr;
            pend = true;
        }
    };

    // ---- cooperative write-back of slot `s` (instance `ib`): solution, info, optional state and rollout ----
    auto store_slot = [&](int s, int64_t ib) {
        const int s_solved = __shfl_sync(0xffffffffu, solved, s * L);
        const int s_it = __shfl_sync(0xffffffffu, it, s * L);
        if (slot == s && l == 0) {
            if (P.iter) P.iter[ib] = it;
            if (P.solved) P.solved[ib] = solved;
            if (P.residuals) {
                T *r = P.residuals + 4 * ib;
                r[0] = res_px; r[1] = res_dx; r[2] = res_pu; r[3] = res_du;
            }
        }
        __syncwarp();
        const int64_t ox = ib * (int64_t)N * NX, ou = ib * (int64_t)(N - 1) * NU;
        // solution->x = vnew, solution->u = znew; work->vnew/znew/g/y; coalesced transposing copy
        for (int e = lane; e < N * NX; e += 32) {
            const int k = e / NX, i = e - k * NX;
            const int w = idx_x(s, k, i);
            const T v = gPA[w];
            if (P.sol_x) P.sol_x[ox + e] = v;
            if (P.s_vnew) P.s_vnew[ox + e] = v;
            if (P.s_g) P.s_g[ox + e] = gPB[w];
            // work->v: previous vnew if the solve converged (staged in the scratch during the last forward pass; unchanged
            // if that was the first iteration of a warm start), else = vnew (admm.cpp:445); untouched when no iteration
            // ran on a warm start
            if (P.s_v && !s_solved && s_it > 0) P.s_v[ox + e] = v;
            else if (P.s_v && s_solved && !(s_it == 1 && !cold)) P.s_v[ox + e] = P.gpi_vscratch[((ib * N + k) * L + i / RX) * PVP + (i % RX)];
            else if (P.s_v && cold && s_it == 0) P.s_v[ox + e] = T(0);
        }
        for (int e = lane; e < (N - 1) * NU; e += 32) {
            const int k = e / NU, j = e - k * NU;
            const int w = idx_u(s, k, j);
            const T z = gPA[w];
            if (P.sol_u) P.sol_u[ou + e] = z;
            if (P.s_znew) P.s_znew[ou + e] = z;
            if (P.s_y) P.s_y[ou + e] = gPB[w];
            if (P.s_z && !s_solved && s_it > 0) P.s_z[ou + e] = z;
            else if (P.s_z && s_solved && !(s_it == 1 && !cold)) P.s_z[ou + e] = P.gpi_vscratch[((ib * N + k) * L + j / RU) * PVP + RX + (j % RU)];
            else if (P.s_z && cold && s_it == 0) P.s_z[ou + e] = T(0);
        }
        // work->u.col(0): one rollout step from d_0 (every lane computes, the lanes of slot s store)
        if constexpr (PS) {
            if (P.u0 || P.s_x || P.s_u) load_fwd_rows(rowsrc);
        }
        if (P.u0) {
            __syncwarp();
            T xo0[RX], Xf0[NX], t10[RX + RU];
#pragma unroll
            for (int a = 0; a < RX; ++a) xo0[a] = x0o[a];
            gather_x(xo0, Xf0);
            T d0[RU];
            load_d(0, d0);
            dots<FAST>(mS1f, Xf0, t10);
#pragma unroll
            for (int b = 0; b < RU; ++b) {
                T u0v = (-t10[RX + b]) - d0[b];
                if (s_it == 0) u0v = (!cold && P.s_u) ? P.s_u[ou + l * RU + b] : T(0);
                if (slot == s && uv[b]) P.u0[ib * NU + l * RU + b] = u0v;
            }
            __syncwarp();
        }
        // work->x / work->u: replay the last rollout from d and x0 (bit-identical to the last forward pass), staging it
        // in this slot's (now dead) primal pack so that the write-back is coalesced too.  Every lane executes the
        // arithmetic (the gathers are warp-wide); only the lanes of slot s store.
        if (P.s_x || P.s_u) {
            __syncwarp();
            T xo[RX], Xf[NX];
#pragma unroll
            for (int a = 0; a < RX; ++a) xo[a] = x0o[a];
            gather_x(xo, Xf);
            for (int k = 0; k < N; ++k) {
                T na[PVP];
#pragma unroll
                for (int e = 0; e < PVP; ++e) na[e] = T(0);
#pragma unroll
                for (int a = 0; a < RX; ++a) na[a] = xo[a];
                if (k < N - 1) {
                    T u[RU], Uf[NU], t1[RX + RU], bu[RX], dk[RU];
                    load_d(k, dk);
                    dots<FAST>(mS1f, Xf, t1);
#pragma unroll
                    for (int b = 0; b < RU; ++b) {
                        u[b] = (-t1[RX + b]) - dk[b];
                        na[RX + b] = u[b];
                    }
                    gather_u(u, Uf);
                    dots<FAST>(mB, Uf, bu);
#pragma unroll
                    for (int a = 0; a < RX; ++a) xo[a] = (t1[a] + bu[a]) + vf[a];
                }
                if (slot == s) store_pack(aPA, k, na);
                if (k < N - 1) gather_x(xo, Xf);
            }
            __syncwarp();
            if (P.s_x)
                for (int e = lane; e < N * NX; e += 32) {
                    const int k = e / NX, i = e - k * NX;
                    if (s_it > 0 || k == 0) P.s_x[ox + e] = gPA[idx_x(s, k, i)];
                    else if (cold) P.s_x[ox + e] = T(0);
                }
            if (P.s_u)
                for (int e = lane; e < (N - 1) * NU; e += 32) {
                    const int k = e / NU, j = e - k * NU;
                    if (s_it > 0) P.s_u[ou + e] = gPA[idx_u(s, k, j)];
                    else if (cold) P.s_u[ou + e] = T(0);
                }
        }
        if constexpr (ADAPT) {  // the adapted cache persists in the instance's blob (after the replay above)
            adapt_blob(slot == s && pend);
            if (slot == s && l == 0) AP.models[ib * (int64_t)MB.model + MB.rho] = rho_m;
            if (slot == s) pend = false;
        }
        __syncwarp();
    };

    // ---- persistent loop: every slot runs its own instance; a slot that terminates (converged or max_iter) is
    // written back and refilled from the global queue immediately, so no lane group waits for the slowest
    // instance of its warp (termination is per instance, admm.cpp:310-328) ----
    for (;;) {
        // 1. retire finished slots / fill empty ones
        const bool fin = busy && (solved || it >= P.max_iter);
        const unsigned todo = __ballot_sync(0xffffffffu, (fin || (!busy && want)) && l == 0);
        for (unsigned m = todo; m; m &= m - 1) {
            const int s = (__ffs(m) - 1) / L;
            const int64_t ib_old = __shfl_sync(0xffffffffu, inst, s * L);
            const int was_busy = __shfl_sync(0xffffffffu, (int)busy, s * L);
            // the queue ticket is requested before the write-back of the finished instance so that the atomic's
            // latency hides behind it.  (Never hold a ticket in advance: a ticket prefetched by every warp keeps instances
            // hostage until a slot frees up, which can cost a whole extra wave per launch.)
            unsigned long long nxt = 0;
            if (lane == 0) nxt = atomicAdd(queue, 1ULL);
            if (was_busy) store_slot(s, ib_old);
            nxt = __shfl_sync(0xffffffffu, nxt, 0);
            if ((int64_t)nxt < P.B) {
                load_slot(s, (int64_t)nxt);
            } else if (slot == s) {
                busy = false;
                want = false;
            }
        }
        if (!__any_sync(0xffffffffu, busy)) break;
        if (__any_sync(0xffffffffu, busy && it >= P.max_iter)) continue;  // max_iter <= 0: retire without iterating
        __syncwarp();

        // 2. ADMM iterations for every busy slot until some slot terminates.  This inner loop has warp-uniform
        // control flow only, so the compiler keeps the warp converged (no divergence bookkeeping around the
        // shared-memory gathers).
        do {
        if constexpr (ADAPT) {
            if (__any_sync(0xffffffffu, pend)) adapt_apply();
        }
        // ---- terminal cost + backward pass (update_linear_cost fused, software-pipelined by one column) ----
        if constexpr (PS) load_bwd_rows(rowsrc);
        T po[RX], Pf[NX];
        {
            T pa[PVP], pb[PVP];
            load_pack(aPA, N - 1, pa);
            load_pb(N - 1, pb);
#pragma unroll
            for (int a = 0; a < RX; ++a) po[a] = nmac<FAST>(pterm[a], rho_(), pa[a] - pb[a]);
        }
        gather_x(po, Pf);
        T q[RX], r[RU], Rf[NU];
        const T *xp = xrefp + (int64_t)(N - 2) * NX;
        const T *up = urefp + (has_uref ? (int64_t)(N - 2) * NU : 0);
        {
            T xr[RX], ur[RU], pa[PVP], pb[PVP];
            cost_load(N - 2, xp, up, xr, ur, pa, pb);
            cost_eval(xr, ur, pa, pb, q, r);
        }
        gather_u(r, Rf);
        // one backward step; MORE = another column follows (its cost inputs are fetched now and consumed at the end of
        // the step).  The last step (k = 0) is peeled so that the loop body carries no k > 0 predicates.
        auto bwd_step = [&](int k, const bool MORE) {  // always inlined with a literal MORE
            T xr_n[RX], ur_n[RU], pa_n[PVP], pb_n[PVP];
            if (MORE) {
                xp -= NX;
                if (has_uref) up -= NU;
                cost_load(k - 1, xp, up, xr_n, ur_n, pa_n, pb_n);
            }
            // d_k = Quu_inv ((B^T p_{k+1} + r_k) + BPf)
            T s_[RU], Sf[NU], acc1[RX + RU], kr[RX], dq[RU];
            dots<FAST>(mS1b, Pf, acc1);  // [AmBKt p_{k+1} ; B^T p_{k+1}]
#pragma unroll
            for (int b = 0; b < RU; ++b) s_[b] = (acc1[RX + b] + r[b]) + vBPf[b];
            gather_u(s_, Sf);
            // p_k = ((q_k + AmBKt p_{k+1}) - Kinf^T r_k) + APf
            dots<FAST>(mKt, Rf, kr);
            {
                T a1[RX], t1_[RX], t2_[RX];
#pragma unroll
                for (int a = 0; a < RX; ++a) a1[a] = acc1[a];
                vadd<T, RX>(q, a1, t1_);
                vsub<T, RX>(t1_, kr, t2_);
                vadd<T, RX>(t2_, vAPf, po);
            }
            if (MORE) gather_x(po, Pf);  // p_0 itself is never used (the forward pass starts from x_0)
            dots<FAST>(mQuu, Sf, dq);
            store_d(k, dq, busy);
            if (MORE) {
                cost_eval(xr_n, ur_n, pa_n, pb_n, q, r);
                gather_u(r, Rf);
            }
        };
        for (int k = N - 2; k >= 1; --k) bwd_step(k, true);
        bwd_step(0, false);
        __syncwarp();

        T rpx = T(0), rdx = T(0), rpu = T(0), rdu = T(0);
        const bool vin = busy && (!cold) && it == 0;  // work->v / work->z come from the caller on the first iteration
        if (keep_v || __any_sync(0xffffffffu, vin)) forward(BoolTag<true>{}, vin, rpx, rdx, rpu, rdu);
        else forward(BoolTag<false>{}, false, rpx, rdx, rpu, rdu);
        __syncwarp();
        // ---- termination_condition (admm.cpp:310-328), per instance ----
        rpx = group_max<T, L>(rpx);
        rdx = group_max<T, L>(rdx);
        rpu = group_max<T, L>(rpu);
        rdu = group_max<T, L>(rdu);
        if constexpr (ADAPT) {  // after update_dual of loop index i = it: adapt when i > 0 && i % 5 == 0 (admm.cpp:407)
            const bool ad = busy && it > 0 && it % 5 == 0;
            if (__any_sync(0xffffffffu, ad)) adapt_sweep(ad);
        }
        if (busy) {
            it += 1;
            if (it % P.check_termination == 0) {
                res_px = rpx;
                res_dx = rdx * rho_();
                res_pu = rpu;
                res_du = rdu * rho_();
                if (res_px < P.pri_tol && res_pu < P.pri_tol && res_dx < P.dua_tol && res_du < P.dua_tol) solved = 1;
            }
        }
        } while (!__any_sync(0xffffffffu, busy && (solved || it >= P.max_iter)));
    }
}

// ---------------------------------------------------------------------------------------------------------
// host side: configuration choice + launch
// ---------------------------------------------------------------------------------------------------------
template <typename T, int NX, int NU, int L>
inline void gpi_consider(int N, int max_smem, GpiPlan &best) {
    if constexpr (gpi_feasible<T, NX, NU, L>()) {
        using Cfg = GpiCfg<NX, NU, L, (int)sizeof(T)>;
        const size_t per_warp = Cfg::warp_elems(N) * sizeof(T);
        // fp32: the TMA staging area aliases the start of the state region (the allocation is at least as large as the blob);
        // fp64: the blob stays resident in front of the state regions (matrix rows are re-read at every sweep start)
        const size_t reserve = cache_reserve_bytes(NX, NU, sizeof(T));
        const size_t blob = reserve + 64;
        const size_t keep = gpi_per_sweep_rows<T>() ? reserve : 0;
        if ((size_t)max_smem < keep + per_warp) return;
        const int w = (int)std::min<size_t>(GPI_MAX_WARPS, ((size_t)max_smem - keep) / per_warp);
        if (w < 1 || blob > (size_t)max_smem) return;
        // score: instances resident per SM, then fewer lanes per instance (less shuffle traffic)
        const int inst = w * Cfg::IPW, binst = best.warps * (best.L ? 32 / best.L : 0);
        const bool better = best.L == 0 || (w >= 4 && best.warps < 4) || (((w >= 4) == (best.warps >= 4)) && inst > binst);
        if (better) {
            best.L = L;
            best.warps = w;
            best.smem = std::max(keep + per_warp * (size_t)w, blob);
            best.instances_per_cta = w * Cfg::IPW;
            best.vscratch_per_instance = (size_t)N * L * Cfg::PVP * sizeof(T);
        }
    }
}

template <typename T, int NX, int NU>
inline GpiPlan gpi_plan(int N, int max_smem) {
    GpiPlan p;
    // L = 16 is only ever needed in fp64 (two registers per matrix entry: L = 4 / 8 exceed the register ceiling from
    // nx = 12 on); for fp32 L = 8 covers every (nx, nu) pair of TM_DIMS, so the fp32 L = 16 kernels are compiled only
    // with -DTM_GPI_L16 (wider states) to keep the build short
    constexpr bool L16 = sizeof(T) == 8
#ifdef TM_GPI_L16
                         || true
#endif
        ;
    // TINYMPC_GPI_LANES=4|8|16 restricts the choice to one group width (A/B switch for measurements)
    const char *e = std::getenv("TINYMPC_GPI_LANES");
    const int only = e ? std::atoi(e) : 0;
    if (!only || only == 4) gpi_consider<T, NX, NU, 4>(N, max_smem, p);
    if (!only || only == 8) gpi_consider<T, NX, NU, 8>(N, max_smem, p);
    if constexpr (L16)
        if (!only || only == 16) gpi_consider<T, NX, NU, 16>(N, max_smem, p);
    return p;
}

template <typename T, int NX, int NU, int L, bool FAST, bool HET, bool MM = false>
int launch_gpi_L(LaunchDesc *d, const GpiPlan &plan, const KParams<T, NX, NU> &P, const T *gmat) {
    if constexpr (gpi_feasible<T, NX, NU, L>()) {
        auto kern = gpi_solve_kernel<T, NX, NU, L, FAST, HET, MM>;
        if (!set_dynamic_smem(kern, plan.smem)) return TINYMPC_ERR_CUDA;
        const int64_t ngroups = (d->io.B + (32 / L) - 1) / (32 / L);
        // ngroups = warps the batch fills.  A batch smaller than one wave is spread over all SMs with fewer warps per CTA
        // (the kernel's carve-up is per warp, any block size up to plan.warps works): the latency of a solve is set by how
        // many warps share a scheduler.
        int warps = plan.warps;
        if ((ngroups + warps - 1) / warps < d->sm_count) warps = (int)std::max<int64_t>(1, (ngroups + d->sm_count - 1) / d->sm_count);
        const int64_t want = (ngroups + warps - 1) / warps;
        const int ctas = (int)std::max<int64_t>(1, std::min<int64_t>(d->sm_count, want));
        kern<<<ctas, warps * 32, plan.smem, d->stream>>>(P, gmat, (unsigned long long *)d->work_queue);
        return launch_done(d, warps * 32, ctas, plan.smem, L, plan.instances_per_cta);
    } else {
        return TINYMPC_ERR_UNSUPPORTED;
    }
}

// the adaptive kernel (plan.smem includes gpi_adapt_bytes); same launch geometry as launch_gpi_L
template <typename T, int NX, int NU, int L>
int launch_gpi_adapt_L(LaunchDesc *d, const GpiPlan &plan, const KParams<T, NX, NU> &P, const T *gmat) {
    static_assert(L < GPI_ADAPT, "the lane count must leave GPI_ADAPT free");
    if constexpr (gpi_feasible<T, NX, NU, L>()) {
        auto kern = gpi_solve_kernel<T, NX, NU, L + GPI_ADAPT, false, true>;
        if (!set_dynamic_smem(kern, plan.smem)) return TINYMPC_ERR_CUDA;
        const int64_t ngroups = (d->io.B + (32 / L) - 1) / (32 / L);
        int warps = plan.warps;
        if ((ngroups + warps - 1) / warps < d->sm_count) warps = (int)std::max<int64_t>(1, (ngroups + d->sm_count - 1) / d->sm_count);
        const int64_t want = (ngroups + warps - 1) / warps;
        const int ctas = (int)std::max<int64_t>(1, std::min<int64_t>(d->sm_count, want));
        kern<<<ctas, warps * 32, plan.smem, d->stream>>>(P, gmat, (unsigned long long *)d->work_queue);
        return launch_done(d, warps * 32, ctas, plan.smem, L, plan.instances_per_cta);
    } else {
        return TINYMPC_ERR_UNSUPPORTED;
    }
}

}  // namespace tmpc
