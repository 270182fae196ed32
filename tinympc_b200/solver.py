"""Host-side mirror of the reference's solver interface for the batched H100 path.

The reference's user-facing calls (src/tinympc/tiny_api.hpp:10-62) map as follows:

    tiny_setup(&solver, A, B, f, Q, R, rho, nx, nu, N, verbose)   -> setup_problem(...) + BatchedTinySolver(problem)
    tiny_set_bound_constraints / _cone_ / _linear_ / _tv_linear_   -> keyword arguments of setup_problem(...)
    tiny_update_settings / solver->settings->max_iter = ...        -> BatchedTinySolver.settings + update_settings()
    tiny_set_x0 / work->Xref = ... / tiny_solve(solver)            -> BatchedTinySolver.solve(x0, Xref, Uref, ...)
    solver->solution->{x,u,iter,solved}, work->{x,u,g,y,...}       -> the dict solve() returns

All heavy lifting happens in libtinympc_b200.so through the C ABI (include/tinympc_b200.h); this file only
moves pointers.  torch is used for device memory and streams only.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import abi
from ._lib import check, load
from .batch import HostBatch
from .problem import MPCProblem, copy_settings, default_settings, dtype_code
from .workloads import ModelSpec


def precompute_cache(nx, nu, rho, A, B, f, Qw, Rw, dtype):
    """tiny_precompute_and_set_cache (tiny_api.cpp:307-381) on the host; Qw/Rw = diag + rho (work->Q/R)."""
    lib = load()
    dt = np.dtype(dtype).type
    A_ = np.asfortranarray(A, dtype=dt)
    B_ = np.asfortranarray(np.asarray(B, dtype=dt).reshape(nx, nu))
    f_ = np.ascontiguousarray(f, dtype=dt)
    Qw = np.ascontiguousarray(Qw, dtype=dt)
    Rw = np.ascontiguousarray(Rw, dtype=dt)
    out = dict(Kinf=np.zeros((nu, nx), dt, order="F"), Pinf=np.zeros((nx, nx), dt, order="F"),
               Quu_inv=np.zeros((nu, nu), dt, order="F"), AmBKt=np.zeros((nx, nx), dt, order="F"),
               APf=np.zeros(nx, dt), BPf=np.zeros(nu, dt))
    vp = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
    sweeps = check(lib.tinympc_b200_precompute_cache(dtype_code(dt), nx, nu, float(dt(rho)), vp(A_), vp(B_), vp(f_),
                                                     vp(Qw), vp(Rw), vp(out["Kinf"]), vp(out["Pinf"]),
                                                     vp(out["Quu_inv"]), vp(out["AmBKt"]), vp(out["APf"]), vp(out["BPf"])))
    return out, sweeps


def setup_problem(spec: ModelSpec, dtype=np.float32) -> MPCProblem:
    """The tiny_setup arithmetic (tiny_api.cpp:117-118,136): work->Q = diag(Q)+rho, work->R = diag(R)+rho, cache."""
    dt = np.dtype(dtype).type
    rho = dt(spec.rho)
    Qw = (np.asarray(spec.Qdiag, dtype=dt) + rho).astype(dt)
    Rw = (np.asarray(spec.Rdiag, dtype=dt) + rho).astype(dt)
    cache, sweeps = precompute_cache(spec.nx, spec.nu, rho, spec.A, spec.B, spec.f, Qw, Rw, dt)
    p = MPCProblem(nx=spec.nx, nu=spec.nu, N=spec.N, dtype=dt, rho=float(rho), A=spec.A, B=spec.B, f=spec.f, Q=Qw, R=Rw,
                   **cache, **spec.constraints)
    p.riccati_sweeps = sweeps
    return p


def setup_models(nx, nu, A, B, f, Qdiag, Rdiag, rho, dtype=np.float32, nthreads=0):
    """tiny_setup's arithmetic for a heterogeneous batch: per-instance A [Bn,nx,nx], B [Bn,nx,nu] (row index first, like the
    reference's examples), f [Bn,nx], user diagonals Qdiag [Bn,nx], Rdiag [Bn,nu], rho [Bn]  ->  packed model blobs
    [Bn, blob] for BatchedTinySolver.solve(..., models=...)  (tinympc_batch_t.models, SURVEY §8f-2)."""
    import os

    lib = load()
    dt = np.dtype(dtype).type
    A = np.asarray(A, dtype=dt)
    Bn = A.shape[0]
    A_ = np.ascontiguousarray(np.transpose(A.reshape(Bn, nx, nx), (0, 2, 1)))          # column-major per instance
    B_ = np.ascontiguousarray(np.transpose(np.asarray(B, dtype=dt).reshape(Bn, nx, nu), (0, 2, 1)))
    f_ = np.ascontiguousarray(np.asarray(f, dtype=dt).reshape(Bn, nx))
    Q_ = np.ascontiguousarray(np.asarray(Qdiag, dtype=dt).reshape(Bn, nx))
    R_ = np.ascontiguousarray(np.asarray(Rdiag, dtype=dt).reshape(Bn, nu))
    r_ = np.ascontiguousarray(np.broadcast_to(np.asarray(rho, dtype=dt), (Bn,)))
    M = int(lib.tinympc_b200_model_blob_elems(nx, nu))
    out = np.zeros((Bn, M), dtype=dt)
    vp = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib.tinympc_b200_precompute_cache_batch(dtype_code(dt), nx, nu, Bn, vp(A_), vp(B_), vp(f_), vp(Q_), vp(R_), vp(r_),
                                                  vp(out), nthreads or (os.cpu_count() or 1)))
    return out


def unpack_model(blob, nx, nu):
    """One per-instance blob -> dict of column-major pieces (for building the equivalent single-model MPCProblem)."""
    sizes = [("A", (nx, nx)), ("B", (nx, nu)), ("f", (nx,)), ("Q", (nx,)), ("R", (nu,)), ("Kinf", (nu, nx)), ("Pinf", (nx, nx)),
             ("Quu_inv", (nu, nu)), ("AmBKt", (nx, nx)), ("APf", (nx,)), ("BPf", (nu,))]
    out, o = {}, 0
    for name, shp in sizes:
        n = int(np.prod(shp))
        out[name] = np.array(blob[o:o + n]).reshape(shp, order="F")
        o += n
    out["rho"] = float(blob[o])
    return out


def pack_models(problem: MPCProblem, B: int):
    """The problem's own model, cache and rho as B identical model blobs [B, blob] (layout: tinympc_batch_t.models,
    csrc/model_blob.h): the starting point of an adaptive-rho batch whose instances share one model."""
    dt = problem.dtype
    pieces = [problem.A, problem.B, problem.f, problem.Q, problem.R, problem.Kinf, problem.Pinf, problem.Quu_inv, problem.AmBKt,
              problem.APf, problem.BPf]
    blob = np.concatenate([np.asarray(a, dtype=dt).reshape(-1, order="F") for a in pieces] + [np.array([problem.rho], dtype=dt)])
    return np.ascontiguousarray(np.tile(blob, (int(B), 1)))


class AdaptiveRho:
    """The reference's adaptive-rho settings (settings->adaptive_rho_min / _max / _enable_clipping) and sensitivity tables
    (cache->dKinf_drho nu x nx, dPinf_drho nx x nx), for BatchedTinySolver.solve(..., adaptive_rho=...)."""

    def __init__(self, dKinf_drho, dPinf_drho, rho_min=1.0, rho_max=100.0, enable_clipping=True):
        self.dKinf_drho, self.dPinf_drho = dKinf_drho, dPinf_drho
        self.rho_min, self.rho_max, self.enable_clipping = float(rho_min), float(rho_max), bool(enable_clipping)

    def to_c(self, problem: MPCProblem, models_ptr) -> abi.AdaptiveRho:
        dt = problem.dtype
        dK = np.asfortranarray(np.asarray(self.dKinf_drho, dtype=dt).reshape(problem.nu, problem.nx))
        dP = np.asfortranarray(np.asarray(self.dPinf_drho, dtype=dt).reshape(problem.nx, problem.nx))
        a = abi.AdaptiveRho()
        a.rho_min, a.rho_max, a.enable_clipping, a.reserved = self.rho_min, self.rho_max, int(self.enable_clipping), 0
        a.dKinf_drho, a.dPinf_drho, a.models = dK.ctypes.data, dP.ctypes.data, models_ptr
        a._owner = (dK, dP)
        return a


class BatchedTinySolver:
    """A TinySolver (types.hpp:213-218) for B independent instances on one H100."""

    def __init__(self, problem: MPCProblem, settings: abi.Settings | None = None, device: int = 0,
                 mode: int = abi.MODE_STRICT, kernel: int = abi.KERNEL_AUTO):
        if not problem.has_cache():
            raise ValueError("problem has no cache (use setup_problem or provide Kinf, Pinf, Quu_inv, AmBKt, APf, BPf)")
        self._lib = load()
        self.problem = problem
        self.device = device
        self._h = C.c_void_p()
        cp = problem.to_c()
        check(self._lib.tinympc_b200_create(C.byref(cp), device, C.byref(self._h)))
        self.settings = copy_settings(settings) if settings is not None else default_settings()
        self.update_settings()
        self.set_mode(mode, kernel)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.tinympc_b200_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def update_settings(self, **kw):
        for k, v in kw.items():
            if not hasattr(self.settings, k):
                raise AttributeError(k)
            setattr(self.settings, k, v)
        check(self._lib.tinympc_b200_update_settings(self._h, C.byref(self.settings)))

    def set_mode(self, mode=abi.MODE_STRICT, kernel=abi.KERNEL_AUTO):
        check(self._lib.tinympc_b200_set_mode(self._h, mode, kernel))
        self.mode, self.kernel = mode, kernel

    def stats(self) -> dict:
        st = abi.Stats()
        check(self._lib.tinympc_b200_get_stats(self._h, C.byref(st)))
        return {n: getattr(st, n) for n, _ in abi.Stats._fields_}

    # ---- host buffers (numpy): the call a reference user would make; H2D/D2H inside ------------------
    def solve(self, x0, Xref, Uref=None, state=None, cold_start=True, want_state=(), models=None,
              adaptive_rho: AdaptiveRho | None = None) -> dict:
        """With adaptive_rho: every instance adapts its own rho / Kinf / Pinf, starting from its blob in `models` (default:
        the problem's own cache, pack_models); the result's "models" holds the adapted blobs, the start of the next solve."""
        if adaptive_rho is None:
            hb = HostBatch(self.problem, x0, Xref, Uref, state=state, cold_start=cold_start, want_state=want_state, models=models)
            cb = hb.to_c()
            check(self._lib.tinympc_b200_solve_host(self._h, C.byref(cb)))
            return hb.result()
        hb = HostBatch(self.problem, x0, Xref, Uref, state=state, cold_start=cold_start, want_state=want_state)
        m = pack_models(self.problem, hb.B) if models is None else np.array(models, dtype=self.problem.dtype).reshape(hb.B, -1)
        cb, ar = hb.to_c(), adaptive_rho.to_c(self.problem, m.ctypes.data)
        check(self._lib.tinympc_b200_solve_adaptive_host(self._h, C.byref(cb), C.byref(ar)))
        out = hb.result()
        out["models"] = m
        return out

    def solve_prepared(self, hb: HostBatch, cb: abi.Batch | None = None):
        """Same as solve() on an already-built HostBatch (bench.py: keeps numpy allocation out of the timed region)."""
        cb = cb if cb is not None else hb.to_c()
        check(self._lib.tinympc_b200_solve_host(self._h, C.byref(cb)))
        return hb

    def setup_models_device(self, A, B, f, Qdiag, Rdiag, rho, want_sweeps=False):
        """setup_models on the GPU (tinympc_b200_precompute_cache_batch_device): inputs as in setup_models (numpy or torch,
        A [Bn,nx,nx] / B [Bn,nx,nu] row index first), result = torch CUDA tensor [Bn, blob] usable as `models=` of
        make_device_batch.  Bit-identical to the host routine."""
        import torch

        p = self.problem
        tdt = torch.float32 if p.dtype == np.float32 else torch.float64
        dev = torch.device("cuda", self.device)
        t = lambda a: torch.as_tensor(a, device=dev).to(tdt)  # noqa: E731
        A_ = t(A).reshape(-1, p.nx, p.nx).transpose(1, 2).contiguous()  # column-major per instance
        Bn = A_.shape[0]
        B_ = t(B).reshape(Bn, p.nx, p.nu).transpose(1, 2).contiguous()
        f_, Q_, R_ = t(f).reshape(Bn, p.nx).contiguous(), t(Qdiag).reshape(Bn, p.nx).contiguous(), t(Rdiag).reshape(Bn, p.nu).contiguous()
        r_ = t(rho).reshape(-1).expand(Bn).contiguous()
        M = int(self._lib.tinympc_b200_model_blob_elems(p.nx, p.nu))
        out = torch.zeros((Bn, M), dtype=tdt, device=dev)
        sweeps = torch.zeros(Bn, dtype=torch.int32, device=dev) if want_sweeps else None
        stream = torch.cuda.current_stream(dev).cuda_stream
        check(self._lib.tinympc_b200_precompute_cache_batch_device(
            self._h, Bn, A_.data_ptr(), B_.data_ptr(), f_.data_ptr(), Q_.data_ptr(), R_.data_ptr(), r_.data_ptr(), out.data_ptr(),
            None if sweeps is None else sweeps.data_ptr(), C.c_void_p(stream)))
        return (out, sweeps) if want_sweeps else out

    # ---- device buffers (torch tensors on cuda:<device>) ---------------------------------------------
    def make_device_batch(self, x0, Xref, Uref=None, state=None, cold_start=True, want_state=(), want_residuals=True,
                          want_u0=False, want_solution=True, models=None):
        """Allocate/adopt torch CUDA tensors and build the device-pointer tinympc_batch_t."""
        import torch

        p = self.problem
        tdt = torch.float32 if p.dtype == np.float32 else torch.float64
        dev = torch.device("cuda", self.device)

        def t(a, shape=None):
            if isinstance(a, torch.Tensor):
                a = a.to(device=dev, dtype=tdt).contiguous()
            else:
                a = torch.as_tensor(np.ascontiguousarray(a, dtype=p.dtype), device=dev)
            return a if shape is None else a.reshape(shape)

        x0 = t(x0).reshape(-1, p.nx)
        B = x0.shape[0]
        Xref = t(Xref)
        per_x = Xref.dim() == 3
        Uref_t = None if Uref is None else t(Uref)
        per_u = Uref_t is not None and Uref_t.dim() == 3
        tens = dict(x0=x0, Xref=Xref, Uref=Uref_t)
        st = {}
        for name in abi.STATE_FIELDS:
            shape = (B, p.N, p.nx) if abi.STATE_IS_X[name] else (B, p.N - 1, p.nu)
            if state is not None and state.get(name) is not None:
                st[name] = t(state[name], shape)
            elif name in want_state:
                st[name] = torch.zeros(shape, dtype=tdt, device=dev)
        out = dict(sol_x=torch.empty((B, p.N, p.nx), dtype=tdt, device=dev) if want_solution else None,
                   sol_u=torch.empty((B, p.N - 1, p.nu), dtype=tdt, device=dev) if want_solution else None,
                   u0=torch.empty((B, p.nu), dtype=tdt, device=dev) if want_u0 else None,
                   iter=torch.zeros(B, dtype=torch.int32, device=dev),
                   solved=torch.zeros(B, dtype=torch.int32, device=dev),
                   residuals=torch.zeros((B, 4), dtype=tdt, device=dev) if want_residuals else None)
        b = abi.Batch()
        b.B = B
        b.x0, b.Xref = x0.data_ptr(), Xref.data_ptr()
        b.xref_per_instance = int(per_x)
        b.Uref = None if Uref_t is None else Uref_t.data_ptr()
        b.uref_per_instance = int(per_u)
        b.cold_start = int(bool(cold_start))
        for name, a in st.items():
            setattr(b.state, name, a.data_ptr())
        b.sol_x = None if out["sol_x"] is None else out["sol_x"].data_ptr()
        b.sol_u = None if out["sol_u"] is None else out["sol_u"].data_ptr()
        b.u0 = None if out["u0"] is None else out["u0"].data_ptr()
        models_t = None if models is None else t(models)
        tens["models"] = models_t
        b.models = None if models_t is None else models_t.data_ptr()
        b.iter, b.solved = out["iter"].data_ptr(), out["solved"].data_ptr()
        b.residuals = None if out["residuals"] is None else out["residuals"].data_ptr()
        res = dict(out)
        res.update(st)
        b._owner = (tens, res)
        return b, res

    def solve_device(self, batch: abi.Batch, stream=None):
        """Enqueue one batched tiny_solve on `stream` (torch.cuda.Stream, default: torch's current stream)."""
        import torch

        s = stream if stream is not None else torch.cuda.current_stream(self.device)
        check(self._lib.tinympc_b200_solve(self._h, C.byref(batch), C.c_void_p(s.cuda_stream)))

    def solve_device_adaptive(self, batch: abi.Batch, models, adaptive_rho: AdaptiveRho, stream=None):
        """solve_device with adaptive rho: `models` = torch CUDA tensor [B, blob] (in/out, e.g. from pack_models), updated in
        place with every instance's adapted rho / Kinf / Pinf."""
        import torch

        p = self.problem
        M = int(self._lib.tinympc_b200_model_blob_elems(p.nx, p.nu))
        if not (isinstance(models, torch.Tensor) and models.is_cuda and models.is_contiguous() and models.numel() == batch.B * M
                and models.dtype == (torch.float32 if p.dtype == np.float32 else torch.float64)):
            raise ValueError(f"models must be a contiguous CUDA tensor of {batch.B} x {M} elements of the problem dtype")
        s = stream if stream is not None else torch.cuda.current_stream(self.device)
        ar = adaptive_rho.to_c(p, models.data_ptr())
        check(self._lib.tinympc_b200_solve_adaptive(self._h, C.byref(batch), C.byref(ar), C.c_void_p(s.cuda_stream)))
