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
from .batch import KINDS, HostBatch, per_instance, problem_dims
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


def _batch_inputs(nx, nu, A, B, f, Qdiag, Rdiag, rho, dt):
    """numpy inputs of the batched precompute: A [Bn,nx,nx], B [Bn,nx,nu] (row index first), f, Qdiag, Rdiag, rho ->
    contiguous arrays of dtype dt, A and B column-major per instance"""
    A = np.asarray(A, dtype=dt)
    Bn = A.shape[0]
    A_ = np.ascontiguousarray(np.transpose(A.reshape(Bn, nx, nx), (0, 2, 1)))          # column-major per instance
    B_ = np.ascontiguousarray(np.transpose(np.asarray(B, dtype=dt).reshape(Bn, nx, nu), (0, 2, 1)))
    f_ = np.ascontiguousarray(np.asarray(f, dtype=dt).reshape(Bn, nx))
    Q_ = np.ascontiguousarray(np.asarray(Qdiag, dtype=dt).reshape(Bn, nx))
    R_ = np.ascontiguousarray(np.asarray(Rdiag, dtype=dt).reshape(Bn, nu))
    r_ = np.ascontiguousarray(np.broadcast_to(np.asarray(rho, dtype=dt), (Bn,)))
    return A_, B_, f_, Q_, R_, r_


def setup_models(nx, nu, A, B, f, Qdiag, Rdiag, rho, dtype=np.float32, nthreads=0):
    """tiny_setup's arithmetic for a heterogeneous batch: per-instance A [Bn,nx,nx], B [Bn,nx,nu] (row index first, like the
    reference's examples), f [Bn,nx], user diagonals Qdiag [Bn,nx], Rdiag [Bn,nu], rho [Bn]  ->  packed model blobs
    [Bn, blob] for BatchedTinySolver.solve(..., models=...)  (tinympc_batch_t.models, SURVEY §8f-2)."""
    import os

    lib = load()
    dt = np.dtype(dtype).type
    ins = _batch_inputs(nx, nu, A, B, f, Qdiag, Rdiag, rho, dt)
    Bn = len(ins[0])
    out = np.zeros((Bn, int(lib.tinympc_b200_model_blob_elems(nx, nu))), dtype=dt)
    vp = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib.tinympc_b200_precompute_cache_batch(dtype_code(dt), nx, nu, Bn, *map(vp, ins), vp(out), nthreads or (os.cpu_count() or 1)))
    return out


def setup_sensitivity(nx, nu, A, B, f, Qdiag, Rdiag, rho, dtype=np.float32, nthreads=0):
    """The adaptive-rho sensitivity tables of Bn models (tinympc_b200_precompute_sensitivity_batch): the derivative with
    respect to rho of the Kinf / Pinf setup_models computes, inputs as in setup_models.  Returns (dKinf_drho [Bn, nu, nx],
    dPinf_drho [Bn, nx, nx]) indexed (instance, row, column), as AdaptiveRho takes them."""
    import os

    lib = load()
    dt = np.dtype(dtype).type
    ins = _batch_inputs(nx, nu, A, B, f, Qdiag, Rdiag, rho, dt)
    Bn = len(ins[0])
    dK, dP = np.zeros((Bn, nx, nu), dtype=dt), np.zeros((Bn, nx, nx), dtype=dt)  # column-major per instance
    vp = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib.tinympc_b200_precompute_sensitivity_batch(dtype_code(dt), nx, nu, Bn, *map(vp, ins), vp(dK), vp(dP),
                                                        nthreads or (os.cpu_count() or 1)))
    return np.transpose(dK, (0, 2, 1)), np.transpose(dP, (0, 2, 1))


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
    (cache->dKinf_drho nu x nx, dPinf_drho nx x nx), for BatchedTinySolver.solve(..., adaptive_rho=...).  Tables with a
    leading batch dimension ([B, nu, nx], [B, nx, nx], e.g. from setup_sensitivity[_device]) give every instance its own
    pair: what a fleet of different models needs."""

    def __init__(self, dKinf_drho, dPinf_drho, rho_min=1.0, rho_max=100.0, enable_clipping=True):
        self.dKinf_drho, self.dPinf_drho = dKinf_drho, dPinf_drho
        self.rho_min, self.rho_max, self.enable_clipping = float(rho_min), float(rho_max), bool(enable_clipping)
        self.per_instance = len(dKinf_drho.shape) == 3 if hasattr(dKinf_drho, "shape") else np.ndim(dKinf_drho) == 3

    def to_c(self, problem: MPCProblem, models_ptr, B=None, device=None) -> abi.AdaptiveRho:
        """device: None = the host entry point (tables as host arrays); a torch device = tinympc_b200_solve_adaptive, whose
        per-instance tables are device arrays (CUDA tensors already in place are passed without a copy)."""
        dt, nx, nu = problem.dtype, problem.nx, problem.nu
        a = abi.AdaptiveRho()
        a.rho_min, a.rho_max, a.enable_clipping, a.reserved = self.rho_min, self.rho_max, int(self.enable_clipping), 0
        a.tables_per_instance = int(self.per_instance)
        if not self.per_instance:
            dK = np.asfortranarray(_host(self.dKinf_drho, dt).reshape(nu, nx))
            dP = np.asfortranarray(_host(self.dPinf_drho, dt).reshape(nx, nx))
            a.dKinf_drho, a.dPinf_drho = dK.ctypes.data, dP.ctypes.data
        else:
            B = self.dKinf_drho.shape[0] if B is None else B
            if tuple(self.dKinf_drho.shape) != (B, nu, nx) or tuple(self.dPinf_drho.shape) != (B, nx, nx):
                raise ValueError(f"per-instance tables must be [{B}, {nu}, {nx}] and [{B}, {nx}, {nx}]")
            if device is None:  # column-major per instance
                dK = np.ascontiguousarray(np.transpose(_host(self.dKinf_drho, dt), (0, 2, 1)))
                dP = np.ascontiguousarray(np.transpose(_host(self.dPinf_drho, dt), (0, 2, 1)))
                a.dKinf_drho, a.dPinf_drho = dK.ctypes.data, dP.ctypes.data
            else:
                import torch

                tdt = torch.float32 if dt == np.float32 else torch.float64
                dK = torch.as_tensor(self.dKinf_drho, device=device).to(tdt).transpose(1, 2).contiguous()
                dP = torch.as_tensor(self.dPinf_drho, device=device).to(tdt).transpose(1, 2).contiguous()
                a.dKinf_drho, a.dPinf_drho = dK.data_ptr(), dP.data_ptr()
        a.models = models_ptr
        a._owner = (dK, dP)
        return a


def _host(a, dt):
    """numpy array of dtype dt from a numpy array or a torch tensor on any device"""
    return np.asarray(a.detach().cpu().numpy() if hasattr(a, "detach") else a, dtype=dt)


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
              adaptive_rho: AdaptiveRho | None = None, bounds: dict | None = None, cones: dict | None = None,
              planes: dict | None = None) -> dict:
        """With adaptive_rho: every instance adapts its own rho / Kinf / Pinf, starting from its blob in `models` (default:
        the problem's own cache, pack_models); the result's "models" holds the adapted blobs, the start of the next solve.
        bounds: per-instance box bounds in place of the problem's, a dict with any of x_min, x_max, u_min, u_max of the
        problem dtype: [B, nx] / [B, nu] (one column per instance) or [B, N, nx] / [B, N-1, nu] (a horizon per instance);
        a side may be absent when its bound is disabled (tinympc_batch_t.bounds_per_instance).
        cones: per-instance cone coefficients in place of the problem's cx / cu, a dict with x_mu [B, num state cones] and / or
        u_mu [B, num input cones] of the problem dtype; a side may be absent when its cone loop does not run
        (tinympc_batch_t.cones_per_instance).
        planes: per-instance static hyperplanes in place of the problem's, a dict with Alin_x [B, nlx, nx] / blin_x [B, nlx]
        and / or Alin_u [B, nlu, nu] / blin_u [B, nlu] of the problem dtype (rows as tiny_set_linear_constraints takes them;
        nlx, nlu: the problem's row counts); a side may be absent when its static hyperplane loop does not run
        (tinympc_batch_t.planes_per_instance)."""
        if adaptive_rho is None:
            hb = HostBatch(self.problem, x0, Xref, Uref, state=state, cold_start=cold_start, want_state=want_state, models=models,
                           bounds=bounds, cones=cones, planes=planes)
            cb = hb.to_c()
            check(self._lib.tinympc_b200_solve_host(self._h, C.byref(cb)))
            return hb.result()
        hb = HostBatch(self.problem, x0, Xref, Uref, state=state, cold_start=cold_start, want_state=want_state, bounds=bounds,
                       cones=cones, planes=planes)
        m = pack_models(self.problem, hb.B) if models is None else np.array(models, dtype=self.problem.dtype).reshape(hb.B, -1)
        cb, ar = hb.to_c(), adaptive_rho.to_c(self.problem, m.ctypes.data, hb.B)
        check(self._lib.tinympc_b200_solve_adaptive_host(self._h, C.byref(cb), C.byref(ar)))
        out = hb.result()
        out["models"] = m
        return out

    def solve_prepared(self, hb: HostBatch, cb: abi.Batch | None = None):
        """Same as solve() on an already-built HostBatch (bench.py: keeps numpy allocation out of the timed region)."""
        cb = cb if cb is not None else hb.to_c()
        check(self._lib.tinympc_b200_solve_host(self._h, C.byref(cb)))
        return hb

    def _device_precompute(self, entry, outputs, A, B, f, Qdiag, Rdiag, rho, want_sweeps):
        """One batched precompute on the GPU through the C entry point `entry`, on the current stream.  Inputs as in
        setup_models (numpy or torch, A [Bn,nx,nx] / B [Bn,nx,nu] row index first); outputs(Bn, dtype=, device=) makes the
        zeroed output tensors.  Returns them and the sweeps [Bn] (int32, None unless want_sweeps)."""
        import torch

        p = self.problem
        like = dict(dtype=torch.float32 if p.dtype == np.float32 else torch.float64, device=torch.device("cuda", self.device))
        t = lambda a: torch.as_tensor(a, device=like["device"]).to(like["dtype"])  # noqa: E731
        A_ = t(A).reshape(-1, p.nx, p.nx).transpose(1, 2).contiguous()  # column-major per instance
        Bn = A_.shape[0]
        B_ = t(B).reshape(Bn, p.nx, p.nu).transpose(1, 2).contiguous()
        f_, Q_, R_ = t(f).reshape(Bn, p.nx).contiguous(), t(Qdiag).reshape(Bn, p.nx).contiguous(), t(Rdiag).reshape(Bn, p.nu).contiguous()
        r_ = t(rho).reshape(-1).expand(Bn).contiguous()
        outs = outputs(Bn, **like)
        sweeps = torch.zeros(Bn, dtype=torch.int32, device=like["device"]) if want_sweeps else None
        stream = torch.cuda.current_stream(like["device"]).cuda_stream
        check(getattr(self._lib, entry)(self._h, Bn, *(a.data_ptr() for a in (A_, B_, f_, Q_, R_, r_)), *(o.data_ptr() for o in outs),
                                        None if sweeps is None else sweeps.data_ptr(), C.c_void_p(stream)))
        return outs, sweeps

    def setup_models_device(self, A, B, f, Qdiag, Rdiag, rho, want_sweeps=False):
        """setup_models on the GPU (tinympc_b200_precompute_cache_batch_device): inputs as in setup_models (numpy or torch,
        A [Bn,nx,nx] / B [Bn,nx,nu] row index first), result = torch CUDA tensor [Bn, blob] usable as `models=` of
        make_device_batch.  Bit-identical to the host routine."""
        import torch

        M = int(self._lib.tinympc_b200_model_blob_elems(self.problem.nx, self.problem.nu))
        (out,), sweeps = self._device_precompute("tinympc_b200_precompute_cache_batch_device",
                                                 lambda Bn, **like: (torch.zeros((Bn, M), **like),), A, B, f, Qdiag, Rdiag, rho, want_sweeps)
        return (out, sweeps) if want_sweeps else out

    def setup_sensitivity_device(self, A, B, f, Qdiag, Rdiag, rho, want_sweeps=False):
        """setup_sensitivity on the GPU (tinympc_b200_precompute_sensitivity_batch_device), inputs as in setup_models_device:
        torch CUDA tensors (dKinf_drho [Bn, nu, nx], dPinf_drho [Bn, nx, nx]) indexed (instance, row, column), views of the
        column-major storage the adaptive solve reads: AdaptiveRho passes them on without a copy.  Bit-identical to the host
        routine."""
        import torch

        nx, nu = self.problem.nx, self.problem.nu
        (dK, dP), sweeps = self._device_precompute(
            "tinympc_b200_precompute_sensitivity_batch_device",
            lambda Bn, **like: (torch.zeros((Bn, nx, nu), **like), torch.zeros((Bn, nx, nx), **like)),  # column-major per instance
            A, B, f, Qdiag, Rdiag, rho, want_sweeps)
        dK, dP = dK.transpose(1, 2), dP.transpose(1, 2)
        return (dK, dP, sweeps) if want_sweeps else (dK, dP)

    # ---- device buffers (torch tensors on cuda:<device>) ---------------------------------------------
    def make_device_batch(self, x0, Xref, Uref=None, state=None, cold_start=True, want_state=(), want_residuals=True,
                          want_u0=False, want_solution=True, models=None, bounds: dict | None = None, cones: dict | None = None,
                          planes: dict | None = None):
        """Allocate/adopt torch CUDA tensors and build the device-pointer tinympc_batch_t.  bounds: per-instance box bounds,
        cones: per-instance cone coefficients, planes: per-instance static hyperplanes, all as in solve(); torch CUDA tensors
        of the problem dtype are used in place (a plane matrix that is the [B, n, nx] view of a contiguous [B, nx, n] tensor
        too), numpy arrays are uploaded."""
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
        for kind, arrays in dict(bounds=bounds, cones=cones, planes=planes).items():
            if arrays is not None:
                mode, abi_arrays = per_instance(kind, arrays, B, problem_dims(p), p.dtype)
                tens[kind] = {f: t(a) for f, a in abi_arrays.items()}
                setattr(b, KINDS[kind].mode_field, mode)
                for f in KINDS[kind].fields.values():
                    setattr(b, f, tens[kind][f].data_ptr() if f in tens[kind] else None)
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
        ar = adaptive_rho.to_c(p, models.data_ptr(), batch.B, models.device)
        check(self._lib.tinympc_b200_solve_adaptive(self._h, C.byref(batch), C.byref(ar), C.c_void_p(s.cuda_stream)))
