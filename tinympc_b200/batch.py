"""Host-side (numpy) construction of a `tinympc_batch_t` (include/tinympc_b200.h).

Layout of every trajectory buffer: [B][N][nx] / [B][N-1][nu], C-contiguous = the reference's column-major
nx x N matrix (types.hpp:94-95) repeated B times.
"""
from __future__ import annotations

import numpy as np

from . import abi
from .problem import MPCProblem


BOUND_NAMES = ("x_min", "x_max", "u_min", "u_max")


def bounds_layout(bounds: dict, B: int, N: int, nx: int, nu: int, dtype) -> int:
    """Check per-instance box bounds (a dict with any of x_min, x_max, u_min, u_max; numpy arrays or torch tensors) against a
    batch of B instances and return their layout (tinympc_batch_t.bounds_per_instance): 1 for [B, nx] / [B, nu] (one column
    per instance), 2 for [B, N, nx] / [B, N-1, nu] (a horizon per instance).  A side may be absent when its bound is
    disabled; min and max of a side come together."""
    unknown = set(bounds) - set(BOUND_NAMES)
    if unknown:
        raise ValueError(f"bounds: unknown keys {sorted(unknown)}; expected any of {BOUND_NAMES}")
    given = {k: v for k, v in bounds.items() if v is not None}
    for lo, hi in (("x_min", "x_max"), ("u_min", "u_max")):
        if (lo in given) != (hi in given):
            raise ValueError(f"bounds: {lo} and {hi} are given together")
    if not given:
        raise ValueError("bounds: give x_min / x_max, u_min / u_max or both")
    want = np.dtype(dtype)
    layouts = set()
    for k, a in given.items():
        dt = a.dtype if hasattr(a, "dtype") else None
        ok_dt = (str(dt).replace("torch.", "") == want.name) if dt is not None else False
        if not ok_dt:
            raise ValueError(f"bounds: {k} must have the problem dtype {want.name}, got {dt}")
        w, kn = (nx, N) if k[0] == "x" else (nu, N - 1)
        shape = tuple(a.shape)
        if shape == (B, w):
            layouts.add(1)
        elif shape == (B, kn, w):
            layouts.add(2)
        else:
            raise ValueError(f"bounds: {k} must be [{B}, {w}] (one column per instance) or [{B}, {kn}, {w}] (a horizon per "
                             f"instance), got {list(shape)}")
    if len(layouts) != 1:
        raise ValueError("bounds: every array takes the same layout ([B, n] or [B, N, n])")
    return layouts.pop()


CONE_NAMES = ("x_mu", "u_mu")


def cones_check(cones: dict, B: int, ncx: int, ncu: int, dtype) -> None:
    """Check per-instance cone coefficients (a dict with x_mu [B, ncx] for the state cones and / or u_mu [B, ncu] for the
    input cones; numpy arrays or torch tensors of the problem dtype) against a batch of B instances of a problem with ncx
    state and ncu input cones (tinympc_batch_t.cone_x_mu / cone_u_mu).  A side may be absent when its cone loop does not run."""
    unknown = set(cones) - set(CONE_NAMES)
    if unknown:
        raise ValueError(f"cones: unknown keys {sorted(unknown)}; expected any of {CONE_NAMES}")
    given = {k: v for k, v in cones.items() if v is not None}
    if not given:
        raise ValueError("cones: give x_mu, u_mu or both")
    want = np.dtype(dtype)
    for k, a in given.items():
        dt = a.dtype if hasattr(a, "dtype") else None
        if dt is None or str(dt).replace("torch.", "") != want.name:
            raise ValueError(f"cones: {k} must have the problem dtype {want.name}, got {dt}")
        nc = ncx if k == "x_mu" else ncu
        if tuple(a.shape) != (B, nc):
            raise ValueError(f"cones: {k} must be [{B}, {nc}] (one mu per instance and {'state' if k == 'x_mu' else 'input'} cone), "
                             f"got {list(a.shape)}")


PLANE_NAMES = ("Alin_x", "blin_x", "Alin_u", "blin_u")


def planes_check(planes: dict, B: int, nlx: int, nlu: int, nx: int, nu: int, dtype) -> None:
    """Check per-instance static hyperplanes (a dict with Alin_x [B, nlx, nx] and blin_x [B, nlx] for the state side and / or
    Alin_u [B, nlu, nu] and blin_u [B, nlu] for the input side, rows as a TinySolver's tiny_set_linear_constraints takes them;
    numpy arrays or torch tensors of the problem dtype) against a batch of B instances of a problem with nlx state and nlu
    input hyperplanes (tinympc_batch_t.Alin_x ... blin_u).  A side may be absent when its static hyperplane loop does not run."""
    unknown = set(planes) - set(PLANE_NAMES)
    if unknown:
        raise ValueError(f"planes: unknown keys {sorted(unknown)}; expected any of {PLANE_NAMES}")
    given = {k: v for k, v in planes.items() if v is not None}
    if not given:
        raise ValueError("planes: give Alin_x / blin_x, Alin_u / blin_u or both pairs")
    for a, b in (("Alin_x", "blin_x"), ("Alin_u", "blin_u")):
        if (a in given) != (b in given):
            raise ValueError(f"planes: {a} and {b} are given in pairs")
    want = np.dtype(dtype)
    shapes = dict(Alin_x=(B, nlx, nx), blin_x=(B, nlx), Alin_u=(B, nlu, nu), blin_u=(B, nlu))
    for k, a in given.items():
        dt = a.dtype if hasattr(a, "dtype") else None
        if dt is None or str(dt).replace("torch.", "") != want.name:
            raise ValueError(f"planes: {k} must have the problem dtype {want.name}, got {dt}")
        if tuple(a.shape) != shapes[k]:
            raise ValueError(f"planes: {k} must be {list(shapes[k])} (one set of the problem's hyperplane rows per instance), "
                             f"got {list(a.shape)}")


def planes_abi(planes: dict) -> dict:
    """the given arrays of a checked planes dict with each instance's matrix in the ABI's column-major order ([B, n, nx] ->
    a [B, nx, n] view; numpy arrays or torch tensors, made contiguous by the caller)"""
    return {k: (v.swapaxes(1, 2) if k.startswith("Alin") else v) for k, v in planes.items() if v is not None}


def num_planes(prob: MPCProblem) -> tuple:
    """(state, input) static hyperplane rows of a problem"""
    return (0 if prob.Alin_x is None else prob.Alin_x.shape[0], 0 if prob.Alin_u is None else prob.Alin_u.shape[0])


class HostBatch:
    """Owns the numpy buffers of one batched solve and the ctypes struct pointing at them."""

    def __init__(self, prob: MPCProblem, x0, Xref, Uref=None, state: dict | None = None, cold_start=True,
                 want_state=(), want_residuals=True, models=None, bounds: dict | None = None, cones: dict | None = None,
                 planes: dict | None = None):
        dt = prob.dtype
        nx, nu, N = prob.nx, prob.nu, prob.N
        self.prob = prob
        self.x0 = np.ascontiguousarray(x0, dtype=dt).reshape(-1, nx)
        B = self.x0.shape[0]
        self.B = B
        Xref = np.ascontiguousarray(Xref, dtype=dt)
        self.xref_per_instance = Xref.ndim == 3
        self.Xref = Xref.reshape((B, N, nx) if self.xref_per_instance else (N, nx))
        if Uref is None:
            self.Uref, self.uref_per_instance = None, False
        else:
            Uref = np.ascontiguousarray(Uref, dtype=dt)
            self.uref_per_instance = Uref.ndim == 3
            self.Uref = Uref.reshape((B, N - 1, nu) if self.uref_per_instance else (N - 1, nu))
        # state: in/out.  Arrays given in `state` are used in place (and updated); names in `want_state`
        # are allocated as zeros.
        self.state = {}
        for name in abi.STATE_FIELDS:
            shape = (B, N, nx) if abi.STATE_IS_X[name] else (B, N - 1, nu)
            if state is not None and name in state and state[name] is not None:
                a = state[name]
                if not (isinstance(a, np.ndarray) and a.dtype == dt and a.flags.c_contiguous and a.shape == shape):
                    a = np.ascontiguousarray(a, dtype=dt).reshape(shape).copy()
                self.state[name] = a
            elif name in want_state:
                self.state[name] = np.zeros(shape, dtype=dt)
        self.cold_start = bool(cold_start)
        self.models = None if models is None else np.ascontiguousarray(models, dtype=dt).reshape(B, -1)
        # per-instance box bounds (see bounds_layout); bounds_per_instance 0 = the problem's
        self.bounds_per_instance, self.bounds = 0, {}
        if bounds is not None:
            self.bounds_per_instance = bounds_layout(bounds, B, N, nx, nu, dt)
            self.bounds = {k: np.ascontiguousarray(v) for k, v in bounds.items() if v is not None}
        # per-instance cone coefficients (see cones_check); cones_per_instance 0 = the problem's cx / cu
        self.cones = None
        if cones is not None:
            cones_check(cones, B, len(prob.Acx), len(prob.Acu), dt)
            self.cones = {k: np.ascontiguousarray(v) for k, v in cones.items() if v is not None}
        # per-instance static hyperplanes (see planes_check), each matrix column-major; planes_per_instance 0 = the problem's
        self.planes = None
        if planes is not None:
            planes_check(planes, B, *num_planes(prob), nx, nu, dt)
            self.planes = {k: np.ascontiguousarray(v) for k, v in planes_abi(planes).items()}
        self.sol_x = np.zeros((B, N, nx), dtype=dt)
        self.sol_u = np.zeros((B, N - 1, nu), dtype=dt)
        self.iter = np.zeros(B, dtype=np.int32)
        self.solved = np.zeros(B, dtype=np.int32)
        self.residuals = np.zeros((B, 4), dtype=dt) if want_residuals else None

    def to_c(self) -> abi.Batch:
        b = abi.Batch()
        b.B = self.B
        b.x0 = self.x0.ctypes.data
        b.Xref = self.Xref.ctypes.data
        b.xref_per_instance = int(self.xref_per_instance)
        b.Uref = None if self.Uref is None else self.Uref.ctypes.data
        b.uref_per_instance = int(self.uref_per_instance)
        b.cold_start = int(self.cold_start)
        for name, a in self.state.items():
            setattr(b.state, name, a.ctypes.data)
        b.sol_x = self.sol_x.ctypes.data
        b.sol_u = self.sol_u.ctypes.data
        b.iter = self.iter.ctypes.data
        b.solved = self.solved.ctypes.data
        b.residuals = None if self.residuals is None else self.residuals.ctypes.data
        b.models = None if self.models is None else self.models.ctypes.data
        b.bounds_per_instance = self.bounds_per_instance
        for k, a in self.bounds.items():
            setattr(b, k, a.ctypes.data)
        if self.cones is not None:
            b.cones_per_instance = 1
            for k, a in self.cones.items():
                setattr(b, "cone_" + k, a.ctypes.data)
        if self.planes is not None:
            b.planes_per_instance = 1
            for k, a in self.planes.items():
                setattr(b, k, a.ctypes.data)
        b._owner = self
        return b

    def result(self) -> dict:
        out = dict(sol_x=self.sol_x, sol_u=self.sol_u, iter=self.iter, solved=self.solved, residuals=self.residuals)
        out.update(self.state)
        return out
