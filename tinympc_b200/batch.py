"""Host-side (numpy) construction of a `tinympc_batch_t` (include/tinympc_b200.h).

Layout of every trajectory buffer: [B][N][nx] / [B][N-1][nu], C-contiguous = the reference's column-major
nx x N matrix (types.hpp:94-95) repeated B times.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable

import numpy as np

from . import abi
from .problem import MPCProblem


@dataclass(frozen=True)
class Kind:
    """One kind of per-instance data of a batch (tinympc_batch_t): the ABI mode field, the user's keys with the ABI field of
    each, the keys that come in pairs, the accepted shapes of every key (shapes(dims, B) -> {key: {shape: mode}}, dims as
    problem_dims gives them) and the
    conversion of an array from the user's layout to the ABI's (an involution, a view)."""
    mode_field: str
    fields: dict
    pairs: tuple
    shapes: Callable
    to_abi: Callable = lambda key, a: a


def _box_shapes(d, B):
    return {k: {(B, w): 1, (B, n, w): 2} for k, w, n in (("x_min", d["nx"], d["N"]), ("x_max", d["nx"], d["N"]),
                                                         ("u_min", d["nu"], d["N"] - 1), ("u_max", d["nu"], d["N"] - 1))}


def _plane_shapes(d, B):
    return {"Alin_x": {(B, d["nlx"], d["nx"]): 1}, "blin_x": {(B, d["nlx"]): 1}, "Alin_u": {(B, d["nlu"], d["nu"]): 1},
            "blin_u": {(B, d["nlu"]): 1}}


# bounds: [B, nx] / [B, nu] (one column per instance, mode 1) or [B, N, nx] / [B, N-1, nu] (a horizon per instance, mode 2);
# cones: x_mu [B, state cones], u_mu [B, input cones]; planes: rows as tiny_set_linear_constraints takes them, Alin_x
# [B, nlx, nx] / blin_x [B, nlx] and Alin_u [B, nlu, nu] / blin_u [B, nlu], each matrix column-major in the ABI
KINDS = {
    "bounds": Kind("bounds_per_instance", {k: k for k in ("x_min", "x_max", "u_min", "u_max")}, (("x_min", "x_max"), ("u_min", "u_max")),
                   _box_shapes),
    "cones": Kind("cones_per_instance", {"x_mu": "cone_x_mu", "u_mu": "cone_u_mu"}, (),
                  lambda d, B: {"x_mu": {(B, d["ncx"]): 1}, "u_mu": {(B, d["ncu"]): 1}}),
    "planes": Kind("planes_per_instance", {k: k for k in ("Alin_x", "blin_x", "Alin_u", "blin_u")},
                   (("Alin_x", "blin_x"), ("Alin_u", "blin_u")), _plane_shapes,
                   lambda key, a: a.swapaxes(1, 2) if key.startswith("Alin") else a),
}


def problem_dims(prob: MPCProblem) -> dict:
    """the sizes the per-instance shapes depend on: horizon, state and input, cones and static hyperplane rows per side"""
    nlx, nlu = (0 if a is None else a.shape[0] for a in (prob.Alin_x, prob.Alin_u))
    return dict(N=prob.N, nx=prob.nx, nu=prob.nu, ncx=len(prob.Acx), ncu=len(prob.Acu), nlx=nlx, nlu=nlu)


def per_instance(kind: str, arrays: dict, B: int, dims: dict, dtype) -> tuple:
    """Check one kind's per-instance arrays (a dict keyed as users write them; numpy arrays or torch tensors of the problem
    dtype) against a batch of B instances of a problem of these dims (problem_dims) -> (the ABI mode, {ABI field: the array
    in ABI layout}).  A side may be absent when its loop does not run; the keys of a pair come together."""
    spec = KINDS[kind]
    unknown = set(arrays) - set(spec.fields)
    if unknown:
        raise ValueError(f"{kind}: unknown keys {sorted(unknown)}; expected any of {tuple(spec.fields)}")
    given = {k: v for k, v in arrays.items() if v is not None}
    if not given:
        raise ValueError(f"{kind}: give any of {tuple(spec.fields)}")
    for a, b in spec.pairs:
        if (a in given) != (b in given):
            raise ValueError(f"{kind}: {a} and {b} are given in pairs")
    want, shapes, modes = np.dtype(dtype), spec.shapes(dims, B), set()
    for k, a in given.items():
        dt = getattr(a, "dtype", None)
        if dt is None or str(dt).replace("torch.", "") != want.name:
            raise ValueError(f"{kind}: {k} must have the problem dtype {want.name}, got {dt}")
        if tuple(a.shape) not in shapes[k]:
            raise ValueError(f"{kind}: {k} must be {' or '.join(str(list(sh)) for sh in shapes[k])}, got {list(a.shape)}")
        modes.add(shapes[k][tuple(a.shape)])
    if len(modes) != 1:
        raise ValueError(f"{kind}: every array takes the same layout, got {sorted(given)} in modes {sorted(modes)}")
    return modes.pop(), {spec.fields[k]: spec.to_abi(k, a) for k, a in given.items()}


# the key lists and the plane check and conversion under the names other modules and the tests import, all views of KINDS
BOUND_NAMES = tuple(KINDS["bounds"].fields)
PLANE_NAMES = tuple(KINDS["planes"].fields)


def planes_check(planes: dict, B: int, nlx: int, nlu: int, nx: int, nu: int, dtype) -> None:
    """per_instance's checks of per-instance static hyperplanes, for a problem with nlx / nlu rows"""
    per_instance("planes", planes, B, dict(nx=nx, nu=nu, nlx=nlx, nlu=nlu), dtype)


def planes_abi(planes: dict) -> dict:
    """the given arrays of a checked planes dict in the ABI's layout (each matrix a column-major view)"""
    return {k: KINDS["planes"].to_abi(k, v) for k, v in planes.items() if v is not None}


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
        # per-instance data (see KINDS): self.bounds / cones / planes = {ABI field: host array in ABI layout}; mode 0 = the problem's
        self.modes = {}
        for kind, arrays in dict(bounds=bounds, cones=cones, planes=planes).items():
            mode, abi_arrays = (0, {}) if arrays is None else per_instance(kind, arrays, B, problem_dims(prob), dt)
            self.modes[kind] = mode
            setattr(self, kind, {f: np.ascontiguousarray(a) for f, a in abi_arrays.items()})
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
        for kind, spec in KINDS.items():
            setattr(b, spec.mode_field, self.modes[kind])
            for f, a in getattr(self, kind).items():
                setattr(b, f, a.ctypes.data)
        b._owner = self
        return b

    def result(self) -> dict:
        out = dict(sol_x=self.sol_x, sol_u=self.sol_u, iter=self.iter, solved=self.solved, residuals=self.residuals)
        out.update(self.state)
        return out
