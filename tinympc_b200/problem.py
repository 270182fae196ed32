"""Host-side problem description for the batched solve path.

`MPCProblem` is the read-only part of the reference's TinyWorkspace + TinyCache
(TinyMPC src/tinympc/types.hpp:43-59, 88-208) as numpy arrays; `Settings` mirrors TinySettings
(types.hpp:63-82, defaults tiny_api_constants.hpp:5-16).  All matrices are stored COLUMN-MAJOR
(Fortran order), exactly as the reference's dynamic Eigen matrices, so that `.ctypes.data` can be handed
straight to the C ABI (include/tinympc_b200.h).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from . import abi

NP_DTYPE = {abi.F32: np.float32, abi.F64: np.float64}


def dtype_code(dt) -> int:
    dt = np.dtype(dt)
    if dt == np.float32:
        return abi.F32
    if dt == np.float64:
        return abi.F64
    raise ValueError(f"unsupported dtype {dt}")


def default_settings() -> abi.Settings:
    """tiny_set_default_settings (tiny_api.cpp:413-441)."""
    return abi.Settings(
        abs_pri_tol=1e-3, abs_dua_tol=1e-3, max_iter=1000, check_termination=1,
        en_state_bound=1, en_input_bound=1, en_state_soc=0, en_input_soc=0,
        en_state_linear=0, en_input_linear=0, en_tv_state_linear=0, en_tv_input_linear=0,
    )


def _f(a, dt, shape=None):
    a = np.asfortranarray(np.asarray(a, dtype=dt))
    if shape is not None:
        a = np.asfortranarray(a.reshape(shape, order="F"))
    return a


@dataclass
class MPCProblem:
    nx: int
    nu: int
    N: int
    dtype: type
    rho: float
    A: np.ndarray
    B: np.ndarray
    f: np.ndarray
    Q: np.ndarray  # work->Q = diag(Q_user) + rho
    R: np.ndarray  # work->R = diag(R_user) + rho
    Kinf: np.ndarray = None
    Pinf: np.ndarray = None
    Quu_inv: np.ndarray = None
    AmBKt: np.ndarray = None
    APf: np.ndarray = None
    BPf: np.ndarray = None
    x_min: Optional[np.ndarray] = None  # nx x N
    x_max: Optional[np.ndarray] = None
    u_min: Optional[np.ndarray] = None  # nu x (N-1)
    u_max: Optional[np.ndarray] = None
    # cones: state triple / input triple (order of the reference DEFINITION, tiny_api.cpp:176-178)
    Acx: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    qcx: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    cx: np.ndarray = field(default_factory=lambda: np.zeros(0))
    Acu: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    qcu: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    cu: np.ndarray = field(default_factory=lambda: np.zeros(0))
    Alin_x: Optional[np.ndarray] = None  # n x nx
    blin_x: Optional[np.ndarray] = None
    Alin_u: Optional[np.ndarray] = None
    blin_u: Optional[np.ndarray] = None
    tv_Alin_x: Optional[np.ndarray] = None  # (n*N) x nx
    tv_blin_x: Optional[np.ndarray] = None  # n x N
    tv_Alin_u: Optional[np.ndarray] = None
    tv_blin_u: Optional[np.ndarray] = None

    def __post_init__(self):
        dt = np.dtype(self.dtype)
        self.dtype = dt.type
        nx, nu, N = self.nx, self.nu, self.N
        self.A = _f(self.A, dt, (nx, nx))
        self.B = _f(self.B, dt, (nx, nu))
        self.f = _f(self.f, dt, (nx,))
        self.Q = _f(self.Q, dt, (nx,))
        self.R = _f(self.R, dt, (nu,))
        for name, shape in (("Kinf", (nu, nx)), ("Pinf", (nx, nx)), ("Quu_inv", (nu, nu)), ("AmBKt", (nx, nx)),
                            ("APf", (nx,)), ("BPf", (nu,))):
            v = getattr(self, name)
            if v is not None:
                setattr(self, name, _f(v, dt, shape))
        for name, shape in (("x_min", (nx, N)), ("x_max", (nx, N)), ("u_min", (nu, N - 1)), ("u_max", (nu, N - 1))):
            v = getattr(self, name)
            if v is not None:
                v = np.asarray(v, dtype=dt)
                if v.ndim <= 1:  # per-row constants replicated over the horizon, as every example does
                    v = np.broadcast_to(v.reshape(-1, 1), shape)
                setattr(self, name, _f(v, dt, shape))
        for name in ("Acx", "qcx", "Acu", "qcu"):
            setattr(self, name, np.ascontiguousarray(getattr(self, name), dtype=np.int32))
        self.cx = _f(self.cx, dt)
        self.cu = _f(self.cu, dt)
        for name in ("Alin_x", "blin_x", "Alin_u", "blin_u", "tv_Alin_x", "tv_blin_x", "tv_Alin_u", "tv_blin_u"):
            v = getattr(self, name)
            if v is not None:
                setattr(self, name, _f(v, dt))

    # ---- shapes -------------------------------------------------------------------------------------
    @property
    def nN(self):
        return self.nx * self.N

    @property
    def mN(self):
        return self.nu * (self.N - 1)

    def astype(self, dt) -> "MPCProblem":
        """Same problem with every floating-point table rounded to `dt` (fp32 copy of an fp64 problem)."""
        kw = {k: getattr(self, k) for k in self.__dataclass_fields__}
        kw["dtype"] = dt
        return MPCProblem(**kw)

    def has_cache(self):
        return self.Kinf is not None

    # ---- C view -------------------------------------------------------------------------------------
    def to_c(self) -> abi.Problem:
        """ctypes view; the returned struct keeps `self` alive through ._owner."""
        p = abi.Problem()
        p.nx, p.nu, p.N = self.nx, self.nu, self.N
        p.dtype = dtype_code(self.dtype)
        p.rho = float(self.dtype(self.rho))

        def ptr(a):
            return None if a is None or a.size == 0 else a.ctypes.data

        p.Adyn, p.Bdyn, p.fdyn, p.Q, p.R = map(ptr, (self.A, self.B, self.f, self.Q, self.R))
        p.Kinf, p.Pinf, p.Quu_inv, p.AmBKt = map(ptr, (self.Kinf, self.Pinf, self.Quu_inv, self.AmBKt))
        p.APf, p.BPf = ptr(self.APf), ptr(self.BPf)
        p.x_min, p.x_max, p.u_min, p.u_max = map(ptr, (self.x_min, self.x_max, self.u_min, self.u_max))
        p.num_state_cones, p.num_input_cones = len(self.Acx), len(self.Acu)
        p.Acx, p.qcx, p.cx = ptr(self.Acx), ptr(self.qcx), ptr(self.cx)
        p.Acu, p.qcu, p.cu = ptr(self.Acu), ptr(self.qcu), ptr(self.cu)
        p.num_state_linear = 0 if self.Alin_x is None else self.Alin_x.shape[0]
        p.num_input_linear = 0 if self.Alin_u is None else self.Alin_u.shape[0]
        p.Alin_x, p.blin_x, p.Alin_u, p.blin_u = map(ptr, (self.Alin_x, self.blin_x, self.Alin_u, self.blin_u))
        p.num_tv_state_linear = 0 if self.tv_Alin_x is None else self.tv_Alin_x.shape[0] // self.N
        p.num_tv_input_linear = 0 if self.tv_Alin_u is None else self.tv_Alin_u.shape[0] // (self.N - 1)
        p.tv_Alin_x, p.tv_blin_x = ptr(self.tv_Alin_x), ptr(self.tv_blin_x)
        p.tv_Alin_u, p.tv_blin_u = ptr(self.tv_Alin_u), ptr(self.tv_blin_u)
        p._owner = self
        return p


def copy_settings(s: abi.Settings) -> abi.Settings:
    out = abi.Settings()
    C.memmove(C.byref(out), C.byref(s), C.sizeof(abi.Settings))
    return out
