"""oracle/oracle.py — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

ctypes front-end to the two CPU checkers:

  * "port"      — oracle/libtinympc_oracle.so, the plain-C restatement (oracle/tinympc_oracle.c);
  * "reference" — oracle/_ref/libtinympc_ref_{f64,f32}[_fast|_fastv3].so, the UNMODIFIED reference
                  (TinyMPC/TinyMPC) compiled by oracle/Makefile + oracle/ref_driver.cpp.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may import this.
The product package (tinympc_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(_HERE))

from tinympc_b200 import abi  # noqa: E402  (struct definitions only)
from tinympc_b200.batch import HostBatch  # noqa: E402
from tinympc_b200.problem import MPCProblem, default_settings, dtype_code  # noqa: E402

_libs = {}


def build(verbose=False):
    """Build the C restatement and, when the TinyMPC checkout (TINYMPC_REFERENCE, default /root/reference) is present,
    the reference libraries."""
    r = subprocess.run(["make", "-C", _HERE, "-j8", "all"], capture_output=True, text=True)
    if verbose or r.returncode:
        print(r.stdout[-4000:], r.stderr[-4000:])
    if r.returncode:
        raise RuntimeError("oracle build failed")


def _load(path):
    if path not in _libs:
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        _libs[path] = C.CDLL(path)
    return _libs[path]


def port_lib():
    path = os.path.join(_HERE, "libtinympc_oracle.so")
    if not os.path.exists(path):
        build()
    lib = _load(path)
    lib.tinympc_oracle_solve_batch.restype = C.c_int
    lib.tinympc_oracle_solve_batch.argtypes = [C.POINTER(abi.Problem), C.POINTER(abi.Settings), C.POINTER(abi.Batch),
                                               C.c_int32]
    lib.tinympc_oracle_precompute_cache.restype = C.c_int
    return lib


def ref_path(dtype, variant=""):
    name = "f64" if np.dtype(dtype) == np.float64 else "f32"
    suffix = f"_{variant}" if variant else ""
    return os.path.join(_HERE, "_ref", f"libtinympc_ref_{name}{suffix}.so")


def ref_available(dtype=np.float64, variant=""):
    return os.path.exists(ref_path(dtype, variant))


def ref_lib(dtype, variant=""):
    lib = _load(ref_path(dtype, variant))
    lib.tinympc_ref_solve_batch.restype = C.c_int
    lib.tinympc_ref_solve_batch.argtypes = [C.POINTER(abi.Problem), C.POINTER(abi.Settings), C.POINTER(abi.Batch),
                                            C.c_int32]
    lib.tinympc_ref_setup_cache.restype = C.c_int
    assert lib.tinympc_ref_dtype() == dtype_code(dtype)
    return lib


def _cache_arrays(nx, nu, dt):
    return dict(Kinf=np.zeros((nu, nx), dt, order="F"), Pinf=np.zeros((nx, nx), dt, order="F"),
                Quu_inv=np.zeros((nu, nu), dt, order="F"), AmBKt=np.zeros((nx, nx), dt, order="F"),
                APf=np.zeros(nx, dt), BPf=np.zeros(nu, dt))


def ref_setup(nx, nu, N, rho, A, B, f, Qdiag, Rdiag, dtype=np.float64, variant="", **constraints) -> MPCProblem:
    """tiny_setup through the compiled reference: returns an MPCProblem whose Q,R and cache are what the
    reference derives (tiny_api.cpp:117-118, 307-381)."""
    dt = np.dtype(dtype).type
    lib = ref_lib(dt, variant)
    A_ = np.asfortranarray(A, dtype=dt)
    B_ = np.asfortranarray(np.asarray(B, dtype=dt).reshape(nx, nu))
    f_ = np.ascontiguousarray(f, dtype=dt)
    Qd = np.ascontiguousarray(Qdiag, dtype=dt)
    Rd = np.ascontiguousarray(Rdiag, dtype=dt)
    Qw, Rw = np.zeros(nx, dt), np.zeros(nu, dt)
    c = _cache_arrays(nx, nu, dt)
    vp = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
    rc = lib.tinympc_ref_setup_cache(C.c_int32(nx), C.c_int32(nu), C.c_int32(N), C.c_double(float(dt(rho))), vp(A_),
                                     vp(B_), vp(f_), vp(Qd), vp(Rd), vp(Qw), vp(Rw), vp(c["Kinf"]), vp(c["Pinf"]),
                                     vp(c["Quu_inv"]), vp(c["AmBKt"]), vp(c["APf"]), vp(c["BPf"]))
    if rc:
        raise RuntimeError(f"tinympc_ref_setup_cache rc={rc}")
    return MPCProblem(nx=nx, nu=nu, N=N, dtype=dt, rho=float(dt(rho)), A=A_, B=B_, f=f_, Q=Qw, R=Rw, **c, **constraints)


def port_setup(nx, nu, N, rho, A, B, f, Qdiag, Rdiag, dtype=np.float64, **constraints) -> MPCProblem:
    """Same as ref_setup with the restated precompute (tolerance-level agreement with Eigen's)."""
    dt = np.dtype(dtype).type
    lib = port_lib()
    A_ = np.asfortranarray(A, dtype=dt)
    B_ = np.asfortranarray(np.asarray(B, dtype=dt).reshape(nx, nu))
    f_ = np.ascontiguousarray(f, dtype=dt)
    rho_t = dt(rho)
    Qw = (np.asarray(Qdiag, dtype=dt) + rho_t).astype(dt)  # tiny_api.cpp:117
    Rw = (np.asarray(Rdiag, dtype=dt) + rho_t).astype(dt)
    c = _cache_arrays(nx, nu, dt)
    vp = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
    rc = lib.tinympc_oracle_precompute_cache(C.c_int32(dtype_code(dt)), C.c_int32(nx), C.c_int32(nu),
                                             C.c_double(float(rho_t)), vp(A_), vp(B_), vp(f_), vp(Qw), vp(Rw),
                                             vp(c["Kinf"]), vp(c["Pinf"]), vp(c["Quu_inv"]), vp(c["AmBKt"]),
                                             vp(c["APf"]), vp(c["BPf"]))
    if rc < 0:
        raise RuntimeError(f"tinympc_oracle_precompute_cache rc={rc}")
    p = MPCProblem(nx=nx, nu=nu, N=N, dtype=dt, rho=float(rho_t), A=A_, B=B_, f=f_, Q=Qw, R=Rw, **c, **constraints)
    p.riccati_iters = rc
    return p


def solve_batch(prob: MPCProblem, settings: abi.Settings | None, x0, Xref, Uref=None, state=None, cold_start=True,
                want_state=(), impl="port", variant="", nthreads=1) -> dict:
    """Batched tiny_solve on the CPU.  impl = "port" (C restatement) or "reference" (compiled reference)."""
    st = settings if settings is not None else default_settings()
    hb = HostBatch(prob, x0, Xref, Uref, state=state, cold_start=cold_start, want_state=want_state)
    cp, cb = prob.to_c(), hb.to_c()
    if impl == "port":
        rc = port_lib().tinympc_oracle_solve_batch(C.byref(cp), C.byref(st), C.byref(cb), nthreads)
    elif impl == "reference":
        rc = ref_lib(prob.dtype, variant).tinympc_ref_solve_batch(C.byref(cp), C.byref(st), C.byref(cb), nthreads)
    else:
        raise ValueError(impl)
    if rc:
        raise RuntimeError(f"{impl} solve_batch rc={rc}")
    return hb.result()


class RefPool:
    """Persistent worker pool around the compiled reference (oracle/ref_driver.cpp: tinympc_ref_pool_*): `nthreads` threads,
    one TinySolver per thread built ONCE through the reference's tiny_setup; used by bench.py's CPU arm so that thread
    spawn and setup stay outside the timed region (BASELINE.md §3.2)."""

    def __init__(self, prob: MPCProblem, settings: abi.Settings | None, nthreads: int, variant=""):
        self.prob = prob
        self.lib = ref_lib(prob.dtype, variant)
        self.lib.tinympc_ref_pool_create.restype = C.c_void_p
        self.lib.tinympc_ref_pool_create.argtypes = [C.POINTER(abi.Problem), C.POINTER(abi.Settings), C.c_int32]
        self.lib.tinympc_ref_pool_solve.restype = C.c_int
        self.lib.tinympc_ref_pool_solve.argtypes = [C.c_void_p, C.POINTER(abi.Batch), C.c_int32, C.POINTER(C.c_double)]
        self.lib.tinympc_ref_pool_destroy.restype = None
        self.lib.tinympc_ref_pool_destroy.argtypes = [C.c_void_p]
        st = settings if settings is not None else default_settings()
        cp = prob.to_c()
        self.nthreads = int(nthreads)
        self.h = self.lib.tinympc_ref_pool_create(C.byref(cp), C.byref(st), self.nthreads)
        if not self.h:
            raise RuntimeError("tinympc_ref_pool_create failed")

    def solve(self, hb: HostBatch, chunk=16):
        """One batched tiny_solve of `hb` on the pool; returns the wall seconds measured inside the driver."""
        cb = hb.to_c()
        sec = C.c_double(0.0)
        rc = self.lib.tinympc_ref_pool_solve(self.h, C.byref(cb), chunk, C.byref(sec))
        if rc:
            raise RuntimeError(f"tinympc_ref_pool_solve rc={rc}")
        return sec.value

    def close(self):
        if self.h:
            self.lib.tinympc_ref_pool_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
