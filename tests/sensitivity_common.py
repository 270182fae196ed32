"""Shared by the sensitivity-table tests (tests/test_sensitivity.py, tests/test_gpu_sensitivity.py): an independent numpy fp64
restatement of the tangent recursion, the model sets, and the adaptive-rho restatement's per-instance-table entry point
(tests/adaptive/adaptive_oracle_per_instance.c, compiled into a temporary directory on first use)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

import adaptive_common as AC
from tinympc_b200 import abi
from tinympc_b200 import workloads as wl

PER_INSTANCE_FN = "tinympc_adaptive_oracle_solve_batch_per_instance"
_lib = {}


def riccati(A, B, Qdiag, Rdiag, rho, sweeps=None):
    """fp64 numpy: Kinf, Pinf of the batched precompute (Q1 = Qdiag + 2 rho, R1 = Rdiag + 2 rho, P0 = rho I) and their
    tangents with respect to rho.  sweeps = None: stop like the library (max|K - K_prev| < 1e-5, at most 1000); else exactly
    that many sweeps.  Returns K, P, dK, dP, sweeps."""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    nx, nu = B.shape
    Q1, R1 = np.diag(np.asarray(Qdiag, np.float64) + 2.0 * rho), np.diag(np.asarray(Rdiag, np.float64) + 2.0 * rho)
    dQ1, dR1 = 2.0 * np.eye(nx), 2.0 * np.eye(nu)
    P, dP, Kprev = rho * np.eye(nx), np.eye(nx), np.zeros((nu, nx))
    it = 0
    while True:
        S = R1 + B.T @ P @ B
        K = np.linalg.solve(S, B.T @ P @ A)
        dS = dR1 + B.T @ dP @ B
        dK = np.linalg.solve(S, B.T @ dP @ A - dS @ K)
        Pn = Q1 + A.T @ P @ (A - B @ K)
        dPn = dQ1 + A.T @ dP @ (A - B @ K) - A.T @ P @ B @ dK
        it += 1
        if (sweeps is None and (np.abs(K - Kprev).max() < 1e-5 or it == 1000)) or it == sweeps:
            return K, Pn, dK, dPn, it
        Kprev, P, dP = K, Pn, dPn


def named_models():
    """name -> ModelSpec: the quadrotor, the cartpole, the rocket and random LTI systems at three (nx, nu) pairs"""
    m = {"quadrotor": wl.quadrotor(N=10), "cartpole": wl.cartpole(N=10), "rocket": wl.rocket(N=10)}
    for nx, nu in ((4, 2), (8, 4), (16, 8)):
        m[f"lti_{nx}_{nu}"] = wl.random_lti(nx, nu, 10, seed=7)
    return m


def lti_batch(nx, nu, B, seed=0, singular_at=None):
    """B random models (A, B, f, Qdiag, Rdiag, rho), row index first; singular_at: that model has B = 0 and R = -2 rho, so
    that R1 + B'PB is the zero matrix from the first sweep on."""
    rng = np.random.default_rng(seed)
    A = np.eye(nx)[None] + 0.03 * rng.standard_normal((B, nx, nx))
    Bm = 0.5 * rng.standard_normal((B, nx, nu))
    f = 0.01 * rng.standard_normal((B, nx))
    Q = rng.uniform(1.0, 10.0, (B, nx))
    R = rng.uniform(0.5, 2.0, (B, nu))
    rho = rng.uniform(0.5, 5.0, B)
    if singular_at is not None:
        Bm[singular_at] = 0.0
        rho[singular_at] = 1.0  # R + rho + rho is exactly 0 in fp32 and fp64
        R[singular_at] = -2.0
    return A, Bm, f, Q, R, rho


def tuned_quadrotor_fleet(N, nm=6):
    """One quadrotor, per-robot tuning: rho and the state weights differ (six models by default).  Returns the spec and
    (A, B, f, Qdiag, Rdiag, rho) with a leading model dimension."""
    sp = wl.quadrotor(N=N)
    k = np.arange(nm)
    t = lambda a: np.tile(np.asarray(a, np.float64)[None], (nm,) + (1,) * np.ndim(a))  # noqa: E731
    return sp, (t(sp.A), t(sp.B), t(sp.f), t(sp.Qdiag) * (1.0 + 0.25 * k)[:, None], t(sp.Rdiag), sp.rho * (0.6 + 0.2 * k))


def deal(B, nm=6, stride=5):
    """instance b uses model (stride * b) % nm: neighbouring slots, and a slot before and after a refill, differ"""
    return (stride * np.arange(B)) % nm


def per_instance_oracle_lib():
    if "lib" not in _lib:
        td = tempfile.mkdtemp(prefix="tinympc_adaptive_oracle_pi_")
        so = os.path.join(td, "libadaptive_oracle_pi.so")
        subprocess.check_call(["gcc", "-std=c11", "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-Wall",
                               "-Wno-unused-function", "-I", os.path.join(AC.ROOT, "include"), "-I", os.path.join(AC.ROOT, "oracle"),
                               "-I", AC.ADIR, "-o", so, os.path.join(AC.ADIR, "adaptive_oracle_per_instance.c"), "-lm"])
        lib = C.CDLL(so)
        fn = getattr(lib, PER_INSTANCE_FN)
        fn.restype = C.c_int
        fn.argtypes = [C.POINTER(abi.Problem), C.POINTER(abi.Settings), C.POINTER(abi.Batch), C.POINTER(abi.AdaptiveRho)]
        _lib["lib"] = lib
        shutil.rmtree(td, ignore_errors=True)  # the mapping stays valid after the file is unlinked
    return _lib["lib"]


def oracle_solve_per_instance(prob, st, x0, Xref, Uref, state, cold, models, ar):
    """AC.oracle_solve through the per-instance-table entry point (ar with shared or per-instance tables)"""
    return AC.oracle_solve(prob, st, x0, Xref, Uref, state, cold, models, ar, lib=per_instance_oracle_lib(), fn=PER_INSTANCE_FN)
