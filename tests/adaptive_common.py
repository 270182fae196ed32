"""Shared by the adaptive-rho tests and tests/golden/make_golden_adaptive.py: the C restatement of the adaptive solve
(tests/adaptive/adaptive_oracle.c, compiled into a temporary directory on first use), the fixture cases and the
closed loop they run."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

import helpers as H
from oracle import oracle
from tinympc_b200 import abi
from tinympc_b200 import workloads as wl
from tinympc_b200.batch import HostBatch
from tinympc_b200.solver import AdaptiveRho, pack_models

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ADIR = os.path.join(HERE, "adaptive")
GOLDEN = os.path.join(HERE, "golden", "adaptive")
BOX = ["x", "u", "v", "z", "vnew", "znew", "g", "y"]
OUT = ["sol_x", "sol_u", "iter", "solved", "residuals"]
_lib = {}


def oracle_lib():
    if "port" not in _lib:
        td = tempfile.mkdtemp(prefix="tinympc_adaptive_oracle_")
        so = os.path.join(td, "libadaptive_oracle.so")
        subprocess.check_call(["gcc", "-std=c11", "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-Wall",
                               "-Wno-unused-function", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "oracle"),
                               "-o", so, os.path.join(ADIR, "adaptive_oracle.c"), "-lm"])
        lib = C.CDLL(so)
        lib.tinympc_adaptive_oracle_solve_batch.restype = C.c_int
        lib.tinympc_adaptive_oracle_solve_batch.argtypes = [C.POINTER(abi.Problem), C.POINTER(abi.Settings), C.POINTER(abi.Batch),
                                                           C.POINTER(abi.AdaptiveRho), C.c_int32]
        _lib["port"] = lib
        shutil.rmtree(td, ignore_errors=True)  # the mapping stays valid after the file is unlinked
    return _lib["port"]


def oracle_solve(prob, st, x0, Xref, Uref, state, cold, models, ar: AdaptiveRho, lib=None, fn="tinympc_adaptive_oracle_solve_batch",
                 nthreads=8):
    """One batched adaptive solve on the CPU; returns (result dict with the box state, adapted models)."""
    hb = HostBatch(prob, x0, Xref, Uref, state=state, cold_start=cold, want_state=BOX)
    m = np.array(models, dtype=prob.dtype).reshape(hb.B, -1)
    cp, cb, ca = prob.to_c(), hb.to_c(), ar.to_c(prob, m.ctypes.data)
    lib = lib if lib is not None else oracle_lib()
    if fn == "tinympc_adaptive_oracle_solve_batch":
        rc = lib.tinympc_adaptive_oracle_solve_batch(C.byref(cp), C.byref(st), C.byref(cb), C.byref(ca), nthreads)
    else:
        rc = getattr(lib, fn)(C.byref(cp), C.byref(st), C.byref(cb), C.byref(ca))
    if rc:
        raise RuntimeError(f"{fn} rc={rc}")
    return hb.result(), m


def advance(prob, x0, u0):
    """x0 <- (A x0 + B u0) + f with ascending sums and no FMA (tinympc_b200_advance's arithmetic)."""
    A, Bm, f = prob.A, prob.B, prob.f
    nxt = np.zeros_like(x0)
    for i in range(prob.nx):
        ax = A[i, 0] * x0[:, 0]
        for m in range(1, prob.nx):
            ax = ax + A[i, m] * x0[:, m]
        bu = Bm[i, 0] * u0[:, 0]
        for j in range(1, prob.nu):
            bu = bu + Bm[i, j] * u0[:, j]
        nxt[:, i] = (ax + bu) + f[i]
    return nxt


def closed_loop(prob, st, c, solve, x0_seq=None):
    """c["steps"] warm-started solves; the adapted models and the box state carry over, x0 advances with u_0.
    solve(prob, st, x0, Xref, Uref, state, cold, models) -> (result, models).  Returns [(result, models)], x0 sequence."""
    x0 = c["x0"].copy()
    models, state, outs, x0s = c["models"].copy(), None, [], []
    for k in range(c["steps"]):
        if x0_seq is not None:
            x0 = np.array(x0_seq[k])
        x0s.append(x0.copy())
        Xref = c["Xref"] if c["Xref"].ndim == 2 else np.ascontiguousarray(np.roll(c["Xref"], -k, axis=1))
        res, models = solve(prob, st, x0, Xref, None, state, state is None, models)
        outs.append((res, models.copy()))
        # copies: a solve updates the state arrays it is given in place, and res must keep this step's values
        state = {n: res[n].copy() for n in BOX}
        x0 = advance(prob, x0, np.ascontiguousarray(res["u"][:, 0, :]))
    return outs, x0s


def quad_tables(dt):
    d = np.load(os.path.join(H.REFERENCE_DIR, "sensitivity_tables.npz"))
    return np.asarray(d["t0"], dtype=dt), np.asarray(d["t1"], dtype=dt)


def _spec_case(spec, dt, B, inst, steps, tables, clip=(1.0, 100.0, True), max_iter=None, tol=None, seed=0):
    prob = H.problem_from_spec(spec, dt, oracle.port_setup)
    st = abi.Settings()
    C.memmove(C.byref(st), C.byref(spec.settings), C.sizeof(abi.Settings))
    if max_iter is not None:
        st.max_iter = max_iter
    if tol is not None:
        st.abs_pri_tol = st.abs_dua_tol = tol
    models = pack_models(prob, B)
    rng = np.random.default_rng(seed)
    # instances start from slightly different rho (and therefore different sensitivity-corrected caches)
    models[:, -1] = (prob.rho * (1.0 + 0.02 * rng.uniform(-1, 1, B))).astype(dt)
    dK, dP = tables
    return dict(prob=prob, st=st, x0=np.ascontiguousarray(inst["x0"], dtype=dt), Xref=np.ascontiguousarray(inst["Xref"], dtype=dt),
                models=models, steps=steps, ar=AdaptiveRho(dK, dP, clip[0], clip[1], clip[2]))


def _lti_tables(nx, nu, dt, seed):
    rng = np.random.default_rng(seed)
    return (0.01 * rng.standard_normal((nu, nx))).astype(dt), (0.01 * rng.standard_normal((nx, nx))).astype(dt)


def make_cases(with_wide=True):
    """name -> case.  The GPU runs every case but the 4-column-block one ("wide_*")."""
    cases = {}
    for dt in (np.float32, np.float64):
        tag = "f32" if dt == np.float32 else "f64"
        tq = quad_tables(dt)
        for N in (10, 50, 100):
            sp = wl.quadrotor(N=N)
            inst = wl.hovering_instances(16, N=N, dtype=dt)
            inst["x0"] = inst["x0"] + (0.3 * np.random.default_rng(N).standard_normal((16, 12))).astype(dt)
            cases[f"hover_N{N}_{tag}"] = _spec_case(sp, dt, 16, inst, 4, tq, seed=N)
        sp = wl.quadrotor(N=50)
        cases[f"track_N50_{tag}"] = _spec_case(sp, dt, 48, wl.tracking_instances(48, N=50, seed=5, dtype=dt), 4, tq, seed=1)
        cases[f"track_clipbind_{tag}"] = _spec_case(sp, dt, 16, wl.tracking_instances(16, N=50, seed=6, dtype=dt), 4, tq,
                                                    clip=(4.99, 5.0, True), seed=2)
        cases[f"track_noclip_{tag}"] = _spec_case(sp, dt, 16, wl.tracking_instances(16, N=50, seed=7, dtype=dt), 4, tq,
                                                  clip=(1.0, 100.0, False), seed=3)
        for mi in (6, 11):
            cases[f"track_maxit{mi}_{tag}"] = _spec_case(sp, dt, 16, wl.tracking_instances(16, N=50, seed=mi, dtype=dt), 4, tq,
                                                         max_iter=mi, seed=mi)
        sp = wl.random_lti(8, 4, 10, seed=2)
        inst = wl.random_instances(16, 8, 10, seed=4, dtype=dt)
        cases[f"lti_8_4_N10_{tag}"] = _spec_case(sp, dt, 16, inst, 4, _lti_tables(8, 4, dt, 11), clip=(0.1, 100.0, True), seed=4)
        if with_wide:
            sp = wl.random_lti(16, 8, 200, seed=3)
            inst = wl.random_instances(4, 16, 200, seed=5, dtype=dt)
            cases[f"wide_16_8_N200_{tag}"] = _spec_case(sp, dt, 4, inst, 2, _lti_tables(16, 8, dt, 12), clip=(0.1, 100.0, True),
                                                         max_iter=20, seed=5)
    return cases


def digests(res, models):
    return [H.digest(res[k]) for k in OUT + BOX] + [H.digest(models)]
