"""CPU-side checks of the C ABI: the shared library loads, exports every symbol include/tinympc_b200.h
declares, the ctypes mirrors match the C structs, and argument errors are reported without a GPU."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from tinympc_b200 import abi
from tinympc_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tinympc_b200.h")


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    declared = set(re.findall(r"\b(tinympc_b200_[a-z_0-9]+)\s*\(", open(HEADER).read()))
    assert declared == set(abi.EXPORTS), declared ^ set(abi.EXPORTS)
    for n in declared:
        assert hasattr(lib, n), n
    assert b"sm_90a" in lib.tinympc_b200_version()


def test_struct_layout_matches_header():
    src = r'''
#include <stdio.h>
#include <stddef.h>
#include "tinympc_b200.h"
int main(void){
  printf("%zu %zu %zu %zu %zu\n", sizeof(tinympc_problem_t), sizeof(tinympc_settings_t), sizeof(tinympc_state_t), sizeof(tinympc_batch_t), sizeof(tinympc_b200_stats_t));
  printf("%zu %zu %zu %zu\n", offsetof(tinympc_problem_t, Kinf), offsetof(tinympc_problem_t, tv_blin_u), offsetof(tinympc_batch_t, state), offsetof(tinympc_batch_t, residuals));
  return 0; }
'''
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "probe.c")
        open(c, "w").write(src)
        exe = os.path.join(td, "probe")
        subprocess.check_call(["/usr/bin/gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = subprocess.check_output([exe], text=True).split()
    sizes = list(map(int, out))
    assert sizes[:5] == [C.sizeof(abi.Problem), C.sizeof(abi.Settings), C.sizeof(abi.State), C.sizeof(abi.Batch), C.sizeof(abi.Stats)]
    assert sizes[5:] == [abi.Problem.Kinf.offset, abi.Problem.tv_blin_u.offset, abi.Batch.state.offset, abi.Batch.residuals.offset]


def test_default_settings_match_reference_constants():
    lib = _lib.load()
    s = abi.Settings()
    assert lib.tinympc_b200_default_settings(C.byref(s)) == 0
    # tiny_api_constants.hpp:5-16
    assert (s.abs_pri_tol, s.abs_dua_tol, s.max_iter, s.check_termination) == (1e-3, 1e-3, 1000, 1)
    assert (s.en_state_bound, s.en_input_bound, s.en_state_soc, s.en_input_soc) == (1, 1, 0, 0)
    assert (s.en_state_linear, s.en_input_linear, s.en_tv_state_linear, s.en_tv_input_linear) == (0, 0, 0, 0)


def test_supported_dims_and_errors():
    lib = _lib.load()
    for nx, nu in ((4, 1), (6, 3), (12, 4), (16, 8), (8, 2)):
        assert lib.tinympc_b200_supported(abi.F32, nx, nu) == 1
        assert lib.tinympc_b200_supported(abi.F64, nx, nu) == 1
    assert lib.tinympc_b200_supported(abi.F32, 5, 7) == 0
    assert lib.tinympc_b200_create(None, 0, None) == abi.ERR_ARG
    assert b"null" in lib.tinympc_b200_last_error()
    p = abi.Problem()
    p.nx, p.nu, p.N, p.dtype = 5, 7, 10, abi.F32
    h = C.c_void_p()
    assert lib.tinympc_b200_create(C.byref(p), 0, C.byref(h)) == abi.ERR_ARG  # null model pointers


def test_product_precompute_matches_oracle_port():
    """tiny_precompute_and_set_cache restated in the product (host C++) vs the oracle's C restatement."""
    import helpers as H
    from oracle import oracle
    from tinympc_b200.solver import setup_problem

    cases = H.make_cases()
    for name in ("cartpole_f64", "quad_hover_N10_f64", "rocket_soc_N10_f64", "lti_8_2_f64", "quad_hover_N10_f32"):
        c = cases[name]
        mine = setup_problem(c["spec"], c["dtype"])
        ref = H.problem_from_spec(c["spec"], c["dtype"], oracle.port_setup)
        tol = 1e-9 if c["dtype"] == np.float64 else 2e-3
        assert mine.riccati_sweeps == ref.riccati_iters or c["dtype"] == np.float32
        for f in ("Q", "R", "Kinf", "Pinf", "Quu_inv", "AmBKt", "APf", "BPf"):
            a, b = getattr(mine, f), getattr(ref, f)
            assert np.allclose(a, b, rtol=tol, atol=tol * max(1.0, float(np.abs(b).max()))), (name, f)


def test_batched_precompute_equals_per_instance_precompute():
    """tinympc_b200_precompute_cache_batch packs, per instance, exactly what the single-model precompute returns."""
    from tinympc_b200 import workloads as wl
    from tinympc_b200.solver import setup_models, setup_problem, unpack_model

    nx, nu, N = 8, 2, 10
    specs = [wl.random_lti(nx, nu, N, seed=100 + i) for i in range(7)]
    for dt in (np.float64, np.float32):
        blobs = setup_models(nx, nu, np.stack([s.A for s in specs]), np.stack([s.B for s in specs]), np.stack([s.f for s in specs]),
                             np.stack([s.Qdiag for s in specs]), np.stack([s.Rdiag for s in specs]),
                             np.array([0.5 + 0.25 * i for i in range(7)]), dtype=dt, nthreads=3)
        assert blobs.shape == (7, 3 * nx * nx + 2 * nx * nu + nu * nu + 3 * nx + 2 * nu + 1)
        for i, sp in enumerate(specs):
            sp.rho = 0.5 + 0.25 * i
            one = setup_problem(sp, dt)
            m = unpack_model(blobs[i], nx, nu)
            for f in ("A", "B", "f", "Q", "R", "Kinf", "Pinf", "Quu_inv", "AmBKt", "APf", "BPf"):
                assert np.array_equal(np.asarray(getattr(one, f)), m[f]), (i, f)
            assert m["rho"] == float(dt(sp.rho))
