"""The adaptive-rho sensitivity tables on the host (tinympc_b200_precompute_sensitivity_batch): the tables are the derivative,
with respect to rho, of the Kinf / Pinf the batched precompute returns.  Checked against an independent numpy restatement of
the tangent recursion and against a finite difference of the primal; plus the test oracle's per-instance-table path."""
import ctypes as C
import os

import numpy as np
import pytest

import adaptive_common as AC
import helpers as H
import sensitivity_common as SC
from tinympc_b200 import abi
from tinympc_b200._lib import TinyMPCError, load
from tinympc_b200.solver import AdaptiveRho, setup_models, setup_sensitivity, unpack_model

MODELS = SC.named_models()


def _one(sp, dt, rho=None, nthreads=1):
    rho = sp.rho if rho is None else rho
    return [a[0] for a in setup_sensitivity(sp.nx, sp.nu, sp.A[None], np.reshape(sp.B, (1, sp.nx, sp.nu)), sp.f[None], sp.Qdiag[None],
                                            sp.Rdiag[None], [rho], dtype=dt, nthreads=nthreads)]


def _rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / np.abs(b).max())


@pytest.mark.parametrize("name", sorted(MODELS))
def test_definition(name):
    """fp64 tables = the numpy tangent recursion (stopped by the same test, so the sweep counts agree too) = a central
    finite difference of the primal at that FIXED sweep count.  (Two independently stopped runs differ by up to the 1e-5 stop
    tolerance, which a difference quotient with h = 1e-4 rho would turn into noise of order 0.1 / rho.)"""
    sp = MODELS[name]
    B = np.reshape(sp.B, (sp.nx, sp.nu))
    dK, dP = _one(sp, np.float64)
    K, P, dK_np, dP_np, sweeps = SC.riccati(sp.A, B, sp.Qdiag, sp.Rdiag, sp.rho)
    blob = setup_models(sp.nx, sp.nu, sp.A[None], B[None], sp.f[None], sp.Qdiag[None], sp.Rdiag[None], [sp.rho], dtype=np.float64)[0]
    m = unpack_model(blob, sp.nx, sp.nu)
    assert _rel(m["Kinf"], K) <= 1e-10 and _rel(m["Pinf"], P) <= 1e-10  # the restatement's primal is the library's
    assert _rel(dK, dK_np) <= 1e-10 and _rel(dP, dP_np) <= 1e-10, (name, _rel(dK, dK_np), _rel(dP, dP_np))
    h = 1e-4 * sp.rho
    Kp, Pp = SC.riccati(sp.A, B, sp.Qdiag, sp.Rdiag, sp.rho + h, sweeps)[:2]
    Km, Pm = SC.riccati(sp.A, B, sp.Qdiag, sp.Rdiag, sp.rho - h, sweeps)[:2]
    assert _rel(dK, (Kp - Km) / (2 * h)) <= 1e-6 and _rel(dP, (Pp - Pm) / (2 * h)) <= 1e-6, name


# fp32 against fp64, relative to the table's largest entry.  Measured on these six models: quadrotor 1.2e-4 (dK and dP) and
# cartpole 1.1e-4 (dK) are the largest, the rocket is at 1.2e-5 and the random LTI systems below 1e-6; the bound leaves a
# factor of about eight.
FP32_TOL = 1e-3


@pytest.mark.parametrize("name", sorted(MODELS))
def test_fp32_tables_against_fp64(name):
    sp = MODELS[name]
    dK32, dP32 = _one(sp, np.float32)
    dK64, dP64 = _one(sp, np.float64)
    assert dK32.dtype == np.float32 and dP32.dtype == np.float32
    print(f"{name}: fp32 vs fp64 dK {_rel(dK32, dK64):.2e} dP {_rel(dP32, dP64):.2e}")
    assert _rel(dK32, dK64) <= FP32_TOL and _rel(dP32, dP64) <= FP32_TOL, name


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_thread_count_invariance_and_batch_order(dt):
    """1 and 8 threads give the same bits, and instance b's tables are those of model b computed alone."""
    A, Bm, f, Q, R, rho = SC.lti_batch(8, 4, 37, seed=3)
    one = setup_sensitivity(8, 4, A, Bm, f, Q, R, rho, dtype=dt, nthreads=1)
    many = setup_sensitivity(8, 4, A, Bm, f, Q, R, rho, dtype=dt, nthreads=8)
    for a, b in zip(one, many):
        assert H.bits_equal(np.ascontiguousarray(a), np.ascontiguousarray(b))
    for b in (0, 17, 36):
        alone = setup_sensitivity(8, 4, A[b:b + 1], Bm[b:b + 1], f[b:b + 1], Q[b:b + 1], R[b:b + 1], rho[b:b + 1], dtype=dt)
        assert H.bits_equal(np.ascontiguousarray(alone[0][0]), np.ascontiguousarray(one[0][b]))
        assert H.bits_equal(np.ascontiguousarray(alone[1][0]), np.ascontiguousarray(one[1][b]))
    assert one[0].shape == (37, 4, 8) and one[1].shape == (37, 8, 8)


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_singular_model_is_reported_like_the_cache_call(dt):
    A, Bm, f, Q, R, rho = SC.lti_batch(4, 2, 9, seed=5, singular_at=6)
    with pytest.raises(TinyMPCError) as e:
        setup_sensitivity(4, 2, A, Bm, f, Q, R, rho, dtype=dt, nthreads=4)
    assert e.value.code == abi.ERR_SINGULAR and "instance 6" in str(e.value)
    with pytest.raises(TinyMPCError) as e2:
        setup_models(4, 2, A, Bm, f, Q, R, rho, dtype=dt, nthreads=4)
    assert e2.value.code == abi.ERR_SINGULAR and "instance 6" in str(e2.value)


def test_argument_errors_and_exports():
    lib = load()
    for n in ("tinympc_b200_precompute_sensitivity_batch", "tinympc_b200_precompute_sensitivity_batch_device"):
        assert hasattr(lib, n) and n in abi.EXPORTS
        assert n in open(os.path.join(AC.ROOT, "include", "tinympc_b200.h")).read()
    a = np.zeros(64)
    p = C.c_void_p(a.ctypes.data)
    call = lib.tinympc_b200_precompute_sensitivity_batch
    assert call(abi.F64, 2, 1, 1, None, p, p, p, p, p, p, p, 1) == abi.ERR_ARG
    assert call(abi.F64, 2, 1, 1, p, p, p, p, p, p, None, p, 1) == abi.ERR_ARG
    assert call(abi.F64, 0, 1, 1, p, p, p, p, p, p, p, p, 1) == abi.ERR_ARG
    assert call(abi.F64, 2, 1, -1, p, p, p, p, p, p, p, p, 1) == abi.ERR_ARG
    assert call(7, 2, 1, 1, p, p, p, p, p, p, p, p, 1) == abi.ERR_ARG
    assert call(abi.F64, 2, 1, 0, p, p, p, p, p, p, p, p, 1) == abi.OK  # an empty batch
    assert lib.tinympc_b200_precompute_sensitivity_batch_device(None, 1, p, p, p, p, p, p, p, p, None, None) == abi.ERR_ARG
    assert C.sizeof(abi.AdaptiveRho) % 8 == 0 and abi.AdaptiveRho.tables_per_instance.offset == abi.AdaptiveRho.models.offset + 8


@pytest.mark.parametrize("name", ["track_N50_f32", "lti_8_4_N10_f64"])
def test_oracle_per_instance_path_equals_shared_path(name):
    """The test oracle's per-instance-table entry point with B equal tables (and with the one shared pair) reproduces its
    shared-table entry point: every output, state field and adapted blob, over the case's closed loop."""
    c = AC.make_cases(with_wide=False)[name]
    ar = c["ar"]
    B = len(c["x0"])
    tile = lambda a: np.ascontiguousarray(np.tile(np.asarray(a)[None], (B, 1, 1)))  # noqa: E731
    ar_b = AdaptiveRho(tile(ar.dKinf_drho), tile(ar.dPinf_drho), ar.rho_min, ar.rho_max, ar.enable_clipping)
    assert ar_b.per_instance and not ar.per_instance
    shared = lambda *a: AC.oracle_solve(*a, ar)  # noqa: E731
    ref, _ = AC.closed_loop(c["prob"], c["st"], c, shared)
    for which in (ar_b, ar):
        got, _ = AC.closed_loop(c["prob"], c["st"], c, lambda *a: SC.oracle_solve_per_instance(*a, which))
        for k in range(c["steps"]):
            H.assert_bits_per_instance(dict(got[k][0], models=got[k][1]), dict(ref[k][0], models=ref[k][1]),
                                       AC.OUT + AC.BOX + ["models"], f"{name} step {k}")


def test_distance_to_the_reference_quadrotor_tables():
    """Informational (printed, not asserted): the reference ships one hard-coded table pair for its quadrotor, produced by a
    script that is not part of it; how far are the tables computed here?"""
    sp = MODELS["quadrotor"]
    t0, t1 = AC.quad_tables(np.float64)
    dK, dP = _one(sp, np.float64)
    print(f"quadrotor rho={sp.rho}: |dK - ref|/|ref| = {_rel(dK, t0):.3e}, |dP - ref|/|ref| = {_rel(dP, t1):.3e}; "
          f"max|dK| {np.abs(dK).max():.4g} (ref {np.abs(t0).max():.4g}), max|dP| {np.abs(dP).max():.4g} (ref {np.abs(t1).max():.4g})")

