"""The scripted driver of the reference interface (tests/shim/shim_script.cpp), built with the unmodified reference
(oracle/_ref/shim_tests/script_ref), held to the batch oracle on the CPU: a bug in the driver must not hide a bug in the
shim that tests/test_gpu_shim_parity.py compares with it.  Plain warm-started closed loops (box, cones, static and
time-varying hyperplanes) must dump exactly what oracle.solve_batch(impl="reference") computes stepping the same loop
through the batch ABI, and the driver's restatement of tiny_solve_batch must equal per-instance cold solves."""
import numpy as np
import pytest

import helpers as H
import shim_common as S
from oracle import oracle
from tinympc_b200 import abi, workloads as wl
from tinympc_b200.problem import MPCProblem

pytestmark = pytest.mark.skipif(not (S.have(S.SCRIPT_REF) and oracle.ref_available(np.float64)),
                                reason="reference builds not present (oracle/Makefile needs a TinyMPC checkout: REF=<path>)")

STATE_FIELDS = list(abi.STATE_FIELDS)


def _settings(d):
    st = abi.Settings()
    for n in S.SETTING_NAMES:
        setattr(st, n, d[n])
    return st


def _plant(A, B, f, x0, u0):
    """tests/shim/shim_script.cpp plant(): ascending index, separate multiply and add"""
    nx, nu = B.shape
    out = np.zeros(nx)
    for i in range(nx):
        ax = A[i, 0] * x0[0]
        for k in range(1, nx):
            ax = ax + A[i, k] * x0[k]
        bu = B[i, 0] * u0[0]
        for j in range(1, nu):
            bu = bu + B[i, j] * u0[j]
        out[i] = (ax + bu) + f[i]
    return out


def _case(name):
    """-> (Model, constraint kwargs of MPCProblem, settings dict, x0, Xref nx x N, Uref nu x N-1 or None, steps)"""
    if name == "box":
        sp = wl.random_lti(8, 2, 12, seed=3)
        m = S.Model.from_spec(sp)
        rng = np.random.default_rng(1)
        cons = dict(x_min=np.full(8, -3.0), x_max=np.full(8, 3.0), u_min=np.full(2, -1.0), u_max=np.full(2, 1.0))
        st = dict(S.DEFAULT_SETTINGS, max_iter=150, abs_pri_tol=1e-2, abs_dua_tol=1e-2)
        return m, cons, st, 1.5 * rng.standard_normal(8), 0.5 * rng.standard_normal((8, 12)), None, 6
    if name == "cones":
        sp = wl.rocket(N=10)
        m = S.Model.from_spec(sp)
        cons = dict(sp.constraints, cx=[0.3], cu=[0.05])
        st = dict(S.DEFAULT_SETTINGS, max_iter=120, abs_pri_tol=1e-2, abs_dua_tol=1e-2, en_state_soc=1, en_input_soc=1)
        inst = wl.rocket_instances(1, N=10, seed=2)
        Uref = np.tile(np.array([[0.0], [0.0], [10.0]]), (1, 9))
        return m, cons, st, inst["x0"][0], inst["Xref"].T if inst["Xref"].ndim == 2 else inst["Xref"][0].T, Uref, 5
    sp = H.quad_linear_spec(tv=(name == "tv_planes"), N=10)
    m = S.Model.from_spec(sp)
    st = dict(S.DEFAULT_SETTINGS)
    st.update({k: getattr(sp.settings, k) for k in S.SETTING_NAMES})
    st.update(abs_pri_tol=1e-2, abs_dua_tol=1e-2)  # converges within max_iter = 60, at different counts
    rng = np.random.default_rng(11)
    return m, dict(sp.constraints), st, 0.3 * rng.standard_normal(12), np.zeros((12, 10)), None, 5


def _script(m, cons, st, x0, Xref, Uref, steps):
    s = S.Script().setup(0, m)
    if "x_min" in cons:
        s.bounds(0, cons["x_min"], cons["x_max"], cons["u_min"], cons["u_max"])
    if "Acx" in cons:
        s.cones(0, cons["Acx"], cons["qcx"], cons["cx"], cons["Acu"], cons["qcu"], cons["cu"])
    if "Alin_x" in cons:
        s.linear(0, cons["Alin_x"], cons["blin_x"], cons["Alin_u"], cons["blin_u"])
    if "tv_Alin_x" in cons:
        s.tv_linear(0, cons["tv_Alin_x"], cons["tv_blin_x"], cons["tv_Alin_u"], cons["tv_blin_u"])
    s.update_settings(0, **{k: st[k] for k in S.SETTING_NAMES})
    s.xref(0, Xref)
    if Uref is not None:
        s.uref(0, Uref)
    s.x0(0, x0)
    for _ in range(steps):
        s.solve(0).plant(0)
    return s


@pytest.mark.parametrize("name", ["box", "cones", "planes", "tv_planes"])
def test_reference_driver_matches_batch_oracle_closed_loop(name, tmp_path):
    m, cons, st, x0, Xref, Uref, steps = _case(name)
    recs, _ = S.run(S.SCRIPT_REF, _script(m, cons, st, x0, Xref, Uref, steps), str(tmp_path), name)
    cache = recs[0]
    assert cache["kind"] == "cache" and cache["rc"] == 0
    base = m.ref_cache()
    prob = MPCProblem(**{k: getattr(base, k) for k in ("nx", "nu", "N", "dtype", "rho", "A", "B", "f", "Q", "R", "Kinf",
                                                        "Pinf", "Quu_inv", "AmBKt", "APf", "BPf")}, **cons)
    settings = _settings(st)
    trees = S.trees(recs)
    assert len(trees) == steps
    state, xk = None, np.asarray(x0, np.float64)
    Uref_b = None if Uref is None else np.ascontiguousarray(Uref.T)
    iters = set()
    for k, t in enumerate(trees):
        r = oracle.solve_batch(prob, settings, xk[None, :], np.ascontiguousarray(Xref.T), Uref_b, state=state,
                               cold_start=state is None, want_state=tuple(STATE_FIELDS), impl="reference")
        where = (name, "step", k)
        assert int(t["iter"][0, 0]) == int(r["iter"][0]) and int(t["solved"][0, 0]) == int(r["solved"][0]), where
        assert t["rc"] == (0 if r["solved"][0] else 1), where
        assert H.bits_equal(t["sol_x"].T, r["sol_x"][0]) and H.bits_equal(t["sol_u"].T, r["sol_u"][0]), where
        for f in STATE_FIELDS:
            assert H.bits_equal(t[f].T, r[f][0]), (where, f)
        res = np.array([t[f][0, 0] for f in ("primal_residual_state", "dual_residual_state", "primal_residual_input",
                                             "dual_residual_input")])
        assert H.bits_equal(res, r["residuals"][0]), where  # check_termination = 1: every solve writes them
        assert int(t["status"][0, 0]) == (1 if r["solved"][0] else 11) and int(t["work_iter"][0, 0]) == int(r["iter"][0])
        iters.add(int(r["iter"][0]))
        state = {f: r[f].copy() for f in STATE_FIELDS}
        xk = _plant(m.A, m.B, m.f, xk, r["u"][0, 0])
    assert len(iters) >= 2, iters  # the loop is not one repeated solve


@pytest.mark.parametrize("name", ["box", "cones"])
def test_reference_driver_batch_emulation_matches_cold_solves(name, tmp_path):
    m, cons, st, x0, Xref, Uref, _ = _case(name)
    B = 7
    rng = np.random.default_rng(5)
    x0s = x0[None, :] * (1.0 + 0.2 * rng.standard_normal((B, m.nx)))
    Xb = np.stack([np.roll(Xref, -k, axis=1).T for k in range(B)])  # (B, N, nx): a different window per instance
    s = _script(m, cons, st, x0, Xref, Uref, 1)
    s.dump(0).batch(0, x0s.T, Xb.reshape(B, -1).T).dump(0)
    recs, ops = S.run(S.SCRIPT_REF, s, str(tmp_path), name)
    before, out, after = recs[-3:]
    assert out["kind"] == "batch" and out["rc"] == 0
    assert ops[s.nops - 2] == []  # the batch prints nothing
    base = m.ref_cache()
    prob = MPCProblem(**{k: getattr(base, k) for k in ("nx", "nu", "N", "dtype", "rho", "A", "B", "f", "Q", "R", "Kinf",
                                                        "Pinf", "Quu_inv", "AmBKt", "APf", "BPf")}, **cons)
    r = oracle.solve_batch(prob, _settings(st), x0s, Xb, None if Uref is None else np.ascontiguousarray(Uref.T),
                           cold_start=True, want_state=("u",), impl="reference")
    assert H.bits_equal(out["u0"].T, np.ascontiguousarray(r["u"][:, 0, :]))
    assert np.array_equal(out["iter"][:, 0].astype(np.int32), r["iter"])
    assert np.array_equal(out["solved"][:, 0].astype(np.int32), r["solved"])
    for f in S.TREE_FIELDS:  # the emulation restores the calling solver's tree
        assert H.bits_equal(before[f], after[f]), f
