"""The acceptance rule of FAST mode (FMA contraction, fmin / fmax clamp) and the cases it is calibrated on.

FAST cannot be bit-identical to any build of the reference (SURVEY B.7), so it is held to an fp64 yardstick:

  O64   = the plain-C restatement (oracle "port") in fp64 on prob.astype(float64) with the inputs upcast: the same cache as
          the kernel, only the arithmetic of the solve differs;
  PIN32 = the pinned fp32 oracle (= STRICT fp32, bit for bit), whose distance to O64 is STRICT's own rounding error.

For every compared field (sol_x, sol_u, every requested state field, residuals):

  fp32:  max|FAST - O64| <= C32 * max|PIN32 - O64| + ULPS32 * eps32 * scale
         and, on sol_x / sol_u / x / u, max|FAST - PIN32| <= 2e-4 * max(1, max|PIN32|)
  fp64:  max|FAST - O64| <= 1e-10 * max(1, scale)

`scale` is the largest magnitude of the field in O64.  A residual is a difference of nearly equal numbers, so its scale is
that of its operands: the state (sol_x) for the primal / dual state residuals and the input (sol_u) for the input ones, times
rho for the dual residuals.  iter and solved are equal to O64's at fixed work (tolerances 0: every solve runs to max_iter).
FAST must differ from the pinned oracle in at least one bit of some field, or the FAST instantiation did not run.  Every
output (FAST and the oracles) satisfies the reference's termination invariants: solved == 1 exactly where the four reported
residuals pass the termination test, and iter == max_iter wherever solved == 0.

Calibration (tests/test_fast_criterion.py, CPU only).  The reference's own FMA builds (-march=x86-64-v3: AVX2 + FMA
contraction) on the cases below (every compiled (nx, nu) at N = 50, quadrotor tracking, every constraint family), cold, warm
and warm at max_iter = 1, measured as max|V3 - O64| / bound:
  fp32: worst ratio 0.414 (C32 = 6, ULPS32 = 8: 2.4x margin; with C32 = 4 it was 0.519, under the 2x margin asked for);
  fp64: worst 1.3e-3 of the 1e-10 bound.
Mutants of the pinned fp32 oracle that model kernel bugs (quadrotor tracking, N = 50) are rejected with these worst ratios
(> 1 is a rejection):
  one Kinf entry x (1 + 1e-3), a wrong register row ............................. 8.55
  Uref shifted by one knot, an off-by-one reference offset ...................... 1.66e3
  v / z zeroed on a warm start at max_iter = 1, a dropped vprev (residuals only) ... 5.99e3
  the last input row's bounds set to +-inf, a lost bound on a lane's last row ... 2.92e4
"""
from __future__ import annotations

import os

import numpy as np

import helpers as H
from oracle import oracle
from tinympc_b200 import abi, workloads as wl

NT = os.cpu_count() or 1
C32 = 6.0
ULPS32 = 8.0
REL64 = 1e-10
REL_XU32 = 2e-4
FIXED_ITERS = 20
EPS = {np.float32: float(np.finfo(np.float32).eps), np.float64: float(np.finfo(np.float64).eps)}
# residual column -> (trajectory field whose magnitude is the operands', times rho?)
RES_OPERANDS = (("sol_x", False), ("sol_x", True), ("sol_u", False), ("sol_u", True))


def fixed_work(settings, max_iter=FIXED_ITERS, **kw):
    """Settings copy with tolerances 0: every instance runs exactly max_iter iterations."""
    st = abi.Settings.from_buffer_copy(settings)
    st.abs_pri_tol = st.abs_dua_tol = 0.0
    st.max_iter = max_iter
    for k, v in kw.items():
        setattr(st, k, v)
    return st


def upcast(d):
    if d is None:
        return None
    return {k: (None if v is None else (np.asarray(v, np.float64) if np.asarray(v).dtype.kind == "f" else v)) for k, v in d.items()}


def oracle_pair(probs, st, model=None, impl="port", variant=""):
    """run(x0, Xref, Uref, state, cold, want) -> (the oracle in the problems' own dtype, O64).  probs: one MPCProblem (shared
    model) or a list of them with model[b] = the problem instance b uses (one oracle run per model).  impl / variant select
    the first result's solver (the pinned restatement by default, or a build of the reference)."""
    shared = not isinstance(probs, (list, tuple))
    plist = [probs] if shared else list(probs)
    p64 = [p.astype(np.float64) for p in plist]

    def solve(ps, x0, Xref, Uref, state, cold, want, imp, var):
        B = len(x0)
        mdl = np.zeros(B, int) if shared else np.asarray(model)
        out = {}
        for m in np.unique(mdl):
            idx = np.flatnonzero(mdl == m)
            sub = None if state is None else {n: np.array(a[idx], copy=True) for n, a in state.items()}
            xr = Xref[idx] if Xref.ndim == 3 else Xref
            ur = None if Uref is None else (Uref[idx] if Uref.ndim == 3 else Uref)
            o = oracle.solve_batch(ps[m], st, x0[idx], xr, ur, state=sub, cold_start=cold, want_state=tuple(want), impl=imp,
                                   variant=var, nthreads=NT)
            for k, v in o.items():
                if v is not None:
                    out.setdefault(k, np.empty((B,) + v.shape[1:], v.dtype))[idx] = v
        return out

    def run(x0, Xref, Uref, state, cold, want):
        a = solve(plist, x0, Xref, Uref, state, cold, want, impl, variant)
        st64 = upcast(state)
        b = solve(p64, np.asarray(x0, np.float64), np.asarray(Xref, np.float64), None if Uref is None else np.asarray(Uref, np.float64),
                  st64, cold, want, "port", "")
        return a, b
    return run


def _scale(key, o64, rho):
    if key == "residuals":
        return np.array([float(np.abs(o64[f]).max()) * (rho if r else 1.0) for f, r in RES_OPERANDS])
    return float(np.abs(o64[key]).max())


def _maxerr(a, b, key):
    d = np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64))
    return d.reshape(-1, 4).max(axis=0) if key == "residuals" else float(d.max())


def rule_ratios(got, pin, o64, keys, dt, rho):
    """key -> worst ratio of the FAST error to what the rule allows (<= 1 passes).  A non-finite FAST value (an element a
    solve never wrote keeps the NaN poison) is an infinite ratio."""
    out = {}
    for key in keys:
        g = np.asarray(got[key])
        if not np.isfinite(g).all():
            out[key] = np.inf
            continue
        scale = _scale(key, o64, rho)
        e_fast = _maxerr(g, o64[key], key)
        if dt == np.float64:
            bound = REL64 * np.maximum(1.0, scale)
        else:
            bound = C32 * _maxerr(pin[key], o64[key], key) + ULPS32 * EPS[np.float32] * scale
        r = float(np.max(e_fast / np.maximum(bound, 1e-300)))
        if dt == np.float32 and key in ("sol_x", "sol_u", "x", "u"):
            p = np.asarray(pin[key], np.float64)
            r = max(r, float(np.abs(g.astype(np.float64) - p).max()) / (REL_XU32 * max(1.0, float(np.abs(p).max()))))
        out[key] = r
    return out


def termination_violations(res, st):
    """The reference's termination invariants on one output: solved == 1 exactly where the four reported residuals pass
    the test (admm.cpp:310-328), iter == max_iter wherever solved == 0.  -> list of messages (empty = holds)."""
    dt = np.asarray(res["residuals"]).dtype.type
    r = np.asarray(res["residuals"])
    tp, td = dt(st.abs_pri_tol), dt(st.abs_dua_tol)
    passes = (r[:, 0] < tp) & (r[:, 2] < tp) & (r[:, 1] < td) & (r[:, 3] < td)
    sv, it = np.asarray(res["solved"]), np.asarray(res["iter"])
    bad = []
    if not np.isin(sv, (0, 1)).all():
        bad.append(f"solved not 0/1: {np.unique(sv)}")
    if not ((sv == 1) == passes).all():
        bad.append(f"solved disagrees with the residual test on {int(((sv == 1) != passes).sum())} instances")
    if not (it[sv == 0] == st.max_iter).all():
        bad.append(f"iter != max_iter on {int((it[sv == 0] != st.max_iter).sum())} unsolved instances")
    return bad


def check_fixed_work(got, pin, o64, keys, dt, rho, st, what):
    """The whole rule on one fixed-work solve; -> the ratios (for reports).  Raises AssertionError naming `what`."""
    for name, res in (("fast", got), ("pinned", pin), ("o64", o64)):
        bad = termination_violations(res, st)
        assert not bad, (what, name, bad)
    for k in ("iter", "solved"):
        assert np.array_equal(got[k], o64[k]), (what, k, np.unique(got[k]), np.unique(o64[k]))
    ratios = rule_ratios(got, pin, o64, keys, dt, rho)
    worst = max(ratios, key=ratios.get)
    assert ratios[worst] <= 1.0, f"{what}: {worst} outside the FAST rule (ratio {ratios[worst]:.3g}; all {fmt(ratios)})"
    assert any(not H.bits_equal(got[k], pin[k]) for k in keys), f"{what}: bit-identical to the pinned oracle: FAST did not run"
    return ratios


def fmt(ratios):
    return " ".join(f"{k}={v:.2g}" for k, v in ratios.items())


# ---------------------------------------------------------------------------------------------------------------------
# cases (shared by the CPU calibration and the GPU suite): -> dict(prob spec, settings, instances, state fields)
# ---------------------------------------------------------------------------------------------------------------------
SOC_LIN_STATE = H.SOC_STATE + ["vlnew", "zlnew", "gl", "yl"]
ROCKET_PLANES = dict(Alin_x=np.array([[1.0, 0, 0, 0, 0, 0]]), blin_x=np.array([4.0]), Alin_u=np.array([[1.0, 1.0, 0]]),
                     blin_u=np.array([5.0]))


def tracking(B, N, dt, seed):
    """Quadrotor tracking with per-instance Xref windows and per-instance Uref; x0 jittered so that the input bounds bite."""
    inst = wl.tracking_instances(B, N=N, seed=seed, dtype=dt, jitter=0.5)
    inst["Uref"] = (0.05 * np.random.default_rng(seed + 1).standard_normal((B, N - 1, 4))).astype(dt)
    return inst


def lti_case(nx, nu, N, B, dt):
    spec = wl.random_lti(nx, nu, N, seed=7 * nx + nu)
    inst = wl.random_instances(B, nx, N, seed=N + nx, dtype=dt)
    inst["x0"] = (3.0 * inst["x0"]).astype(dt)  # the input bounds bite
    return spec, inst, H.BOX_STATE


def family_case(name, B, dt):
    """The constraint-family cases: -> (spec, inst, state fields)."""
    rng = np.random.default_rng(31)
    if name in ("cones", "cones_tight"):
        spec = wl.rocket(N=20)
        spread = 0.3
        if name == "cones_tight":  # both cone branches active (helpers.make_cases)
            spec.constraints = dict(spec.constraints, cx=[0.1], cu=[0.02], Acx=[1], Acu=[0])
            spread = 0.5
        return spec, wl.rocket_instances(B, N=20, seed=4, dtype=dt, spread=spread, per_instance_refs=True), H.SOC_STATE
    if name in ("lin", "tvlin"):
        spec = H.quad_linear_spec(tv=name == "tvlin")
        inst = dict(x0=(0.3 * rng.standard_normal((B, 12))).astype(dt), Xref=(0.05 * rng.standard_normal((B, spec.N, 12))).astype(dt),
                    Uref=(0.02 * rng.standard_normal((B, spec.N - 1, 4))).astype(dt))
        return spec, inst, (H.TVLIN_STATE if name == "tvlin" else H.LIN_STATE)
    if name == "cones_lin":
        spec = wl.rocket(N=20)
        spec.constraints = dict(spec.constraints, **ROCKET_PLANES)
        spec.settings.en_state_linear = spec.settings.en_input_linear = 1
        return spec, wl.rocket_instances(B, N=20, seed=6, dtype=dt, spread=0.3, per_instance_refs=True), SOC_LIN_STATE
    raise KeyError(name)


FAMILY_CASES = ["cones", "cones_tight", "lin", "tvlin", "cones_lin"]


def warm_inputs(x0, res, want, seed):
    """Next MPC step from an oracle's state: perturbed x0, duals reset on every third instance, v / z included."""
    rng = np.random.default_rng(seed)
    x0b = (x0 + 0.02 * rng.standard_normal(x0.shape)).astype(x0.dtype)
    state = {n: np.array(res[n], copy=True) for n in want}
    for n in ("g", "y"):
        state[n][::3] = 0
    return x0b, state


def three_solves(run, inst, want, st, st1):
    """The oracle side of a FAST case: a cold solve, a warm step from the oracle's own state, and the same warm step at
    max_iter = 1.  run(settings) -> oracle_pair runner.  -> [(label, settings, x0, state, cold, (pin, o64))]"""
    x0, Xref, Uref = inst["x0"], inst["Xref"], inst.get("Uref")
    r = run(st)
    pin1, o1 = r(x0, Xref, Uref, None, True, want)
    x0b, state = warm_inputs(x0, pin1, want, seed=len(x0))
    pin2, o2 = r(x0b, Xref, Uref, state, False, want)
    pin3, o3 = run(st1)(x0b, Xref, Uref, state, False, want)
    return [("cold", st, x0, None, True, (pin1, o1)), ("warm", st, x0b, state, False, (pin2, o2)),
            ("warm max_iter=1", st1, x0b, state, False, (pin3, o3))]
