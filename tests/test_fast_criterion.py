"""Calibration of the FAST acceptance rule (tests/fast_common.py) on the CPU, no GPU needed.

The rule must accept what FMA contraction legitimately does, and reject what a kernel bug does:
  * the reference's own FMA builds (oracle/_ref/libtinympc_ref_{f32,f64}_fastv3.so, -march=x86-64-v3) pass it with at
    least 2x margin on the cases the GPU suite uses: cold, warm, and warm at max_iter = 1;
  * mutants of the pinned fp32 oracle, each a plausible kernel bug reproduced by altering the oracle's inputs, fail it.
"""
import numpy as np
import pytest

import fast_common as F
import helpers as H
from oracle import oracle
from tinympc_b200.solver import setup_problem

DIMS = [(4, 1), (6, 3), (12, 4), (4, 2), (4, 4), (4, 8), (8, 2), (8, 4), (8, 8), (12, 2), (12, 8), (16, 2), (16, 4), (16, 8)]
B = 45


def _cases(dt):
    """name -> (problem, fixed-work settings, instances, state fields): every compiled (nx, nu) at N = 50, quadrotor tracking
    with per-instance references, and every constraint family."""
    out = {}
    for nx, nu in DIMS:
        spec, inst, want = F.lti_case(nx, nu, 50, B, dt)
        out[f"box_{nx}_{nu}"] = (spec, inst, want)
    from tinympc_b200 import workloads as wl
    out["box_quad_track"] = (wl.quadrotor(N=50), F.tracking(B, 50, dt, seed=3), H.BOX_STATE)
    for name in F.FAMILY_CASES:
        out[name] = F.family_case(name, B, dt)
    return out


def _ratios(prob, st, inst, want, variant):
    """Worst rule ratio of the reference build `variant` over the three solves of a case."""
    st1 = F.fixed_work(st, max_iter=1)
    worst = {}
    ref = lambda s: F.oracle_pair(prob, s, impl="reference", variant=variant)  # noqa: E731
    port = lambda s: F.oracle_pair(prob, s)  # noqa: E731
    for label, s, x0, state, cold, (pin, o64) in F.three_solves(port, inst, want, st, st1):
        v, _ = ref(s)(x0, inst["Xref"], inst.get("Uref"), state, cold, want)
        keys = ["sol_x", "sol_u", "residuals"] + list(want)
        for name, res in (("v3", v), ("pin", pin), ("o64", o64)):
            assert not F.termination_violations(res, s), (label, name)
        r = F.rule_ratios(v, pin, o64, keys, prob.dtype, prob.rho)
        for k, x in r.items():
            worst[(label, k)] = max(worst.get((label, k), 0.0), x)
    return worst


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_reference_fma_build_accepted_with_margin(dt):
    if not oracle.ref_available(dt, "fastv3"):
        pytest.skip("the reference's -march=x86-64-v3 build is not available (no TinyMPC checkout at build time)")
    lines, worst_all = [], 0.0
    for name, (spec, inst, want) in _cases(dt).items():
        prob = setup_problem(spec, dt)
        st = F.fixed_work(spec.settings)
        worst = _ratios(prob, st, inst, want, "fastv3")
        (label, key), w = max(worst.items(), key=lambda kv: kv[1])
        lines.append(f"{name:16s} worst {w:.3g} ({label}: {key})")
        worst_all = max(worst_all, w)
        assert w <= 0.5, f"{name}: the reference's FMA build uses {w:.3g} of the FAST rule's bound ({label}: {key})"
    print(f"\nfastv3 {dt.__name__}: worst ratio {worst_all:.3g}\n" + "\n".join(lines))


# ---------------------------------------------------------------------------------------------------------------------
# mutants: the pinned fp32 oracle on altered inputs, judged by the rule against the unaltered oracles
# ---------------------------------------------------------------------------------------------------------------------
def _quad_case():
    from tinympc_b200 import workloads as wl
    dt = np.float32
    spec = wl.quadrotor(N=50)
    prob = setup_problem(spec, dt)
    return prob, F.fixed_work(spec.settings), F.tracking(B, 50, dt, seed=3)


def _judge(prob, st, inst, want, mutant_fn, solves=("cold", "warm", "warm max_iter=1")):
    """Worst rule ratio of the mutant over the chosen solves (> 1 = rejected), and whether it changed any output."""
    st1 = F.fixed_work(st, max_iter=1)
    worst, changed = 0.0, False
    for label, s, x0, state, cold, (pin, o64) in F.three_solves(lambda s: F.oracle_pair(prob, s), inst, want, st, st1):
        if label not in solves:
            continue
        m = mutant_fn(prob, s, x0, inst, state, cold, want)
        keys = ["sol_x", "sol_u", "residuals"] + list(want)
        changed |= any(not H.bits_equal(m[k], pin[k]) for k in keys)
        worst = max(worst, max(F.rule_ratios(m, pin, o64, keys, np.float32, prob.rho).values()))
    return worst, changed


def _solve(prob, s, x0, Xref, Uref, state, cold, want):
    state = None if state is None else {n: np.array(a, copy=True) for n, a in state.items()}
    return oracle.solve_batch(prob, s, x0, Xref, Uref, state=state, cold_start=cold, want_state=tuple(want), impl="port",
                              nthreads=F.NT)


def _kinf_row(prob, s, x0, inst, state, cold, want):
    """A wrong register row: one Kinf entry (the largest of the last row) x (1 + 1e-3)."""
    p = prob.astype(prob.dtype)
    K = p.Kinf.copy(order="F")
    j = int(np.argmax(np.abs(K[-1])))
    K[-1, j] *= prob.dtype(1.001)
    p.Kinf = K
    return _solve(p, s, x0, inst["Xref"], inst["Uref"], state, cold, want)


def _uref_shift(prob, s, x0, inst, state, cold, want):
    """An off-by-one reference offset: every instance reads Uref one knot late."""
    U = np.array(inst["Uref"], copy=True)
    U[:, 1:] = inst["Uref"][:, :-1]
    return _solve(prob, s, x0, inst["Xref"], U, state, cold, want)


def _vz_dropped(prob, s, x0, inst, state, cold, want):
    """A dropped vprev: the warm start's work->v / work->z read as zero."""
    if state is not None:
        state = dict(state, v=np.zeros_like(state["v"]), z=np.zeros_like(state["z"]))
    return _solve(prob, s, x0, inst["Xref"], inst["Uref"], state, cold, want)


def _lost_bound(prob, s, x0, inst, state, cold, want):
    """A lost bound on a lane's last row: the last input row's bounds are +-inf."""
    p = prob.astype(prob.dtype)
    lo, hi = p.u_min.copy(order="F"), p.u_max.copy(order="F")
    lo[-1], hi[-1] = -np.inf, np.inf
    p.u_min, p.u_max = lo, hi
    return _solve(p, s, x0, inst["Xref"], inst["Uref"], state, cold, want)


MUTANTS = {"kinf_row": (_kinf_row, ("cold", "warm")), "uref_shift": (_uref_shift, ("cold", "warm")),
           "vz_dropped": (_vz_dropped, ("warm max_iter=1",)), "lost_bound": (_lost_bound, ("cold", "warm"))}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_mutant_rejected(mutant):
    prob, st, inst = _quad_case()
    fn, solves = MUTANTS[mutant]
    worst, changed = _judge(prob, st, inst, H.BOX_STATE, fn, solves)
    print(f"\n{mutant}: worst ratio {worst:.3g}")
    assert changed, f"{mutant}: the mutation did not change any output (the case does not exercise it)"
    assert worst > 1.0, f"{mutant}: accepted by the FAST rule (worst ratio {worst:.3g})"


def test_vz_dropped_only_visible_in_residuals():
    """v / z reach only the first iteration's dual residual (admm.cpp:315,317): at max_iter = 1 the dropped-vprev mutant
    moves the residuals and nothing else, so the residual check is what catches it."""
    prob, st, inst = _quad_case()
    st1 = F.fixed_work(st, max_iter=1)
    (_, _, x0, state, cold, (pin, o64)), = [c for c in F.three_solves(lambda s: F.oracle_pair(prob, s), inst, H.BOX_STATE, st, st1)
                                            if c[0] == "warm max_iter=1"]
    m = _vz_dropped(prob, st1, x0, inst, state, cold, H.BOX_STATE)
    for k in ["sol_x", "sol_u"] + [n for n in H.BOX_STATE if n not in ("v", "z")]:
        assert H.bits_equal(m[k], pin[k]), k
    r = F.rule_ratios(m, pin, o64, ["residuals"], np.float32, prob.rho)
    assert r["residuals"] > 1.0, r
