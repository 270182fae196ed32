"""FAST mode (FMA contraction, fmin / fmax clamp) on every kernel variant it compiles, held to the fp64 oracle.

The rule is tests/fast_common.py's (calibrated on the CPU by tests/test_fast_criterion.py): in fp32 FAST's distance to the fp64
restatement (O64) is at most C32 times the pinned fp32 oracle's (STRICT's own error) plus a few ulps, on the trajectories, every
requested state field, u0 and the residuals; in fp64 it is 1e-10 of the field's scale.  Every fixed-work case (tolerances 0,
20 iterations, a ragged batch) runs on NaN-poisoned outputs:
  1. a cold solve;
  2. a warm step from the pinned oracle's state (perturbed x0, duals reset on every third instance, v / z present, so the
     kernels' first-iteration path with the caller's previous slacks runs); the oracles get the same state (O64 upcast);
  3. the same warm step at max_iter = 1, where v / z decide the dual residuals.
To-convergence cases bound the iteration-count shifts against the pinned oracle and print them.  Every solve records which
instantiation ran (stats()); test_fast_suite_reaches_every_fast_instantiation, the last test of the file, asserts that the
set reached is the set the library compiles.
"""
import numpy as np
import pytest

import fast_common as F
import helpers as H
import test_gpu_het_streamed as HS
import test_gpu_multiwave as MW
from tinympc_b200 import abi, workloads as wl
from tinympc_b200.problem import copy_settings
from tinympc_b200.solver import BatchedTinySolver, setup_problem

pytestmark = pytest.mark.gpu

ALL_DIMS = [(4, 1), (6, 3), (12, 4), (4, 2), (4, 4), (4, 8), (8, 2), (8, 4), (8, 8), (12, 2), (12, 8), (16, 2), (16, 4), (16, 8)]
KERNELS = {"tpi": abi.KERNEL_TPI, "gpi": abi.KERNEL_GPI, "gps": abi.KERNEL_GPS, "auto": abi.KERNEL_AUTO}
B_RAGGED = 45  # not a multiple of 32 / L for any lane count
DT = {"f32": np.float32, "f64": np.float64}

# instantiations reached in this session: ("gpi", dtype, L, het) / ("gps", family mask, "shared" or "het") / ("tpi", ext)
REACHED = set()
NI_SEEN = set()  # instances per lane group of the shared-model streamed solves


def _record(stt, mask, het):
    fam = stt["kernel_family"]
    if fam == abi.KERNEL_GPI:
        REACHED.add(("gpi", stt["_dt"], stt["lanes_per_instance"], het))
    elif fam == abi.KERNEL_GPS:
        # instances per lane group: the planner's choice for the shape (1 or 2) with a shared model, 1 with per-instance models
        ni = stt["instances_per_cta"] * stt["lanes_per_instance"] // stt["threads_per_cta"]
        assert ni in ((1,) if het else (1, 2)), stt
        REACHED.add(("gps", mask, "het" if het else "shared"))
        NI_SEEN.add(ni)
    elif fam == abi.KERNEL_TPI:
        REACHED.add(("tpi", mask != 0))


def _mask(st):
    soc = bool(st.en_state_soc or st.en_input_soc)
    lin = bool(st.en_state_linear or st.en_input_linear or st.en_tv_state_linear or st.en_tv_input_linear)
    return 0 if not (soc or lin) else (1 if not lin else (6 if not soc else 7))


def _solver(prob, st, kernel):
    return BatchedTinySolver(prob, st, mode=abi.MODE_FAST, kernel=KERNELS[kernel])


def _device(solver, s, x0, inst, state, cold, want, models):
    """One FAST solve on the device path with poisoned outputs, under settings s; records the instantiation."""
    solver.settings = copy_settings(s)
    solver.update_settings()
    g, stt = MW._device_solve(solver, x0, inst["Xref"], inst.get("Uref"), state, cold, want, models=models)
    stt["_dt"] = solver.problem.dtype.__name__
    _record(stt, _mask(s), models is not None)
    return g, stt


def _with_u0(o):
    return dict(o, u0=np.ascontiguousarray(o["u"][:, 0, :]))


def _fixed_work_case(prob_or_probs, st, inst, want, kernels, what, model=None, models=None, expect=None):
    """Steps 1-3 of the module docstring on each kernel, against oracles computed once.  -> {(kernel, label): ratios}"""
    probs = prob_or_probs
    p0 = probs[0] if isinstance(probs, (list, tuple)) else probs
    rho = max(p.rho for p in probs) if isinstance(probs, (list, tuple)) else p0.rho
    st = F.fixed_work(st)
    st1 = F.fixed_work(st, max_iter=1)
    solves = F.three_solves(lambda s: F.oracle_pair(probs, s, model=model), inst, want, st, st1)
    keys = ["sol_x", "sol_u", "residuals", "u0"] + list(want)
    out = {}
    for kernel in kernels:
        solver = _solver(p0, st, kernel)
        for label, s, x0, state, cold, (pin, o64) in solves:
            g, stt = _device(solver, s, x0, inst, state, cold, want, models)
            if expect is not None:
                expect(kernel, stt)
            out[(kernel, label)] = F.check_fixed_work(g, _with_u0(pin), _with_u0(o64), keys, p0.dtype, rho, s,
                                                      f"{what} [{kernel}] {label}")
        solver.close()
    return out


def _family_is(kernel, stt):
    if kernel != "auto":
        assert stt["kernel_family"] == KERNELS[kernel], (kernel, stt)


# ---------------------------------------------------------------------------------------------------------------------
# 1. box constraints, shared model: every compiled (nx, nu), fp32 / fp64, all three kernel families
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("dims", ALL_DIMS)
def test_box_every_shape(dims, dt):
    """N = 50: the fp32 on-chip plans use L = 4 and L = 8, the fp64 ones L = 4, 8 and 16; padded shapes ((6,3), (4,1),
    (12,8), ...) put padding rows next to real ones."""
    dt = DT[dt]
    nx, nu = dims
    spec, inst, want = F.lti_case(nx, nu, 50, B_RAGGED, dt)
    prob = setup_problem(spec, dt)
    _fixed_work_case(prob, spec.settings, inst, want, ["tpi", "gpi", "gps"], f"box ({nx},{nu}) {dt.__name__}",
                     expect=lambda k, stt: _family_is(k, stt) if k != "gpi" else None)


@pytest.mark.parametrize("dt", ["f32", "f64"])
def test_box_tracking_per_instance_references(dt):
    """Quadrotor tracking: per-instance Xref windows and per-instance Uref; the input bounds bite."""
    dt = DT[dt]
    spec = wl.quadrotor(N=50)
    prob = setup_problem(spec, dt)
    _fixed_work_case(prob, spec.settings, F.tracking(77, 50, dt, seed=3), H.BOX_STATE, ["tpi", "gpi", "gps"],
                     f"quad tracking {dt.__name__}", expect=_family_is)


@pytest.mark.parametrize("dt", ["f32", "f64"])
def test_box_time_varying_bounds(dt):
    dt = DT[dt]
    spec = wl.quadrotor(N=20)
    rng = np.random.default_rng(3)
    N = spec.N
    cons = dict(spec.constraints)
    cons["x_min"] = -5.0 - rng.uniform(0, 1, (12, N))
    cons["x_max"] = 5.0 + rng.uniform(0, 1, (12, N))
    cons["u_min"] = -0.5 + 0.3 * rng.uniform(0, 1, (4, N - 1))
    cons["u_max"] = 0.5 - 0.3 * rng.uniform(0, 1, (4, N - 1))
    spec.constraints = cons
    prob = setup_problem(spec, dt)
    _fixed_work_case(prob, spec.settings, F.tracking(61, N, dt, seed=4), H.BOX_STATE, ["tpi", "gpi", "gps"],
                     f"time-varying bounds {dt.__name__}", expect=_family_is)


def test_box_bounds_with_signed_zeros():
    """Bounds at +-0 (test_gpu_parity.test_bounds_with_signed_zeros): FAST clamps with fmin / fmax, which may return the
    other zero; the values stay within the rule."""
    dt = np.float32
    spec = wl.quadrotor(N=10)
    spec.constraints = dict(x_min=np.array([-5, -5, 0.0, -5, -5, -5, -0.0, -5, -5, -5, -5, -5]),
                            x_max=np.array([5, 5, 5, 5, -0.0, 5, 5, 5, 5, 5, 0.0, 5]),
                            u_min=np.array([-0.0, -0.5, 0.0, -0.5]), u_max=np.array([0.5, 0.0, 0.5, -0.0]))
    prob = setup_problem(spec, dt)
    inst = wl.tracking_instances(77, N=10, seed=9, dtype=dt)
    inst["x0"][:38] = -inst["x0"][:38]
    _fixed_work_case(prob, spec.settings, inst, H.BOX_STATE, ["tpi", "gpi", "gps"], "signed-zero bounds", expect=_family_is)


# ---------------------------------------------------------------------------------------------------------------------
# 2. constraint families: cones (incl. both branches active), static / time-varying hyperplanes, cones + hyperplanes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("case", F.FAMILY_CASES)
def test_constraint_families(case, dt):
    dt = DT[dt]
    spec, inst, want = F.family_case(case, 53, dt)
    prob = setup_problem(spec, dt)
    _fixed_work_case(prob, spec.settings, inst, want, ["tpi", "gps"], f"{case} {dt.__name__}", expect=_family_is)


# ---------------------------------------------------------------------------------------------------------------------
# 3. per-instance models: on-chip (GPI HET) and streamed (GPS HET, every family mask)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt,dims,L", [("f32", (12, 4), 4), ("f32", (16, 8), 8), ("f64", (4, 2), 4), ("f64", (8, 4), 8),
                                       ("f64", (12, 4), 16)])
def test_gpi_per_instance_models(dt, dims, L):
    dt = DT[dt]
    nx, nu = dims
    B = 75
    sp, (blobs, probs) = HS._lti_fleet(nx, nu, 50, dt, wl.random_lti(nx, nu, 50).constraints)
    model = HS._assign(B)
    inst = wl.random_instances(B, nx, 50, seed=11 + nx, dtype=dt)
    inst["x0"] = (3.0 * inst["x0"]).astype(dt)

    def expect(kernel, stt):
        assert stt["kernel_family"] == abi.KERNEL_GPI and stt["lanes_per_instance"] == L, stt

    _fixed_work_case(probs, sp.settings, inst, H.BOX_STATE, ["gpi"], f"gpi het ({nx},{nu}) {dt.__name__}", model=model,
                     models=blobs[model], expect=expect)


def _gps_het_case(mask, dt):
    B = 75
    model = HS._assign(B)
    if mask == 0:
        sp = wl.quadrotor(N=50)
        blobs, probs = HS._tuned_fleet(sp, dt)
        return sp, blobs, probs, model, F.tracking(B, 50, dt, seed=5), H.BOX_STATE, "gps"
    if mask == 1:
        sp, blobs, probs = HS._rocket_fleet(dt, 20)
        return sp, blobs, probs, model, wl.rocket_instances(B, N=20, seed=4, dtype=dt, spread=0.3, per_instance_refs=True), H.SOC_STATE, "auto"
    if mask == 6:
        sp = H.quad_linear_spec(tv=True)
        blobs, probs = HS._tuned_fleet(sp, dt)
        return sp, blobs, probs, model, MW._hyperplane_instances(B, sp.N, dt, seed=31), H.TVLIN_STATE, "auto"
    spec = wl.rocket(N=20)
    sp, blobs, probs = HS._rocket_fleet(dt, 20, cons=dict(spec.constraints, **F.ROCKET_PLANES))
    sp.settings.en_state_linear = sp.settings.en_input_linear = 1
    return sp, blobs, probs, model, wl.rocket_instances(B, N=20, seed=6, dtype=dt, spread=0.3, per_instance_refs=True), F.SOC_LIN_STATE, "auto"


@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("mask", [0, 1, 6, 7])
def test_gps_per_instance_models(mask, dt):
    dt = DT[dt]
    sp, blobs, probs, model, inst, want, kernel = _gps_het_case(mask, dt)

    def expect(kernel, stt):
        HS._expect_het_plan(stt)

    _fixed_work_case(probs, sp.settings, inst, want, [kernel], f"gps het mask {mask} {dt.__name__}", model=model,
                     models=blobs[model], expect=expect)


# ---------------------------------------------------------------------------------------------------------------------
# 4. to convergence: termination invariants, distance to O64, iteration-count shifts against the pinned oracle
# ---------------------------------------------------------------------------------------------------------------------
F32_SHIFT_MAX = 0.6   # fp32: the iteration count is rounding-sensitive (the reference's own FMA build moves it on 45 % of box_quad_f32)
F64_SHIFT_MAX = 0.01


def check_converged(g, pin, o64, st, dt, what):
    """-> (instances whose iter differs from the pinned oracle, batch size).  Prints the count."""
    for name, res in (("fast", g), ("pinned", pin), ("o64", o64)):
        bad = F.termination_violations(res, st)
        assert not bad, (what, name, bad)
    shifted = g["iter"] != pin["iter"]
    n = int(shifted.sum())
    shifts = np.unique(g["iter"][shifted] - pin["iter"][shifted]).tolist()
    print(f"{what}: iter differs from the pinned oracle on {n} of {len(shifted)} instances, shifts {shifts}")
    if dt == np.float64:
        assert n <= F64_SHIFT_MAX * len(shifted), (what, n)
        assert all(abs(s) == st.check_termination for s in shifts), (what, shifts)
    else:
        assert n <= F32_SHIFT_MAX * len(shifted), (what, n)
    same = ~shifted
    for key in ("sol_x", "sol_u"):
        a, p, r = (np.asarray(v[key], np.float64) for v in (g, pin, o64))
        scale = float(np.abs(r).max())
        if dt == np.float64:
            assert np.abs(a - r)[same].max(initial=0.0) <= F.REL64 * max(1.0, scale), (what, key)
        else:
            assert np.abs(a - p)[same].max(initial=0.0) <= F.REL_XU32 * max(1.0, float(np.abs(p).max())), (what, key)
            # on the same instances: an iteration more or less moves a solution by up to the tolerance, in either build
            e_fast, e_pin = float(np.abs(a - r)[same].max(initial=0.0)), float(np.abs(p - r)[same].max(initial=0.0))
            assert e_fast <= 2.0 * e_pin + F.ULPS32 * F.EPS[np.float32] * scale, (what, key, e_fast, e_pin)
    return n, len(shifted)


CONVERGED = {
    "box_quad_f32": ("f32", ["tpi", "gpi", "gps"]),
    "box_quad_f64": ("f64", ["tpi", "gpi", "gps"]),
    "cones_f64": ("f64", ["tpi", "gps"]),
    "cones_f32": ("f32", ["tpi", "gps"]),
    "lin_f32": ("f32", ["tpi", "gps"]),
}


@pytest.mark.parametrize("case", list(CONVERGED))
def test_to_convergence(case):
    tag, kernels = CONVERGED[case]
    dt = DT[tag]
    B = 301
    if case.startswith("box"):
        spec = wl.quadrotor(N=50)
        inst, want = wl.tracking_instances(B, N=50, seed=5, dtype=dt), ()
    else:
        spec, inst, _ = F.family_case(case.rsplit("_", 1)[0], B, dt)
        want = ()
    prob = setup_problem(spec, dt)
    st = spec.settings
    pin, o64 = F.oracle_pair(prob, st)(inst["x0"], inst["Xref"], inst.get("Uref"), None, True, want)
    for kernel in kernels:
        solver = _solver(prob, st, kernel)
        g, stt = _device(solver, st, inst["x0"], inst, None, True, want, None)
        _family_is(kernel, stt)
        check_converged(g, pin, o64, st, dt, f"{case} [{kernel}]")
        solver.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. slot refill across >= 3 waves, mixed termination
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", ["gpi", "gps"])
def test_multiwave_refill(kernel, monkeypatch):
    """GPI: quadrotor N = 50 fp32 (32 instances per SM); GPS: one warp per SM.  Cold then warm with v / z, every instance
    judged by the to-convergence rule (refill faults show as instances far outside it)."""
    if kernel == "gps":
        monkeypatch.setenv("TINYMPC_GPS_WARPS", "1")
    dt = np.float32
    prob, st = MW._quad(50, dt)
    fam = KERNELS[kernel]
    B = 3 * MW._capacity(prob, st, fam) + 37
    inst = MW._tracking(B, 50, dt, seed=41)
    want = H.BOX_STATE
    run = F.oracle_pair(prob, st)
    pin1, o1 = run(inst["x0"], inst["Xref"], inst["Uref"], None, True, want)
    H.assert_mixed_termination(pin1)
    solver = _solver(prob, st, kernel)
    g1, stt = _device(solver, st, inst["x0"], inst, None, True, want, None)
    MW._assert_multiwave(stt, B, fam, 3.0)
    check_converged(g1, pin1, o1, st, dt, f"multiwave {kernel} cold")
    H.assert_mixed_termination(g1)
    x0b, state = F.warm_inputs(inst["x0"], pin1, want, seed=B)
    pin2, o2 = run(x0b, inst["Xref"], inst["Uref"], state, False, want)
    g2, stt = _device(solver, st, x0b, inst, state, False, want, None)
    MW._assert_multiwave(stt, B, fam, 3.0)
    check_converged(g2, pin2, o2, st, dt, f"multiwave {kernel} warm")
    solver.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. device-resident closed loop, 15 steps
# ---------------------------------------------------------------------------------------------------------------------
def _plant(A, Bm, f, x0, u0):
    """x <- (A x + B u0) + f: ascending sums, no FMA (tinympc_b200_advance's arithmetic), in the dtype of the operands."""
    nx, nu = A.shape[0], Bm.shape[1]
    nxt = np.zeros_like(x0)
    for i in range(nx):
        ax = A[i, 0] * x0[:, 0]
        for m in range(1, nx):
            ax = ax + A[i, m] * x0[:, m]
        bu = Bm[i, 0] * u0[:, 0]
        for j in range(1, nu):
            bu = bu + Bm[i, j] * u0[:, j]
        nxt[:, i] = (ax + bu) + f[i]
    return nxt


@pytest.mark.parametrize("case", ["quad_tracking_f32", "rocket_cones_f64"])
def test_device_closed_loop(case):
    """A FAST DeviceMPCLoop against (1) an fp64 oracle loop with an fp64 plant and (2) the pinned loop with the same plant
    arithmetic as the device: at every step FAST's x0 and u0 error against (1) <= C32 x the pinned loop's + a few ulps
    (fp64: 1e-10 relative)."""
    from tinympc_b200.closed_loop import DeviceMPCLoop

    steps = 15
    if case.startswith("quad"):
        dt = np.float32
        spec = wl.quadrotor(N=10)
        inst = wl.tracking_instances(150, N=10, seed=12, dtype=dt)
        extra = ()
        fields, reset, roll = ("v", "z", "vnew", "znew", "g", "y"), True, True
    else:
        dt = np.float64
        spec = wl.rocket(N=20)
        inst = wl.rocket_instances(90, N=20, seed=4, dtype=dt)
        extra = ("x", "u", "vcnew", "zcnew", "gc", "yc")
        fields, reset, roll = ("v", "z", "vnew", "znew", "g", "y") + extra, False, False
    prob = setup_problem(spec, dt)
    st = F.fixed_work(spec.settings)
    solver = _solver(prob, st, "auto")
    loop = DeviceMPCLoop(solver, inst["x0"], reset_duals=reset, extra_state=extra)
    p64 = prob.astype(np.float64)
    run = F.oracle_pair(prob, st)
    x_pin, x_64 = inst["x0"].copy(), inst["x0"].astype(np.float64)
    s_pin = s_64 = None
    worst = 0.0
    for k in range(steps):
        Xref = np.ascontiguousarray(np.roll(inst["Xref"], -k, axis=1 if inst["Xref"].ndim == 3 else 0)) if roll else inst["Xref"]
        x0_fast = loop.x0.cpu().numpy().copy()
        out = loop.step(Xref, inst.get("Uref"))
        stt = solver.stats()
        stt["_dt"] = dt.__name__
        _record(stt, _mask(st), False)
        u0_fast = out["u0"].cpu().numpy()
        for s in (s_pin, s_64):
            if s is not None and reset:
                s["g"], s["y"] = np.zeros_like(s["g"]), np.zeros_like(s["y"])
        # the two reference loops, each from its own state
        want = fields + (() if "u" in fields else ("u",))
        pin, _ = run(x_pin, Xref, inst.get("Uref"), s_pin, s_pin is None, want)
        _, o64 = run(x_64, Xref, inst.get("Uref"), s_64, s_64 is None, want)  # O64 from the fp64 loop's own x0 / state
        u_pin, u_64 = pin["u"][:, 0, :], o64["u"][:, 0, :]
        for name, a, p, r in (("x0", x0_fast, x_pin, x_64), ("u0", u0_fast, u_pin, u_64)):
            e_fast = float(np.abs(a.astype(np.float64) - r).max())
            e_pin = float(np.abs(p.astype(np.float64) - r).max())
            scale = float(np.abs(r).max())
            bound = F.REL64 * max(1.0, scale) if dt == np.float64 else F.C32 * e_pin + F.ULPS32 * F.EPS[np.float32] * scale
            worst = max(worst, e_fast / bound)
            assert e_fast <= bound, (case, k, name, e_fast, e_pin, bound)
        s_pin = {n: pin[n] for n in fields}
        s_64 = {n: o64[n] for n in fields}
        x_pin = _plant(prob.A, prob.B, prob.f, x_pin, np.ascontiguousarray(u_pin))
        x_64 = _plant(p64.A, p64.B, p64.f, x_64, np.ascontiguousarray(u_64))
    print(f"closed loop {case}: worst ratio {worst:.3g} over {steps} steps")
    solver.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. coverage: every FAST instantiation the library compiles was reached above
# ---------------------------------------------------------------------------------------------------------------------
def _compiled():
    gpi = {("gpi", "float32", L, het) for L in (4, 8) for het in (False, True)}
    gpi |= {("gpi", "float64", L, het) for L in (4, 8, 16) for het in (False, True)}
    gps = {("gps", m, v) for m in (0, 1, 6, 7) for v in ("shared", "het")}
    return gpi | gps | {("tpi", False), ("tpi", True)}


def test_fast_suite_reaches_every_fast_instantiation():
    if not REACHED:
        pytest.skip("the coverage record is filled by the other tests of this file: run the whole file")
    print("reached:", sorted(REACHED, key=str))
    assert REACHED == _compiled(), (sorted(_compiled() - REACHED, key=str), sorted(REACHED - _compiled(), key=str))
