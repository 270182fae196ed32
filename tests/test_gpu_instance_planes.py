"""Per-instance static hyperplanes (tinympc_batch_t.planes_per_instance) on the streamed (GPS) lane-group kernel, through the
device entry point, the host path, the Python layer and the device closed loop.

Every instance is compared bit for bit, on every output and requested state field, with the oracle run once per distinct
plane set over the instances that use it (planes_common.grouped_oracle).  The plane sets are dealt with a stride, so
neighbouring slots, the two instances of a lane group and the refills of a slot change planes.  Outputs and, on cold starts,
the requested state arrays are filled with a NaN bit pattern before each solve (H.poison), so an element a solve never writes
cannot match an oracle value by accident.  The launch plan is asserted through stats()."""
import ctypes as C
import os

import numpy as np
import pytest

import bounds_common as BC
import cones_common as CC
import helpers as H
import planes_common as PC
from tinympc_b200 import abi, workloads as wl
from tinympc_b200._lib import TinyMPCError
from tinympc_b200.batch import HostBatch
from tinympc_b200.solver import AdaptiveRho, BatchedTinySolver, pack_models, setup_models, setup_problem

pytestmark = pytest.mark.gpu

NT = os.cpu_count() or 1
OUTS = ("sol_x", "sol_u", "iter", "solved", "residuals", "u0")
WANT = tuple(H.LIN_STATE)
TV_WANT = WANT + ("vlnew_tv", "zlnew_tv", "gl_tv", "yl_tv")
DTS = [np.float32, np.float64]
PLAN = ("kernel_family", "lanes_per_instance", "instances_per_cta", "threads_per_cta", "ctas", "smem_bytes_per_cta")


# ---------------------------------------------------------------------------------------------------------------------
# problems, instances, the two solve paths
# ---------------------------------------------------------------------------------------------------------------------
def _settings(spec, **kw):
    st = abi.Settings.from_buffer_copy(spec.settings)
    for k, v in kw.items():
        setattr(st, k, v)
    return st


def _quad(dt, N, tv=False, **kw):
    """the hyperplane quadrotor (helpers.quad_linear_spec); tv: the time-varying hyperplanes of the handle run too (mask 6,
    both families)"""
    spec = H.quad_linear_spec(N=N)
    if tv:
        spec.constraints = dict(spec.constraints, **H.quad_linear_spec(tv=True, N=N).constraints)
        spec.settings.en_tv_state_linear = 1
        spec.settings.en_tv_input_linear = 1
    return spec, setup_problem(spec, dt), _settings(spec, **dict(dict(max_iter=40), **kw))


def _quad_instances(B, N, dt, seed):
    inst = wl.tracking_instances(B, N=N, seed=seed, dtype=dt, jitter=0.3)
    return dict(x0=inst["x0"], Xref=inst["Xref"], Uref=None)


def _sides(st):
    """the plane sides whose loops run under the settings"""
    return tuple(k for k, on in (("x", st.en_state_linear), ("u", st.en_input_linear)) if on)


def _expect(o, want):
    ref = {k: o[k] for k in H.OUT_KEYS + list(want)}
    ref["u0"] = np.ascontiguousarray(o["u"][:, 0, :])
    return ref


def _check(got, o, want, what):
    H.assert_bits_per_instance(got, _expect(o, want), H.OUT_KEYS + list(want) + ["u0"], what)


def _device(solver, x0, Xref, Uref, state, cold, want=WANT, models=None, planes=None, **kw):
    """tinympc_b200_solve on tensors from make_device_batch -> (numpy results, stats)"""
    import torch

    batch, out = solver.make_device_batch(x0, Xref, Uref, state=state, cold_start=cold, want_state=tuple(want), want_u0=True,
                                          models=models, planes=planes, **kw)
    for k in OUTS:
        H.poison(out[k])
    if cold:
        for n in want:
            H.poison(out[n])
    solver.solve_device(batch)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items() if v is not None}, solver.stats()


def _pinned(a, keep):
    import torch

    t = torch.empty(a.nbytes, dtype=torch.uint8, pin_memory=True)
    keep.append(t)
    p = t.numpy().view(a.dtype).reshape(a.shape)
    p[...] = a
    return p


def _host(solver, x0, Xref, Uref, state, cold, want=WANT, planes=None, models=None, pin=False):
    """tinympc_b200_solve_host on a HostBatch (u0 requested too); pin: every caller buffer page-locked"""
    p = solver.problem
    state = None if state is None else {n: np.array(a, copy=True) for n, a in state.items()}
    hb = HostBatch(p, x0, Xref, Uref, state=state, cold_start=cold, want_state=tuple(want), models=models, planes=planes)
    hb.u0 = np.empty((hb.B, p.nu), p.dtype)
    keep = []
    if pin:
        for n in ("x0", "Xref", "Uref", "sol_x", "sol_u", "iter", "solved", "residuals", "u0", "models"):
            if getattr(hb, n) is not None:
                setattr(hb, n, _pinned(getattr(hb, n), keep))
        hb.state = {n: _pinned(a, keep) for n, a in hb.state.items()}
        hb.planes = {n: _pinned(a, keep) for n, a in hb.planes.items()}
    for k in OUTS:
        H.poison(getattr(hb, k))
    if cold:
        for n in want:
            H.poison(hb.state[n])
    cb = hb.to_c()
    cb.u0 = hb.u0.ctypes.data
    solver.solve_prepared(hb, cb)
    return {k: np.array(v, copy=True) for k, v in dict(hb.result(), u0=hb.u0).items() if v is not None}, solver.stats()


def _warm_inputs(x0, res, seed, want=WANT):
    """the next MPC step: perturbed measurements, the returned state, duals reset on every third instance"""
    rng = np.random.default_rng(seed)
    x0b = (x0 + 0.02 * rng.standard_normal(x0.shape)).astype(x0.dtype)
    state = {n: np.array(res[n], copy=True) for n in want}
    for n in ("g", "y", "gl", "yl", "gl_tv", "yl_tv", "gc", "yc"):
        if n in state:
            state[n][::3] = 0
    return x0b, state


def _cold_warm(solver, inst, planes, what, models=None, model_of=None, want=WANT):
    """cold solve, then a warm step from the returned state with the duals reset on every third instance; every instance vs
    the grouped oracle; returns the two oracle results and the stats of the cold solve"""
    port = PC.grouped_oracle(solver.problem, solver.settings, planes, models=models, model_of=model_of, nthreads=NT)
    m = None if models is None else models[model_of]
    x0, Xref, Uref = inst["x0"], inst["Xref"], inst.get("Uref")
    o1 = port(x0, Xref, Uref, None, True, want)
    g1, st1 = _device(solver, x0, Xref, Uref, None, True, want, models=m, planes=planes)
    assert st1["kernel_family"] == abi.KERNEL_GPS and st1["kernel_launches"] == 1, st1
    _check(g1, o1, want, what + " cold")
    x0b, state = _warm_inputs(x0, o1, seed=len(x0), want=want)
    o2 = port(x0b, Xref, Uref, state, False, want)
    g2, st2 = _device(solver, x0b, Xref, Uref, state, False, want, models=m, planes=planes)
    assert st2["kernel_family"] == abi.KERNEL_GPS, st2
    _check(g2, o2, want, what + " warm")
    return o1, o2, st1


def _plan(stt):
    return {k: stt[k] for k in PLAN}


def _shared_plan(solver, inst, want=WANT, models=None):
    """the launch statistics of the same batch without per-instance planes"""
    _device(solver, inst["x0"], inst["Xref"], inst.get("Uref"), None, True, want, models=models)
    return solver.stats()


def _same_plan(shared, stt):
    """per-instance planes kept the shared solve's plan, shared memory included: they add no table"""
    assert _plan(stt) == _plan(shared), (stt, shared)


def _one_per_group(stt):
    assert stt["kernel_family"] == abi.KERNEL_GPS, stt
    assert stt["instances_per_cta"] == stt["threads_per_cta"] // stt["lanes_per_instance"], stt


def _fleet_palette(spec, prob, K, seed):
    """K robots' planes from workloads.plane_fleet, in the problem dtype"""
    f = wl.plane_fleet(spec, K, seed=seed, dtype=prob.dtype)
    return [{k: v[i] for k, v in f.items()} for i in range(K)]


def _quad_models(spec, dt, nm=4):
    """nm quadrotors of different masses (input matrix scaled by 1 / m): per-instance models"""
    rng = np.random.default_rng(11)
    m = 1.0 + 0.2 * rng.uniform(-1.0, 1.0, size=nm)
    tile = lambda a: np.tile(np.asarray(a, dtype=np.float64)[None], (nm,) + (1,) * np.ndim(a))  # noqa: E731
    return setup_models(spec.nx, spec.nu, tile(spec.A), tile(spec.B) / m[:, None, None], tile(spec.f), tile(spec.Qdiag),
                        tile(spec.Rdiag), np.full(nm, spec.rho), dtype=dt)


# ---------------------------------------------------------------------------------------------------------------------
# 1. every instance given the handle's planes: the shared solve's bits and plan
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
def test_equal_planes_equal_shared_solve(dt):
    spec, prob, st = _quad(dt, 50)
    s = BatchedTinySolver(prob, st)
    B = 1500
    inst = _quad_instances(B, 50, dt, seed=1)
    planes = PC.batch_planes([PC.own_planes(prob)], np.zeros(B, int))
    x0, state = inst["x0"], None
    for cold in (True, False):
        shared, s0 = _device(s, x0, inst["Xref"], None, state, cold)
        got, s1 = _device(s, x0, inst["Xref"], None, state, cold, planes=planes)
        _same_plan(s0, s1)
        H.assert_bits_per_instance(got, shared, list(shared), f"cold={cold}")
        x0, state = _warm_inputs(inst["x0"], shared, seed=2)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. quadrotor fleets: state planes only, input planes only, both
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("sides", ["x", "u", "xu"])
def test_quad_fleet(sides, dt):
    spec, prob, st = _quad(dt, 50, en_state_linear=int("x" in sides), en_input_linear=int("u" in sides))
    s = BatchedTinySolver(prob, st)
    B = 1200
    inst = _quad_instances(B, 50, dt, seed=3)
    pal = _fleet_palette(spec, prob, 7, seed=4)
    planes = PC.batch_planes(pal, BC.deal(B, 7, stride=3), sides=_sides(st))
    off = {"x": ("zlnew", "yl"), "u": ("vlnew", "gl"), "xu": ()}[sides]  # a side whose loop does not run: fields left unwritten
    want = tuple(n for n in WANT if n not in off)
    plan0 = _shared_plan(s, inst, want)
    o1, _, stt = _cold_warm(s, inst, planes, f"quad fleet {sides}", want=want)
    _same_plan(plan0, stt)
    # the planes bite: most instances end with a slack on one of their own planes
    act = PC.active_rows(planes, o1.get("vlnew"), o1.get("zlnew"))
    assert act.mean() >= 0.5, act.mean()
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. more than 2.5 waves of slot refills in one launch
# ---------------------------------------------------------------------------------------------------------------------
def _capacity(solver):
    """instances one wave of the solver's persistent kernel holds (ctas x instances_per_cta), from a one-iteration probe solve
    with per-instance planes that fills every SM"""
    import torch

    p = solver.problem
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    B = 256 * sm
    mi = solver.settings.max_iter
    solver.update_settings(max_iter=1)
    planes = PC.batch_planes([PC.own_planes(p)], np.zeros(B, int))
    batch, _ = solver.make_device_batch(np.zeros((B, p.nx), p.dtype), np.zeros((p.N, p.nx), p.dtype), cold_start=True, planes=planes)
    solver.solve_device(batch)
    torch.cuda.synchronize()
    solver.update_settings(max_iter=mi)
    stt = solver.stats()
    assert stt["ctas"] == sm, stt
    return stt["ctas"] * stt["instances_per_cta"]


@pytest.mark.parametrize("dt,warps", [(np.float64, None), (np.float32, "1"), (np.float64, "1")])
def test_multiwave(dt, warps, monkeypatch):
    if warps:
        monkeypatch.setenv("TINYMPC_GPS_WARPS", warps)
    spec, prob, st = _quad(dt, 20, max_iter=25)
    s = BatchedTinySolver(prob, st)
    B = int(2.6 * _capacity(s)) + 37
    K = 5
    pal = PC.plane_palette(prob, K - 1, seed=20) + PC.plane_palette(prob, 1, seed=22, pad=1)  # one robot pads a row of each side
    o1, _, stt = _cold_warm(s, _quad_instances(B, 20, dt, seed=21), PC.batch_planes(pal, BC.deal(B, K)), "multiwave")
    assert B >= 2.5 * stt["ctas"] * stt["instances_per_cta"], (B, stt)
    assert len(np.unique(o1["iter"])) >= 3, np.unique(o1["iter"])  # slots retire at different times
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. with per-instance models: one instance per lane group, the gps_het_slots plan
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
def test_with_models(dt):
    spec, prob, st = _quad(dt, 30)
    s = BatchedTinySolver(prob, st)
    B = 900
    inst = _quad_instances(B, 30, dt, seed=5)
    models = _quad_models(spec, dt)
    model_of = (np.arange(B) * 3) % 4
    plan0 = _shared_plan(s, inst, models=models[model_of])
    pal = PC.plane_palette(prob, 6, seed=6)
    _, _, stt = _cold_warm(s, inst, PC.batch_planes(pal, BC.deal(B, 6)), "planes + models", models=models, model_of=model_of)
    _one_per_group(stt)
    _same_plan(plan0, stt)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. static per-instance planes with the handle's time-varying planes (mask 6, both families); rocket with cones (mask 7)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
def test_with_time_varying_planes(dt):
    spec, prob, st = _quad(dt, 20, tv=True)
    s = BatchedTinySolver(prob, st)
    B = 700
    inst = _quad_instances(B, 20, dt, seed=7)
    plan0 = _shared_plan(s, inst, TV_WANT)
    pal = _fleet_palette(spec, prob, 5, seed=8)
    _, _, stt = _cold_warm(s, inst, PC.batch_planes(pal, BC.deal(B, 5, stride=3)), "static + tv planes", want=TV_WANT)
    _same_plan(plan0, stt)
    s.close()


def _rocket_planes_spec(N):
    """the conic rocket with a static state plane (a lateral corridor, x + 0.5 y <= 1) and an input plane (u0 + u1 <= 4)"""
    spec = wl.rocket(N=N)
    Ax = np.array([[1.0, 0.5, 0.0, 0.0, 0.0, 0.0]])
    Au = np.array([[1.0, 1.0, 0.0]])
    spec.constraints = dict(spec.constraints, Alin_x=Ax, blin_x=np.array([1.0]), Alin_u=Au, blin_u=np.array([4.0]))
    spec.settings.en_state_linear = 1
    spec.settings.en_input_linear = 1
    return spec


@pytest.mark.parametrize("dt", DTS)
def test_rocket_cones_and_planes(dt):
    spec = _rocket_planes_spec(50)
    prob = setup_problem(spec, dt)
    st = _settings(spec, max_iter=40, abs_pri_tol=0.1, abs_dua_tol=0.1)
    s = BatchedTinySolver(prob, st)
    B = 800
    inst = wl.rocket_instances(B, N=50, seed=9, dtype=dt, spread=0.3, per_instance_refs=True)
    want = tuple(H.SOC_STATE) + ("vlnew", "zlnew", "gl", "yl")
    plan0 = _shared_plan(s, inst, want)
    pal = PC.plane_palette(prob, 6, seed=10, shift=(-1.0, 0.2))
    _, _, stt = _cold_warm(s, inst, PC.batch_planes(pal, BC.deal(B, 6, stride=5)), "rocket cones + planes", want=want)
    _same_plan(plan0, stt)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. every compiled (nx, nu): covered shapes against the oracle, the others refused
# ---------------------------------------------------------------------------------------------------------------------
DIMS = [(4, 1), (6, 3), (12, 4), (4, 2), (4, 4), (4, 8), (8, 2), (8, 4), (8, 8), (12, 2), (12, 8), (16, 2), (16, 4), (16, 8)]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("nx,nu", DIMS)
def test_every_shape(nx, nu, dt):
    spec = wl.random_lti(nx, nu, 30, seed=300 + nx * 10 + nu)
    rng = np.random.default_rng(nx * 100 + nu)
    spec.constraints = dict(spec.constraints, Alin_x=rng.standard_normal((2, nx)), blin_x=np.array([0.2, 0.1]),
                            Alin_u=rng.standard_normal((1, nu)), blin_u=np.array([0.1]))
    spec.settings.en_state_linear = 1
    spec.settings.en_input_linear = 1
    prob = setup_problem(spec, dt)
    st = _settings(spec, max_iter=30)
    s = BatchedTinySolver(prob, st)
    B = 300
    inst = dict(x0=(0.5 * rng.standard_normal((B, nx))).astype(dt), Xref=(0.1 * rng.standard_normal((B, 30, nx))).astype(dt))
    _, sh = _device(s, inst["x0"], inst["Xref"], None, None, True)
    pal = PC.plane_palette(prob, 3, seed=nx + nu)
    planes = PC.batch_planes(pal, BC.deal(B, 3, stride=2))
    if sh["kernel_family"] != abi.KERNEL_GPS:
        with pytest.raises(TinyMPCError) as e:
            _device(s, inst["x0"], inst["Xref"], None, None, True, planes=planes)
        assert e.value.code == abi.ERR_UNSUPPORTED
        pytest.skip(f"({nx},{nu}) is not covered by the streamed kernel in this precision")
    _, _, stt = _cold_warm(s, inst, planes, f"({nx},{nu})")
    _same_plan(sh, stt)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. the host path in 11 chunks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pin", [False, True])
@pytest.mark.parametrize("dt,with_models", [(np.float32, False), (np.float64, False), (np.float32, True)])
def test_host_path_chunks(dt, with_models, pin, monkeypatch):
    spec, prob, st = _quad(dt, 20)
    s = BatchedTinySolver(prob, st)
    B = 11 * 96 - 40
    monkeypatch.setenv("TINYMPC_HOST_CHUNK", "96")
    pal = PC.plane_palette(prob, 7, seed=30)
    planes = PC.batch_planes(pal, BC.deal(B, 7, stride=3))
    models = _quad_models(spec, dt) if with_models else None
    model_of = None if models is None else np.arange(B) % 4
    m = None if models is None else models[model_of]
    port = PC.grouped_oracle(prob, st, planes, models=models, model_of=model_of, nthreads=NT)
    inst = _quad_instances(B, 20, dt, seed=31)
    o1 = port(inst["x0"], inst["Xref"], None, None, True, WANT)
    g1, stt = _host(s, inst["x0"], inst["Xref"], None, None, True, planes=planes, models=m, pin=pin)
    assert stt["kernel_launches"] == 11, stt
    _check(g1, o1, WANT, "host cold")
    x0b, state = _warm_inputs(inst["x0"], o1, seed=32)
    o2 = port(x0b, inst["Xref"], None, state, False, WANT)
    g2, stt = _host(s, x0b, inst["Xref"], None, state, False, planes=planes, models=m, pin=pin)
    _check(g2, o2, WANT, "host warm")
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 8. the device closed loop, one step's planes overridden (a moving obstacle)
# ---------------------------------------------------------------------------------------------------------------------
def _advance(prob, x0, u0):
    """tinympc_b200_advance's arithmetic: ascending sums, no FMA"""
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


@pytest.mark.parametrize("dt", DTS)
def test_closed_loop(dt):
    from tinympc_b200.closed_loop import DeviceMPCLoop

    spec, prob, st = _quad(dt, 30)
    s = BatchedTinySolver(prob, st)
    B = 400
    inst = _quad_instances(B, 30, dt, seed=42)
    pal = PC.plane_palette(prob, 4, seed=40)
    pal2 = PC.plane_palette(prob, 4, seed=41, shift=(-0.6, -0.2))  # one step with the obstacles closer
    which = BC.deal(B, 4, stride=3)
    extra = ("x", "u", "vlnew", "zlnew", "gl", "yl")
    loop = DeviceMPCLoop(s, inst["x0"], reset_duals=True, extra_state=extra, planes=PC.batch_planes(pal, which))
    want = loop.fields
    x0 = inst["x0"].copy()
    state = None
    for k in range(4):
        p_ = pal2 if k == 2 else pal
        out = loop.step(inst["Xref"], None, planes=PC.batch_planes(pal2, which) if k == 2 else None)
        if state is not None:
            state["g"] = np.zeros_like(state["g"])
            state["y"] = np.zeros_like(state["y"])
        o = PC.grouped_oracle(prob, st, PC.batch_planes(p_, which), nthreads=NT)(x0, inst["Xref"], None, state, state is None, want)
        got = {key: out[key].cpu().numpy() for key in H.OUT_KEYS + list(want) + ["u0"]}
        _check(got, o, want, f"closed loop step {k}")
        state = {n: o[n] for n in want}
        x0 = _advance(prob, x0, o["u"][:, 0, :])
        assert H.bits_equal(loop.x0.cpu().numpy(), x0), ("advance", k)
    with pytest.raises(ValueError):
        loop.rollout(inst["Xref"], 3)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 9. queued solves with different planes on one handle
# ---------------------------------------------------------------------------------------------------------------------
def test_queued_solves_different_planes():
    import torch

    dt = np.float32
    spec, prob, st = _quad(dt, 50)
    s = BatchedTinySolver(prob, st)
    B = 6000
    inst = _quad_instances(B, 50, dt, seed=50)
    pals = [PC.plane_palette(prob, 5, seed=51), PC.plane_palette(prob, 5, seed=52, shift=(-0.6, 0.0))]
    which = BC.deal(B, 5)
    dev = torch.device("cuda", 0)
    pls = [{k: torch.as_tensor(v, device=dev) for k, v in PC.batch_planes(p, which).items()} for p in pals]

    def run(sync):
        res = []
        for pl in pls:
            batch, out = s.make_device_batch(inst["x0"], inst["Xref"], None, cold_start=True, want_state=WANT, want_u0=True,
                                             planes=pl)
            for k in OUTS + WANT:
                H.poison(out[k])
            s.solve_device(batch)
            if sync:
                torch.cuda.synchronize()
            res.append((batch, out))
        torch.cuda.synchronize()
        return [{k: v.cpu().numpy() for k, v in out.items() if v is not None} for _, out in res]

    queued, synced = run(False), run(True)
    for q, y, p in zip(queued, synced, pals):
        H.assert_bits_per_instance(q, y, list(y), "queued vs synchronised")
        o = PC.grouped_oracle(prob, st, PC.batch_planes(p, which), nthreads=NT)(inst["x0"], inst["Xref"], None, None, True, WANT)
        _check(q, o, WANT, "queued vs oracle")
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 10. per-instance planes on a problem whose static hyperplane loops do not run: the solve without them
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
def test_plane_loops_off(dt):
    spec, prob, st = _quad(dt, 30, en_state_linear=0, en_input_linear=0)
    s = BatchedTinySolver(prob, st)
    B = 500
    inst = _quad_instances(B, 30, dt, seed=60)
    planes = PC.batch_planes(PC.plane_palette(prob, 3, seed=61), BC.deal(B, 3, stride=2))
    want = tuple(H.BOX_STATE)
    for pl in (planes, {k: planes[k] for k in ("Alin_x", "blin_x")}):
        shared, s0 = _device(s, inst["x0"], inst["Xref"], None, None, True, want)
        got, s1 = _device(s, inst["x0"], inst["Xref"], None, None, True, want, planes=pl)
        assert _plan(s0) == _plan(s1), (s0, s1)
        H.assert_bits_per_instance(got, shared, list(shared), "plane loops off")
    # the rocket has no hyperplane rows at all: no pointer is needed either
    rs = wl.rocket(N=20)
    r = BatchedTinySolver(setup_problem(rs, dt), rs.settings)
    rinst = wl.rocket_instances(64, N=20, seed=62, dtype=dt)
    batch, _ = r.make_device_batch(rinst["x0"], rinst["Xref"], rinst["Uref"], cold_start=True)
    batch.planes_per_instance = 1
    assert r._lib.tinympc_b200_solve(r._h, C.byref(batch), None) == abi.OK
    r.close()
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 11. loud errors
# ---------------------------------------------------------------------------------------------------------------------
def test_errors():
    import torch

    dt = np.float64
    spec = _rocket_planes_spec(20)
    prob = setup_problem(spec, dt)
    st = _settings(spec, max_iter=20)
    s = BatchedTinySolver(prob, st)
    B = 64
    inst = wl.rocket_instances(B, N=20, seed=70, dtype=dt)
    planes = PC.batch_planes(PC.plane_palette(prob, 2, seed=71), BC.deal(B, 2, stride=1))
    batch, _ = s.make_device_batch(inst["x0"], inst["Xref"], inst["Uref"], cold_start=True, planes=planes)

    def rc(b=batch):
        r = s._lib.tinympc_b200_solve(s._h, C.byref(b), None)
        torch.cuda.synchronize()
        return r

    def err():
        return s._lib.tinympc_b200_last_error()

    assert rc() == abi.OK
    # a missing pointer for a side whose loop runs; a bad mode; reserved4
    for field, val in (("Alin_x", None), ("blin_x", None), ("Alin_u", None), ("blin_u", None), ("planes_per_instance", 2),
                       ("planes_per_instance", -1), ("reserved4", 1)):
        b = abi.Batch.from_buffer_copy(batch)
        setattr(b, field, val)
        assert rc(b) == abi.ERR_ARG, field
    # the missing side's loop switched off: its pointers are never needed
    b = abi.Batch.from_buffer_copy(batch)
    b.Alin_u = b.blin_u = None
    s.update_settings(en_input_linear=0)
    assert rc(b) == abi.OK
    s.update_settings(en_input_linear=1)
    # FAST mode, explicit thread per instance
    s.set_mode(abi.MODE_FAST)
    assert rc() == abi.ERR_UNSUPPORTED and b"STRICT" in err()
    s.set_mode(abi.MODE_STRICT, abi.KERNEL_TPI)
    assert rc() == abi.ERR_UNSUPPORTED and b"thread per instance" in err()
    s.set_mode(abi.MODE_STRICT, abi.KERNEL_AUTO)
    # per-instance bounds or cones in the same batch
    bb, _ = s.make_device_batch(inst["x0"], inst["Xref"], inst["Uref"], cold_start=True, planes=planes,
                                bounds=dict(u_min=np.full((B, 3), -10.0), u_max=np.full((B, 3), 105.0),
                                            x_min=np.tile(prob.x_min[:, 0], (B, 1)), x_max=np.tile(prob.x_max[:, 0], (B, 1))))
    assert rc(bb) == abi.ERR_UNSUPPORTED and b"bounds or cones" in err()
    cb, _ = s.make_device_batch(inst["x0"], inst["Xref"], inst["Uref"], cold_start=True, planes=planes,
                                cones=CC.batch_cones(CC.mu_palette(prob, 1, seed=72), np.zeros(B, int)))
    assert rc(cb) == abi.ERR_UNSUPPORTED and b"bounds or cones" in err()
    # adaptive rho and rollouts
    models = torch.as_tensor(pack_models(prob, B), device="cuda")
    dK, dP = np.zeros((prob.nu, prob.nx), dt), np.zeros((prob.nx, prob.nx), dt)
    ar = AdaptiveRho(dK, dP).to_c(prob, models.data_ptr(), B, models.device)
    assert s._lib.tinympc_b200_solve_adaptive(s._h, C.byref(batch), C.byref(ar), None) == abi.ERR_UNSUPPORTED
    assert b"hyperplanes" in err()
    rb = abi.Batch.from_buffer_copy(batch)
    rb.Xref = rb.Uref = rb.iter = rb.solved = rb.residuals = rb.u0 = None
    rb.sol_x = rb.sol_u = None
    r = abi.Rollout()
    X = torch.as_tensor(np.ascontiguousarray(inst["Xref"]), device="cuda")
    r.T, r.Xref = 1, X.data_ptr()
    assert s._lib.tinympc_b200_rollout(s._h, C.byref(rb), C.byref(r), None) == abi.ERR_UNSUPPORTED
    assert b"rollout" in err()
    # Python checks: shapes, dtype, keys, pairs
    bad = [dict(planes, Alin_x=planes["Alin_x"][:, :, :-1]), dict(planes, blin_u=planes["blin_u"][:-1]),
           dict(planes, Alin_x=planes["Alin_x"].astype(np.float32)), {"Alin_x": planes["Alin_x"]},
           dict(planes, A=planes["Alin_x"]), {}]
    for pp in bad:
        with pytest.raises(ValueError):
            s.make_device_batch(inst["x0"], inst["Xref"], cold_start=True, planes=pp)
        with pytest.raises(ValueError):
            s.solve(inst["x0"], inst["Xref"], planes=pp)
    s.close()
