"""Per-instance cone coefficients (tinympc_batch_t.cones_per_instance) on the streamed (GPS) lane-group kernel, through the device
entry point, the host path, the Python layer and the device closed loop.

Every instance is compared bit for bit, on every output and requested state field, with the oracle run once per distinct mu
set over the instances that use it (cones_common.grouped_oracle).  The mu sets are dealt with a stride, so neighbouring slots,
the two instances of a lane group and the refills of a slot change mu.  Outputs and, on cold starts, the requested state
arrays are filled with a NaN bit pattern before each solve (H.poison), so an element a solve never writes cannot match an
oracle value by accident.  The launch plan is asserted through stats()."""
import os

import numpy as np
import pytest

import bounds_common as BC
import cones_common as CC
import helpers as H
from tinympc_b200 import abi, workloads as wl
from tinympc_b200._lib import TinyMPCError
from tinympc_b200.batch import HostBatch
from tinympc_b200.solver import AdaptiveRho, BatchedTinySolver, pack_models, setup_models, setup_problem

pytestmark = pytest.mark.gpu

NT = os.cpu_count() or 1
OUTS = ("sol_x", "sol_u", "iter", "solved", "residuals", "u0")
WANT = tuple(H.SOC_STATE)
DTS = [np.float32, np.float64]
PLAN = ("kernel_family", "lanes_per_instance", "instances_per_cta", "threads_per_cta", "ctas")


# ---------------------------------------------------------------------------------------------------------------------
# problems, instances, the two solve paths
# ---------------------------------------------------------------------------------------------------------------------
def _settings(spec, **kw):
    st = abi.Settings.from_buffer_copy(spec.settings)
    for k, v in kw.items():
        setattr(st, k, v)
    return st


def _rocket(dt, N, **kw):
    spec = wl.rocket(N=N)
    return setup_problem(spec, dt), _settings(spec, **dict(dict(max_iter=40, abs_pri_tol=0.1, abs_dua_tol=0.1), **kw))


def _rocket_instances(B, N, dt, seed):
    return wl.rocket_instances(B, N=N, seed=seed, dtype=dt, spread=0.3, per_instance_refs=True)


def _sides(st):
    """the cone sides whose loops run under the settings"""
    return tuple(k for k, on in (("x_mu", st.en_state_soc), ("u_mu", st.en_input_soc)) if on)


def _expect(o, want):
    ref = {k: o[k] for k in H.OUT_KEYS + list(want)}
    ref["u0"] = np.ascontiguousarray(o["u"][:, 0, :])
    return ref


def _check(got, o, want, what):
    H.assert_bits_per_instance(got, _expect(o, want), H.OUT_KEYS + list(want) + ["u0"], what)


def _device(solver, x0, Xref, Uref, state, cold, want=WANT, models=None, bounds=None, cones=None):
    """tinympc_b200_solve on tensors from make_device_batch -> (numpy results, stats)"""
    import torch

    batch, out = solver.make_device_batch(x0, Xref, Uref, state=state, cold_start=cold, want_state=tuple(want), want_u0=True,
                                          models=models, bounds=bounds, cones=cones)
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


def _host(solver, x0, Xref, Uref, state, cold, want=WANT, cones=None, models=None, pin=False):
    """tinympc_b200_solve_host on a HostBatch (u0 requested too); pin: every caller buffer page-locked"""
    p = solver.problem
    state = None if state is None else {n: np.array(a, copy=True) for n, a in state.items()}
    hb = HostBatch(p, x0, Xref, Uref, state=state, cold_start=cold, want_state=tuple(want), models=models, cones=cones)
    hb.u0 = np.empty((hb.B, p.nu), p.dtype)
    keep = []
    if pin:
        for n in ("x0", "Xref", "Uref", "sol_x", "sol_u", "iter", "solved", "residuals", "u0", "models"):
            if getattr(hb, n) is not None:
                setattr(hb, n, _pinned(getattr(hb, n), keep))
        hb.state = {n: _pinned(a, keep) for n, a in hb.state.items()}
        hb.cones = {n: _pinned(a, keep) for n, a in hb.cones.items()}
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
    for n in ("g", "y", "gc", "yc"):
        if n in state:
            state[n][::3] = 0
    return x0b, state


def _cold_warm(solver, inst, cones, what, models=None, model_of=None, bpal=None, bwhich=None, want=WANT):
    """cold solve, then a warm step from the returned state with the duals reset on every third instance; every instance vs
    the grouped oracle; returns the two oracle results and the stats of the cold solve"""
    port = CC.grouped_oracle(solver.problem, solver.settings, cones, models=models, model_of=model_of, bpal=bpal, bwhich=bwhich,
                             nthreads=NT)
    m = None if models is None else models[model_of]
    bounds = None if bpal is None else BC.batch_bounds(bpal, bwhich)
    x0, Xref, Uref = inst["x0"], inst["Xref"], inst.get("Uref")
    o1 = port(x0, Xref, Uref, None, True, want)
    g1, st1 = _device(solver, x0, Xref, Uref, None, True, want, models=m, bounds=bounds, cones=cones)
    assert st1["kernel_family"] == abi.KERNEL_GPS and st1["kernel_launches"] == 1, st1
    _check(g1, o1, want, what + " cold")
    x0b, state = _warm_inputs(x0, o1, seed=len(x0), want=want)
    o2 = port(x0b, Xref, Uref, state, False, want)
    g2, st2 = _device(solver, x0b, Xref, Uref, state, False, want, models=m, bounds=bounds, cones=cones)
    assert st2["kernel_family"] == abi.KERNEL_GPS, st2
    _check(g2, o2, want, what + " warm")
    return o1, o2, st1


def _plan(stt):
    return {k: stt[k] for k in PLAN}


def _shared_plan(solver, inst, models=None):
    """the launch statistics of the same batch without per-instance cones"""
    _device(solver, inst["x0"], inst["Xref"], inst.get("Uref"), None, True, models=models)
    return solver.stats()


def _same_plan(shared, stt, dt):
    """per-instance cones kept the shared solve's plan (lanes, instances per lane group, warps, CTAs); shared memory grew by
    the cone-coefficient table alone: MAX_CONES (4) mu per side and slot"""
    assert _plan(stt) == _plan(shared), (stt, shared)
    assert stt["smem_bytes_per_cta"] - shared["smem_bytes_per_cta"] == stt["instances_per_cta"] * 2 * 4 * np.dtype(dt).itemsize, (stt, shared)


def _one_per_group(stt):
    assert stt["kernel_family"] == abi.KERNEL_GPS, stt
    assert stt["instances_per_cta"] == stt["threads_per_cta"] // stt["lanes_per_instance"], stt


def _two_per_group(stt):
    assert stt["kernel_family"] == abi.KERNEL_GPS, stt
    assert stt["instances_per_cta"] == 2 * (stt["threads_per_cta"] // stt["lanes_per_instance"]), stt


def _rocket_models(dt, nm=4):
    """nm rockets of different masses (wl.rocket_fleet): per-instance models"""
    f = wl.rocket_fleet(nm, N=10, seed=3)
    spec = f["spec"]
    return setup_models(spec.nx, spec.nu, f["A"], f["B"], f["f"], f["Qdiag"], f["Rdiag"], f["rho"], dtype=dt)


def _thrust_palette(prob, K, layout, seed):
    """K rockets' thrust limits (the problem's u bounds scaled by 0.6 .. 1.0) and the problem's state bounds"""
    pal = BC.palette(prob, K, layout, seed, scale=1.0, tight=0.4)
    for d in pal:
        for k in ("x_min", "x_max"):
            a = np.asarray(getattr(prob, k))
            d[k] = np.ascontiguousarray(a[:, 0] if layout == 1 else a.T, dtype=prob.dtype)
    return pal


# ---------------------------------------------------------------------------------------------------------------------
# 1. every instance given the handle's mu: the shared solve's bits and plan (two instances per lane group kept)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
def test_equal_mu_equal_shared_solve(dt):
    prob, st = _rocket(dt, 100)
    s = BatchedTinySolver(prob, st)
    B = 700
    inst = _rocket_instances(B, 100, dt, seed=1)
    cones = CC.batch_cones([dict(x_mu=prob.cx, u_mu=prob.cu)], np.zeros(B, int))
    x0, state = inst["x0"], None
    for cold in (True, False):
        shared, s0 = _device(s, x0, inst["Xref"], inst["Uref"], state, cold)
        got, s1 = _device(s, x0, inst["Xref"], inst["Uref"], state, cold, cones=cones)
        _same_plan(s0, s1, dt)
        _two_per_group(s1)
        H.assert_bits_per_instance(got, shared, list(shared), f"cold={cold}")
        x0, state = _warm_inputs(inst["x0"], shared, seed=2)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. a fleet on the rocket shape, N = 100: state cones only, input cones only, both
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("sides", ["x", "u", "xu"])
def test_rocket_fleet(sides, dt):
    prob, st = _rocket(dt, 100, en_state_soc=int("x" in sides), en_input_soc=int("u" in sides))
    s = BatchedTinySolver(prob, st)
    B = 900
    inst = _rocket_instances(B, 100, dt, seed=3)
    fleet = wl.cone_fleet(wl.rocket(N=100), 7, seed=4, dtype=dt)  # 7 robots' mu (x 0.6 .. 1.0), dealt with a stride
    pal = [dict(x_mu=fleet["x_mu"][i], u_mu=fleet["u_mu"][i]) for i in range(7)]
    cones = CC.batch_cones(pal, BC.deal(B, 7, stride=3), sides=_sides(st))
    plan0 = _shared_plan(s, inst)
    off = {"x": ("zcnew", "yc"), "u": ("vcnew", "gc"), "xu": ()}[sides]  # a side whose loop does not run: fields left unwritten
    o1, _, stt = _cold_warm(s, inst, cones, f"rocket fleet {sides}", want=tuple(n for n in WANT if n not in off))
    _same_plan(plan0, stt, dt)
    _two_per_group(stt)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. more than 2.5 waves of slot refills in one launch
# ---------------------------------------------------------------------------------------------------------------------
def _capacity(solver):
    """instances one wave of the solver's persistent kernel holds (ctas x instances_per_cta), from a one-iteration probe solve
    with per-instance cones that fills every SM"""
    import torch

    p = solver.problem
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    B = 256 * sm
    mi = solver.settings.max_iter
    solver.update_settings(max_iter=1)
    cones = CC.batch_cones([dict(x_mu=p.cx, u_mu=p.cu)], np.zeros(B, int))
    batch, _ = solver.make_device_batch(np.zeros((B, p.nx), p.dtype), np.zeros((p.N, p.nx), p.dtype), cold_start=True, cones=cones)
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
    prob, st = _rocket(dt, 20, max_iter=25)
    s = BatchedTinySolver(prob, st)
    B = int(2.6 * _capacity(s)) + 37
    K = 5
    pal = CC.mu_palette(prob, K, seed=20, scale=(0.4, 1.0))
    o1, _, stt = _cold_warm(s, _rocket_instances(B, 20, dt, seed=21), CC.batch_cones(pal, BC.deal(B, K)), "multiwave")
    assert B >= 2.5 * stt["ctas"] * stt["instances_per_cta"], (B, stt)
    assert len(np.unique(o1["iter"])) > 3, np.unique(o1["iter"])  # slots retire at different times
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. with per-instance models, per-instance bounds (both layouts), and both
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("combo", ["models", "bounds1", "bounds2", "models+bounds2"])
def test_with_models_and_bounds(combo, dt):
    prob, st = _rocket(dt, 50)
    s = BatchedTinySolver(prob, st)
    B = 700
    inst = _rocket_instances(B, 50, dt, seed=5)
    pal = CC.mu_palette(prob, 6, seed=6)
    cones = CC.batch_cones(pal, BC.deal(B, 6))
    kw = {}
    if "models" in combo:
        kw.update(models=_rocket_models(dt), model_of=(np.arange(B) * 3) % 4)
    if "bounds" in combo:
        layout = int(combo[-1])
        kw.update(bpal=_thrust_palette(prob, 5, layout, seed=7), bwhich=BC.deal(B, 5, stride=3))
    _, _, stt = _cold_warm(s, inst, cones, f"cones + {combo}", **kw)
    _one_per_group(stt)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. cones together with static and time-varying hyperplanes (family mask 7)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("tv", [False, True])
def test_cones_with_hyperplanes(tv, dt):
    spec = H.quad_linear_spec(tv=tv, N=20)
    spec.constraints = dict(spec.constraints, Acx=[0], qcx=[3], cx=[0.8], Acu=[1], qcu=[3], cu=[1.5])
    spec.settings.en_state_soc = 1
    spec.settings.en_input_soc = 1
    prob = setup_problem(spec, dt)
    st = _settings(spec, max_iter=40, abs_pri_tol=1e-2, abs_dua_tol=1e-2)
    s = BatchedTinySolver(prob, st)
    rng = np.random.default_rng(3)
    B, N = 500, spec.N
    inst = dict(x0=(0.3 * rng.standard_normal((B, 12))).astype(dt), Xref=(0.05 * rng.standard_normal((B, N, 12))).astype(dt),
                Uref=(0.02 * rng.standard_normal((B, N - 1, 4))).astype(dt))
    inst["Xref"][:, :, 2] += 0.5  # the state cone's axis: altitude
    pal = CC.mu_palette(prob, 4, seed=8, scale=(0.3, 1.5))
    plan0 = _shared_plan(s, inst)
    _, _, stt = _cold_warm(s, inst, CC.batch_cones(pal, BC.deal(B, 4, stride=3)), f"cones + hyperplanes tv={tv}")
    _same_plan(plan0, stt, dt)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. every compiled (nx, nu) the streamed kernel covers; input cones where nu >= 3
# ---------------------------------------------------------------------------------------------------------------------
DIMS = [(4, 1), (6, 3), (12, 4), (4, 2), (4, 4), (4, 8), (8, 2), (8, 4), (8, 8), (12, 2), (12, 8), (16, 2), (16, 4), (16, 8)]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("nx,nu", DIMS)
def test_every_shape(nx, nu, dt):
    spec = wl.random_lti(nx, nu, 30, seed=200 + nx * 10 + nu)
    cons = dict(Acx=[0, nx - 3], qcx=[3, 3], cx=[0.7, 1.3])
    spec.settings.en_state_soc = 1
    if nu >= 3:
        cons.update(Acu=[0], qcu=[3], cu=[0.9])
        spec.settings.en_input_soc = 1
    spec.constraints = dict(spec.constraints, **cons)
    prob = setup_problem(spec, dt)
    st = _settings(spec, max_iter=30)
    s = BatchedTinySolver(prob, st)
    B = 300
    rng = np.random.default_rng(nx * nu)
    inst = dict(x0=(0.5 * rng.standard_normal((B, nx))).astype(dt), Xref=(0.1 * rng.standard_normal((B, 30, nx))).astype(dt))
    inst["x0"][:, 2] += 0.3
    _, sh = _device(s, inst["x0"], inst["Xref"], None, None, True)
    if sh["kernel_family"] != abi.KERNEL_GPS:
        pal = CC.mu_palette(prob, 3, seed=nx + nu)
        with pytest.raises(TinyMPCError) as e:
            _device(s, inst["x0"], inst["Xref"], None, None, True, cones=CC.batch_cones(pal, BC.deal(B, 3, stride=2), _sides(st)))
        assert e.value.code == abi.ERR_UNSUPPORTED
        pytest.skip(f"({nx},{nu}) is not covered by the streamed kernel in this precision")
    pal = CC.mu_palette(prob, 3, seed=nx + nu, scale=(0.3, 1.2))
    want = WANT if nu >= 3 else tuple(n for n in WANT if n not in ("zcnew", "yc"))  # no input cones: their fields stay unwritten
    _, _, stt = _cold_warm(s, inst, CC.batch_cones(pal, BC.deal(B, 3, stride=2), _sides(st)), f"({nx},{nu})", want=want)
    _same_plan(sh, stt, dt)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. the host path in 11 chunks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pin", [False, True])
@pytest.mark.parametrize("dt,with_models", [(np.float32, False), (np.float64, False), (np.float64, True)])
def test_host_path_chunks(dt, with_models, pin, monkeypatch):
    prob, st = _rocket(dt, 20)
    s = BatchedTinySolver(prob, st)
    B = 11 * 96 - 40
    monkeypatch.setenv("TINYMPC_HOST_CHUNK", "96")
    pal = CC.mu_palette(prob, 7, seed=30)
    cones = CC.batch_cones(pal, BC.deal(B, 7, stride=3))
    models = _rocket_models(dt) if with_models else None
    model_of = None if models is None else np.arange(B) % 4
    m = None if models is None else models[model_of]
    port = CC.grouped_oracle(prob, st, cones, models=models, model_of=model_of, nthreads=NT)
    inst = _rocket_instances(B, 20, dt, seed=31)
    o1 = port(inst["x0"], inst["Xref"], inst["Uref"], None, True, WANT)
    g1, stt = _host(s, inst["x0"], inst["Xref"], inst["Uref"], None, True, cones=cones, models=m, pin=pin)
    assert stt["kernel_launches"] == 11, stt
    _check(g1, o1, WANT, "host cold")
    x0b, state = _warm_inputs(inst["x0"], o1, seed=32)
    o2 = port(x0b, inst["Xref"], inst["Uref"], state, False, WANT)
    g2, stt = _host(s, x0b, inst["Xref"], inst["Uref"], state, False, cones=cones, models=m, pin=pin)
    _check(g2, o2, WANT, "host warm")
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 8. the device closed loop
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

    prob, st = _rocket(dt, 30)
    s = BatchedTinySolver(prob, st)
    B = 400
    inst = _rocket_instances(B, 30, dt, seed=42)
    pal = CC.mu_palette(prob, 4, seed=40)
    pal2 = CC.mu_palette(prob, 4, seed=41, scale=(0.3, 0.6))  # one step with tighter cones
    which = BC.deal(B, 4, stride=3)
    extra = ("x", "u", "vcnew", "zcnew", "gc", "yc")
    loop = DeviceMPCLoop(s, inst["x0"], reset_duals=True, extra_state=extra, cones=CC.batch_cones(pal, which))
    want = loop.fields
    x0 = inst["x0"].copy()
    state = None
    for k in range(4):
        p_ = pal2 if k == 2 else pal
        out = loop.step(inst["Xref"], inst["Uref"], cones=CC.batch_cones(pal2, which) if k == 2 else None)
        if state is not None:
            state["g"] = np.zeros_like(state["g"])
            state["y"] = np.zeros_like(state["y"])
        o = CC.grouped_oracle(prob, st, CC.batch_cones(p_, which), nthreads=NT)(x0, inst["Xref"], inst["Uref"], state, state is None, want)
        got = {key: out[key].cpu().numpy() for key in H.OUT_KEYS + list(want) + ["u0"]}
        _check(got, o, want, f"closed loop step {k}")
        state = {n: o[n] for n in want}
        x0 = _advance(prob, x0, o["u"][:, 0, :])
        assert H.bits_equal(loop.x0.cpu().numpy(), x0), ("advance", k)
    with pytest.raises(ValueError):
        loop.rollout(inst["Xref"], 3)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 9. queued solves with different mu on one handle
# ---------------------------------------------------------------------------------------------------------------------
def test_queued_solves_different_mu():
    import torch

    dt = np.float64
    prob, st = _rocket(dt, 50)
    s = BatchedTinySolver(prob, st)
    B = 3000
    inst = _rocket_instances(B, 50, dt, seed=50)
    pals = [CC.mu_palette(prob, 5, seed=51), CC.mu_palette(prob, 5, seed=52, scale=(0.3, 0.7))]
    which = BC.deal(B, 5)
    dev = torch.device("cuda", 0)
    cns = [{k: torch.as_tensor(v, device=dev) for k, v in CC.batch_cones(p, which).items()} for p in pals]

    def run(sync):
        res = []
        for c in cns:
            batch, out = s.make_device_batch(inst["x0"], inst["Xref"], inst["Uref"], cold_start=True, want_state=WANT, want_u0=True,
                                             cones=c)
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
        o = CC.grouped_oracle(prob, st, CC.batch_cones(p, which), nthreads=NT)(inst["x0"], inst["Xref"], inst["Uref"], None, True, WANT)
        _check(q, o, WANT, "queued vs oracle")
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 10. per-instance cones on a problem whose cone loops do not run: the solve without them
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
def test_cone_loops_off(dt):
    prob, st = _rocket(dt, 50, en_state_soc=0, en_input_soc=0)
    s = BatchedTinySolver(prob, st)
    B = 500
    inst = _rocket_instances(B, 50, dt, seed=60)
    cones = CC.batch_cones(CC.mu_palette(prob, 3, seed=61), BC.deal(B, 3, stride=2))
    want = tuple(H.BOX_STATE)
    for c in (cones, {"x_mu": cones["x_mu"]}):
        shared, s0 = _device(s, inst["x0"], inst["Xref"], inst["Uref"], None, True, want)
        got, s1 = _device(s, inst["x0"], inst["Xref"], inst["Uref"], None, True, want, cones=c)
        assert _plan(s0) == _plan(s1) and s0["smem_bytes_per_cta"] == s1["smem_bytes_per_cta"], (s0, s1)
        H.assert_bits_per_instance(got, shared, list(shared), "cone loops off")
    # a box-only problem without any cones: no pointer is needed either
    import ctypes as C

    batch, _ = s.make_device_batch(inst["x0"], inst["Xref"], inst["Uref"], cold_start=True)
    batch.cones_per_instance = 1
    assert s._lib.tinympc_b200_solve(s._h, C.byref(batch), None) == abi.OK
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 11. loud errors
# ---------------------------------------------------------------------------------------------------------------------
def test_errors():
    import ctypes as C

    import torch

    dt = np.float64
    prob, st = _rocket(dt, 20)
    s = BatchedTinySolver(prob, st)
    B = 64
    inst = _rocket_instances(B, 20, dt, seed=70)
    cones = CC.batch_cones(CC.mu_palette(prob, 2, seed=71), BC.deal(B, 2, stride=1))
    batch, _ = s.make_device_batch(inst["x0"], inst["Xref"], inst["Uref"], cold_start=True, cones=cones)

    def rc(b=batch):
        r = s._lib.tinympc_b200_solve(s._h, C.byref(b), None)
        torch.cuda.synchronize()
        return r

    def err():
        return s._lib.tinympc_b200_last_error()

    assert rc() == abi.OK
    # a missing pointer for a side whose loop runs; a bad mode; reserved3
    for field, val in (("cone_x_mu", None), ("cone_u_mu", None), ("cones_per_instance", 2), ("cones_per_instance", -1), ("reserved3", 1)):
        b = abi.Batch.from_buffer_copy(batch)
        setattr(b, field, val)
        assert rc(b) == abi.ERR_ARG, field
    # the missing side's loop switched off: its pointer is never needed
    b = abi.Batch.from_buffer_copy(batch)
    b.cone_u_mu = None
    s.update_settings(en_input_soc=0)
    assert rc(b) == abi.OK
    s.update_settings(en_input_soc=1)
    # FAST mode, explicit thread per instance
    s.set_mode(abi.MODE_FAST)
    assert rc() == abi.ERR_UNSUPPORTED and b"STRICT" in err()
    s.set_mode(abi.MODE_STRICT, abi.KERNEL_TPI)
    assert rc() == abi.ERR_UNSUPPORTED and b"thread per instance" in err()
    s.set_mode(abi.MODE_STRICT, abi.KERNEL_AUTO)
    # adaptive rho and rollouts
    models = torch.as_tensor(pack_models(prob, B), device="cuda")
    dK, dP = np.zeros((prob.nu, prob.nx), dt), np.zeros((prob.nx, prob.nx), dt)
    ar = AdaptiveRho(dK, dP).to_c(prob, models.data_ptr(), B, models.device)
    assert s._lib.tinympc_b200_solve_adaptive(s._h, C.byref(batch), C.byref(ar), None) == abi.ERR_UNSUPPORTED
    assert b"cone" in err()
    rb = abi.Batch.from_buffer_copy(batch)
    rb.Xref = rb.Uref = rb.iter = rb.solved = rb.residuals = rb.u0 = None
    rb.sol_x = rb.sol_u = None
    r = abi.Rollout()
    X = torch.as_tensor(np.ascontiguousarray(inst["Xref"][0]), device="cuda")
    r.T, r.Xref = 1, X.data_ptr()
    assert s._lib.tinympc_b200_rollout(s._h, C.byref(rb), C.byref(r), None) == abi.ERR_UNSUPPORTED
    assert b"rollout" in err()
    # Python checks: shapes, dtype, keys
    bad = [dict(cones, x_mu=cones["x_mu"][:, :0]), dict(cones, u_mu=cones["u_mu"][:-1]), dict(cones, x_mu=cones["x_mu"].astype(np.float32)),
           dict(cones, x_mu=cones["x_mu"][:, :, None]), dict(cones, mu=cones["x_mu"]), {}]
    for cc in bad:
        with pytest.raises(ValueError):
            s.make_device_batch(inst["x0"], inst["Xref"], cold_start=True, cones=cc)
        with pytest.raises(ValueError):
            s.solve(inst["x0"], inst["Xref"], cones=cc)
    s.close()
