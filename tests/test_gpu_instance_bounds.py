"""Per-instance box bounds (tinympc_batch_t.bounds_per_instance) on the on-chip (GPI) and streamed (GPS) lane-group kernels,
through the device entry point, the host path, the Python layer and the device closed loop.

Every instance is compared bit for bit, on every output and requested state field, with the oracle run once per bound set over
the instances that use it (bounds_common.grouped_oracle).  The bound sets are dealt with a stride, so neighbouring slots and
the refills of a slot change bounds.  Outputs and, on cold starts, the requested state arrays are filled with a NaN bit
pattern before each solve (H.poison), so an element a solve never writes cannot match an oracle value by accident.  The
launch plan is asserted through stats()."""
import os

import numpy as np
import pytest

import bounds_common as BC
import helpers as H
from tinympc_b200 import abi, workloads as wl
from tinympc_b200._lib import TinyMPCError
from tinympc_b200.batch import HostBatch
from tinympc_b200.solver import AdaptiveRho, BatchedTinySolver, pack_models, setup_models, setup_problem

pytestmark = pytest.mark.gpu

NT = os.cpu_count() or 1
OUTS = ("sol_x", "sol_u", "iter", "solved", "residuals", "u0")
WANT = tuple(H.BOX_STATE)
DTS = [np.float32, np.float64]


# ---------------------------------------------------------------------------------------------------------------------
# problems, instances, the two solve paths
# ---------------------------------------------------------------------------------------------------------------------
def _settings(spec, **kw):
    st = abi.Settings.from_buffer_copy(spec.settings)
    for k, v in kw.items():
        setattr(st, k, v)
    return st


def _quad(N, dt, max_iter=15):
    """Quadrotor tracking; with x0 jittered by 0.5 and max_iter = 15 instances converge after 7..15 iterations or stop at
    max_iter, so the slots of a warp retire at different times."""
    spec = wl.quadrotor(N=N)
    return setup_problem(spec, dt), _settings(spec, max_iter=max_iter)


def _tracking(B, N, dt, seed):
    inst = wl.tracking_instances(B, N=N, seed=seed, dtype=dt, jitter=0.5)
    inst["Uref"] = (0.05 * np.random.default_rng(seed + 1).standard_normal((B, N - 1, 4))).astype(dt)
    return inst


def _rocket(dt, N, **cons):
    spec = wl.rocket(N=N)
    if cons:
        spec.constraints = dict(spec.constraints, **cons)
    return setup_problem(spec, dt), _settings(spec, max_iter=40, abs_pri_tol=0.1, abs_dua_tol=0.1)


def _rocket_instances(B, N, dt, seed):
    return wl.rocket_instances(B, N=N, seed=seed, dtype=dt, spread=0.3, per_instance_refs=True)


def _thrust_palette(prob, K, layout, seed):
    """K rockets' thrust limits (the problem's u bounds scaled by 0.6 .. 1.0) and the problem's state bounds"""
    pal = BC.palette(prob, K, layout, seed, scale=1.0, tight=0.4)
    for d in pal:
        for k in ("x_min", "x_max"):
            a = np.asarray(getattr(prob, k))
            d[k] = np.ascontiguousarray(a[:, 0] if layout == 1 else a.T, dtype=prob.dtype)
    return pal


def _expect(o, want):
    ref = {k: o[k] for k in H.OUT_KEYS + list(want)}
    ref["u0"] = np.ascontiguousarray(o["u"][:, 0, :])
    return ref


def _check(got, o, want, what):
    H.assert_bits_per_instance(got, _expect(o, want), H.OUT_KEYS + list(want) + ["u0"], what)


def _device(solver, x0, Xref, Uref, state, cold, want=WANT, models=None, bounds=None):
    """tinympc_b200_solve on tensors from make_device_batch -> (numpy results, stats)"""
    import torch

    batch, out = solver.make_device_batch(x0, Xref, Uref, state=state, cold_start=cold, want_state=tuple(want), want_u0=True,
                                          models=models, bounds=bounds)
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


def _host(solver, x0, Xref, Uref, state, cold, want=WANT, bounds=None, pin=False):
    """tinympc_b200_solve_host on a HostBatch (u0 requested too); pin: every caller buffer page-locked"""
    p = solver.problem
    state = None if state is None else {n: np.array(a, copy=True) for n, a in state.items()}
    hb = HostBatch(p, x0, Xref, Uref, state=state, cold_start=cold, want_state=tuple(want), bounds=bounds)
    hb.u0 = np.empty((hb.B, p.nu), p.dtype)
    keep = []
    if pin:
        for n in ("x0", "Xref", "Uref", "sol_x", "sol_u", "iter", "solved", "residuals", "u0"):
            if getattr(hb, n) is not None:
                setattr(hb, n, _pinned(getattr(hb, n), keep))
        hb.state = {n: _pinned(a, keep) for n, a in hb.state.items()}
        hb.bounds = {n: _pinned(a, keep) for n, a in hb.bounds.items()}
    for k in OUTS:
        H.poison(getattr(hb, k))
    if cold:
        for n in want:
            H.poison(hb.state[n])
    cb = hb.to_c()
    cb.u0 = hb.u0.ctypes.data
    solver.solve_prepared(hb, cb)
    return {k: np.array(v, copy=True) for k, v in dict(hb.result(), u0=hb.u0).items() if v is not None}, solver.stats()


def _warm_inputs(x0, res, seed):
    """the next MPC step: perturbed measurements, the returned state, duals reset on every third instance"""
    rng = np.random.default_rng(seed)
    x0b = (x0 + 0.02 * rng.standard_normal(x0.shape)).astype(x0.dtype)
    state = {n: np.array(res[n], copy=True) for n in WANT}
    for n in ("g", "y"):
        state[n][::3] = 0
    return x0b, state


def _capacity(solver, bounds_fn, models=None):
    """instances one wave of the solver's persistent kernel holds with per-instance bounds (ctas x instances_per_cta), from a
    one-iteration probe solve that fills every SM"""
    import torch

    p = solver.problem
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    B = 64 * sm
    mi = solver.settings.max_iter
    solver.update_settings(max_iter=1)
    m = None if models is None else models[np.zeros(B, int)]
    batch, _ = solver.make_device_batch(np.zeros((B, p.nx), p.dtype), np.zeros((p.N, p.nx), p.dtype), cold_start=True,
                                        models=m, bounds=bounds_fn(B))
    solver.solve_device(batch)
    torch.cuda.synchronize()
    solver.update_settings(max_iter=mi)
    stt = solver.stats()
    assert stt["ctas"] == sm, stt
    return stt["ctas"] * stt["instances_per_cta"]


def _cold_warm(solver, inst, pal, which, family, what, models=None, model_of=None, mult=None):
    """cold solve, then a warm step from the returned state with the duals reset on every third instance; every instance vs
    the grouped oracle; the plan is `family`, with `mult` waves in one launch when given"""
    port = BC.grouped_oracle(solver.problem, solver.settings, pal, which, models=models, model_of=model_of, nthreads=NT)
    bounds = BC.batch_bounds(pal, which)
    m = None if models is None else models[model_of]
    x0, Xref, Uref = inst["x0"], inst["Xref"], inst.get("Uref")
    B = len(x0)
    o1 = port(x0, Xref, Uref, None, True, WANT)
    g1, stt = _device(solver, x0, Xref, Uref, None, True, models=m, bounds=bounds)
    assert stt["kernel_family"] == family and stt["kernel_launches"] == 1, stt
    if mult:
        assert B >= mult * stt["ctas"] * stt["instances_per_cta"], (B, stt)
    _check(g1, o1, WANT, what + " cold")
    x0b, state = _warm_inputs(x0, o1, seed=B)
    o2 = port(x0b, Xref, Uref, state, False, WANT)
    g2, stt = _device(solver, x0b, Xref, Uref, state, False, models=m, bounds=bounds)
    assert stt["kernel_family"] == family, stt
    _check(g2, o2, WANT, what + " warm")
    return o1, o2


def _one_per_group(stt):
    """the streamed kernel ran a one-instance-per-lane-group variant"""
    assert stt["kernel_family"] == abi.KERNEL_GPS, stt
    assert stt["instances_per_cta"] == stt["threads_per_cta"] // stt["lanes_per_instance"], stt


def _quad_fleet(dt, nm=4):
    """nm quadrotors of different masses (input matrix scaled) and tunings: per-instance models"""
    spec = wl.quadrotor(N=50)
    k = np.arange(nm)
    t = lambda a: np.tile(np.asarray(a, np.float64)[None], (nm,) + (1,) * np.ndim(a))  # noqa: E731
    Bm = t(spec.B) / (1.0 + 0.15 * (k - 1.5))[:, None, None]
    return setup_models(spec.nx, spec.nu, t(spec.A), Bm, t(spec.f), t(spec.Qdiag) * (1.0 + 0.2 * k)[:, None], t(spec.Rdiag),
                        spec.rho * (0.8 + 0.2 * k), dtype=dt)


# ---------------------------------------------------------------------------------------------------------------------
# 1. bounds equal to the handle's
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("kernel", [abi.KERNEL_GPI, abi.KERNEL_GPS])
@pytest.mark.parametrize("layout", [1, 2])
def test_equal_bounds_equal_shared_solve(layout, kernel, dt):
    prob, st = _quad(50, dt)
    s = BatchedTinySolver(prob, st, kernel=kernel)
    inst = _tracking(300, 50, dt, seed=1)
    pal = BC.equal_palette(prob, layout)
    bounds = BC.batch_bounds(pal, np.zeros(300, int))
    x0, state = inst["x0"], None
    for cold in (True, False):
        shared, s0 = _device(s, x0, inst["Xref"], inst["Uref"], state, cold)
        got, s1 = _device(s, x0, inst["Xref"], inst["Uref"], state, cold, bounds=bounds)
        assert s0["kernel_family"] == s1["kernel_family"] == kernel, (s0, s1)
        H.assert_bits_per_instance(got, shared, list(shared), f"layout {layout} cold={cold}")
        o = BC.grouped_oracle(prob, st, pal, np.zeros(300, int), nthreads=NT)(x0, inst["Xref"], inst["Uref"], state, cold, WANT)
        _check(got, o, WANT, f"layout {layout} cold={cold} vs oracle")
        x0, state = _warm_inputs(inst["x0"], shared, seed=2)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. a fleet of limits on chip, > 2.5 waves
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("layout", [1, 2])
@pytest.mark.parametrize("with_models", [False, True])
def test_fleet_on_chip_multiwave(with_models, layout, dt):
    prob, st = _quad(50, dt)
    s = BatchedTinySolver(prob, st)
    K = 5
    pal = BC.palette(prob, K, layout, seed=10 + layout, scale=1.0, tight=0.7)
    models = _quad_fleet(dt) if with_models else None
    cap = _capacity(s, lambda B: BC.batch_bounds(pal, BC.deal(B, K)), models)
    B = int(2.6 * cap) + 37
    which = BC.deal(B, K)
    model_of = None if models is None else (np.arange(B) * 3) % len(models)
    inst = _tracking(B, 50, dt, seed=20 + layout)
    o1, o2 = _cold_warm(s, inst, pal, which, abi.KERNEL_GPI, f"fleet layout {layout}", models=models, model_of=model_of, mult=2.5)
    H.assert_mixed_termination(o1)
    if layout == 2:  # the horizons really vary over k and between sets
        assert not np.array_equal(pal[0]["u_max"][0], pal[0]["u_max"][5]) and not np.array_equal(pal[0]["u_max"], pal[1]["u_max"])
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. every compiled (nx, nu) with an on-chip plan at N = 50
# ---------------------------------------------------------------------------------------------------------------------
DIMS = [(4, 1), (6, 3), (12, 4), (4, 2), (4, 4), (4, 8), (8, 2), (8, 4), (8, 8), (12, 2), (12, 8), (16, 2), (16, 4), (16, 8)]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("nx,nu", DIMS)
def test_every_shape_on_chip(nx, nu, dt):
    spec = wl.random_lti(nx, nu, 50, seed=100 + nx * 10 + nu)
    prob = setup_problem(spec, dt)
    st = _settings(spec, max_iter=30)
    s = BatchedTinySolver(prob, st, kernel=abi.KERNEL_GPI)
    pal = BC.palette(prob, 3, 1 + (nx + nu) % 2, seed=nx + nu, scale=0.3, tight=0.5)
    which = BC.deal(160, 3, stride=2)
    rng = np.random.default_rng(nx * nu)
    inst = dict(x0=(0.5 * rng.standard_normal((160, nx))).astype(dt), Xref=(0.1 * rng.standard_normal((160, 50, nx))).astype(dt))
    _, stt = _device(s, inst["x0"], inst["Xref"], None, None, True, bounds=BC.batch_bounds(pal, which))
    if stt["kernel_family"] != abi.KERNEL_GPI:
        pytest.skip(f"({nx},{nu}) has no on-chip plan at N = 50 in this precision")
    _cold_warm(s, inst, pal, which, abi.KERNEL_GPI, f"({nx},{nu})")
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. the streamed kernel
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("N", [20, 100])
@pytest.mark.parametrize("layout", [1, 2])
def test_rocket_fleet_cones(layout, N, dt):
    prob, st = _rocket(dt, N)
    s = BatchedTinySolver(prob, st)
    pal = _thrust_palette(prob, 6, layout, seed=N + layout)
    which = BC.deal(700, 6)
    o1, _ = _cold_warm(s, _rocket_instances(700, N, dt, seed=N), pal, which, abi.KERNEL_GPS, f"rocket N={N} layout {layout}")
    _one_per_group(s.stats())
    s.close()


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("tv", [False, True])
def test_hyperplanes(tv, dt):
    spec = H.quad_linear_spec(tv=tv)
    spec.settings.en_state_bound = 1
    spec.settings.en_input_bound = 1
    prob = setup_problem(spec, dt)
    st = _settings(spec, max_iter=40, abs_pri_tol=1e-2, abs_dua_tol=1e-2)
    s = BatchedTinySolver(prob, st)
    pal = BC.palette(prob, 4, 2 if tv else 1, seed=7, scale=0.2, tight=0.6)
    rng = np.random.default_rng(3)
    B, N = 500, spec.N
    inst = dict(x0=(0.3 * rng.standard_normal((B, 12))).astype(dt), Xref=(0.05 * rng.standard_normal((B, N, 12))).astype(dt),
                Uref=(0.02 * rng.standard_normal((B, N - 1, 4))).astype(dt))
    _cold_warm(s, inst, pal, BC.deal(B, 4, stride=3), abi.KERNEL_GPS, f"hyperplanes tv={tv}")
    _one_per_group(s.stats())
    s.close()


@pytest.mark.parametrize("layout", [1, 2])
def test_box_horizon_off_chip(layout):
    """Quadrotor fp64, N = 1000: no on-chip plan, so the batch streams"""
    dt = np.float64
    prob, st = _quad(1000, dt, max_iter=30)
    s = BatchedTinySolver(prob, st)
    pal = BC.palette(prob, 3, layout, seed=5, scale=0.5, tight=0.5)
    inst = wl.hovering_instances(64, N=1000, dtype=dt)
    inst["x0"] = (inst["x0"] + 0.2 * np.random.default_rng(3).standard_normal(inst["x0"].shape)).astype(dt)
    _cold_warm(s, inst, pal, BC.deal(64, 3, stride=2), abi.KERNEL_GPS, "N=1000")
    s.close()


@pytest.mark.parametrize("dt", DTS)
def test_explicit_gps_box_with_models(dt):
    prob, st = _quad(50, dt)
    s = BatchedTinySolver(prob, st, kernel=abi.KERNEL_GPS)
    pal = BC.palette(prob, 5, 2, seed=8, scale=0.8, tight=0.6)
    inst = _tracking(600, 50, dt, seed=9)
    which = BC.deal(600, 5)
    _cold_warm(s, inst, pal, which, abi.KERNEL_GPS, "explicit GPS")
    _one_per_group(s.stats())
    models = _quad_fleet(dt)
    _cold_warm(s, inst, pal, which, abi.KERNEL_GPS, "explicit GPS + models", models=models, model_of=np.arange(600) % 4)
    s.close()


@pytest.mark.parametrize("dt", DTS)
def test_streamed_multiwave_one_warp(dt, monkeypatch):
    """TINYMPC_GPS_WARPS=1: one warp per SM, > 2.5 waves plus a ragged remainder in one launch"""
    monkeypatch.setenv("TINYMPC_GPS_WARPS", "1")
    prob, st = _rocket(dt, 20)
    s = BatchedTinySolver(prob, st)
    pal = _thrust_palette(prob, 5, 1, seed=12)
    cap = _capacity(s, lambda B: BC.batch_bounds(pal, BC.deal(B, 5)))
    B = int(2.6 * cap) + 5
    o1, _ = _cold_warm(s, _rocket_instances(B, 20, dt, seed=13), pal, BC.deal(B, 5), abi.KERNEL_GPS, "GPS 1 warp", mult=2.5)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. signed zeros: the shared fp32 solve of this problem clamps with min / max; per-instance bounds at +-0 must not
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", [1, 2])
def test_signed_zero_bounds(layout):
    dt = np.float32
    prob, st = _quad(50, dt)
    s = BatchedTinySolver(prob, st)
    pal = BC.palette(prob, 3, layout, seed=6, scale=0.3, zeros=True)
    assert any(np.signbit(d["u_min"]).any() and (d["u_min"] == 0).any() for d in pal)
    o1, _ = _cold_warm(s, _tracking(400, 50, dt, seed=6), pal, BC.deal(400, 3, stride=2), abi.KERNEL_GPI, "+-0 bounds")
    assert (o1["znew"] == 0).any() and np.signbit(o1["znew"][o1["znew"] == 0]).any()  # slacks land on -0
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. the host path in 11 chunks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pin", [False, True])
@pytest.mark.parametrize("layout", [1, 2])
def test_host_path_chunks(layout, pin, monkeypatch):
    dt = np.float32
    prob, st = _quad(50, dt)
    s = BatchedTinySolver(prob, st)
    B = 11 * 96 - 40
    monkeypatch.setenv("TINYMPC_HOST_CHUNK", "96")
    pal = BC.palette(prob, 7, layout, seed=30, scale=0.7, tight=0.6)
    which = BC.deal(B, 7, stride=3)
    bounds = BC.batch_bounds(pal, which)
    port = BC.grouped_oracle(prob, st, pal, which, nthreads=NT)
    inst = _tracking(B, 50, dt, seed=31)
    o1 = port(inst["x0"], inst["Xref"], inst["Uref"], None, True, WANT)
    g1, stt = _host(s, inst["x0"], inst["Xref"], inst["Uref"], None, True, bounds=bounds, pin=pin)
    assert stt["kernel_launches"] == 11, stt
    _check(g1, o1, WANT, "host cold")
    x0b, state = _warm_inputs(inst["x0"], o1, seed=32)
    o2 = port(x0b, inst["Xref"], inst["Uref"], state, False, WANT)
    g2, stt = _host(s, x0b, inst["Xref"], inst["Uref"], state, False, bounds=bounds, pin=pin)
    _check(g2, o2, WANT, "host warm")
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. the device closed loop
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


@pytest.mark.parametrize("with_models", [False, True])
def test_closed_loop(with_models):
    from tinympc_b200.closed_loop import DeviceMPCLoop

    dt = np.float32
    prob, st = _quad(50, dt)
    s = BatchedTinySolver(prob, st)
    B = 300
    pal = BC.palette(prob, 4, 1, seed=40, scale=0.6, tight=0.5)
    pal2 = BC.palette(prob, 4, 2, seed=41, scale=0.4, tight=0.5)  # one step in a moving corridor
    which = BC.deal(B, 4, stride=3)
    models = _quad_fleet(dt) if with_models else None
    model_of = None if models is None else np.arange(B) % 4
    inst = _tracking(B, 50, dt, seed=42)
    loop = DeviceMPCLoop(s, inst["x0"], reset_duals=True, bounds=BC.batch_bounds(pal, which),
                         models=None if models is None else models[model_of])
    x0 = inst["x0"].copy()
    state = None
    for k in range(5):
        Xref = np.ascontiguousarray(np.roll(inst["Xref"], -k, axis=1))
        p_ = pal2 if k == 2 else pal
        out = loop.step(Xref, bounds=BC.batch_bounds(pal2, which) if k == 2 else None)
        if state is not None:
            state["g"] = np.zeros_like(state["g"])
            state["y"] = np.zeros_like(state["y"])
        o = BC.grouped_oracle(prob, st, p_, which, models=models, model_of=model_of, nthreads=NT)(x0, Xref, None, state,
                                                                                                 state is None, WANT)
        got = {key: out[key].cpu().numpy() for key in H.OUT_KEYS + list(loop.fields) + ["u0"]}
        _check(got, o, loop.fields, f"closed loop step {k}")
        state = {n: o[n] for n in WANT}
        u0 = o["u"][:, 0, :]
        if models is None:
            x0 = _advance(prob, x0, u0)
        else:
            nxt = np.empty_like(x0)
            for m in range(len(models)):
                idx = np.flatnonzero(model_of == m)
                nxt[idx] = _advance(BC.with_model(prob, models[m]), x0[idx], u0[idx])
            x0 = nxt
        assert H.bits_equal(loop.x0.cpu().numpy(), x0), ("advance", k)
    with pytest.raises(ValueError):
        loop.rollout(inst["Xref"], 3)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 8. queued solves with different bound arrays
# ---------------------------------------------------------------------------------------------------------------------
def test_queued_solves_different_bounds():
    import torch

    dt = np.float32
    prob, st = _quad(50, dt)
    s = BatchedTinySolver(prob, st)
    B = 3000
    inst = _tracking(B, 50, dt, seed=50)
    pals = [BC.palette(prob, 5, 1, seed=51, scale=0.7, tight=0.6), BC.palette(prob, 5, 2, seed=52, scale=0.5, tight=0.6)]
    which = BC.deal(B, 5)
    dev = torch.device("cuda", 0)
    bnd = [{k: torch.as_tensor(v, device=dev) for k, v in BC.batch_bounds(p, which).items()} for p in pals]

    def run(sync):
        res = []
        for b in bnd:
            batch, out = s.make_device_batch(inst["x0"], inst["Xref"], inst["Uref"], cold_start=True, want_state=WANT, want_u0=True,
                                             bounds=b)
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
        o = BC.grouped_oracle(prob, st, p, which, nthreads=NT)(inst["x0"], inst["Xref"], inst["Uref"], None, True, WANT)
        _check(q, o, WANT, "queued vs oracle")
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 9. loud errors
# ---------------------------------------------------------------------------------------------------------------------
def test_errors():
    import ctypes as C

    import torch

    dt = np.float32
    prob, st = _quad(50, dt)
    s = BatchedTinySolver(prob, st)
    B = 64
    inst = _tracking(B, 50, dt, seed=60)
    pal = BC.palette(prob, 2, 1, seed=61, scale=0.5)
    bounds = BC.batch_bounds(pal, BC.deal(B, 2, stride=1))
    batch, _ = s.make_device_batch(inst["x0"], inst["Xref"], cold_start=True, bounds=bounds)

    def rc(b=batch):
        r = s._lib.tinympc_b200_solve(s._h, C.byref(b), None)
        torch.cuda.synchronize()
        return r

    assert rc() == abi.OK
    # FAST mode, explicit thread per instance
    s.set_mode(abi.MODE_FAST)
    assert rc() == abi.ERR_UNSUPPORTED and b"STRICT" in s._lib.tinympc_b200_last_error()
    s.set_mode(abi.MODE_STRICT, abi.KERNEL_TPI)
    assert rc() == abi.ERR_UNSUPPORTED and b"thread per instance" in s._lib.tinympc_b200_last_error()
    s.set_mode(abi.MODE_STRICT, abi.KERNEL_AUTO)
    # adaptive rho and rollouts
    models = torch.as_tensor(pack_models(prob, B), device="cuda")
    dK, dP = np.zeros((prob.nu, prob.nx), dt), np.zeros((prob.nx, prob.nx), dt)
    ar = AdaptiveRho(dK, dP).to_c(prob, models.data_ptr(), B, models.device)
    assert s._lib.tinympc_b200_solve_adaptive(s._h, C.byref(batch), C.byref(ar), None) == abi.ERR_UNSUPPORTED
    assert b"adaptive" in s._lib.tinympc_b200_last_error()
    rb = abi.Batch.from_buffer_copy(batch)
    rb.Xref = rb.Uref = rb.iter = rb.solved = rb.residuals = rb.u0 = None
    rb.sol_x = rb.sol_u = None
    r = abi.Rollout()
    X = torch.as_tensor(np.ascontiguousarray(inst["Xref"][0]), device="cuda")
    r.T, r.Xref = 1, X.data_ptr()
    assert s._lib.tinympc_b200_rollout(s._h, C.byref(rb), C.byref(r), None) == abi.ERR_UNSUPPORTED
    assert b"rollout" in s._lib.tinympc_b200_last_error()
    # bad mode, half pair, reserved2
    for field, val in (("bounds_per_instance", 3), ("bounds_per_instance", -1), ("reserved2", 1), ("x_max", None), ("u_min", None)):
        b = abi.Batch.from_buffer_copy(batch)
        setattr(b, field, val)
        assert rc(b) == abi.ERR_ARG, field
    # an enabled side without its pair; a disabled side's pair is never needed
    b = abi.Batch.from_buffer_copy(batch)
    b.x_min = b.x_max = None
    assert rc(b) == abi.ERR_NO_BOUNDS
    s.update_settings(en_state_bound=0)
    assert rc(b) == abi.OK
    s.update_settings(en_state_bound=1)
    # Python checks: shapes, dtype, pairs, mixed layouts
    bad = [dict(bounds, x_min=bounds["x_min"][:, :5]), dict(bounds, x_min=bounds["x_min"].astype(np.float64)),
           {"x_min": bounds["x_min"]}, dict(bounds, u_min=np.stack([pal[0]["u_min"]] * B)[:, None, :].repeat(49, 1)),
           dict(bounds, q=bounds["x_min"]), {}]
    for bb in bad:
        with pytest.raises(ValueError):
            s.make_device_batch(inst["x0"], inst["Xref"], cold_start=True, bounds=bb)
        with pytest.raises(ValueError):
            s.solve(inst["x0"], inst["Xref"], bounds=bb)
    s.close()
    # a handle created without bounds, solved with per-instance bounds
    kw = {k: getattr(prob, k) for k in prob.__dataclass_fields__}
    kw.update(x_min=None, x_max=None, u_min=None, u_max=None)
    bare = BatchedTinySolver(type(prob)(**kw), st)
    with pytest.raises(TinyMPCError) as e:
        bare.solve(inst["x0"], inst["Xref"])
    assert e.value.code == abi.ERR_NO_BOUNDS
    got = bare.solve(inst["x0"], inst["Xref"], bounds=bounds)
    o = BC.grouped_oracle(prob, st, pal, BC.deal(B, 2, stride=1), nthreads=NT)(inst["x0"], inst["Xref"], None, None, True, ())
    H.assert_bits_per_instance(got, o, H.OUT_KEYS, "handle without bounds")
    bare.close()
