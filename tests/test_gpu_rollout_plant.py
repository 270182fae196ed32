"""Closed loops against plants of their own (tinympc_rollout_t.plant / noise, DeviceMPCLoop(plant=...), step(noise=...),
tinympc_b200_advance_plant): every robot's real dynamics differ from the controller's model and it sees its state through a noisy
sensor.  The rollout's GPI_PLANT variant is held bit for bit to DeviceMPCLoop stepping the same loop, and both to a host loop of
the CPU oracle with a numpy plant step.  Every output buffer of a rollout is filled with a NaN bit pattern first."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest

import adaptive_common as AC
import helpers as H
from oracle import oracle
from tinympc_b200 import abi, workloads as wl
from tinympc_b200._lib import TinyMPCError, check
from tinympc_b200.closed_loop import DeviceMPCLoop, pack_plant
from tinympc_b200.solver import AdaptiveRho, BatchedTinySolver, setup_models, setup_problem

pytestmark = pytest.mark.gpu

NT = os.cpu_count() or 1
FIELDS = ("v", "z", "vnew", "znew", "g", "y")
PER_STEP = ("x", "u", "iter", "solved", "residuals")
PLAN = ("kernel_family", "lanes_per_instance", "instances_per_cta", "smem_bytes_per_cta", "ctas", "threads_per_cta")
DIMS = [(4, 1), (6, 3), (12, 4), (4, 2), (4, 4), (4, 8), (8, 2), (8, 4), (8, 8), (12, 2), (12, 8), (16, 2), (16, 4), (16, 8)]


def _torch():
    import torch

    return torch


def _settings(spec, **kw):
    st = abi.Settings.from_buffer_copy(spec.settings)
    for k, v in kw.items():
        setattr(st, k, v)
    return st


def _quad(dt, N=50, **kw):
    spec = wl.quadrotor(N=N)
    return spec, setup_problem(spec, dt), _settings(spec, **dict(dict(max_iter=15), **kw))


def _episode(B, N, T, dt, seed):
    """Per-robot sliding tracking references of T+N-1 knots, an input reference, jittered start states."""
    inst = wl.tracking_instances(B, N=T + N - 1, seed=seed, dtype=dt, jitter=0.5)
    U = (0.05 * np.random.default_rng(seed + 1).standard_normal((B, T + N - 2, 4))).astype(dt)
    return np.ascontiguousarray(inst["x0"]), inst["Xref"], U


def _noise(B, T, nx, dt, seed, scale=0.01):
    return (scale * np.random.default_rng(seed).standard_normal((B, T, nx))).astype(dt)


def _plant(spec, B, dt, seed=0, drift=0.02, shared=False):
    """plant_fleet rounded to dt (the records the device reads); shared: robot 0's plant for the whole batch"""
    pl = wl.plant_fleet(spec, B, seed=seed, drift=drift)
    pl = {k: pl[k].astype(dt) for k in ("A", "B", "f")}
    return {k: np.ascontiguousarray(v[0]) for k, v in pl.items()} if shared else pl


def _capacity(solver):
    """Instances one wave of the on-chip kernel holds."""
    torch = _torch()
    p = solver.problem
    B = 64 * torch.cuda.get_device_properties(0).multi_processor_count
    st1 = abi.Settings.from_buffer_copy(solver.settings)
    st1.max_iter = 1
    s = BatchedTinySolver(p, st1, kernel=abi.KERNEL_GPI)
    batch, _ = s.make_device_batch(np.zeros((B, p.nx), p.dtype), np.zeros((p.N, p.nx), p.dtype), cold_start=True)
    s.solve_device(batch)
    torch.cuda.synchronize()
    stt = s.stats()
    s.close()
    return stt["ctas"] * stt["instances_per_cta"]


def _advance_ref(plant, x0, u0):
    """x <- (A_p x + B_p u0) + f_p per robot with ascending sums from the first product, no FMA (advance_kernel's arithmetic)"""
    A, Bm, f = plant["A"], plant["B"], plant["f"]
    if A.ndim == 2:
        A, Bm, f = A[None], Bm[None], f[None]
    nx, nu = A.shape[1], Bm.shape[2]
    nxt = np.zeros_like(x0)
    for i in range(nx):
        ax = A[:, i, 0] * x0[:, 0]
        for m in range(1, nx):
            ax = ax + A[:, i, m] * x0[:, m]
        bu = Bm[:, i, 0] * u0[:, 0]
        for j in range(1, nu):
            bu = bu + Bm[:, i, j] * u0[:, j]
        nxt[:, i] = (ax + bu) + f[:, i]
    return nxt


# ---------------------------------------------------------------------------------------------------------------------
# the three ways of running an episode
# ---------------------------------------------------------------------------------------------------------------------
def _loop(solver, x0, X, U, T, plant=None, noise=None, w=None, models=None, loop=None, t0=0):
    """DeviceMPCLoop.step(noise=n[:, t]) T times with the sliding window, then x0 += w[:, t] -> per-step outputs and the loop"""
    torch = _torch()
    N = solver.problem.N
    if loop is None:
        loop = DeviceMPCLoop(solver, x0, reset_duals=True, models=models, plant=plant)
    per = {k: [] for k in PER_STEP}
    for t in range(t0, t0 + T):
        per["x"].append(loop.x0.clone())
        out = loop.step(X[..., t:t + N, :], None if U is None else U[..., t:t + N - 1, :],
                        noise=None if noise is None else noise[:, t])
        for k, o in (("u", "u0"), ("iter", "iter"), ("solved", "solved"), ("residuals", "residuals")):
            per[k].append(out[o].clone())
        if w is not None:
            loop.x0 += torch.as_tensor(w[:, t], device=loop.x0.device)
    per["x"].append(loop.x0.clone())
    torch.cuda.synchronize()
    return {k: torch.stack(v, 1).cpu().numpy() for k, v in per.items()}, loop


def _final(loop):
    _torch().cuda.synchronize()
    d = {n: loop.state[n].cpu().numpy() for n in loop.fields}
    d.update(x0=loop.x0.cpu().numpy(), sol_x=loop.out["sol_x"].cpu().numpy(), sol_u=loop.out["sol_u"].cpu().numpy())
    return d


def _rollout_c(solver, x0, X, U, T, plant=None, noise=None, w=None, models=None, ro_extra=None):
    """tinympc_b200_rollout (duals reset, v / z carried) on poisoned device buffers -> (rc, per-step outputs, final state, stats)"""
    torch = _torch()
    p = solver.problem
    dev = torch.device("cuda", solver.device)
    tdt = torch.float32 if p.dtype == np.float32 else torch.float64
    t = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a, dtype=p.dtype), device=dev)  # noqa: E731
    B = len(x0)
    x0_t, X_t, U_t, w_t, n_t, M = t(x0), t(X), t(U), t(w), t(noise), t(models)
    rec, per = (None, False) if plant is None else pack_plant(plant, p.nx, p.nu, B, tdt, dev)
    st = {n: H.poison(torch.empty((B, p.N, p.nx) if abi.STATE_IS_X[n] else (B, p.N - 1, p.nu), dtype=tdt, device=dev))
          for n in FIELDS}
    out = dict(x=torch.empty((B, T + 1, p.nx), dtype=tdt, device=dev), u=torch.empty((B, T, p.nu), dtype=tdt, device=dev),
               iter=torch.empty((B, T), dtype=torch.int32, device=dev), solved=torch.empty((B, T), dtype=torch.int32, device=dev),
               residuals=torch.empty((B, T, 4), dtype=tdt, device=dev), sol_x=torch.empty((B, p.N, p.nx), dtype=tdt, device=dev),
               sol_u=torch.empty((B, p.N - 1, p.nu), dtype=tdt, device=dev))
    for v in out.values():
        H.poison(v)
    x0_before = x0_t.clone()
    b = abi.Batch()
    b.B, b.x0, b.cold_start = B, x0_t.data_ptr(), 1
    for n, a in st.items():
        setattr(b.state, n, a.data_ptr())
    b.sol_x, b.sol_u = out["sol_x"].data_ptr(), out["sol_u"].data_ptr()
    b.models = None if M is None else M.data_ptr()
    r = abi.Rollout()
    r.T, r.reset_duals, r.carry_v = T, 1, 1
    r.Xref, r.xref_per_instance = X_t.data_ptr(), int(X_t.dim() == 3)
    r.Uref, r.uref_per_instance = (None, 0) if U_t is None else (U_t.data_ptr(), int(U_t.dim() == 3))
    r.w = None if w_t is None else w_t.data_ptr()
    r.x_traj, r.u_traj, r.residuals_traj = out["x"].data_ptr(), out["u"].data_ptr(), out["residuals"].data_ptr()
    r.iter_traj, r.solved_traj = out["iter"].data_ptr(), out["solved"].data_ptr()
    r.plant, r.plant_per_instance = (None, 0) if rec is None else (rec.data_ptr(), int(per))
    r.noise = None if n_t is None else n_t.data_ptr()
    for k, v in (ro_extra or {}).items():
        setattr(r, k, v)
    rc = solver._lib.tinympc_b200_rollout(solver._h, C.byref(b), C.byref(r), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize()
    assert torch.equal(x0_before.view(torch.uint8), x0_t.view(torch.uint8)), "io->x0 must not be modified"
    return rc, {k: v.cpu().numpy() for k, v in out.items()}, {n: a.cpu().numpy() for n, a in st.items()}, solver.stats()


def _oracle_episode(prob, st, x0, X, U, T, plant, noise=None, w=None, state_fields=FIELDS):
    """The loop on the host: the oracle solves each window from x + n warm-started with the duals reset, the plant advances
    the true state with numpy's ascending sums."""
    N, dt = prob.N, prob.dtype
    state = None
    per = {k: [] for k in PER_STEP}
    for t in range(T):
        per["x"].append(x0.copy())
        if state is not None:
            state["g"] = np.zeros_like(state["g"])
            state["y"] = np.zeros_like(state["y"])
        xm = x0 if noise is None else x0 + noise[:, t]
        Xw = np.ascontiguousarray(X[..., t:t + N, :])
        Uw = None if U is None else np.ascontiguousarray(U[..., t:t + N - 1, :])
        o = oracle.solve_batch(prob, st, xm, Xw, Uw, state=state, cold_start=state is None,
                               want_state=tuple(dict.fromkeys(state_fields + ("u",))), impl="port", nthreads=NT)
        state = {n: np.array(o[n], copy=True) for n in state_fields}
        u0 = np.ascontiguousarray(o["u"][:, 0, :])
        per["u"].append(u0)
        for k in ("iter", "solved", "residuals"):
            per[k].append(o[k])
        x0 = _advance_ref(plant, x0, u0)
        if w is not None:
            x0 = (x0 + w[:, t]).astype(dt)
    per["x"].append(x0.copy())
    return {k: np.stack(v, 1) for k, v in per.items()}, state, o


def _compare(got, ref, fin_got, loop, what):
    H.assert_bits_per_instance(got, ref, PER_STEP, what)
    H.assert_bits_per_instance(dict(fin_got, x0=got["x"][:, -1], sol_x=got["sol_x"], sol_u=got["sol_u"]), _final(loop),
                               list(FIELDS) + ["x0", "sol_x", "sol_u"], what + " final")


def _sample(d, idx):
    return {k: v[idx] for k, v in d.items()}


# ---------------------------------------------------------------------------------------------------------------------
# 1. a per-robot plant fleet with noise and disturbance
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_plant_fleet_noise_matches_loop_and_oracle(dt):
    """(12,4,50) tracking, about 2.6 waves of the on-chip plan, T = 5: plant_fleet with drift, noise and w; the rollout equals
    DeviceMPCLoop.step x5 and, for a sample of robots, the oracle's host loop."""
    spec, prob, st = _quad(dt)
    solver = BatchedTinySolver(prob, st)
    B = int(2.6 * _capacity(solver)) + 11
    T = 5
    x0, X, U = _episode(B, prob.N, T, dt, seed=71)
    plant = _plant(spec, B, dt, seed=1)
    noise = _noise(B, T, 12, dt, seed=2)
    w = _noise(B, T, 12, dt, seed=3, scale=0.005)
    rc, got, fin, stt = _rollout_c(solver, x0, X, U, T, plant=plant, noise=noise, w=w)
    check(rc)
    assert stt["kernel_family"] == abi.KERNEL_GPI and stt["kernel_launches"] == 1, stt
    assert B >= 2.5 * stt["ctas"] * stt["instances_per_cta"], (B, stt)
    ref, loop = _loop(solver, x0, X, U, T, plant=plant, noise=noise, w=w)
    H.assert_mixed_termination(dict(iter=ref["iter"].ravel(), solved=ref["solved"].ravel()))
    _compare(got, ref, fin, loop, f"plant fleet {dt.__name__}")
    idx = np.r_[0:24, B - 24:B]
    oref, state, last = _oracle_episode(prob, st, x0[idx], X[idx], U[idx], T, _sample(plant, idx), noise[idx], w[idx])
    H.assert_bits_per_instance(_sample(got, idx), oref, PER_STEP, f"plant fleet oracle {dt.__name__}")
    H.assert_bits_per_instance(dict(_sample(fin, idx), sol_x=got["sol_x"][idx], sol_u=got["sol_u"][idx]),
                               dict(state, sol_x=last["sol_x"], sol_u=last["sol_u"]), list(FIELDS) + ["sol_x", "sol_u"],
                               f"plant fleet oracle {dt.__name__} final")


# ---------------------------------------------------------------------------------------------------------------------
# 2. a shared plant, a plant without noise, noise without a plant, a controller fleet with plants
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["shared_plant", "plant_no_noise", "noise_no_plant", "models_and_plants"])
def test_rollout_plant_variants(case):
    dt = np.float32
    spec, prob, st = _quad(dt)
    solver = BatchedTinySolver(prob, st)
    B, T = 700, 4
    x0, X, U = _episode(B, prob.N, T, dt, seed=81)
    plant = None if case == "noise_no_plant" else _plant(spec, B, dt, seed=4, shared=case == "shared_plant")
    noise = None if case == "plant_no_noise" else _noise(B, T, 12, dt, seed=5)
    models = None
    if case == "models_and_plants":
        M = 6
        blobs = setup_models(12, 4, np.stack([spec.A] * M), np.stack([spec.B * (1.0 + 0.05 * i) for i in range(M)]),
                             np.stack([spec.f] * M), np.stack([spec.Qdiag * (1.0 + 0.2 * i) for i in range(M)]),
                             np.stack([spec.Rdiag] * M), np.array([spec.rho * (1.0 + 0.25 * i) for i in range(M)]), dtype=dt)
        models = blobs[(5 * np.arange(B)) % M]
    rc, got, fin, stt = _rollout_c(solver, x0, X, U, T, plant=plant, noise=noise, models=models)
    check(rc)
    assert stt["kernel_family"] == abi.KERNEL_GPI, stt
    ref, loop = _loop(solver, x0, X, U, T, plant=plant, noise=noise, models=models)
    _compare(got, ref, fin, loop, case)
    if case != "models_and_plants":  # the oracle solves with the handle's model
        idx = np.r_[0:16, B - 16:B]
        truth = {k: v[idx] for k, v in plant.items()} if plant is not None and case != "shared_plant" else plant
        if truth is None:
            truth = dict(A=np.asarray(prob.A, dt), B=np.asarray(prob.B, dt), f=np.asarray(prob.f, dt))
        oref, _, _ = _oracle_episode(prob, st, x0[idx], X[idx], U[idx], T, truth, None if noise is None else noise[idx])
        H.assert_bits_per_instance(_sample(got, idx), oref, PER_STEP, case + " oracle")


# ---------------------------------------------------------------------------------------------------------------------
# 3. every compiled shape
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_rollout_plant_every_shape(dt):
    """Every compiled (nx, nu) at N = 50, T = 3 with per-robot plants and noise: the plain rollout's plan, equal to the loop;
    a shape without an on-chip plan is refused."""
    N, T, B = 50, 3, 300
    served = 0
    for nx, nu in DIMS:
        spec = wl.random_lti(nx, nu, N, seed=nx * 31 + nu)
        spec.settings.max_iter = 30
        prob = setup_problem(spec, dt)
        solver = BatchedTinySolver(prob, spec.settings, kernel=abi.KERNEL_GPI)
        rng = np.random.default_rng(nx + nu)
        x0 = (3.0 * rng.standard_normal((B, nx))).astype(dt)
        X = (0.3 * rng.standard_normal((B, T + N - 1, nx))).astype(dt)
        pl = wl.plant_fleet(spec, B, seed=nx, drift=0.01)
        pl["A"] = pl["A"] * (1.0 + 0.01 * rng.standard_normal(pl["A"].shape))
        plant = {k: pl[k].astype(dt) for k in ("A", "B", "f")}
        noise = _noise(B, T, nx, dt, seed=nu)
        rc0, _, _, plain = _rollout_c(solver, x0, X, None, T)
        rc, got, fin, stt = _rollout_c(solver, x0, X, None, T, plant=plant, noise=noise)
        if rc0 == abi.ERR_UNSUPPORTED:  # no on-chip plan for this horizon
            assert rc == abi.ERR_UNSUPPORTED and b"horizon" in solver._lib.tinympc_b200_last_error(), (nx, nu, rc)
            continue
        check(rc0)
        check(rc)
        served += 1
        assert {k: stt[k] for k in PLAN} == {k: plain[k] for k in PLAN}, (nx, nu, stt, plain)
        ref, loop = _loop(solver, x0, X, None, T, plant=plant, noise=noise)
        _compare(got, ref, fin, loop, f"shape ({nx},{nu}) {dt.__name__}")
    assert served >= 5, served


# ---------------------------------------------------------------------------------------------------------------------
# 4. edges
# ---------------------------------------------------------------------------------------------------------------------
def test_rollout_plant_t0_writes_nothing():
    spec, prob, st = _quad(np.float32)
    x0, X, U = _episode(50, prob.N, 0, np.float32, seed=2)
    solver = BatchedTinySolver(prob, st)
    rc, got, fin, _ = _rollout_c(solver, x0, X, U, 0, plant=_plant(spec, 50, np.float32), noise=_noise(50, 0, 12, np.float32, 1))
    check(rc)
    for k, v in list(got.items()) + list(fin.items()):
        assert H.bits_equal(v, H.poison(np.empty_like(v))), k


@pytest.mark.parametrize("case", ["T1", "max_iter0", "check3"])
def test_rollout_plant_edges(case):
    dt = np.float64
    kw = dict(T1=dict(), max_iter0=dict(max_iter=0), check3=dict(max_iter=20, check_termination=3))[case]
    spec, prob, st = _quad(dt, **kw)
    T, B = (1 if case == "T1" else 4), 300
    x0, X, U = _episode(B, prob.N, T, dt, seed=40)
    plant = _plant(spec, B, dt, seed=6)
    noise, w = _noise(B, T, 12, dt, seed=7), _noise(B, T, 12, dt, seed=8, scale=0.005)
    solver = BatchedTinySolver(prob, st)
    rc, got, fin, _ = _rollout_c(solver, x0, X, U, T, plant=plant, noise=noise, w=w)
    check(rc)
    ref, loop = _loop(solver, x0, X, U, T, plant=plant, noise=noise, w=w)
    _compare(got, ref, fin, loop, case)
    if case == "max_iter0":  # no iteration: u0 = 0, so x1 = A_p x0 + f_p (+ w)
        assert not got["u"].any() and not got["iter"].any()
        x1 = _advance_ref(plant, x0, np.zeros((B, 4), dt)) + w[:, 0]
        assert H.bits_equal(got["x"][:, 1], x1)


def test_rollout_plant_continues_loop_and_step_continues_rollout():
    """step, step, rollout(3), step with a plant fleet and noise, against step x6, through DeviceMPCLoop.rollout."""
    torch = _torch()
    dt = np.float32
    spec, prob, st = _quad(dt)
    B = 500
    x0, X, U = _episode(B, prob.N, 6, dt, seed=50)
    plant, noise = _plant(spec, B, dt, seed=9), _noise(B, 6, 12, dt, seed=10)
    solver = BatchedTinySolver(prob, st)
    ref, ref_loop = _loop(solver, x0, X, U, 6, plant=plant, noise=noise)
    a = DeviceMPCLoop(solver, x0, reset_duals=True, plant=plant)
    _, a = _loop(solver, None, X, U, 2, noise=noise, loop=a)
    res = a.rollout(torch.as_tensor(X[:, 2:], device="cuda"), 3, Uref_traj=U[:, 2:], noise=noise[:, 2:5])
    torch.cuda.synchronize()
    got = {k: res[k].cpu().numpy() for k in PER_STEP}
    H.assert_bits_per_instance(got, {k: v[:, 2:5] if k != "x" else v[:, 2:6] for k, v in ref.items()}, PER_STEP, "rollout after steps")
    _, a = _loop(solver, None, X, U, 1, noise=noise, loop=a, t0=5)
    H.assert_bits_per_instance(_final(a), _final(ref_loop), list(a.fields) + ["x0", "sol_x", "sol_u"], "step after rollout")


# ---------------------------------------------------------------------------------------------------------------------
# 5. the step path where rollouts do not go: cones, adaptive rho
# ---------------------------------------------------------------------------------------------------------------------
def test_step_rocket_cones_plant_fleet_vs_oracle():
    """A nominal rocket controller with cones (streamed kernel) driving rocket_fleet's rockets through a noisy sensor, every
    step against the oracle's host loop."""
    dt = np.float64
    spec = wl.rocket(N=20)
    st = _settings(spec, max_iter=40)
    prob = setup_problem(spec, dt)
    B, T = 120, 4
    fl = wl.rocket_fleet(B, N=20, seed=5)
    plant = {k: fl[k].astype(dt) for k in ("A", "B", "f")}
    inst = wl.rocket_instances(B, N=20 + T, seed=11, dtype=dt, spread=0.3, per_instance_refs=True)
    X, U = inst["Xref"], inst["Uref"]
    noise = _noise(B, T, 6, dt, seed=12, scale=0.02)
    solver = BatchedTinySolver(prob, st)
    cone_fields = ("x", "u", "vcnew", "zcnew", "gc", "yc")
    loop = DeviceMPCLoop(solver, inst["x0"], reset_duals=True, extra_state=cone_fields, plant=plant)
    got, _ = _loop(solver, None, X, U, T, noise=noise, loop=loop)
    assert solver.stats()["kernel_family"] == abi.KERNEL_GPS
    ref, state, last = _oracle_episode(prob, st, inst["x0"].copy(), X, U, T, plant, noise, state_fields=loop.fields)
    H.assert_bits_per_instance(got, ref, PER_STEP, "rocket cones plant fleet")
    H.assert_bits_per_instance(_final(loop), dict(state, x0=ref["x"][:, -1], sol_x=last["sol_x"], sol_u=last["sol_u"]),
                               list(loop.fields) + ["x0", "sol_x", "sol_u"], "rocket cones final")


def test_step_adaptive_rho_plant_fleet_vs_oracle():
    """DeviceMPCLoop(adaptive_rho=..., plant=...) with noise: the adaptive C oracle solves from the measurement, the plants step
    the true state."""
    dt = np.float64
    sp = wl.quadrotor(N=50)
    prob = H.problem_from_spec(sp, dt, oracle.port_setup)
    ar = AdaptiveRho(*AC.quad_tables(dt))
    B, T = 300, 4
    inst = wl.tracking_instances(B, N=50, seed=12, dtype=dt)
    plant = _plant(sp, B, dt, seed=13)
    noise = _noise(B, T, 12, dt, seed=14)
    s = BatchedTinySolver(prob, sp.settings, device=0)
    loop = DeviceMPCLoop(s, inst["x0"], adaptive_rho=ar, plant=plant)
    x0, state, models = inst["x0"].copy(), None, AC.pack_models(prob, B)
    for k in range(T):
        Xref = np.ascontiguousarray(np.roll(inst["Xref"], -k, axis=1))
        out = loop.step(Xref, noise=noise[:, k])
        ref, models = AC.oracle_solve(prob, sp.settings, x0 + noise[:, k], Xref, None, state, state is None, models, ar)
        got = {key: out[key].cpu().numpy() for key in AC.OUT + list(loop.fields)}
        got["models"] = loop.models.cpu().numpy()
        H.assert_bits_per_instance(got, dict(ref, models=models), AC.OUT + list(loop.fields) + ["models"], f"step {k}")
        state = {n: ref[n] for n in AC.BOX}
        x0 = _advance_ref(plant, x0, np.ascontiguousarray(ref["u"][:, 0, :]))
        assert H.bits_equal(loop.x0.cpu().numpy(), x0), k
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. tinympc_b200_advance_plant
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.float32, np.float64])
@pytest.mark.parametrize("per_instance", [False, True])
def test_advance_plant(dt, per_instance):
    torch = _torch()
    nx, nu, N, B = 12, 4, 10, 333
    spec = wl.quadrotor(N=N)
    solver = BatchedTinySolver(setup_problem(spec, dt), spec.settings)
    plant = _plant(spec, B, dt, seed=15, shared=not per_instance)
    tdt = torch.float32 if dt == np.float32 else torch.float64
    rec, per = pack_plant(plant, nx, nu, B, tdt, "cuda")
    assert per == per_instance
    rng = np.random.default_rng(16)
    x0 = rng.standard_normal((B, nx)).astype(dt)
    for stride in (nu, (N - 1) * nu):
        u = rng.standard_normal((B, stride)).astype(dt)
        x_t, u_t = torch.as_tensor(x0, device="cuda"), torch.as_tensor(u, device="cuda")
        check(solver._lib.tinympc_b200_advance_plant(solver._h, B, C.c_void_p(x_t.data_ptr()), C.c_void_p(u_t.data_ptr()), stride,
                                                     C.c_void_p(rec.data_ptr()), int(per), None))
        torch.cuda.synchronize()
        assert H.bits_equal(x_t.cpu().numpy(), _advance_ref(plant, x0, np.ascontiguousarray(u[:, :nu]))), stride
    solver.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. errors
# ---------------------------------------------------------------------------------------------------------------------
def _err(solver, T=2, **kw):
    p = solver.problem
    x0 = np.random.default_rng(0).standard_normal((8, p.nx)).astype(p.dtype)
    X = np.zeros((8, T + p.N - 1, p.nx), p.dtype)
    rc, *_ = _rollout_c(solver, x0, X, None, T, **kw)
    return rc


def test_rollout_plant_errors():
    torch = _torch()
    spec, prob, st = _quad(np.float32)
    s = BatchedTinySolver(prob, st)
    lib = s._lib
    plant, noise = _plant(spec, 8, np.float32), _noise(8, 2, 12, np.float32, 0)
    kw = dict(plant=plant, noise=noise)
    rec = torch.zeros(12 * 12 + 12 * 4 + 12, device="cuda")
    for ro in ({"plant_per_instance": 2}, {"plant_per_instance": -1}, {"reserved2": 1}, {"plant": None, "plant_per_instance": 1}):
        assert _err(s, ro_extra=ro, **kw) == abi.ERR_ARG, ro
    assert _err(s, ro_extra={"plant": rec.data_ptr(), "plant_per_instance": 0}) == abi.OK  # a shared record
    s.set_mode(abi.MODE_FAST)
    assert _err(s, **kw) == abi.ERR_UNSUPPORTED and b"STRICT" in lib.tinympc_b200_last_error()
    for fam in (abi.KERNEL_TPI, abi.KERNEL_GPS):
        s.set_mode(abi.MODE_STRICT, fam)
        assert _err(s, **kw) == abi.ERR_UNSUPPORTED and b"GPI" in lib.tinympc_b200_last_error()
    s.set_mode(abi.MODE_STRICT, abi.KERNEL_AUTO)
    rspec = wl.rocket(N=20)
    rs = BatchedTinySolver(setup_problem(rspec, np.float64), rspec.settings)
    assert _err(rs, plant=_plant(rspec, 8, np.float64), noise=_noise(8, 2, 6, np.float64, 0)) == abi.ERR_UNSUPPORTED and b"cones" in lib.tinympc_b200_last_error()
    _, lprob, lst = _quad(np.float32, N=1000)
    ls = BatchedTinySolver(lprob, lst)
    assert _err(ls, **kw) == abi.ERR_UNSUPPORTED and b"horizon" in lib.tinympc_b200_last_error()
    # tinympc_b200_advance_plant
    x = torch.zeros((8, 12), device="cuda")
    u = torch.zeros((8, 4), device="cuda")
    args = (s._h, 8, C.c_void_p(x.data_ptr()), C.c_void_p(u.data_ptr()), 4)
    assert lib.tinympc_b200_advance_plant(*args, None, 0, None) == abi.ERR_ARG
    assert lib.tinympc_b200_advance_plant(*args, C.c_void_p(rec.data_ptr()), 2, None) == abi.ERR_ARG
    # Python: missing keys, shapes, dtypes
    x0 = np.zeros((8, 12), np.float32)
    for bad in (dict(A=plant["A"], B=plant["B"]), dict(plant, A=plant["A"][:, :11]), dict(plant, f=plant["f"][0]),
                dict(plant, B=plant["B"].astype(np.int32)), [plant["A"], plant["B"], plant["f"]]):
        with pytest.raises(ValueError):
            DeviceMPCLoop(s, x0, plant=bad)
    loop = DeviceMPCLoop(s, x0, plant=plant)
    with pytest.raises(ValueError):
        loop.step(np.zeros((50, 12), np.float32), noise=np.zeros((8, 11), np.float32))
    with pytest.raises(ValueError):
        loop.step(np.zeros((50, 12), np.float32), noise=np.zeros((8, 12), np.int64))
    with pytest.raises(ValueError):
        loop.rollout(np.zeros((51, 12), np.float32), 2, noise=np.zeros((8, 3, 12), np.float32))
    # the existing refusals hold with a plant
    dK, dP = np.zeros((4, 12)), np.zeros((12, 12))
    with pytest.raises(ValueError):
        DeviceMPCLoop(s, x0, adaptive_rho=AdaptiveRho(dK, dP), plant=plant).rollout(np.zeros((60, 12), np.float32), 2)
    with pytest.raises(ValueError):
        DeviceMPCLoop(s, x0, extra_state=("x", "u"), plant=plant).rollout(np.zeros((60, 12), np.float32), 2)
    with pytest.raises(TinyMPCError):
        s.set_mode(abi.MODE_FAST)
        DeviceMPCLoop(s, x0, plant=plant).rollout(np.zeros((60, 12), np.float32), 2, noise=np.zeros((8, 2, 12), np.float32))
