"""Closed-loop rollouts (tinympc_b200_rollout, DeviceMPCLoop.rollout): T warm-started MPC steps per robot in one launch of the
on-chip kernel's rollout variant, held bit for bit to DeviceMPCLoop stepping the same loop one launch at a time, and to the CPU
oracle stepping it on the host.  Every output buffer of the rollout is filled with a NaN bit pattern first."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest

import helpers as H
from oracle import oracle
from tinympc_b200 import abi, workloads as wl
from tinympc_b200._lib import TinyMPCError, check
from tinympc_b200.closed_loop import DeviceMPCLoop
from tinympc_b200.solver import AdaptiveRho, BatchedTinySolver, setup_models, setup_problem

pytestmark = pytest.mark.gpu

NT = os.cpu_count() or 1
FIELDS = ("v", "z", "vnew", "znew", "g", "y")
FIELDS_FAST = ("vnew", "znew", "g", "y")
PER_STEP = ("x", "u", "iter", "solved", "residuals")
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
    return setup_problem(spec, dt), _settings(spec, **dict(dict(max_iter=15), **kw))


def _episode(B, N, T, dt, seed, per_robot=True, uref=True):
    """Sliding tracking references of T+N-1 knots (per robot or one shared), an input reference, jittered start states."""
    inst = wl.tracking_instances(B, N=T + N - 1, seed=seed, dtype=dt, jitter=0.5)
    rng = np.random.default_rng(seed + 1)
    X = inst["Xref"] if per_robot else np.ascontiguousarray(inst["Xref"][0])
    U = None
    if uref:
        U = (0.05 * rng.standard_normal((B, T + N - 2, 4) if per_robot else (T + N - 2, 4))).astype(dt)
    return np.ascontiguousarray(inst["x0"]), X, U


def _capacity(solver):
    """Instances one wave of the on-chip kernel holds, from a one-iteration solve large enough to fill every SM."""
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


# ---------------------------------------------------------------------------------------------------------------------
# the two ways of running an episode
# ---------------------------------------------------------------------------------------------------------------------
def _loop(solver, x0, X, U, T, reset, exact, models=None, w=None, loop=None):
    """DeviceMPCLoop.step T times with the sliding window -> per-step outputs [B, T(+1), ...] and the final loop."""
    torch = _torch()
    N = solver.problem.N
    if loop is None:
        loop = DeviceMPCLoop(solver, x0, reset_duals=reset, exact_first_residual=exact, models=models)
    per = {k: [] for k in PER_STEP}
    for t in range(T):
        per["x"].append(loop.x0.clone())
        out = loop.step(X[..., t:t + N, :], None if U is None else U[..., t:t + N - 1, :])
        for k, o in (("u", "u0"), ("iter", "iter"), ("solved", "solved"), ("residuals", "residuals")):
            per[k].append(out[o].clone())
        if w is not None:
            loop.x0 += torch.as_tensor(w[:, t], device=loop.x0.device)
    per["x"].append(loop.x0.clone())
    torch.cuda.synchronize()
    res = {k: torch.stack(v, 1).cpu().numpy() for k, v in per.items() if v}
    return res, loop


def _final(loop):
    torch = _torch()
    torch.cuda.synchronize()
    d = {n: loop.state[n].cpu().numpy() for n in loop.fields}
    d.update(x0=loop.x0.cpu().numpy(), sol_x=loop.out["sol_x"].cpu().numpy(), sol_u=loop.out["sol_u"].cpu().numpy())
    return d


def _rollout_c(solver, x0, X, U, T, reset, carry, fields, cold=True, state=None, models=None, w=None, io_extra=None, ro_extra=None):
    """tinympc_b200_rollout on poisoned device buffers -> (rc, per-step outputs, final state, stats)."""
    torch = _torch()
    p = solver.problem
    dev = torch.device("cuda", solver.device)
    tdt = torch.float32 if p.dtype == np.float32 else torch.float64
    t = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a, dtype=p.dtype), device=dev)  # noqa: E731
    B = len(x0)
    x0_t, X_t, U_t, w_t = t(x0), t(X), t(U), t(w)
    M = None if models is None else torch.as_tensor(np.ascontiguousarray(models, dtype=p.dtype), device=dev)
    st = {}
    for n in fields:
        shape = (B, p.N, p.nx) if abi.STATE_IS_X[n] else (B, p.N - 1, p.nu)
        st[n] = H.poison(torch.empty(shape, dtype=tdt, device=dev)) if state is None else t(state[n]).clone()
    out = dict(x=torch.empty((B, T + 1, p.nx), dtype=tdt, device=dev), u=torch.empty((B, T, p.nu), dtype=tdt, device=dev),
               iter=torch.empty((B, T), dtype=torch.int32, device=dev), solved=torch.empty((B, T), dtype=torch.int32, device=dev),
               residuals=torch.empty((B, T, 4), dtype=tdt, device=dev), sol_x=torch.empty((B, p.N, p.nx), dtype=tdt, device=dev),
               sol_u=torch.empty((B, p.N - 1, p.nu), dtype=tdt, device=dev))
    for v in out.values():
        H.poison(v)
    x0_before = x0_t.clone()
    b = abi.Batch()
    b.B, b.x0, b.cold_start = B, x0_t.data_ptr(), int(cold)
    for n, a in st.items():
        setattr(b.state, n, a.data_ptr())
    b.sol_x, b.sol_u = out["sol_x"].data_ptr(), out["sol_u"].data_ptr()
    b.models = None if M is None else M.data_ptr()
    r = abi.Rollout()
    r.T, r.reset_duals, r.carry_v = T, int(reset), int(carry)
    r.Xref, r.xref_per_instance = (None, 0) if X_t is None else (X_t.data_ptr(), int(X_t.dim() == 3))
    r.Uref, r.uref_per_instance = (None, 0) if U_t is None else (U_t.data_ptr(), int(U_t.dim() == 3))
    r.w = None if w_t is None else w_t.data_ptr()
    r.x_traj, r.u_traj, r.residuals_traj = out["x"].data_ptr(), out["u"].data_ptr(), out["residuals"].data_ptr()
    r.iter_traj, r.solved_traj = out["iter"].data_ptr(), out["solved"].data_ptr()
    for k, v in (io_extra or {}).items():
        setattr(b, k, v)
    for k, v in (ro_extra or {}).items():
        setattr(r, k, v)
    rc = solver._lib.tinympc_b200_rollout(solver._h, C.byref(b), C.byref(r), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize()
    assert torch.equal(x0_before.view(torch.uint8), x0_t.view(torch.uint8)), "io->x0 must not be modified"
    res = {k: v.cpu().numpy() for k, v in out.items()}
    fin = {n: a.cpu().numpy() for n, a in st.items()}
    return rc, res, fin, solver.stats()


def _compare(got, ref, fin_got, loop, what, fields):
    H.assert_bits_per_instance(got, ref, PER_STEP, what)
    f = _final(loop)
    H.assert_bits_per_instance(dict(fin_got, x0=got["x"][:, -1], sol_x=got["sol_x"], sol_u=got["sol_u"]), f,
                               list(fields) + ["x0", "sol_x", "sol_u"], what + " final")


def _mixed(res):
    """Steps end both converged and at max_iter, at >= 5 different iteration counts."""
    H.assert_mixed_termination(dict(iter=res["iter"].ravel(), solved=res["solved"].ravel()))


# ---------------------------------------------------------------------------------------------------------------------
# against the loop
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.float32, np.float64])
@pytest.mark.parametrize("per_robot,reset,exact", [(True, True, True), (False, False, True), (True, False, False), (False, True, False)])
def test_rollout_matches_loop(dt, per_robot, reset, exact):
    """(12,4,50) tracking with an input reference, 2.5 waves of the plan plus a ragged remainder, T = 5."""
    prob, st = _quad(dt)
    solver = BatchedTinySolver(prob, st)
    cap = _capacity(solver)
    B = int(2.5 * cap) + 37
    T = 5
    x0, X, U = _episode(B, prob.N, T, dt, seed=11 + int(per_robot) + 2 * int(reset), per_robot=per_robot)
    fields = FIELDS if exact else FIELDS_FAST
    rc, got, fin, stt = _rollout_c(solver, x0, X, U, T, reset, exact, fields)
    check(rc)
    assert stt["kernel_family"] == abi.KERNEL_GPI and stt["kernel_launches"] == 1, stt
    assert B >= 2.5 * stt["ctas"] * stt["instances_per_cta"], (B, stt)
    ref, loop = _loop(solver, x0, X, U, T, reset, exact)
    _mixed(ref)
    _compare(got, ref, fin, loop, f"rollout {dt.__name__} per_robot={per_robot} reset={reset} exact={exact}", fields)


def _oracle_episode(prob, st, x0, X, U, T, w=None):
    """The loop on the host: the oracle solves each window warm-started with the duals reset, the plant advances with the
    ascending-k, no-FMA arithmetic of tinympc_b200_advance."""
    N, dt = prob.N, prob.dtype
    A, Bm, f = np.asarray(prob.A, dt), np.asarray(prob.B, dt), np.asarray(prob.f, dt)
    state = None
    per = {k: [] for k in PER_STEP}
    for t in range(T):
        per["x"].append(x0.copy())
        if state is not None:
            state["g"] = np.zeros_like(state["g"])
            state["y"] = np.zeros_like(state["y"])
        Xw = np.ascontiguousarray(X[..., t:t + N, :])
        Uw = None if U is None else np.ascontiguousarray(U[..., t:t + N - 1, :])
        o = oracle.solve_batch(prob, st, x0, Xw, Uw, state=state, cold_start=state is None, want_state=FIELDS + ("u",),
                               impl="port", nthreads=NT)
        state = {n: np.array(o[n], copy=True) for n in FIELDS}
        u0 = np.ascontiguousarray(o["u"][:, 0, :])
        per["u"].append(u0)
        per["iter"].append(o["iter"])
        per["solved"].append(o["solved"])
        per["residuals"].append(o["residuals"])
        nxt = np.zeros_like(x0)
        for i in range(prob.nx):
            ax = A[i, 0] * x0[:, 0]
            for m in range(1, prob.nx):
                ax = ax + A[i, m] * x0[:, m]
            bu = Bm[i, 0] * u0[:, 0]
            for j in range(1, prob.nu):
                bu = bu + Bm[i, j] * u0[:, j]
            nxt[:, i] = (ax + bu) + f[i]
        x0 = nxt if w is None else (nxt + w[:, t]).astype(dt)
    per["x"].append(x0.copy())
    return {k: np.stack(v, 1) for k, v in per.items()}, state, o


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_rollout_matches_oracle(dt):
    """64 robots, duals reset, v / z carried: every step against the oracle stepping the loop on the host."""
    prob, st = _quad(dt)
    T, B = 4, 64
    x0, X, U = _episode(B, prob.N, T, dt, seed=5)
    solver = BatchedTinySolver(prob, st)
    rc, got, fin, _ = _rollout_c(solver, x0, X, U, T, True, True, FIELDS)
    check(rc)
    ref, state, last = _oracle_episode(prob, st, x0, X, U, T)
    H.assert_bits_per_instance(got, ref, PER_STEP, f"oracle {dt.__name__}")
    H.assert_bits_per_instance(dict(fin, sol_x=got["sol_x"], sol_u=got["sol_u"]), dict(state, sol_x=last["sol_x"], sol_u=last["sol_u"]),
                               list(FIELDS) + ["sol_x", "sol_u"], f"oracle {dt.__name__} final")


# ---------------------------------------------------------------------------------------------------------------------
# fleets and disturbances
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_rollout_fleet(dt):
    """Six tuned quadrotors dealt with a stride of five, against DeviceMPCLoop(models=...), per-robot references."""
    spec = wl.quadrotor(N=50)
    st = _settings(spec, max_iter=15)
    M = 6
    rng = np.random.default_rng(3)
    A = np.stack([spec.A] * M)
    Bm = np.stack([spec.B * (1.0 + 0.05 * i) for i in range(M)])
    f = np.stack([spec.f] * M)
    Q = np.stack([spec.Qdiag * (1.0 + 0.2 * i) for i in range(M)])
    R = np.stack([spec.Rdiag * (1.0 + 0.1 * rng.random()) for _ in range(M)])
    blobs = setup_models(12, 4, A, Bm, f, Q, R, np.array([spec.rho * (1.0 + 0.25 * i) for i in range(M)]), dtype=dt)
    prob = setup_problem(spec, dt)
    solver = BatchedTinySolver(prob, st)
    B = int(2.5 * _capacity(solver)) + 37
    models = blobs[(5 * np.arange(B)) % M]
    T = 4
    x0, X, U = _episode(B, 50, T, dt, seed=21)
    rc, got, fin, stt = _rollout_c(solver, x0, X, U, T, True, True, FIELDS, models=models)
    check(rc)
    assert stt["kernel_family"] == abi.KERNEL_GPI, stt
    ref, loop = _loop(solver, x0, X, U, T, True, True, models=models)
    _mixed(ref)
    _compare(got, ref, fin, loop, f"fleet {dt.__name__}", FIELDS)


def test_rollout_disturbance():
    dt = np.float32
    prob, st = _quad(dt)
    T, B = 5, 700
    x0, X, U = _episode(B, prob.N, T, dt, seed=31)
    w = (0.01 * np.random.default_rng(4).standard_normal((B, T, 12))).astype(dt)
    solver = BatchedTinySolver(prob, st)
    rc, got, fin, _ = _rollout_c(solver, x0, X, U, T, True, True, FIELDS, w=w)
    check(rc)
    ref, loop = _loop(solver, x0, X, U, T, True, True, w=w)
    _compare(got, ref, fin, loop, "disturbance", FIELDS)
    oref, _, _ = _oracle_episode(prob, st, x0[:64], X[:64], U[:64], T, w=w[:64])
    H.assert_bits_per_instance({k: v[:64] for k, v in got.items()}, oref, PER_STEP, "disturbance oracle")


# ---------------------------------------------------------------------------------------------------------------------
# every compiled shape
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_rollout_every_shape(dt):
    """Every compiled (nx, nu) at N = 50, T = 3: the rollout runs with the plan a fixed-step solve of the same batch gets on the
    on-chip kernel and equals the loop; a shape without an on-chip plan is refused."""
    torch = _torch()
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
        batch, _ = solver.make_device_batch(x0, X[:, :N], cold_start=True)
        solver.solve_device(batch)
        torch.cuda.synchronize()
        plan = solver.stats()
        rc, got, fin, stt = _rollout_c(solver, x0, X, None, T, True, True, FIELDS)
        if plan["kernel_family"] != abi.KERNEL_GPI:  # no on-chip plan for this horizon
            assert rc == abi.ERR_UNSUPPORTED, (nx, nu, rc)
            continue
        check(rc)
        served += 1
        keys = ("kernel_family", "lanes_per_instance", "instances_per_cta", "smem_bytes_per_cta", "ctas", "threads_per_cta")
        assert {k: stt[k] for k in keys} == {k: plan[k] for k in keys}, (nx, nu, stt, plan)
        ref, loop = _loop(solver, x0, X, None, T, True, True)
        _compare(got, ref, fin, loop, f"shape ({nx},{nu}) {dt.__name__}", FIELDS)
    assert served >= 5, served


# ---------------------------------------------------------------------------------------------------------------------
# edges
# ---------------------------------------------------------------------------------------------------------------------
def test_rollout_t0_writes_nothing():
    prob, st = _quad(np.float32)
    x0, X, U = _episode(50, prob.N, 0, np.float32, seed=2)
    solver = BatchedTinySolver(prob, st)
    rc, got, fin, _ = _rollout_c(solver, x0, X, U, 0, True, True, FIELDS)
    check(rc)
    for k, v in list(got.items()) + list(fin.items()):
        assert H.bits_equal(v, H.poison(np.empty_like(v))), k


@pytest.mark.parametrize("case", ["T1", "max_iter0", "check3"])
def test_rollout_edges(case):
    dt = np.float64
    kw = dict(T1=dict(), max_iter0=dict(max_iter=0), check3=dict(max_iter=20, check_termination=3))[case]
    prob, st = _quad(dt, **kw)
    T = 1 if case == "T1" else 4
    x0, X, U = _episode(300, prob.N, T, dt, seed=40)
    solver = BatchedTinySolver(prob, st)
    rc, got, fin, _ = _rollout_c(solver, x0, X, U, T, True, True, FIELDS)
    check(rc)
    ref, loop = _loop(solver, x0, X, U, T, True, True)
    _compare(got, ref, fin, loop, case, FIELDS)


@pytest.mark.parametrize("exact", [True, False])
def test_rollout_continues_loop_and_step_continues_rollout(exact):
    """step, step, rollout(3), step against step x6, through DeviceMPCLoop.rollout."""
    torch = _torch()
    dt = np.float32
    prob, st = _quad(dt)
    N, B = prob.N, 500
    x0, X, U = _episode(B, N, 6, dt, seed=50)
    solver = BatchedTinySolver(prob, st)
    ref, ref_loop = _loop(solver, x0, X, U, 6, True, exact)
    a = DeviceMPCLoop(solver, x0, reset_duals=True, exact_first_residual=exact)
    _, a = _loop(solver, x0, X, U, 2, True, exact, loop=a)
    res = a.rollout(torch.as_tensor(X[:, 2:], device="cuda"), 3, Uref_traj=U[:, 2:])
    torch.cuda.synchronize()
    got = {k: res[k].cpu().numpy() for k in PER_STEP}
    H.assert_bits_per_instance(got, {k: v[:, 2:5] if k != "x" else v[:, 2:6] for k, v in ref.items()}, PER_STEP, "rollout after steps")
    _, a = _loop(solver, None, X[:, 5:], U[:, 5:], 1, True, exact, loop=a)
    fa, fr = _final(a), _final(ref_loop)
    H.assert_bits_per_instance(fa, fr, list(a.fields) + ["x0", "sol_x", "sol_u"], "step after rollout")


# ---------------------------------------------------------------------------------------------------------------------
# loud errors
# ---------------------------------------------------------------------------------------------------------------------
def _err(solver, T=2, **kw):
    """The return code of a small rollout (an error leaves every buffer as it was)."""
    p = solver.problem
    x0 = np.random.default_rng(0).standard_normal((8, p.nx)).astype(p.dtype)
    X = np.zeros((8, T + p.N - 1, p.nx), p.dtype)
    rc, *_ = _rollout_c(solver, x0, X, None, T, True, True, FIELDS, **kw)
    return rc


def test_rollout_errors():
    prob, st = _quad(np.float32)
    s = BatchedTinySolver(prob, st)
    lib = s._lib
    s.set_mode(abi.MODE_FAST)
    assert _err(s) == abi.ERR_UNSUPPORTED and b"STRICT" in lib.tinympc_b200_last_error()
    for fam in (abi.KERNEL_TPI, abi.KERNEL_GPS):
        s.set_mode(abi.MODE_STRICT, fam)
        assert _err(s) == abi.ERR_UNSUPPORTED and b"GPI" in lib.tinympc_b200_last_error()
    s.set_mode(abi.MODE_STRICT, abi.KERNEL_AUTO)
    dummy = _torch().zeros(64, device="cuda").data_ptr()  # any device buffer: the call must refuse it before reading
    for field in ("Xref", "iter", "u0"):
        assert _err(s, io_extra={field: dummy}) == abi.ERR_ARG, field
    assert _err(s, ro_extra={"Xref": None}) == abi.ERR_ARG
    assert _err(s, ro_extra={"T": -1}) == abi.ERR_ARG
    assert _err(s, ro_extra={"reserved": 1}) == abi.ERR_ARG
    assert _err(s, ro_extra={"reserved1": (C.c_int64 * 2)(0, 5)}) == abi.ERR_ARG
    rspec = wl.rocket(N=20)
    rs = BatchedTinySolver(setup_problem(rspec, np.float64), rspec.settings)
    assert _err(rs) == abi.ERR_UNSUPPORTED and b"cones" in lib.tinympc_b200_last_error()
    lprob, lst = _quad(np.float32, N=1000)
    ls = BatchedTinySolver(lprob, lst)
    assert _err(ls) == abi.ERR_UNSUPPORTED and b"horizon" in lib.tinympc_b200_last_error()
    # Python: adaptive rho and extra state are refused
    dK, dP = np.zeros((4, 12)), np.zeros((12, 12))
    loop = DeviceMPCLoop(s, np.zeros((4, 12), np.float32), adaptive_rho=AdaptiveRho(dK, dP))
    with pytest.raises(ValueError):
        loop.rollout(np.zeros((60, 12), np.float32), 2)
    loop = DeviceMPCLoop(s, np.zeros((4, 12), np.float32), extra_state=("x", "u"))
    with pytest.raises(ValueError):
        loop.rollout(np.zeros((60, 12), np.float32), 2)
    with pytest.raises(TinyMPCError):
        s.set_mode(abi.MODE_FAST)
        DeviceMPCLoop(s, np.zeros((4, 12), np.float32)).rollout(np.zeros((60, 12), np.float32), 2)
