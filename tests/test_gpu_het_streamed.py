"""Per-instance models (tinympc_batch_t.models) on the streamed lane-group kernel (GPS), bit for bit against the oracle.

A heterogeneous batch runs on the streamed kernel whenever the on-chip kernel cannot serve it: cones or hyperplanes, a
horizon that does not fit on chip, or an explicit GPS request.  The checker is the pinned restatement run once per model
over the instances that use it.  The instances are dealt to a handful of distinct models with a stride co-prime to the
model count, so that neighbouring slots, and a slot before and after a refill, hold different models.  Every scalar is
compared: the outputs, every requested state field (family slacks and duals included) and u0.
"""
import ctypes as C
import os

import numpy as np
import pytest

import helpers as H
import test_gpu_multiwave as MW
from oracle import oracle
from tinympc_b200 import abi, workloads as wl
from tinympc_b200._lib import TinyMPCError
from tinympc_b200.problem import MPCProblem
from tinympc_b200.solver import BatchedTinySolver, pack_models, setup_models, setup_problem, unpack_model

pytestmark = pytest.mark.gpu

NT = os.cpu_count() or 1
NM = 6      # distinct models of a batch
STRIDE = 5  # instance b uses model (STRIDE * b) % NM
DIMS = [(4, 1), (6, 3), (12, 4), (4, 2), (4, 4), (4, 8), (8, 2), (8, 4), (8, 8), (12, 2), (12, 8), (16, 2), (16, 4), (16, 8)]
SOC_LIN_STATE = H.SOC_STATE + ["vlnew", "zlnew", "gl", "yl"]


# ---------------------------------------------------------------------------------------------------------------------
# models, oracle, plan
# ---------------------------------------------------------------------------------------------------------------------
def _assign(B, nm=NM):
    return (STRIDE * np.arange(B)) % nm


def _models(nx, nu, N, dt, A, B, f, Qdiag, Rdiag, rho, cons):
    """setup_models blobs and, per blob, the single-model MPCProblem the oracle solves it with."""
    blobs = setup_models(nx, nu, A, B, f, Qdiag, Rdiag, rho, dtype=dt)
    probs = []
    for b in blobs:
        m = unpack_model(b, nx, nu)
        r = m.pop("rho")
        probs.append(MPCProblem(nx=nx, nu=nu, N=N, dtype=dt, rho=r, **m, **cons))
    return blobs, probs


def _rocket_fleet(dt, N, cons=None, seed=1):
    fl = wl.rocket_fleet(NM, N=N, seed=seed, mass_spread=0.3)
    sp = fl["spec"]
    cons = sp.constraints if cons is None else cons
    blobs, probs = _models(6, 3, N, dt, fl["A"], fl["B"], fl["f"], fl["Qdiag"], fl["Rdiag"], fl["rho"], cons)
    return sp, blobs, probs


def _tuned_fleet(spec, dt, nm=NM):
    """One model shared by every robot, per-robot tuning: rho and the state weights differ."""
    k = np.arange(nm)
    t = lambda a: np.tile(np.asarray(a, np.float64)[None], (nm,) + (1,) * np.ndim(a))  # noqa: E731
    Q = t(spec.Qdiag) * (1.0 + 0.25 * k)[:, None]
    rho = spec.rho * (0.6 + 0.2 * k)
    return _models(spec.nx, spec.nu, spec.N, dt, t(spec.A), t(spec.B), t(spec.f), Q, t(spec.Rdiag), rho, spec.constraints)


def _lti_fleet(nx, nu, N, dt, cons, seed=500):
    specs = [wl.random_lti(nx, nu, N, seed=seed + i) for i in range(NM)]
    rho = np.array([0.5 + 0.3 * i for i in range(NM)])
    st = lambda k: np.stack([getattr(s, k) for s in specs])  # noqa: E731
    return specs[0], _models(nx, nu, N, dt, st("A"), st("B"), st("f"), st("Qdiag"), st("Rdiag"), rho, cons)


def _port_grouped(probs, model, st):
    """One oracle run per model over the instances that use it; shared references are passed through."""
    def run(x0, Xref, Uref, state, cold, want):
        out = {}
        for m in np.unique(model):
            idx = np.flatnonzero(model == m)
            sub = None if state is None else {n: np.array(a[idx], copy=True) for n, a in state.items()}
            xr = Xref[idx] if Xref.ndim == 3 else Xref
            ur = None if Uref is None else (Uref[idx] if Uref.ndim == 3 else Uref)
            o = oracle.solve_batch(probs[m], st, x0[idx], xr, ur, state=sub, cold_start=cold, want_state=tuple(want),
                                   impl="port", nthreads=NT)
            for k, v in o.items():
                if v is not None:
                    out.setdefault(k, np.empty((len(x0),) + v.shape[1:], v.dtype))[idx] = v
        return out
    return run


def _expect_het_plan(stt):
    """The streamed kernel ran its per-instance-model variant: one instance per lane group."""
    assert stt["kernel_family"] == abi.KERNEL_GPS, stt
    assert stt["instances_per_cta"] == stt["threads_per_cta"] // stt["lanes_per_instance"], stt
    assert stt["workspace_bytes"] > 0, stt


def _cold_then_warm(solver, inst, models, port, want, what):
    """Cold solve and one warm step (duals reset on every third instance) on the device path with poisoned outputs."""
    x0, Xref, Uref = inst["x0"], inst["Xref"], inst.get("Uref")
    o1 = port(x0, Xref, Uref, None, True, want)
    g1, stt = MW._device_solve(solver, x0, Xref, Uref, None, True, want, models=models)
    _expect_het_plan(stt)
    MW._check(g1, o1, want, what + " cold")
    x0b, state = MW._warm_inputs(x0, o1, want, seed=len(x0))
    o2 = port(x0b, Xref, Uref, state, False, want)
    g2, stt = MW._device_solve(solver, x0b, Xref, Uref, state, False, want, models=models)
    _expect_het_plan(stt)
    MW._check(g2, o2, want, what + " warm")
    return o1, stt


def _het_capacity(prob, st, blob):
    """Instances one wave of the per-instance-model variant holds (ctas x instances_per_cta), from a one-iteration probe."""
    import torch

    sm = torch.cuda.get_device_properties(0).multi_processor_count
    st1 = abi.Settings.from_buffer_copy(st)
    st1.max_iter = 1
    s = BatchedTinySolver(prob, st1)
    B = 64 * sm
    batch, _ = s.make_device_batch(np.zeros((B, prob.nx), prob.dtype), np.zeros((prob.N, prob.nx), prob.dtype), cold_start=True,
                                   models=np.tile(blob, (B, 1)))
    s.solve_device(batch)
    torch.cuda.synchronize()
    stt = s.stats()
    s.close()
    _expect_het_plan(stt)
    assert stt["ctas"] == sm, stt
    return stt["ctas"] * stt["instances_per_cta"]


# ---------------------------------------------------------------------------------------------------------------------
# 1-3. constraint families
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [20, 100])
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_rocket_fleet_cones(dt, N):
    """Rockets of different masses with cones (C4's problem): AUTO picks the streamed kernel's NI = 1 variant."""
    sp, blobs, probs = _rocket_fleet(dt, N)
    st = MW._settings(sp)
    B = 150
    model = _assign(B)
    inst = wl.rocket_instances(B, N=N, seed=4, dtype=dt, spread=0.3, per_instance_refs=True)
    solver = BatchedTinySolver(probs[0], st)
    o1, _ = _cold_then_warm(solver, inst, blobs[model], _port_grouped(probs, model, st), H.SOC_STATE, f"rocket fleet N={N}")
    # the models really differ: every rocket that is not of model 0 gets another input sequence than model 0 would give it
    o0 = _port_grouped(probs, np.zeros(B, int), st)(inst["x0"], inst["Xref"], inst["Uref"], None, True, ())
    other = model != 0
    assert (np.abs(o1["sol_u"][other] - o0["sol_u"][other]).reshape(other.sum(), -1).max(axis=1) > 0).all()
    solver.close()


@pytest.mark.parametrize("tv", [False, True])
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_hyperplanes_per_robot_tuning(dt, tv):
    """Static / time-varying hyperplanes on the quadrotor, per-instance models that vary rho and the state weights."""
    sp = H.quad_linear_spec(tv=tv)
    blobs, probs = _tuned_fleet(sp, dt)
    st = MW._settings(sp, max_iter=40, abs_pri_tol=1e-2, abs_dua_tol=1e-2)
    B = 150
    model = _assign(B)
    inst = MW._hyperplane_instances(B, sp.N, dt, seed=31)
    solver = BatchedTinySolver(probs[0], st)
    want = H.TVLIN_STATE if tv else H.LIN_STATE
    _cold_then_warm(solver, inst, blobs[model], _port_grouped(probs, model, st), want, f"hyperplanes tv={tv}")
    solver.close()


ROCKET_PLANES = dict(Alin_x=np.array([[1.0, 0, 0, 0, 0, 0]]), blin_x=np.array([4.0]), Alin_u=np.array([[1.0, 1.0, 0]]),
                     blin_u=np.array([5.0]))


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_rocket_fleet_cones_and_hyperplanes(dt):
    """Cones and static hyperplanes together (every family of the kernel's mask 7) on the rocket fleet."""
    spec = wl.rocket(N=20)
    cons = dict(spec.constraints, **ROCKET_PLANES)
    sp, blobs, probs = _rocket_fleet(dt, 20, cons=cons)
    st = MW._settings(sp, en_state_linear=1, en_input_linear=1)
    B = 150
    model = _assign(B)
    inst = wl.rocket_instances(B, N=20, seed=6, dtype=dt, spread=0.3, per_instance_refs=True)
    solver = BatchedTinySolver(probs[0], st)
    _cold_then_warm(solver, inst, blobs[model], _port_grouped(probs, model, st), SOC_LIN_STATE, "rocket cones + hyperplanes")
    solver.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. every compiled shape, box only and with one static hyperplane
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("plane", [False, True])
@pytest.mark.parametrize("dt", [np.float32, np.float64])
@pytest.mark.parametrize("nx,nu", DIMS)
def test_every_shape_explicit_gps(nx, nu, dt, plane):
    N, B = 10, 40
    cons = wl.random_lti(nx, nu, N).constraints
    if plane:
        a = np.random.default_rng(nx * 17 + nu).uniform(-1.0, 1.0, (1, nx))
        cons = dict(cons, Alin_x=a, blin_x=np.array([0.5]))
    sp, (blobs, probs) = _lti_fleet(nx, nu, N, dt, cons)
    st = MW._settings(sp, max_iter=25, en_state_linear=int(plane))
    model = _assign(B)
    inst = wl.random_instances(B, nx, N, seed=70 + nx + nu, dtype=dt)
    inst["x0"] = (3.0 * inst["x0"]).astype(dt)
    solver = BatchedTinySolver(probs[0], st, kernel=abi.KERNEL_GPS)
    want = H.BOX_STATE + (["vlnew", "gl"] if plane else [])  # a state hyperplane: the input-side family stays disabled
    _cold_then_warm(solver, inst, blobs[model], _port_grouped(probs, model, st), want, f"({nx},{nu}) plane={plane}")
    solver.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. a box problem whose horizon does not fit on chip
# ---------------------------------------------------------------------------------------------------------------------
def test_box_horizon_off_chip():
    """Quadrotor fp64, N = 1000: no on-chip plan, so a heterogeneous batch streams."""
    dt = np.float64
    sp = wl.quadrotor(N=1000)
    blobs, probs = _tuned_fleet(sp, dt)
    st = MW._settings(sp, max_iter=30)
    B = 64
    model = _assign(B)
    inst = wl.hovering_instances(B, N=1000, dtype=dt)
    inst["x0"] = (inst["x0"] + 0.2 * np.random.default_rng(3).standard_normal(inst["x0"].shape)).astype(dt)
    solver = BatchedTinySolver(probs[0], st)
    _cold_then_warm(solver, inst, blobs[model], _port_grouped(probs, model, st), H.BOX_STATE, "quadrotor N=1000")
    solver.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. identical models = the shared-model solve
# ---------------------------------------------------------------------------------------------------------------------
def test_identical_models_equal_shared_model_solve():
    """pack_models blobs on the per-instance-model variant (NI = 1) give the bits of the shared-model streamed solve (NI = 2)."""
    dt = np.float64
    spec = wl.rocket(N=100)
    prob = setup_problem(spec, dt)
    B = 300
    inst = wl.rocket_instances(B, N=100, seed=8, dtype=dt, per_instance_refs=True)
    want = H.SOC_STATE
    solver = BatchedTinySolver(prob, spec.settings)
    shared, st_s = MW._device_solve(solver, inst["x0"], inst["Xref"], inst["Uref"], None, True, want)
    het, st_h = MW._device_solve(solver, inst["x0"], inst["Xref"], inst["Uref"], None, True, want, models=pack_models(prob, B))
    assert st_s["kernel_family"] == abi.KERNEL_GPS and st_s["instances_per_cta"] == 2 * st_s["threads_per_cta"] // st_s["lanes_per_instance"]
    _expect_het_plan(st_h)
    H.assert_bits_per_instance(het, shared, MW.OUTS + tuple(want), "identical models vs shared model")
    solver.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. slot refill across waves
# ---------------------------------------------------------------------------------------------------------------------
def _multiwave_rocket():
    dt = np.float64
    sp, blobs, probs = _rocket_fleet(dt, 20, seed=2)
    st = MW._settings(sp, max_iter=40, abs_pri_tol=0.1, abs_dua_tol=0.1)
    return probs, blobs, st, lambda B: MW._rocket_instances(B, 20, dt, seed=6), H.SOC_STATE


def _multiwave_box_off_chip():
    """Quadrotor tracking fp64, N = 200: the on-chip kernel has no plan for this horizon."""
    dt = np.float64
    sp = wl.quadrotor(N=200)
    blobs, probs = _tuned_fleet(sp, dt)
    st = MW._settings(sp, max_iter=15)
    return probs, blobs, st, lambda B: MW._tracking(B, 200, dt, seed=14), H.BOX_STATE


@pytest.mark.parametrize("case", ["rocket_cones_N20", "box_quad_N200"])
def test_multiwave_refill_cold_then_warm(case, monkeypatch):
    """TINYMPC_GPS_WARPS=1: one warp per SM, > 2.5 waves plus a ragged remainder in one launch; a refill loads a different
    model into the slot."""
    monkeypatch.setenv("TINYMPC_GPS_WARPS", "1")
    probs, blobs, st, gen, want = _multiwave_rocket() if case.startswith("rocket") else _multiwave_box_off_chip()
    B = 3 * _het_capacity(probs[0], st, blobs[0]) + 37
    model = _assign(B)
    solver = BatchedTinySolver(probs[0], st)
    stt = MW._cold_warm(solver, gen(B), want, abi.KERNEL_GPS, "het multiwave " + case, _port_grouped(probs, model, st),
                        models=blobs[model])
    _expect_het_plan(stt)
    assert stt["threads_per_cta"] == 32, stt
    solver.close()


# ---------------------------------------------------------------------------------------------------------------------
# 8. host path
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pin", [None, "all"])
def test_host_path_chunks(pin, monkeypatch):
    """tinympc_b200_solve_host with models on the streamed kernel: 11 chunks, page-locked or pageable caller buffers."""
    monkeypatch.setenv("TINYMPC_HOST_CHUNK", "96")
    dt = np.float64
    sp, blobs, probs = _rocket_fleet(dt, 20, seed=3)
    st = MW._settings(sp, max_iter=40, abs_pri_tol=0.1, abs_dua_tol=0.1)
    B = 1000
    model = _assign(B)
    inst = MW._rocket_instances(B, 20, dt, seed=9)
    port = _port_grouped(probs, model, st)
    want = H.SOC_STATE
    solver = BatchedTinySolver(probs[0], st)
    o1 = port(inst["x0"], inst["Xref"], inst["Uref"], None, True, want)
    x0b, state = MW._warm_inputs(inst["x0"], o1, want, seed=10)
    o2 = port(x0b, inst["Xref"], inst["Uref"], state, False, want)
    for step, (x0, s_in, o) in enumerate(((inst["x0"], None, o1), (x0b, state, o2))):
        h, stt = MW._host_solve(solver, x0, inst["Xref"], inst["Uref"], s_in, s_in is None, want, models=blobs[model], pin=pin)
        assert stt["kernel_launches"] == 11 and stt["kernel_family"] == abi.KERNEL_GPS, stt
        MW._check(h, o, want, f"host pin={pin} step {step}")


# ---------------------------------------------------------------------------------------------------------------------
# 9. FAST mode
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["box_quad_f32", "box_quad_f64", "rocket_cones_f64"])
def test_fast_mode_within_reference_scatter(case):
    """FAST (FMA contraction) at fixed work (tolerances 0, 20 iterations): x, u within 2e-4 relative of the STRICT oracle
    in fp32, 1e-10 in fp64 (the criterion of the shared-model kernels)."""
    dt = np.float32 if case.endswith("f32") else np.float64
    B = 150
    model = _assign(B)
    if case.startswith("box"):
        sp = wl.quadrotor(N=50)
        blobs, probs = _tuned_fleet(sp, dt)
        inst = wl.tracking_instances(B, N=50, seed=5, dtype=dt)
        kernel = abi.KERNEL_GPS
    else:
        sp, blobs, probs = _rocket_fleet(dt, 20)
        inst = wl.rocket_instances(B, N=20, seed=5, dtype=dt, per_instance_refs=True)
        kernel = abi.KERNEL_AUTO
    st = MW._settings(sp, abs_pri_tol=0.0, abs_dua_tol=0.0, max_iter=20)
    solver = BatchedTinySolver(probs[0], st, mode=abi.MODE_FAST, kernel=kernel)
    g = solver.solve(inst["x0"], inst["Xref"], inst["Uref"], cold_start=True, want_state=("x", "u"), models=blobs[model])
    _expect_het_plan(solver.stats())
    o = _port_grouped(probs, model, st)(inst["x0"], inst["Xref"], inst["Uref"], None, True, ("x", "u"))
    tol = 2e-4 if dt == np.float32 else 1e-10
    assert (g["iter"] == 20).all() and not g["solved"].any()
    for key in ("sol_x", "sol_u", "x", "u"):
        a, b = g[key].astype(np.float64), o[key].astype(np.float64)
        assert np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max()), (key, np.abs(a - b).max())
    solver.close()


# ---------------------------------------------------------------------------------------------------------------------
# 10. device closed loop of a heterogeneous fleet
# ---------------------------------------------------------------------------------------------------------------------
def _advance_ref(A, Bm, f, x0, u0):
    """x0 <- (A x0 + B u0) + f per instance (A [B,nx,nx], Bm [B,nx,nu] row index first): ascending sums, no FMA."""
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


def _blob_abf(blobs, nx, nu):
    ms = [unpack_model(b, nx, nu) for b in blobs]
    return np.stack([m["A"] for m in ms]), np.stack([m["B"] for m in ms]), np.stack([m["f"] for m in ms])


def test_device_closed_loop_fleet():
    """DeviceMPCLoop(models=...) without adaptive rho: solve with every plant's own model and advance it with its own
    A, B, f; every step against an oracle loop, x0 bit for bit."""
    from tinympc_b200.closed_loop import DeviceMPCLoop

    dt = np.float64
    sp, blobs, probs = _rocket_fleet(dt, 20, seed=5)
    st = MW._settings(sp, max_iter=40)
    B = 120
    model = _assign(B)
    inst = wl.rocket_instances(B, N=20, seed=11, dtype=dt, spread=0.3, per_instance_refs=True)
    solver = BatchedTinySolver(probs[0], st)
    cone_fields = ("x", "u", "vcnew", "zcnew", "gc", "yc")
    loop = DeviceMPCLoop(solver, inst["x0"], reset_duals=True, extra_state=cone_fields, models=blobs[model])
    port = _port_grouped(probs, model, st)
    A, Bm, f = (a[model] for a in _blob_abf(blobs, 6, 3))
    x0, state = inst["x0"].copy(), None
    for k in range(4):
        Xref = np.ascontiguousarray(np.roll(inst["Xref"], -k, axis=1))
        out = loop.step(Xref, inst["Uref"])
        if state is not None:
            state["g"] = np.zeros_like(state["g"])
            state["y"] = np.zeros_like(state["y"])
        o = port(x0, Xref, inst["Uref"], state, state is None, loop.fields)
        got = {key: out[key].cpu().numpy() for key in H.OUT_KEYS + list(loop.fields) + ["u0"]}
        _expect_het_plan(solver.stats())
        MW._check(got, o, loop.fields, f"closed loop step {k}")
        state = {n: o[n] for n in loop.fields}
        x0 = _advance_ref(A, Bm, f, x0, np.ascontiguousarray(o["u"][:, 0, :]))
        assert H.bits_equal(loop.x0.cpu().numpy(), x0), ("advance", k)
    solver.close()


# ---------------------------------------------------------------------------------------------------------------------
# 11. tinympc_b200_advance_models
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_advance_models(dt):
    import torch

    nx, nu, N, B = 8, 4, 10, 77
    sp, (blobs, probs) = _lti_fleet(nx, nu, N, dt, wl.random_lti(nx, nu, N).constraints)
    model = _assign(B)
    solver = BatchedTinySolver(probs[0], sp.settings)
    lib, h = solver._lib, solver._h
    rng = np.random.default_rng(2)
    x0 = rng.standard_normal((B, nx)).astype(dt)
    U = rng.standard_normal((B, N - 1, nu)).astype(dt)
    A, Bm, f = (a[model] for a in _blob_abf(blobs, nx, nu))
    dev = lambda a: torch.as_tensor(np.ascontiguousarray(a), device="cuda:0")  # noqa: E731
    tm = dev(blobs[model])
    stream = C.c_void_p(torch.cuda.current_stream(0).cuda_stream)
    # u_stride = nu (a u0 buffer) and (N-1)*nu (a work->u buffer): the first control of every instance
    for u, stride in ((np.ascontiguousarray(U[:, 0, :]), nu), (U, (N - 1) * nu)):
        tx, tu = dev(x0), dev(u)
        assert lib.tinympc_b200_advance_models(h, B, C.c_void_p(tx.data_ptr()), C.c_void_p(tu.data_ptr()), stride,
                                               C.c_void_p(tm.data_ptr()), stream) == abi.OK
        torch.cuda.synchronize()
        assert H.bits_equal(tx.cpu().numpy(), _advance_ref(A, Bm, f, x0, U[:, 0, :])), stride
    # pack_models blobs: the handle's own step
    prob = setup_problem(sp, dt)
    s2 = BatchedTinySolver(prob, sp.settings)
    tp = dev(pack_models(prob, B))
    ta, tb, tu = dev(x0), dev(x0), dev(U[:, 0, :])
    assert s2._lib.tinympc_b200_advance(s2._h, B, C.c_void_p(ta.data_ptr()), C.c_void_p(tu.data_ptr()), nu, stream) == abi.OK
    assert s2._lib.tinympc_b200_advance_models(s2._h, B, C.c_void_p(tb.data_ptr()), C.c_void_p(tu.data_ptr()), nu,
                                               C.c_void_p(tp.data_ptr()), stream) == abi.OK
    torch.cuda.synchronize()
    assert H.bits_equal(ta.cpu().numpy(), tb.cpu().numpy())
    assert not H.bits_equal(ta.cpu().numpy(), x0)
    # null pointers
    p = C.c_void_p(ta.data_ptr())
    assert lib.tinympc_b200_advance_models(h, B, p, p, nu, None, stream) == abi.ERR_ARG
    assert lib.tinympc_b200_advance_models(h, B, None, p, nu, p, stream) == abi.ERR_ARG
    assert lib.tinympc_b200_advance_models(h, B, p, None, nu, p, stream) == abi.ERR_ARG
    assert lib.tinympc_b200_advance_models(None, B, p, p, nu, p, stream) == abi.ERR_ARG
    s2.close()
    solver.close()


# ---------------------------------------------------------------------------------------------------------------------
# routing
# ---------------------------------------------------------------------------------------------------------------------
def test_routing():
    """Box constraints with an on-chip plan keep the on-chip kernel (AUTO and GPI); explicit GPS streams; TPI refuses."""
    dt = np.float32
    sp = wl.quadrotor(N=20)
    blobs, probs = _tuned_fleet(sp, dt)
    B = 64
    model = _assign(B)
    inst = wl.tracking_instances(B, N=20, seed=2, dtype=dt)
    st = MW._settings(sp, max_iter=30)
    port = _port_grouped(probs, model, st)
    o = port(inst["x0"], inst["Xref"], None, None, True, H.BOX_STATE)
    for kernel, fam in ((abi.KERNEL_AUTO, abi.KERNEL_GPI), (abi.KERNEL_GPI, abi.KERNEL_GPI), (abi.KERNEL_GPS, abi.KERNEL_GPS)):
        s = BatchedTinySolver(probs[0], st, kernel=kernel)
        g, stt = MW._device_solve(s, inst["x0"], inst["Xref"], None, None, True, H.BOX_STATE, models=blobs[model])
        assert stt["kernel_family"] == fam, (kernel, stt)
        MW._check(g, o, H.BOX_STATE, f"routing kernel={kernel}")
        s.close()
    s = BatchedTinySolver(probs[0], st, kernel=abi.KERNEL_TPI)
    with pytest.raises(TinyMPCError) as e:
        s.solve(inst["x0"], inst["Xref"], None, models=blobs[model])
    assert e.value.code == abi.ERR_UNSUPPORTED
    s.close()
