"""Per-instance static hyperplanes (tinympc_batch_t.planes_per_instance) on the streamed (GPS) lane-group kernel, through the
device entry point, the host path, the Python layer and the device closed loop.

Every instance is compared bit for bit, on every output and requested state field, with the oracle run once per distinct
plane set over the instances that use it (instance_common.grouped_oracle), NaN-poisoned as instance_common describes.  The
plane sets are dealt with a stride, so neighbouring slots, the two instances of a lane group and the refills of a slot change
planes.  The launch plan is asserted through stats(); per-instance planes add no shared-memory table."""
import ctypes as C

import numpy as np
import pytest

import helpers as H
import instance_common as IC
from tinympc_b200 import abi, workloads as wl
from tinympc_b200._lib import TinyMPCError
from tinympc_b200.solver import BatchedTinySolver, setup_models, setup_problem

pytestmark = pytest.mark.gpu

WANT = tuple(H.LIN_STATE)
TV_WANT = WANT + ("vlnew_tv", "zlnew_tv", "gl_tv", "yl_tv")
DTS = [np.float32, np.float64]


# ---------------------------------------------------------------------------------------------------------------------
# problems and instances
# ---------------------------------------------------------------------------------------------------------------------
def _quad(dt, N, tv=False, **kw):
    """the hyperplane quadrotor (helpers.quad_linear_spec); tv: the time-varying hyperplanes of the handle run too (mask 6,
    both families)"""
    spec = H.quad_linear_spec(N=N)
    if tv:
        spec.constraints = dict(spec.constraints, **H.quad_linear_spec(tv=True, N=N).constraints)
        spec.settings.en_tv_state_linear = 1
        spec.settings.en_tv_input_linear = 1
    return spec, setup_problem(spec, dt), IC.settings(spec, **dict(dict(max_iter=40), **kw))


def _quad_instances(B, N, dt, seed):
    inst = wl.tracking_instances(B, N=N, seed=seed, dtype=dt, jitter=0.3)
    return dict(x0=inst["x0"], Xref=inst["Xref"], Uref=None)


def _sides(st):
    """the plane sides whose loops run under the settings"""
    return tuple(k for k, on in (("x", st.en_state_linear), ("u", st.en_input_linear)) if on)


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
    planes = IC.batch_planes([IC.own_planes(prob)], np.zeros(B, int))
    x0, state = inst["x0"], None
    for cold in (True, False):
        shared, s0 = IC.device(s, x0, inst["Xref"], None, state, cold, WANT)
        got, s1 = IC.device(s, x0, inst["Xref"], None, state, cold, WANT, planes=planes)
        IC.same_plan(s0, s1)
        H.assert_bits_per_instance(got, shared, list(shared), f"cold={cold}")
        x0, state = IC.warm_inputs(inst["x0"], shared, seed=2, want=WANT)
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
    planes = IC.batch_planes(pal, IC.deal(B, 7, stride=3), sides=_sides(st))
    off = {"x": ("zlnew", "yl"), "u": ("vlnew", "gl"), "xu": ()}[sides]  # a side whose loop does not run: fields left unwritten
    want = tuple(n for n in WANT if n not in off)
    plan0 = IC.shared_plan(s, inst, want)
    o1, _, stt = IC.cold_warm(s, inst, f"quad fleet {sides}", want, planes=planes)
    IC.same_plan(plan0, stt)
    # the planes bite: most instances end with a slack on one of their own planes
    act = IC.active_rows(planes, o1.get("vlnew"), o1.get("zlnew"))
    assert act.mean() >= 0.5, act.mean()
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. more than 2.5 waves of slot refills in one launch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt,warps", [(np.float64, None), (np.float32, "1"), (np.float64, "1")])
def test_multiwave(dt, warps, monkeypatch):
    if warps:
        monkeypatch.setenv("TINYMPC_GPS_WARPS", warps)
    spec, prob, st = _quad(dt, 20, max_iter=25)
    s = BatchedTinySolver(prob, st)
    B = int(2.6 * IC.capacity(s, lambda B: dict(planes=IC.batch_planes([IC.own_planes(prob)], np.zeros(B, int))))) + 37
    K = 5
    pal = IC.plane_palette(prob, K - 1, seed=20) + IC.plane_palette(prob, 1, seed=22, pad=1)  # one robot pads a row of each side
    o1, _, _ = IC.cold_warm(s, _quad_instances(B, 20, dt, seed=21), "multiwave", WANT, mult=2.5,
                            planes=IC.batch_planes(pal, IC.deal(B, K)))
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
    plan0 = IC.shared_plan(s, inst, WANT, models=models[model_of])
    pal = IC.plane_palette(prob, 6, seed=6)
    _, _, stt = IC.cold_warm(s, inst, "planes + models", WANT, models=models, model_of=model_of,
                             planes=IC.batch_planes(pal, IC.deal(B, 6)))
    IC.one_per_group(stt)
    IC.same_plan(plan0, stt)
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
    plan0 = IC.shared_plan(s, inst, TV_WANT)
    pal = _fleet_palette(spec, prob, 5, seed=8)
    _, _, stt = IC.cold_warm(s, inst, "static + tv planes", TV_WANT, planes=IC.batch_planes(pal, IC.deal(B, 5, stride=3)))
    IC.same_plan(plan0, stt)
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
    st = IC.settings(spec, max_iter=40, abs_pri_tol=0.1, abs_dua_tol=0.1)
    s = BatchedTinySolver(prob, st)
    B = 800
    inst = wl.rocket_instances(B, N=50, seed=9, dtype=dt, spread=0.3, per_instance_refs=True)
    want = tuple(H.SOC_STATE) + ("vlnew", "zlnew", "gl", "yl")
    plan0 = IC.shared_plan(s, inst, want)
    pal = IC.plane_palette(prob, 6, seed=10, shift=(-1.0, 0.2))
    _, _, stt = IC.cold_warm(s, inst, "rocket cones + planes", want, planes=IC.batch_planes(pal, IC.deal(B, 6, stride=5)))
    IC.same_plan(plan0, stt)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. every compiled (nx, nu): covered shapes against the oracle, the others refused
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("nx,nu", IC.DIMS)
def test_every_shape(nx, nu, dt):
    spec = wl.random_lti(nx, nu, 30, seed=300 + nx * 10 + nu)
    rng = np.random.default_rng(nx * 100 + nu)
    spec.constraints = dict(spec.constraints, Alin_x=rng.standard_normal((2, nx)), blin_x=np.array([0.2, 0.1]),
                            Alin_u=rng.standard_normal((1, nu)), blin_u=np.array([0.1]))
    spec.settings.en_state_linear = 1
    spec.settings.en_input_linear = 1
    prob = setup_problem(spec, dt)
    st = IC.settings(spec, max_iter=30)
    s = BatchedTinySolver(prob, st)
    B = 300
    inst = dict(x0=(0.5 * rng.standard_normal((B, nx))).astype(dt), Xref=(0.1 * rng.standard_normal((B, 30, nx))).astype(dt))
    _, sh = IC.device(s, inst["x0"], inst["Xref"], None, None, True, WANT)
    pal = IC.plane_palette(prob, 3, seed=nx + nu)
    planes = IC.batch_planes(pal, IC.deal(B, 3, stride=2))
    if sh["kernel_family"] != abi.KERNEL_GPS:
        with pytest.raises(TinyMPCError) as e:
            IC.device(s, inst["x0"], inst["Xref"], None, None, True, WANT, planes=planes)
        assert e.value.code == abi.ERR_UNSUPPORTED
        pytest.skip(f"({nx},{nu}) is not covered by the streamed kernel in this precision")
    _, _, stt = IC.cold_warm(s, inst, f"({nx},{nu})", WANT, planes=planes)
    IC.same_plan(sh, stt)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. the host path in 11 chunks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pin", [False, True])
@pytest.mark.parametrize("dt,with_models", [(np.float32, False), (np.float64, False), (np.float32, True)])
def test_host_path_chunks(dt, with_models, pin, monkeypatch):
    spec, prob, st = _quad(dt, 20)
    s = BatchedTinySolver(prob, st)
    B = IC.HOST_B
    planes = IC.batch_planes(IC.plane_palette(prob, 7, seed=30), IC.deal(B, 7, stride=3))
    models = _quad_models(spec, dt) if with_models else None
    model_of = None if models is None else np.arange(B) % 4
    IC.host_path_chunks(s, _quad_instances(B, 20, dt, seed=31), WANT, pin, monkeypatch, models=models, model_of=model_of, planes=planes)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 8. the device closed loop: four steps, one with the obstacles closer
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
def test_closed_loop(dt):
    spec, prob, st = _quad(dt, 30)
    s = BatchedTinySolver(prob, st)
    B = 400
    inst = _quad_instances(B, 30, dt, seed=42)
    pal = IC.plane_palette(prob, 4, seed=40)
    pal2 = IC.plane_palette(prob, 4, seed=41, shift=(-0.6, -0.2))
    which = IC.deal(B, 4, stride=3)
    IC.closed_loop(s, inst, "planes", IC.batch_planes(pal, which), IC.batch_planes(pal2, which), 4,
                   extra_state=("x", "u", "vlnew", "zlnew", "gl", "yl"))
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 9. queued solves with different planes on one handle
# ---------------------------------------------------------------------------------------------------------------------
def test_queued_solves_different_planes():
    dt = np.float32
    spec, prob, st = _quad(dt, 50)
    s = BatchedTinySolver(prob, st)
    B = 6000
    inst = _quad_instances(B, 50, dt, seed=50)
    pals = [IC.plane_palette(prob, 5, seed=51), IC.plane_palette(prob, 5, seed=52, shift=(-0.6, 0.0))]
    IC.queued_solves(s, inst, WANT, "planes", [IC.batch_planes(p, IC.deal(B, 5)) for p in pals])
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
    planes = IC.batch_planes(IC.plane_palette(prob, 3, seed=61), IC.deal(B, 3, stride=2))
    want = tuple(H.BOX_STATE)
    for pl in (planes, {k: planes[k] for k in ("Alin_x", "blin_x")}):
        shared, s0 = IC.device(s, inst["x0"], inst["Xref"], None, None, True, want)
        got, s1 = IC.device(s, inst["x0"], inst["Xref"], None, None, True, want, planes=pl)
        IC.same_plan(s0, s1)
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
    dt = np.float64
    spec = _rocket_planes_spec(20)
    prob = setup_problem(spec, dt)
    st = IC.settings(spec, max_iter=20)
    s = BatchedTinySolver(prob, st)
    B = 64
    inst = wl.rocket_instances(B, N=20, seed=70, dtype=dt)
    planes = IC.batch_planes(IC.plane_palette(prob, 2, seed=71), IC.deal(B, 2, stride=1))
    batch, _ = s.make_device_batch(inst["x0"], inst["Xref"], inst["Uref"], cold_start=True, planes=planes)
    assert IC.solve_rc(s, batch) == abi.OK
    # a missing pointer for a side whose loop runs; a bad mode; reserved4
    for field, val in (("Alin_x", None), ("blin_x", None), ("Alin_u", None), ("blin_u", None), ("planes_per_instance", 2),
                       ("planes_per_instance", -1), ("reserved4", 1)):
        b = abi.Batch.from_buffer_copy(batch)
        setattr(b, field, val)
        assert IC.solve_rc(s, b) == abi.ERR_ARG, field
    # the missing side's loop switched off: its pointers are never needed
    b = abi.Batch.from_buffer_copy(batch)
    b.Alin_u = b.blin_u = None
    s.update_settings(en_input_linear=0)
    assert IC.solve_rc(s, b) == abi.OK
    s.update_settings(en_input_linear=1)
    # per-instance bounds or cones in the same batch
    bb, _ = s.make_device_batch(inst["x0"], inst["Xref"], inst["Uref"], cold_start=True, planes=planes,
                                bounds=dict(u_min=np.full((B, 3), -10.0), u_max=np.full((B, 3), 105.0),
                                            x_min=np.tile(prob.x_min[:, 0], (B, 1)), x_max=np.tile(prob.x_max[:, 0], (B, 1))))
    assert IC.solve_rc(s, bb) == abi.ERR_UNSUPPORTED and b"bounds or cones" in s._lib.tinympc_b200_last_error()
    cb, _ = s.make_device_batch(inst["x0"], inst["Xref"], inst["Uref"], cold_start=True, planes=planes,
                                cones=IC.batch_cones(IC.mu_palette(prob, 1, seed=72), np.zeros(B, int)))
    assert IC.solve_rc(s, cb) == abi.ERR_UNSUPPORTED and b"bounds or cones" in s._lib.tinympc_b200_last_error()
    IC.assert_refused(s, batch, inst["Xref"], b"hyperplanes")
    # Python checks: shapes, dtype, keys, pairs
    IC.assert_python_rejects(s, inst, "planes", [
        dict(planes, Alin_x=planes["Alin_x"][:, :, :-1]), dict(planes, blin_u=planes["blin_u"][:-1]),
        dict(planes, Alin_x=planes["Alin_x"].astype(np.float32)), {"Alin_x": planes["Alin_x"]}, dict(planes, A=planes["Alin_x"]), {}])
    s.close()
