"""Per-instance cone coefficients (tinympc_batch_t.cones_per_instance) on the streamed (GPS) lane-group kernel, through the device
entry point, the host path, the Python layer and the device closed loop.

Every instance is compared bit for bit, on every output and requested state field, with the oracle run once per distinct mu
set over the instances that use it (instance_common.grouped_oracle), NaN-poisoned as instance_common describes.  The mu sets
are dealt with a stride, so neighbouring slots, the two instances of a lane group and the refills of a slot change mu.  The
launch plan is asserted through stats()."""
import ctypes as C

import numpy as np
import pytest

import helpers as H
import instance_common as IC
from tinympc_b200 import abi, workloads as wl
from tinympc_b200._lib import TinyMPCError
from tinympc_b200.solver import BatchedTinySolver, setup_models, setup_problem

pytestmark = pytest.mark.gpu

WANT = tuple(H.SOC_STATE)
DTS = [np.float32, np.float64]


# ---------------------------------------------------------------------------------------------------------------------
# problems and instances
# ---------------------------------------------------------------------------------------------------------------------
def _rocket(dt, N, **kw):
    spec = wl.rocket(N=N)
    return setup_problem(spec, dt), IC.settings(spec, **dict(dict(max_iter=40, abs_pri_tol=0.1, abs_dua_tol=0.1), **kw))


def _rocket_instances(B, N, dt, seed):
    return wl.rocket_instances(B, N=N, seed=seed, dtype=dt, spread=0.3, per_instance_refs=True)


def _sides(st):
    """the cone sides whose loops run under the settings"""
    return tuple(k for k, on in (("x_mu", st.en_state_soc), ("u_mu", st.en_input_soc)) if on)


def _table(dt):
    """the cone-coefficient table's bytes per instance: MAX_CONES (4) mu per side"""
    return 2 * 4 * np.dtype(dt).itemsize


def _rocket_models(dt, nm=4):
    """nm rockets of different masses (wl.rocket_fleet): per-instance models"""
    f = wl.rocket_fleet(nm, N=10, seed=3)
    spec = f["spec"]
    return setup_models(spec.nx, spec.nu, f["A"], f["B"], f["f"], f["Qdiag"], f["Rdiag"], f["rho"], dtype=dt)


# ---------------------------------------------------------------------------------------------------------------------
# 1. every instance given the handle's mu: the shared solve's bits and plan (two instances per lane group kept)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
def test_equal_mu_equal_shared_solve(dt):
    prob, st = _rocket(dt, 100)
    s = BatchedTinySolver(prob, st)
    B = 700
    inst = _rocket_instances(B, 100, dt, seed=1)
    cones = IC.batch_cones([dict(x_mu=prob.cx, u_mu=prob.cu)], np.zeros(B, int))
    x0, state = inst["x0"], None
    for cold in (True, False):
        shared, s0 = IC.device(s, x0, inst["Xref"], inst["Uref"], state, cold, WANT)
        got, s1 = IC.device(s, x0, inst["Xref"], inst["Uref"], state, cold, WANT, cones=cones)
        IC.same_plan(s0, s1, _table(dt))
        IC.two_per_group(s1)
        H.assert_bits_per_instance(got, shared, list(shared), f"cold={cold}")
        x0, state = IC.warm_inputs(inst["x0"], shared, seed=2, want=WANT)
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
    cones = IC.batch_cones(pal, IC.deal(B, 7, stride=3), sides=_sides(st))
    plan0 = IC.shared_plan(s, inst, WANT)
    off = {"x": ("zcnew", "yc"), "u": ("vcnew", "gc"), "xu": ()}[sides]  # a side whose loop does not run: fields left unwritten
    _, _, stt = IC.cold_warm(s, inst, f"rocket fleet {sides}", tuple(n for n in WANT if n not in off), cones=cones)
    IC.same_plan(plan0, stt, _table(dt))
    IC.two_per_group(stt)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. more than 2.5 waves of slot refills in one launch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt,warps", [(np.float64, None), (np.float32, "1"), (np.float64, "1")])
def test_multiwave(dt, warps, monkeypatch):
    if warps:
        monkeypatch.setenv("TINYMPC_GPS_WARPS", warps)
    prob, st = _rocket(dt, 20, max_iter=25)
    s = BatchedTinySolver(prob, st)
    B = int(2.6 * IC.capacity(s, lambda B: dict(cones=IC.batch_cones([dict(x_mu=prob.cx, u_mu=prob.cu)], np.zeros(B, int))))) + 37
    K = 5
    pal = IC.mu_palette(prob, K, seed=20, scale=(0.4, 1.0))
    o1, _, _ = IC.cold_warm(s, _rocket_instances(B, 20, dt, seed=21), "multiwave", WANT, mult=2.5,
                            cones=IC.batch_cones(pal, IC.deal(B, K)))
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
    pal = IC.mu_palette(prob, 6, seed=6)
    kw = dict(cones=IC.batch_cones(pal, IC.deal(B, 6)))
    if "models" in combo:
        kw.update(models=_rocket_models(dt), model_of=(np.arange(B) * 3) % 4)
    if "bounds" in combo:
        kw.update(bounds=IC.batch_bounds(IC.thrust_palette(prob, 5, int(combo[-1]), seed=7), IC.deal(B, 5, stride=3)))
    _, _, stt = IC.cold_warm(s, inst, f"cones + {combo}", WANT, **kw)
    IC.one_per_group(stt)
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
    st = IC.settings(spec, max_iter=40, abs_pri_tol=1e-2, abs_dua_tol=1e-2)
    s = BatchedTinySolver(prob, st)
    rng = np.random.default_rng(3)
    B, N = 500, spec.N
    inst = dict(x0=(0.3 * rng.standard_normal((B, 12))).astype(dt), Xref=(0.05 * rng.standard_normal((B, N, 12))).astype(dt),
                Uref=(0.02 * rng.standard_normal((B, N - 1, 4))).astype(dt))
    inst["Xref"][:, :, 2] += 0.5  # the state cone's axis: altitude
    pal = IC.mu_palette(prob, 4, seed=8, scale=(0.3, 1.5))
    plan0 = IC.shared_plan(s, inst, WANT)
    _, _, stt = IC.cold_warm(s, inst, f"cones + hyperplanes tv={tv}", WANT, cones=IC.batch_cones(pal, IC.deal(B, 4, stride=3)))
    IC.same_plan(plan0, stt, _table(dt))
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. every compiled (nx, nu) the streamed kernel covers; input cones where nu >= 3
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("nx,nu", IC.DIMS)
def test_every_shape(nx, nu, dt):
    spec = wl.random_lti(nx, nu, 30, seed=200 + nx * 10 + nu)
    cons = dict(Acx=[0, nx - 3], qcx=[3, 3], cx=[0.7, 1.3])
    spec.settings.en_state_soc = 1
    if nu >= 3:
        cons.update(Acu=[0], qcu=[3], cu=[0.9])
        spec.settings.en_input_soc = 1
    spec.constraints = dict(spec.constraints, **cons)
    prob = setup_problem(spec, dt)
    st = IC.settings(spec, max_iter=30)
    s = BatchedTinySolver(prob, st)
    B = 300
    rng = np.random.default_rng(nx * nu)
    inst = dict(x0=(0.5 * rng.standard_normal((B, nx))).astype(dt), Xref=(0.1 * rng.standard_normal((B, 30, nx))).astype(dt))
    inst["x0"][:, 2] += 0.3
    _, sh = IC.device(s, inst["x0"], inst["Xref"], None, None, True, WANT)
    if sh["kernel_family"] != abi.KERNEL_GPS:
        pal = IC.mu_palette(prob, 3, seed=nx + nu)
        with pytest.raises(TinyMPCError) as e:
            IC.device(s, inst["x0"], inst["Xref"], None, None, True, WANT, cones=IC.batch_cones(pal, IC.deal(B, 3, stride=2), _sides(st)))
        assert e.value.code == abi.ERR_UNSUPPORTED
        pytest.skip(f"({nx},{nu}) is not covered by the streamed kernel in this precision")
    pal = IC.mu_palette(prob, 3, seed=nx + nu, scale=(0.3, 1.2))
    want = WANT if nu >= 3 else tuple(n for n in WANT if n not in ("zcnew", "yc"))  # no input cones: their fields stay unwritten
    _, _, stt = IC.cold_warm(s, inst, f"({nx},{nu})", want, cones=IC.batch_cones(pal, IC.deal(B, 3, stride=2), _sides(st)))
    IC.same_plan(sh, stt, _table(dt))
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. the host path in 11 chunks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pin", [False, True])
@pytest.mark.parametrize("dt,with_models", [(np.float32, False), (np.float64, False), (np.float64, True)])
def test_host_path_chunks(dt, with_models, pin, monkeypatch):
    prob, st = _rocket(dt, 20)
    s = BatchedTinySolver(prob, st)
    B = IC.HOST_B
    cones = IC.batch_cones(IC.mu_palette(prob, 7, seed=30), IC.deal(B, 7, stride=3))
    models = _rocket_models(dt) if with_models else None
    model_of = None if models is None else np.arange(B) % 4
    IC.host_path_chunks(s, _rocket_instances(B, 20, dt, seed=31), WANT, pin, monkeypatch, models=models, model_of=model_of, cones=cones)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 8. the device closed loop: four steps, one with tighter cones
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
def test_closed_loop(dt):
    prob, st = _rocket(dt, 30)
    s = BatchedTinySolver(prob, st)
    B = 400
    inst = _rocket_instances(B, 30, dt, seed=42)
    pal = IC.mu_palette(prob, 4, seed=40)
    pal2 = IC.mu_palette(prob, 4, seed=41, scale=(0.3, 0.6))
    which = IC.deal(B, 4, stride=3)
    IC.closed_loop(s, inst, "cones", IC.batch_cones(pal, which), IC.batch_cones(pal2, which), 4,
                   extra_state=("x", "u", "vcnew", "zcnew", "gc", "yc"))
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 9. queued solves with different mu on one handle
# ---------------------------------------------------------------------------------------------------------------------
def test_queued_solves_different_mu():
    dt = np.float64
    prob, st = _rocket(dt, 50)
    s = BatchedTinySolver(prob, st)
    B = 3000
    inst = _rocket_instances(B, 50, dt, seed=50)
    pals = [IC.mu_palette(prob, 5, seed=51), IC.mu_palette(prob, 5, seed=52, scale=(0.3, 0.7))]
    IC.queued_solves(s, inst, WANT, "cones", [IC.batch_cones(p, IC.deal(B, 5)) for p in pals])
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
    cones = IC.batch_cones(IC.mu_palette(prob, 3, seed=61), IC.deal(B, 3, stride=2))
    want = tuple(H.BOX_STATE)
    for c in (cones, {"x_mu": cones["x_mu"]}):
        shared, s0 = IC.device(s, inst["x0"], inst["Xref"], inst["Uref"], None, True, want)
        got, s1 = IC.device(s, inst["x0"], inst["Xref"], inst["Uref"], None, True, want, cones=c)
        IC.same_plan(s0, s1)
        H.assert_bits_per_instance(got, shared, list(shared), "cone loops off")
    # a box-only problem without any cones: no pointer is needed either
    batch, _ = s.make_device_batch(inst["x0"], inst["Xref"], inst["Uref"], cold_start=True)
    batch.cones_per_instance = 1
    assert s._lib.tinympc_b200_solve(s._h, C.byref(batch), None) == abi.OK
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 11. loud errors
# ---------------------------------------------------------------------------------------------------------------------
def test_errors():
    dt = np.float64
    prob, st = _rocket(dt, 20)
    s = BatchedTinySolver(prob, st)
    B = 64
    inst = _rocket_instances(B, 20, dt, seed=70)
    cones = IC.batch_cones(IC.mu_palette(prob, 2, seed=71), IC.deal(B, 2, stride=1))
    batch, _ = s.make_device_batch(inst["x0"], inst["Xref"], inst["Uref"], cold_start=True, cones=cones)
    assert IC.solve_rc(s, batch) == abi.OK
    # a missing pointer for a side whose loop runs; a bad mode; reserved3
    for field, val in (("cone_x_mu", None), ("cone_u_mu", None), ("cones_per_instance", 2), ("cones_per_instance", -1), ("reserved3", 1)):
        b = abi.Batch.from_buffer_copy(batch)
        setattr(b, field, val)
        assert IC.solve_rc(s, b) == abi.ERR_ARG, field
    # the missing side's loop switched off: its pointer is never needed
    b = abi.Batch.from_buffer_copy(batch)
    b.cone_u_mu = None
    s.update_settings(en_input_soc=0)
    assert IC.solve_rc(s, b) == abi.OK
    s.update_settings(en_input_soc=1)
    IC.assert_refused(s, batch, inst["Xref"], b"cone")
    # Python checks: shapes, dtype, keys
    IC.assert_python_rejects(s, inst, "cones", [
        dict(cones, x_mu=cones["x_mu"][:, :0]), dict(cones, u_mu=cones["u_mu"][:-1]), dict(cones, x_mu=cones["x_mu"].astype(np.float32)),
        dict(cones, x_mu=cones["x_mu"][:, :, None]), dict(cones, mu=cones["x_mu"]), {}])
    s.close()
