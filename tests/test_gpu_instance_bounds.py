"""Per-instance box bounds (tinympc_batch_t.bounds_per_instance) on the on-chip (GPI) and streamed (GPS) lane-group kernels,
through the device entry point, the host path, the Python layer and the device closed loop.

Every instance is compared bit for bit, on every output and requested state field, with the oracle run once per bound set over
the instances that use it (instance_common.grouped_oracle), NaN-poisoned as instance_common describes.  The bound sets are
dealt with a stride, so neighbouring slots and the refills of a slot change bounds.  The launch plan is asserted through
stats()."""
import numpy as np
import pytest

import helpers as H
import instance_common as IC
from tinympc_b200 import abi, workloads as wl
from tinympc_b200._lib import TinyMPCError
from tinympc_b200.solver import BatchedTinySolver, setup_models, setup_problem

pytestmark = pytest.mark.gpu

WANT = tuple(H.BOX_STATE)
DTS = [np.float32, np.float64]


# ---------------------------------------------------------------------------------------------------------------------
# problems and instances
# ---------------------------------------------------------------------------------------------------------------------
def _quad(N, dt, max_iter=15):
    """Quadrotor tracking; with x0 jittered by 0.5 and max_iter = 15 instances converge after 7..15 iterations or stop at
    max_iter, so the slots of a warp retire at different times."""
    spec = wl.quadrotor(N=N)
    return setup_problem(spec, dt), IC.settings(spec, max_iter=max_iter)


def _tracking(B, N, dt, seed):
    inst = wl.tracking_instances(B, N=N, seed=seed, dtype=dt, jitter=0.5)
    inst["Uref"] = (0.05 * np.random.default_rng(seed + 1).standard_normal((B, N - 1, 4))).astype(dt)
    return inst


def _rocket(dt, N):
    spec = wl.rocket(N=N)
    return setup_problem(spec, dt), IC.settings(spec, max_iter=40, abs_pri_tol=0.1, abs_dua_tol=0.1)


def _rocket_instances(B, N, dt, seed):
    return wl.rocket_instances(B, N=N, seed=seed, dtype=dt, spread=0.3, per_instance_refs=True)


def _cold_warm(solver, inst, pal, which, family, what, **kw):
    return IC.cold_warm(solver, inst, what, WANT, family, bounds=IC.batch_bounds(pal, which), **kw)


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
    bounds = IC.batch_bounds(IC.equal_palette(prob, layout), np.zeros(300, int))
    x0, state = inst["x0"], None
    for cold in (True, False):
        shared, s0 = IC.device(s, x0, inst["Xref"], inst["Uref"], state, cold, WANT)
        got, s1 = IC.device(s, x0, inst["Xref"], inst["Uref"], state, cold, WANT, bounds=bounds)
        assert s0["kernel_family"] == s1["kernel_family"] == kernel, (s0, s1)
        H.assert_bits_per_instance(got, shared, list(shared), f"layout {layout} cold={cold}")
        o = IC.grouped_oracle(prob, st, bounds=bounds, nthreads=IC.NT)(x0, inst["Xref"], inst["Uref"], state, cold, WANT)
        IC.check(got, o, WANT, f"layout {layout} cold={cold} vs oracle")
        x0, state = IC.warm_inputs(inst["x0"], shared, seed=2, want=WANT)
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
    pal = IC.palette(prob, K, layout, seed=10 + layout, scale=1.0, tight=0.7)
    models = _quad_fleet(dt) if with_models else None
    cap = IC.capacity(s, lambda B: dict(bounds=IC.batch_bounds(pal, IC.deal(B, K))), models, per_sm=64)
    B = int(2.6 * cap) + 37
    which = IC.deal(B, K)
    model_of = None if models is None else (np.arange(B) * 3) % len(models)
    inst = _tracking(B, 50, dt, seed=20 + layout)
    o1, _, _ = _cold_warm(s, inst, pal, which, abi.KERNEL_GPI, f"fleet layout {layout}", models=models, model_of=model_of, mult=2.5)
    H.assert_mixed_termination(o1)
    if layout == 2:  # the horizons really vary over k and between sets
        assert not np.array_equal(pal[0]["u_max"][0], pal[0]["u_max"][5]) and not np.array_equal(pal[0]["u_max"], pal[1]["u_max"])
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. every compiled (nx, nu) with an on-chip plan at N = 50
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("nx,nu", IC.DIMS)
def test_every_shape_on_chip(nx, nu, dt):
    spec = wl.random_lti(nx, nu, 50, seed=100 + nx * 10 + nu)
    prob = setup_problem(spec, dt)
    st = IC.settings(spec, max_iter=30)
    s = BatchedTinySolver(prob, st, kernel=abi.KERNEL_GPI)
    pal = IC.palette(prob, 3, 1 + (nx + nu) % 2, seed=nx + nu, scale=0.3, tight=0.5)
    which = IC.deal(160, 3, stride=2)
    rng = np.random.default_rng(nx * nu)
    inst = dict(x0=(0.5 * rng.standard_normal((160, nx))).astype(dt), Xref=(0.1 * rng.standard_normal((160, 50, nx))).astype(dt))
    _, stt = IC.device(s, inst["x0"], inst["Xref"], None, None, True, WANT, bounds=IC.batch_bounds(pal, which))
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
    pal = IC.thrust_palette(prob, 6, layout, seed=N + layout)
    _cold_warm(s, _rocket_instances(700, N, dt, seed=N), pal, IC.deal(700, 6), abi.KERNEL_GPS, f"rocket N={N} layout {layout}")
    IC.one_per_group(s.stats())
    s.close()


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("tv", [False, True])
def test_hyperplanes(tv, dt):
    spec = H.quad_linear_spec(tv=tv)
    spec.settings.en_state_bound = 1
    spec.settings.en_input_bound = 1
    prob = setup_problem(spec, dt)
    st = IC.settings(spec, max_iter=40, abs_pri_tol=1e-2, abs_dua_tol=1e-2)
    s = BatchedTinySolver(prob, st)
    pal = IC.palette(prob, 4, 2 if tv else 1, seed=7, scale=0.2, tight=0.6)
    rng = np.random.default_rng(3)
    B, N = 500, spec.N
    inst = dict(x0=(0.3 * rng.standard_normal((B, 12))).astype(dt), Xref=(0.05 * rng.standard_normal((B, N, 12))).astype(dt),
                Uref=(0.02 * rng.standard_normal((B, N - 1, 4))).astype(dt))
    _cold_warm(s, inst, pal, IC.deal(B, 4, stride=3), abi.KERNEL_GPS, f"hyperplanes tv={tv}")
    IC.one_per_group(s.stats())
    s.close()


@pytest.mark.parametrize("layout", [1, 2])
def test_box_horizon_off_chip(layout):
    """Quadrotor fp64, N = 1000: no on-chip plan, so the batch streams"""
    dt = np.float64
    prob, st = _quad(1000, dt, max_iter=30)
    s = BatchedTinySolver(prob, st)
    pal = IC.palette(prob, 3, layout, seed=5, scale=0.5, tight=0.5)
    inst = wl.hovering_instances(64, N=1000, dtype=dt)
    inst["x0"] = (inst["x0"] + 0.2 * np.random.default_rng(3).standard_normal(inst["x0"].shape)).astype(dt)
    _cold_warm(s, inst, pal, IC.deal(64, 3, stride=2), abi.KERNEL_GPS, "N=1000")
    s.close()


@pytest.mark.parametrize("dt", DTS)
def test_explicit_gps_box_with_models(dt):
    prob, st = _quad(50, dt)
    s = BatchedTinySolver(prob, st, kernel=abi.KERNEL_GPS)
    pal = IC.palette(prob, 5, 2, seed=8, scale=0.8, tight=0.6)
    inst = _tracking(600, 50, dt, seed=9)
    which = IC.deal(600, 5)
    _cold_warm(s, inst, pal, which, abi.KERNEL_GPS, "explicit GPS")
    IC.one_per_group(s.stats())
    models = _quad_fleet(dt)
    _cold_warm(s, inst, pal, which, abi.KERNEL_GPS, "explicit GPS + models", models=models, model_of=np.arange(600) % 4)
    s.close()


@pytest.mark.parametrize("dt", DTS)
def test_streamed_multiwave_one_warp(dt, monkeypatch):
    """TINYMPC_GPS_WARPS=1: one warp per SM, > 2.5 waves plus a ragged remainder in one launch"""
    monkeypatch.setenv("TINYMPC_GPS_WARPS", "1")
    prob, st = _rocket(dt, 20)
    s = BatchedTinySolver(prob, st)
    pal = IC.thrust_palette(prob, 5, 1, seed=12)
    cap = IC.capacity(s, lambda B: dict(bounds=IC.batch_bounds(pal, IC.deal(B, 5))), per_sm=64)
    B = int(2.6 * cap) + 5
    _cold_warm(s, _rocket_instances(B, 20, dt, seed=13), pal, IC.deal(B, 5), abi.KERNEL_GPS, "GPS 1 warp", mult=2.5)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. signed zeros: the shared fp32 solve of this problem clamps with min / max; per-instance bounds at +-0 must not
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", [1, 2])
def test_signed_zero_bounds(layout):
    dt = np.float32
    prob, st = _quad(50, dt)
    s = BatchedTinySolver(prob, st)
    pal = IC.palette(prob, 3, layout, seed=6, scale=0.3, zeros=True)
    assert any(np.signbit(d["u_min"]).any() and (d["u_min"] == 0).any() for d in pal)
    o1, _, _ = _cold_warm(s, _tracking(400, 50, dt, seed=6), pal, IC.deal(400, 3, stride=2), abi.KERNEL_GPI, "+-0 bounds")
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
    pal = IC.palette(prob, 7, layout, seed=30, scale=0.7, tight=0.6)
    bounds = IC.batch_bounds(pal, IC.deal(IC.HOST_B, 7, stride=3))
    IC.host_path_chunks(s, _tracking(IC.HOST_B, 50, dt, seed=31), WANT, pin, monkeypatch, bounds=bounds)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. the device closed loop: five steps, the reference window moving, one step in a moving corridor
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_models", [False, True])
def test_closed_loop(with_models):
    dt = np.float32
    prob, st = _quad(50, dt)
    s = BatchedTinySolver(prob, st)
    B = 300
    pal = IC.palette(prob, 4, 1, seed=40, scale=0.6, tight=0.5)
    pal2 = IC.palette(prob, 4, 2, seed=41, scale=0.4, tight=0.5)
    which = IC.deal(B, 4, stride=3)
    models = _quad_fleet(dt) if with_models else None
    model_of = None if models is None else np.arange(B) % 4
    inst = _tracking(B, 50, dt, seed=42)
    IC.closed_loop(s, dict(x0=inst["x0"], Xref=inst["Xref"]), "bounds", IC.batch_bounds(pal, which), IC.batch_bounds(pal2, which),
                   5, want=WANT, roll=True, models=models, model_of=model_of)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 8. queued solves with different bound arrays
# ---------------------------------------------------------------------------------------------------------------------
def test_queued_solves_different_bounds():
    dt = np.float32
    prob, st = _quad(50, dt)
    s = BatchedTinySolver(prob, st)
    B = 3000
    inst = _tracking(B, 50, dt, seed=50)
    pals = [IC.palette(prob, 5, 1, seed=51, scale=0.7, tight=0.6), IC.palette(prob, 5, 2, seed=52, scale=0.5, tight=0.6)]
    IC.queued_solves(s, inst, WANT, "bounds", [IC.batch_bounds(p, IC.deal(B, 5)) for p in pals])
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 9. loud errors
# ---------------------------------------------------------------------------------------------------------------------
def test_errors():
    dt = np.float32
    prob, st = _quad(50, dt)
    s = BatchedTinySolver(prob, st)
    B = 64
    inst = _tracking(B, 50, dt, seed=60)
    pal = IC.palette(prob, 2, 1, seed=61, scale=0.5)
    bounds = IC.batch_bounds(pal, IC.deal(B, 2, stride=1))
    batch, _ = s.make_device_batch(inst["x0"], inst["Xref"], cold_start=True, bounds=bounds)
    assert IC.solve_rc(s, batch) == abi.OK
    IC.assert_refused(s, batch, inst["Xref"], b"adaptive")
    # bad mode, half pair, reserved2
    for field, val in (("bounds_per_instance", 3), ("bounds_per_instance", -1), ("reserved2", 1), ("x_max", None), ("u_min", None)):
        b = abi.Batch.from_buffer_copy(batch)
        setattr(b, field, val)
        assert IC.solve_rc(s, b) == abi.ERR_ARG, field
    # an enabled side without its pair; a disabled side's pair is never needed
    b = abi.Batch.from_buffer_copy(batch)
    b.x_min = b.x_max = None
    assert IC.solve_rc(s, b) == abi.ERR_NO_BOUNDS
    s.update_settings(en_state_bound=0)
    assert IC.solve_rc(s, b) == abi.OK
    s.update_settings(en_state_bound=1)
    # Python checks: shapes, dtype, pairs, mixed layouts
    IC.assert_python_rejects(s, inst, "bounds", [
        dict(bounds, x_min=bounds["x_min"][:, :5]), dict(bounds, x_min=bounds["x_min"].astype(np.float64)), {"x_min": bounds["x_min"]},
        dict(bounds, u_min=np.stack([pal[0]["u_min"]] * B)[:, None, :].repeat(49, 1)), dict(bounds, q=bounds["x_min"]), {}])
    s.close()
    # a handle created without bounds, solved with per-instance bounds
    kw = {k: getattr(prob, k) for k in prob.__dataclass_fields__}
    kw.update(x_min=None, x_max=None, u_min=None, u_max=None)
    bare = BatchedTinySolver(type(prob)(**kw), st)
    with pytest.raises(TinyMPCError) as e:
        bare.solve(inst["x0"], inst["Xref"])
    assert e.value.code == abi.ERR_NO_BOUNDS
    got = bare.solve(inst["x0"], inst["Xref"], bounds=bounds)
    o = IC.grouped_oracle(prob, st, bounds=bounds, nthreads=IC.NT)(inst["x0"], inst["Xref"], None, None, True, ())
    H.assert_bits_per_instance(got, o, H.OUT_KEYS, "handle without bounds")
    bare.close()
