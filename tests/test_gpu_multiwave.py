"""Multi-wave parity: the paths a batch takes once it no longer fits in one wave, against the oracle on EVERY instance.

  * GPI / GPS are persistent kernels: a lane group that finishes an instance writes it back and takes the next ticket from
    a global queue, so a batch larger than the resident capacity (ctas x instances_per_cta) reloads slots that held another
    instance a moment ago (state zeroed or warm-loaded, v-scratch staged, per-instance model rows re-read, counters reset).
  * tinympc_b200_solve_host cuts a batch into chunks over three pipeline slots and DMAs straight to / from page-locked
    caller buffers.

Every test sizes its batch from the launch plan (a one-iteration probe solve), asserts that the batch really spans
several waves in ONE launch (or the expected number of chunks), that instances of a warp retire at different iterations
(>= 5 distinct iteration counts, converged and max_iter-capped ones), and compares every scalar: the outputs, every
requested state field and u0.  Before each solve the outputs are filled with a NaN bit pattern (H.poison), on cold starts
the requested state arrays too, so an element a solve never writes cannot pass by matching an oracle zero.
"""
import functools
import os

import numpy as np
import pytest

import helpers as H
from oracle import oracle
from tinympc_b200 import abi, workloads as wl
from tinympc_b200.batch import HostBatch
from tinympc_b200.problem import MPCProblem
from tinympc_b200.solver import BatchedTinySolver, setup_models, setup_problem, unpack_model

pytestmark = pytest.mark.gpu

NT = os.cpu_count() or 1
OUTS = ("sol_x", "sol_u", "iter", "solved", "residuals", "u0")


# ---------------------------------------------------------------------------------------------------------------------
# problems and instances
# ---------------------------------------------------------------------------------------------------------------------
def _settings(spec, **kw):
    st = abi.Settings.from_buffer_copy(spec.settings)
    for k, v in kw.items():
        setattr(st, k, v)
    return st


def _quad(N, dt, max_iter=15, check=1):
    """Quadrotor tracking: with x0 jittered by 0.5 and max_iter = 15 the instances converge after 7..15 iterations or
    stop at max_iter, so the slots of one warp retire at different times."""
    spec = wl.quadrotor(N=N)
    return setup_problem(spec, dt), _settings(spec, max_iter=max_iter, check_termination=check)


def _tracking(B, N, dt, seed):
    inst = wl.tracking_instances(B, N=N, seed=seed, dtype=dt, jitter=0.5)
    inst["Uref"] = (0.05 * np.random.default_rng(seed + 1).standard_normal((B, N - 1, 4))).astype(dt)
    return inst


def _rocket(dt, N=20):
    """Rocket landing with cones; tolerances loosened (0.1) so that part of the batch converges before max_iter."""
    spec = wl.rocket(N=N)
    return setup_problem(spec, dt), _settings(spec, max_iter=40, abs_pri_tol=0.1, abs_dua_tol=0.1)


def _rocket_instances(B, N, dt, seed):
    return wl.rocket_instances(B, N=N, seed=seed, dtype=dt, spread=0.3, per_instance_refs=True)


def _hyperplanes(tv, dt):
    spec = H.quad_linear_spec(tv=tv)
    return setup_problem(spec, dt), _settings(spec, max_iter=40, abs_pri_tol=1e-2, abs_dua_tol=1e-2)


def _hyperplane_instances(B, N, dt, seed):
    rng = np.random.default_rng(seed)
    return dict(x0=(0.3 * rng.standard_normal((B, 12))).astype(dt), Xref=(0.05 * rng.standard_normal((B, N, 12))).astype(dt),
                Uref=(0.02 * rng.standard_normal((B, N - 1, 4))).astype(dt))


def _warm_inputs(x0, res, want, seed):
    """Next MPC step: perturbed measurements, the returned state, duals reset on every third instance
    (examples/quadrotor_tracking.cpp:92-93 resets them on every instance)."""
    rng = np.random.default_rng(seed)
    x0b = (x0 + 0.02 * rng.standard_normal(x0.shape)).astype(x0.dtype)
    state = {n: np.array(res[n], copy=True) for n in want}
    for n in ("g", "y"):
        state[n][::3] = 0
    return x0b, state


# ---------------------------------------------------------------------------------------------------------------------
# oracle
# ---------------------------------------------------------------------------------------------------------------------
def _port(prob, st):
    def run(x0, Xref, Uref, state, cold, want):
        state = None if state is None else {n: np.array(a, copy=True) for n, a in state.items()}
        return oracle.solve_batch(prob, st, x0, Xref, Uref, state=state, cold_start=cold, want_state=tuple(want), impl="port",
                                  nthreads=NT)
    return run


def _port_grouped(probs, model, st):
    """Heterogeneous batch: one oracle run per model over the instances that use it."""
    def run(x0, Xref, Uref, state, cold, want):
        out = {}
        for m in np.unique(model):
            idx = np.flatnonzero(model == m)
            sub = None if state is None else {n: a[idx] for n, a in state.items()}
            o = oracle.solve_batch(probs[m], st, x0[idx], Xref[idx], Uref[idx], state=sub, cold_start=cold,
                                   want_state=tuple(want), impl="port", nthreads=NT)
            for k, v in o.items():
                if v is not None:
                    out.setdefault(k, np.empty((len(x0),) + v.shape[1:], v.dtype))[idx] = v
        return out
    return run


def _expect(o, want):
    ref = {k: o[k] for k in H.OUT_KEYS + list(want)}
    ref["u0"] = np.ascontiguousarray(o["u"][:, 0, :])  # work->u.col(0)
    return ref


def _check(got, o, want, what):
    H.assert_bits_per_instance(got, _expect(o, want), H.OUT_KEYS + list(want) + ["u0"], what)


# ---------------------------------------------------------------------------------------------------------------------
# the two solve paths, with poisoned outputs
# ---------------------------------------------------------------------------------------------------------------------
def _device_solve(solver, x0, Xref, Uref, state, cold, want, models=None):
    """tinympc_b200_solve on tensors from make_device_batch -> (numpy results, stats)."""
    import torch

    batch, out = solver.make_device_batch(x0, Xref, Uref, state=state, cold_start=cold, want_state=tuple(want), want_u0=True,
                                          models=models)
    for k in OUTS:
        H.poison(out[k])
    if cold:  # cold_start ignores the state on input and writes every requested field
        for n in want:
            H.poison(out[n])
    solver.solve_device(batch)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items() if v is not None}, solver.stats()


def _pin(hb, mode):
    """Move the buffers of a HostBatch to page-locked memory: "all"; "in" = x0 / references / models and every other state
    field; "out" = the outputs and the remaining state fields (so that pinned and pageable outputs interleave)."""
    import torch

    keep = []

    def pinned(a):
        t = torch.empty(a.nbytes, dtype=torch.uint8, pin_memory=True)
        keep.append(t)
        p = t.numpy().view(a.dtype).reshape(a.shape)
        p[...] = a
        return p

    ins = [n for n in ("x0", "Xref", "Uref", "models") if getattr(hb, n) is not None]
    outs = [n for n in OUTS if getattr(hb, n) is not None]
    for n in (ins if mode in ("all", "in") else []) + (outs if mode in ("all", "out") else []):
        setattr(hb, n, pinned(getattr(hb, n)))
    for i, n in enumerate(abi.STATE_FIELDS):
        if n in hb.state and (mode == "all" or (mode == "in") == (i % 2 == 0)):
            hb.state[n] = pinned(hb.state[n])
    hb._pinned = keep


def _host_solve(solver, x0, Xref, Uref, state, cold, want, models=None, pin=None):
    """tinympc_b200_solve_host on a HostBatch (u0 requested too) -> (numpy results, stats)."""
    p = solver.problem
    state = None if state is None else {n: np.array(a, copy=True) for n, a in state.items()}
    hb = HostBatch(p, x0, Xref, Uref, state=state, cold_start=cold, want_state=tuple(want), models=models)
    hb.u0 = np.empty((hb.B, p.nu), p.dtype)
    if pin:
        _pin(hb, pin)
    for k in OUTS:
        H.poison(getattr(hb, k))
    if cold:
        for n in want:
            H.poison(hb.state[n])
    cb = hb.to_c()
    cb.u0 = hb.u0.ctypes.data
    solver.solve_prepared(hb, cb)
    res = dict(hb.result(), u0=hb.u0)
    return {k: np.array(v, copy=True) for k, v in res.items() if v is not None}, solver.stats()


# ---------------------------------------------------------------------------------------------------------------------
# launch plan
# ---------------------------------------------------------------------------------------------------------------------
def _capacity(prob, st, kernel):
    """Instances one wave of the persistent kernel holds (ctas x instances_per_cta), read from a one-iteration probe solve
    large enough to fill every SM."""
    import torch

    sm = torch.cuda.get_device_properties(0).multi_processor_count
    st1 = abi.Settings.from_buffer_copy(st)
    st1.max_iter = 1
    s = BatchedTinySolver(prob, st1, kernel=kernel)
    B = 64 * sm
    batch, _ = s.make_device_batch(np.zeros((B, prob.nx), prob.dtype), np.zeros((prob.N, prob.nx), prob.dtype), cold_start=True)
    s.solve_device(batch)
    torch.cuda.synchronize()
    stt = s.stats()
    s.close()
    assert stt["ctas"] == sm, stt
    return stt["ctas"] * stt["instances_per_cta"]


def _assert_multiwave(stt, B, family, mult=2.5):
    """One launch of `family` served B instances, at least `mult` times what its slots hold at once: slots were refilled."""
    assert stt["kernel_family"] == family, stt
    assert stt["kernel_launches"] == 1, stt
    cap = stt["ctas"] * stt["instances_per_cta"]
    assert B >= mult * cap, (B, cap, stt)


def _cold_warm(solver, inst, want, family, what, port, models=None, mult=3.0):
    """Cold solve, then a warm-started step from the returned state, on the device path; every instance vs the oracle."""
    B = len(inst["x0"])
    o1 = port(inst["x0"], inst["Xref"], inst["Uref"], None, True, want)
    H.assert_mixed_termination(o1)
    g1, stt = _device_solve(solver, inst["x0"], inst["Xref"], inst["Uref"], None, True, want, models=models)
    _assert_multiwave(stt, B, family, mult)
    _check(g1, o1, want, what + " cold")
    x0b, state = _warm_inputs(inst["x0"], o1, want, seed=B)
    o2 = port(x0b, inst["Xref"], inst["Uref"], state, False, want)
    H.assert_mixed_termination(o2)
    g2, stt = _device_solve(solver, x0b, inst["Xref"], inst["Uref"], state, False, want, models=models)
    _assert_multiwave(stt, B, family, mult)
    _check(g2, o2, want, what + " warm")
    return stt


# ---------------------------------------------------------------------------------------------------------------------
# A. on-chip lane groups (GPI): slot refill
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt,N,check", [(np.float32, 50, 1), (np.float64, 20, 1), (np.float32, 50, 3)])
def test_gpi_refill_cold_then_warm(dt, N, check):
    """3 waves + a ragged remainder in one launch; BOX_STATE with v / z (staged through the v-scratch) and u0.
    check_termination = 3: residuals are refreshed only every third iteration, so a refilled slot must not report its
    previous instance's values (max_iter 20 leaves five iteration counts that occur: 9, 12, 15, 18, 20)."""
    prob, st = _quad(N, dt, max_iter=15 if check == 1 else 20, check=check)
    B = 3 * _capacity(prob, st, abi.KERNEL_GPI) + 37
    inst = _tracking(B, N, dt, seed=N + check)
    solver = BatchedTinySolver(prob, st, kernel=abi.KERNEL_GPI)
    stt = _cold_warm(solver, inst, H.BOX_STATE, abi.KERNEL_GPI, f"gpi N={N} {dt.__name__} check={check}", _port(prob, st))
    if dt == np.float32 and N == 50:
        assert (stt["lanes_per_instance"], stt["instances_per_cta"]) == (4, 32)


# ---------------------------------------------------------------------------------------------------------------------
# B. GPI with per-instance models: a refill brings a different model into a slot
# ---------------------------------------------------------------------------------------------------------------------
HET_M = 50


@functools.lru_cache(maxsize=None)
def _het_models(dt):
    nx, nu, N = 12, 4, 20
    specs = [wl.random_lti(nx, nu, N, seed=300 + i) for i in range(HET_M)]
    rhos = np.array([0.5 + 0.1 * (i % 9) for i in range(HET_M)])
    blobs = setup_models(nx, nu, np.stack([s.A for s in specs]), np.stack([s.B for s in specs]), np.stack([s.f for s in specs]),
                         np.stack([s.Qdiag for s in specs]), np.stack([s.Rdiag for s in specs]), rhos, dtype=dt)
    probs = []
    for i in range(HET_M):
        m = unpack_model(blobs[i], nx, nu)
        rho = m.pop("rho")
        probs.append(MPCProblem(nx=nx, nu=nu, N=N, dtype=dt, rho=rho, **m, **specs[0].constraints))
    return specs, blobs, probs


def _het_case(dt):
    specs, blobs, probs = _het_models(dt)
    st = _settings(specs[0], max_iter=40)
    B = 3 * _capacity(probs[0], st, abi.KERNEL_GPI) + 37
    model = (17 * np.arange(B)) % HET_M  # neighbouring tickets use different models
    rng = np.random.default_rng(9)
    inst = dict(x0=(2.0 * rng.standard_normal((B, 12))).astype(dt), Xref=(0.1 * rng.standard_normal((B, 20, 12))).astype(dt),
                Uref=(0.05 * rng.standard_normal((B, 19, 4))).astype(dt))
    return probs, st, inst, blobs[model], _port_grouped(probs, model, st)


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_gpi_heterogeneous_refill(dt):
    """(12,4,20): fp32 keeps a slot's matrix rows in registers, fp64 re-reads them from the slot's own blob every sweep;
    both must switch to the new instance's model on a refill."""
    probs, st, inst, models, port = _het_case(dt)
    solver = BatchedTinySolver(probs[0], st)
    _cold_warm(solver, inst, H.BOX_STATE, abi.KERNEL_GPI, f"het {dt.__name__}", port, models=models)


# ---------------------------------------------------------------------------------------------------------------------
# C. streamed lane groups (GPS) with one warp per SM: many waves for every feature family
# ---------------------------------------------------------------------------------------------------------------------
GPS_CASES = {
    "box_quad_N50_f32": (lambda: _quad(50, np.float32), lambda B, N, dt: _tracking(B, N, dt, seed=5), H.BOX_STATE),
    "soc_rocket_N20_f64": (lambda: _rocket(np.float64), lambda B, N, dt: _rocket_instances(B, N, dt, seed=6), H.SOC_STATE),
    "lin_quad_f32": (lambda: _hyperplanes(False, np.float32), lambda B, N, dt: _hyperplane_instances(B, N, dt, seed=7), H.LIN_STATE),
    "tvlin_quad_f64": (lambda: _hyperplanes(True, np.float64), lambda B, N, dt: _hyperplane_instances(B, N, dt, seed=8), H.TVLIN_STATE),
}


@pytest.mark.parametrize("case", list(GPS_CASES))
def test_gps_refill_cold_then_warm(case, monkeypatch):
    """TINYMPC_GPS_WARPS=1 caps the resident slots at one warp per SM; the box quadrotor runs two instances per lane group
    (NI = 2), whose service order refills the second instance of a group independently of the first.  Region B (previous
    slacks, family slacks) is in use because v / z and the family slacks are requested."""
    monkeypatch.setenv("TINYMPC_GPS_WARPS", "1")
    make, gen, want = GPS_CASES[case]
    prob, st = make()
    B = 3 * _capacity(prob, st, abi.KERNEL_GPS) + 37
    inst = gen(B, prob.N, prob.dtype)
    solver = BatchedTinySolver(prob, st, kernel=abi.KERNEL_GPS)
    stt = _cold_warm(solver, inst, want, abi.KERNEL_GPS, "gps " + case, _port(prob, st))
    assert stt["threads_per_cta"] == 32, stt
    if case.startswith("box"):
        assert stt["instances_per_cta"] == 2 * (32 // stt["lanes_per_instance"]), stt  # two instances per lane group


# ---------------------------------------------------------------------------------------------------------------------
# D. device-resident closed loop across waves
# ---------------------------------------------------------------------------------------------------------------------
def test_device_closed_loop_across_waves():
    """DeviceMPCLoop on AUTO (on-chip lane groups) with 2.5 waves of plants: warm starts with v / z (exact first residual)
    land in refilled slots at every step."""
    dt = np.float32
    prob, st = _quad(10, dt)
    B = int(np.ceil(2.5 * _capacity(prob, st, abi.KERNEL_AUTO))) + 37
    inst = wl.tracking_instances(B, N=10, seed=13, dtype=dt, jitter=0.5)
    solver = BatchedTinySolver(prob, st)
    port = _port(prob, st)
    outs = H.device_closed_loop_vs_oracle(solver, inst, 3, lambda p, s, *a: port(*a))
    for o in outs:
        H.assert_mixed_termination(o)
    _assert_multiwave(solver.stats(), B, abi.KERNEL_GPI)


# ---------------------------------------------------------------------------------------------------------------------
# E. host path: chunks over three pipeline slots, page-locked caller buffers
# ---------------------------------------------------------------------------------------------------------------------
HOST_KERNELS = {"tpi": abi.KERNEL_TPI, "gpi": abi.KERNEL_GPI, "gps": abi.KERNEL_GPS}


@functools.lru_cache(maxsize=None)
def _host_case():
    """1000 distinct tracking instances (N = 50, fp32): oracle cold step and warm step."""
    prob, st = _quad(50, np.float32)
    inst = _tracking(1000, 50, np.float32, seed=17)
    port = _port(prob, st)
    want = H.BOX_STATE
    o1 = port(inst["x0"], inst["Xref"], inst["Uref"], None, True, want)
    x0b, state = _warm_inputs(inst["x0"], o1, want, seed=18)
    o2 = port(x0b, inst["Xref"], inst["Uref"], state, False, want)
    return prob, st, inst, o1, x0b, state, o2


@pytest.mark.parametrize("pin", [None, "all", "in", "out"])
@pytest.mark.parametrize("kernel", list(HOST_KERNELS))
def test_host_path_chunks_and_pinned_buffers(kernel, pin, monkeypatch):
    """TINYMPC_HOST_CHUNK=96 cuts B = 1000 into 11 chunks (every pipeline slot reused three times or more); cold + warm with
    all state in / out and u0, bit-equal to the oracle and to the device path.  pin: page-locked caller buffers (DMA straight
    to / from them) — all of them, or only the inputs / only the outputs, with the in / out state fields split between the two."""
    monkeypatch.setenv("TINYMPC_HOST_CHUNK", "96")
    prob, st, inst, o1, x0b, state, o2 = _host_case()
    want = H.BOX_STATE
    for o in (o1, o2):
        H.assert_mixed_termination(o)
    solver = BatchedTinySolver(prob, st, kernel=HOST_KERNELS[kernel])
    what = f"host {kernel} pin={pin}"
    for step, (x0, stt_in, o) in enumerate(((inst["x0"], None, o1), (x0b, state, o2))):
        cold = stt_in is None
        h, stt = _host_solve(solver, x0, inst["Xref"], inst["Uref"], stt_in, cold, want, pin=pin)
        assert stt["kernel_launches"] == 11, stt
        _check(h, o, want, f"{what} step {step}")
        d, _ = _device_solve(solver, x0, inst["Xref"], inst["Uref"], stt_in, cold, want)
        H.assert_bits_per_instance(h, d, H.OUT_KEYS + want + ["u0"], f"{what} step {step}: host vs device path")


def test_host_path_default_chunking_gpi(monkeypatch):
    """B = 20 037 on the on-chip kernel: the host path's default chunking (B > 16 384), rounded to whole waves; cold + warm,
    every instance against the oracle."""
    monkeypatch.delenv("TINYMPC_HOST_CHUNK", raising=False)
    dt = np.float32
    prob, st = _quad(50, dt)
    wave = _capacity(prob, st, abi.KERNEL_GPI)
    B = 20037
    # the chunk rule of tinympc_b200_solve_host (csrc/capi.cu, "chunking: big enough to fill the GPU ..."), restated: an eighth
    # of the batch but at least 8192, rounded up to 32, then to the nearest whole number of GPI waves
    chunk = (max(8192, (B + 7) // 8) + 31) // 32 * 32
    chunk = max(1, (chunk + wave // 2) // wave) * wave
    assert B > chunk > 0 and chunk % wave == 0
    nchunks = -(-B // chunk)
    inst = _tracking(B, 50, dt, seed=19)
    port = _port(prob, st)
    want = H.BOX_STATE
    solver = BatchedTinySolver(prob, st, kernel=abi.KERNEL_GPI)
    o1 = port(inst["x0"], inst["Xref"], inst["Uref"], None, True, want)
    H.assert_mixed_termination(o1)
    h1, stt = _host_solve(solver, inst["x0"], inst["Xref"], inst["Uref"], None, True, want)
    assert stt["kernel_family"] == abi.KERNEL_GPI, stt
    assert stt["kernel_launches"] == nchunks > 1, ("one launch per chunk of whole waves; has the chunk rule changed?", nchunks, stt)
    _check(h1, o1, want, "host default chunking cold")
    x0b, state = _warm_inputs(inst["x0"], o1, want, seed=20)
    o2 = port(x0b, inst["Xref"], inst["Uref"], state, False, want)
    H.assert_mixed_termination(o2)
    h2, stt = _host_solve(solver, x0b, inst["Xref"], inst["Uref"], state, False, want)
    assert stt["kernel_launches"] == nchunks, stt
    _check(h2, o2, want, "host default chunking warm")


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_host_path_heterogeneous_chunks(dt, monkeypatch):
    """The heterogeneous batch of test_gpi_heterogeneous_refill through the chunked host path: the models field is sliced per
    chunk like every other per-instance buffer; three chunks, each a little over one wave."""
    probs, st, inst, models, port = _het_case(dt)
    B = len(inst["x0"])
    chunk = ((B - 37) // 3 + 64 + 31) // 32 * 32  # a little over one wave, a multiple of 32 (the host path rounds up to 32)
    monkeypatch.setenv("TINYMPC_HOST_CHUNK", str(chunk))
    want = H.BOX_STATE
    solver = BatchedTinySolver(probs[0], st)
    o1 = port(inst["x0"], inst["Xref"], inst["Uref"], None, True, want)
    H.assert_mixed_termination(o1)
    h1, stt = _host_solve(solver, inst["x0"], inst["Xref"], inst["Uref"], None, True, want, models=models)
    assert stt["kernel_launches"] == -(-B // chunk) == 3 and stt["kernel_family"] == abi.KERNEL_GPI, stt
    _check(h1, o1, want, f"host het {dt.__name__} cold")
    x0b, state = _warm_inputs(inst["x0"], o1, want, seed=21)
    o2 = port(x0b, inst["Xref"], inst["Uref"], state, False, want)
    H.assert_mixed_termination(o2)
    h2, stt = _host_solve(solver, x0b, inst["Xref"], inst["Uref"], state, False, want, models=models)
    assert stt["kernel_launches"] == 3, stt
    _check(h2, o2, want, f"host het {dt.__name__} warm")


DISABLED_CASES = {  # (problem, instances, fields of the enabled families, kernels)
    "box_quad_N50_f32": (lambda: _quad(50, np.float32), lambda B, N, dt: _tracking(B, N, dt, seed=25), H.BOX_STATE, ["tpi", "gpi", "gps"]),
    "soc_rocket_N20_f64": (lambda: _rocket(np.float64), lambda B, N, dt: _rocket_instances(B, N, dt, seed=26), H.SOC_STATE, ["tpi", "gps"]),
}


@pytest.mark.parametrize("case,kernel", [(c, k) for c, v in DISABLED_CASES.items() for k in v[3]])
def test_disabled_family_state_fields_left_alone(case, kernel, monkeypatch):
    """include/tinympc_b200.h: the slack / dual fields of a constraint family the settings leave disabled are neither read nor
    written.  tinympc_b200_solve returns such buffers unchanged on cold and warm starts, tinympc_b200_solve_host on warm
    starts (its cold start leaves them unspecified); the enabled fields still equal the oracle."""
    monkeypatch.setenv("TINYMPC_HOST_CHUNK", "96")
    make, gen, want, _ = DISABLED_CASES[case]
    prob, st = make()
    B = 1000
    inst = gen(B, prob.N, prob.dtype)
    off = [n for n in abi.STATE_FIELDS if n not in want]
    every = list(want) + off

    def poisoned(n):
        return H.poison(np.empty((B, prob.N, prob.nx) if abi.STATE_IS_X[n] else (B, prob.N - 1, prob.nu), prob.dtype))

    port = _port(prob, st)
    solver = BatchedTinySolver(prob, st, kernel=HOST_KERNELS[kernel])
    o1 = port(inst["x0"], inst["Xref"], inst["Uref"], None, True, want)
    g1, _ = _device_solve(solver, inst["x0"], inst["Xref"], inst["Uref"], None, True, every)  # poisons every field first
    _check(g1, o1, want, f"{case} {kernel} device cold")
    H.assert_bits_per_instance(g1, {n: poisoned(n) for n in off}, off, f"{case} {kernel} device cold: disabled families")
    h1, _ = _host_solve(solver, inst["x0"], inst["Xref"], inst["Uref"], None, True, every)
    _check(h1, o1, want, f"{case} {kernel} host cold")
    x0b, state = _warm_inputs(inst["x0"], o1, want, seed=27)
    o2 = port(x0b, inst["Xref"], inst["Uref"], state, False, want)
    state_all = dict(state, **{n: poisoned(n) for n in off})
    for path, solve in (("device", _device_solve), ("host", _host_solve)):
        r, _ = solve(solver, x0b, inst["Xref"], inst["Uref"], state_all, False, every)
        _check(r, o2, want, f"{case} {kernel} {path} warm")
        H.assert_bits_per_instance(r, {n: poisoned(n) for n in off}, off, f"{case} {kernel} {path} warm: disabled families")

