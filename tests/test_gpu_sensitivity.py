"""Sensitivity tables on the H100 (tinympc_b200_precompute_sensitivity_batch_device) and per-instance tables in the adaptive
solve (tinympc_adaptive_rho_t.tables_per_instance): device tables bit for bit against the host routine, the adaptive solve bit
for bit against the C restatement's per-instance-table entry point (tests/adaptive/adaptive_oracle_per_instance.c)."""
import ctypes as C

import numpy as np
import pytest

import adaptive_common as AC
import helpers as H
import sensitivity_common as SC
from oracle import oracle
from tinympc_b200 import abi
from tinympc_b200 import workloads as wl
from tinympc_b200._lib import load
from tinympc_b200.batch import HostBatch
from tinympc_b200.solver import AdaptiveRho, BatchedTinySolver, pack_models, setup_models, setup_problem, setup_sensitivity

pytestmark = pytest.mark.gpu

KEYS = AC.OUT + AC.BOX
DIMS = [(4, 1), (6, 3), (12, 4), (4, 2), (4, 4), (4, 8), (8, 2), (8, 4), (8, 8), (12, 2), (12, 8), (16, 2), (16, 4), (16, 8)]


def _cm(a):
    """the column-major storage behind a (instance, row, column) view, as a contiguous array whose bytes can be compared:
    every NaN gets one bit pattern (a NaN the arithmetic produces has another payload on the CPU than on the GPU; a model
    with few inputs whose fp32 recursion never settles can overflow its tangent within the 1000 sweeps)"""
    a = np.array(np.transpose(np.asarray(a), (0, 2, 1)), order="C")  # a copy
    a[np.isnan(a)] = np.nan
    return a


@pytest.mark.parametrize("dt", [np.float32, np.float64])
@pytest.mark.parametrize("nx,nu", DIMS)
def test_device_tables_equal_host_tables(nx, nu, dt):
    """B = 1, 33 and 4 097 (more warps than one launch holds at once); the 4 097 batch has one singular model in the middle:
    sweeps_out = -1 there, its tables untouched, the neighbours unaffected, and the cache kernel flags the same model."""
    import torch

    s = BatchedTinySolver(setup_problem(wl.random_lti(nx, nu, 10), dt), device=0)
    for B, bad in ((1, None), (33, None), (4097, 2048)):
        A, Bm, f, Q, R, rho = SC.lti_batch(nx, nu, B, seed=nx * 100 + nu + B, singular_at=bad)
        dK, dP, sw = s.setup_sensitivity_device(A, Bm, f, Q, R, rho, want_sweeps=True)
        _, sw_cache = s.setup_models_device(A, Bm, f, Q, R, rho, want_sweeps=True)
        torch.cuda.synchronize()
        dK, dP, sw, sw_cache = dK.cpu().numpy(), dP.cpu().numpy(), sw.cpu().numpy(), sw_cache.cpu().numpy()
        assert dK.shape == (B, nu, nx) and dP.shape == (B, nx, nx)
        assert np.array_equal(sw, sw_cache)  # the same sweeps, and -1 for the same models, as the cache precompute
        good = np.ones(B, bool)
        if bad is not None:
            assert sw[bad] == -1 and not dK[bad].any() and not dP[bad].any()
            good[bad] = False
        assert (sw[good] > 0).all()
        hK, hP = setup_sensitivity(nx, nu, A[good], Bm[good], f[good], Q[good], R[good], rho[good], dtype=dt)
        H.assert_bits_per_instance(dict(dK=_cm(dK[good]), dP=_cm(dP[good])), dict(dK=_cm(hK), dP=_cm(hP)), ["dK", "dP"],
                                   f"({nx},{nu}) {np.dtype(dt).name} B={B}")
        finite = np.isfinite(hK).reshape(len(hK), -1).all(axis=1)
        assert finite.mean() > 0.8 and (dt == np.float32 or finite.all()), finite.mean()  # the comparison is about numbers
    s.close()


def _tiled(ar, B):
    tile = lambda a: np.ascontiguousarray(np.tile(np.asarray(a)[None], (B, 1, 1)))  # noqa: E731
    return AdaptiveRho(tile(ar.dKinf_drho), tile(ar.dPinf_drho), ar.rho_min, ar.rho_max, ar.enable_clipping)


@pytest.mark.parametrize("name", ["track_N50_f32", "track_N50_f64"])
def test_equal_per_instance_tables_match_the_shared_table_solve(name):
    """B copies of one table pair, read per instance from global memory, against the same pair staged in shared memory: every
    output, state field and adapted blob over the case's closed loop, through the host and the device entry points."""
    import torch

    c = AC.make_cases(with_wide=False)[name]
    prob, st, ar = c["prob"], c["st"], c["ar"]
    ar_b = _tiled(ar, len(c["x0"]))
    s = BatchedTinySolver(prob, st, device=0)

    def host(which):
        def fn(p, st_, x0, Xref, Uref, state, cold, models):
            o = s.solve(x0, Xref, Uref, state=state, cold_start=cold, want_state=AC.BOX, models=models, adaptive_rho=which)
            return o, o["models"]
        return fn

    def device(p, st_, x0, Xref, Uref, state, cold, models):
        tm = torch.as_tensor(models, device="cuda:0").contiguous()
        batch, out = s.make_device_batch(x0, Xref, state=state, cold_start=cold, want_state=AC.BOX)
        s.solve_device_adaptive(batch, tm, ar_b)
        torch.cuda.synchronize()
        return {k: out[k].cpu().numpy() for k in KEYS}, tm.cpu().numpy()

    ref, _ = AC.closed_loop(prob, st, c, host(ar))
    for what, fn in (("host", host(ar_b)), ("device", device)):
        got, _ = AC.closed_loop(prob, st, c, fn)
        for k in range(c["steps"]):
            H.assert_bits_per_instance(dict(got[k][0], models=got[k][1]), dict(ref[k][0], models=ref[k][1]), KEYS + ["models"],
                                       f"{name} {what} step {k}")
    assert np.any(ref[-1][1][:, -1] != c["models"][:, -1])  # rho did adapt
    s.close()


def _fleet(dt, N=50):
    """Six differently tuned quadrotors: model blobs and sensitivity tables per model, from the device calls, checked against
    the host calls; the handle they were computed on."""
    import torch

    sp, (A, Bm, f, Q, R, rho) = SC.tuned_quadrotor_fleet(N)
    prob = H.problem_from_spec(sp, dt, oracle.port_setup)
    st = abi.Settings()
    C.memmove(C.byref(st), C.byref(sp.settings), C.sizeof(abi.Settings))
    st.max_iter = 16  # loop index 15 adapts: adaptation also lands on the last iteration of the capped instances
    s = BatchedTinySolver(prob, st, device=0)
    blobs = s.setup_models_device(A, Bm, f, Q, R, rho)
    dK, dP = s.setup_sensitivity_device(A, Bm, f, Q, R, rho)
    torch.cuda.synchronize()
    assert H.bits_equal(blobs.cpu().numpy(), setup_models(12, 4, A, Bm, f, Q, R, rho, dtype=dt))
    hK, hP = setup_sensitivity(12, 4, A, Bm, f, Q, R, rho, dtype=dt)
    assert H.bits_equal(_cm(dK.cpu().numpy()), _cm(hK)) and H.bits_equal(_cm(dP.cpu().numpy()), _cm(hP))
    assert len({hK[m].tobytes() for m in range(6)}) == 6  # six different table pairs
    return sp, prob, st, s, blobs, dK, dP


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_fleet_device_cold_then_two_warm_steps(dt):
    """A fleet of six models dealt with a stride of five over more than 2.5 waves of the persistent kernel, tables and blobs
    from the device calls and never copied to the host, outputs poisoned: every instance and scalar, models included."""
    import torch

    sp, prob, st, s, blobs, dK, dP = _fleet(dt)
    s.solve(np.zeros((64, 12), dt), np.zeros((50, 12), dt), adaptive_rho=AdaptiveRho(dK[:1].expand(64, -1, -1), dP[:1].expand(64, -1, -1)))
    stt = s.stats()
    assert stt["kernel_family"] == abi.KERNEL_GPI
    B = int(2.6 * torch.cuda.get_device_properties(0).multi_processor_count * stt["instances_per_cta"])
    model = torch.as_tensor(SC.deal(B), device="cuda:0")
    tm = blobs[model].contiguous()
    ar = AdaptiveRho(dK[model], dP[model], 1.0, 100.0, True)
    ar_ref = AdaptiveRho(ar.dKinf_drho.cpu().numpy(), ar.dPinf_drho.cpu().numpy(), 1.0, 100.0, True)
    inst = wl.tracking_instances(B, N=50, seed=21, dtype=dt)
    start = tm.cpu().numpy()
    state, ref_models = None, start
    for step in range(3):
        x0 = inst["x0"] if step == 0 else AC.advance(prob, x0, ref["u"][:, 0, :])
        batch, out = s.make_device_batch(x0, inst["Xref"], state=state, cold_start=state is None, want_state=AC.BOX)
        ref, ref_models = SC.oracle_solve_per_instance(prob, st, x0, inst["Xref"], None, state, state is None, ref_models, ar_ref)
        for key in AC.OUT:
            H.poison(out[key])
        if state is None:
            for key in AC.BOX:
                H.poison(out[key])
        s.solve_device_adaptive(batch, tm, ar)
        torch.cuda.synchronize()
        assert s.stats()["ctas"] * s.stats()["instances_per_cta"] * 2.5 < B
        got = {k: out[k].cpu().numpy() for k in KEYS}
        got["models"] = tm.cpu().numpy()
        H.assert_bits_per_instance(got, dict(ref, models=ref_models), KEYS + ["models"], f"fleet step {step}")
        if step == 0:
            H.assert_mixed_termination(ref)
        state = {k: ref[k] for k in AC.BOX}
    assert np.any(ref_models[:, -1] != start[:, -1])
    # the tables matter: with every instance on model 0's pair, instances of other models get another adapted cache
    wrong, m0 = SC.oracle_solve_per_instance(prob, st, inst["x0"], inst["Xref"], None, None, True, start,
                                             AdaptiveRho(ar_ref.dKinf_drho[:1].repeat(B, 0), ar_ref.dPinf_drho[:1].repeat(B, 0)))
    right, m1 = SC.oracle_solve_per_instance(prob, st, inst["x0"], inst["Xref"], None, None, True, start, ar_ref)
    assert np.any(m0[SC.deal(B) != 0] != m1[SC.deal(B) != 0])
    s.close()


@pytest.mark.parametrize("pinned", [False, True])
def test_fleet_host_path_in_11_chunks(monkeypatch, pinned):
    """tinympc_b200_solve_adaptive_host slices the per-instance tables per chunk as it slices the models; pageable and
    page-locked caller buffers (the latter are read by DMA straight from the caller's memory)."""
    import torch

    dt = np.float32
    sp, prob, st, s, blobs, dK, dP = _fleet(dt)
    B = 11 * 256
    model = SC.deal(B)
    inst = wl.tracking_instances(B, N=50, seed=22, dtype=dt)
    hK, hP = dK.cpu().numpy()[model], dP.cpu().numpy()[model]
    models = np.ascontiguousarray(blobs.cpu().numpy()[model])
    ar_ref = AdaptiveRho(hK, hP)
    ref, rm = SC.oracle_solve_per_instance(prob, st, inst["x0"], inst["Xref"], None, None, True, models, ar_ref)
    hb = HostBatch(prob, inst["x0"], inst["Xref"], None, cold_start=True, want_state=AC.BOX)
    keep = []

    def buf(a):  # column-major per instance is what the C call takes
        a = np.ascontiguousarray(a)
        if not pinned:
            return a
        t = torch.from_numpy(a).pin_memory()
        keep.append(t)
        return t.numpy()

    m, cK, cP = buf(models.copy()), buf(_cm(hK)), buf(_cm(hP))
    a = AdaptiveRho(hK, hP).to_c(prob, m.ctypes.data, B)
    a.dKinf_drho, a.dPinf_drho = cK.ctypes.data, cP.ctypes.data
    cb = hb.to_c()
    monkeypatch.setenv("TINYMPC_HOST_CHUNK", "256")
    rc = load().tinympc_b200_solve_adaptive_host(s._h, C.byref(cb), C.byref(a))
    assert rc == 0, load().tinympc_b200_last_error()
    assert s.stats()["kernel_launches"] == 11
    H.assert_bits_per_instance(dict(hb.result(), models=m), dict(ref, models=rm), KEYS + ["models"], f"host chunks pinned={pinned}")
    s.close()


def test_fleet_device_closed_loop():
    """DeviceMPCLoop(adaptive_rho=<per-instance tables>, models=<fleet>): tables and models stay on the GPU for 5 steps."""
    from tinympc_b200.closed_loop import DeviceMPCLoop

    dt = np.float64
    sp, prob, st, s, blobs, dK, dP = _fleet(dt)
    B = 300
    model = SC.deal(B)
    inst = wl.tracking_instances(B, N=50, seed=23, dtype=dt)
    ar = AdaptiveRho(dK[model], dP[model])
    loop = DeviceMPCLoop(s, inst["x0"], adaptive_rho=ar, models=blobs[model])
    assert loop.adaptive_rho.dKinf_drho.is_cuda
    ar_ref = AdaptiveRho(ar.dKinf_drho.cpu().numpy(), ar.dPinf_drho.cpu().numpy())
    x0, state, models = inst["x0"].copy(), None, blobs.cpu().numpy()[model]
    for k in range(5):
        Xref = np.ascontiguousarray(np.roll(inst["Xref"], -k, axis=1))
        out = loop.step(Xref)
        ref, models = SC.oracle_solve_per_instance(prob, st, x0, Xref, None, state, state is None, models, ar_ref)
        got = {key: out[key].cpu().numpy() for key in AC.OUT + list(loop.fields)}
        got["models"] = loop.models.cpu().numpy()
        H.assert_bits_per_instance(got, dict(ref, models=models), AC.OUT + list(loop.fields) + ["models"], f"step {k}")
        state = {n: ref[n] for n in AC.BOX}
        x0 = AC.advance(prob, x0, np.ascontiguousarray(ref["u"][:, 0, :]))  # the fleet shares A, B, f: one plant model
        assert H.bits_equal(loop.x0.cpu().numpy(), x0)
    s.close()


def test_loud_errors():
    lib = load()
    dt = np.float32
    sp = wl.quadrotor(N=50)
    prob = H.problem_from_spec(sp, dt, oracle.port_setup)
    inst = wl.tracking_instances(8, N=50, seed=1, dtype=dt)
    s = BatchedTinySolver(prob, sp.settings, device=0)
    models = pack_models(prob, 8)
    cb = HostBatch(prob, inst["x0"], inst["Xref"]).to_c()
    dK, dP = np.zeros((8, 4, 12), dt), np.zeros((8, 12, 12), dt)

    def call(per=1, null=None):
        a = AdaptiveRho(dK, dP).to_c(prob, models.ctypes.data, 8)
        a.tables_per_instance = per
        if null:
            setattr(a, null, None)
        return lib.tinympc_b200_solve_adaptive_host(s._h, C.byref(cb), C.byref(a))

    assert call(null="dKinf_drho") == abi.ERR_ARG
    assert call(null="dPinf_drho") == abi.ERR_ARG
    assert call(per=2) == abi.ERR_ARG and b"tables_per_instance" in lib.tinympc_b200_last_error()
    assert call(per=-1) == abi.ERR_ARG
    assert call() == abi.OK
    with pytest.raises(ValueError):
        AdaptiveRho(dK[:7], dP[:7]).to_c(prob, models.ctypes.data, 8)
    s.close()
