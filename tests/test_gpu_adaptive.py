"""Adaptive rho on the H100 (tinympc_b200_solve_adaptive[_host], the adaptive variant of the on-chip kernel), bit for bit against
the C restatement (tests/adaptive/adaptive_oracle.c), which tests/test_oracle_adaptive.py pins to the unmodified reference: every
output, requested state array and adapted model blob of every instance."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import adaptive_common as AC
import helpers as H
from tinympc_b200 import abi
from tinympc_b200 import workloads as wl
from tinympc_b200._lib import TinyMPCError
from tinympc_b200.solver import AdaptiveRho, BatchedTinySolver, pack_models

pytestmark = pytest.mark.gpu

KEYS = AC.OUT + AC.BOX


def gpu_solve(solver, ar):
    def fn(prob, st, x0, Xref, Uref, state, cold, models):
        out = solver.solve(x0, Xref, Uref, state=state, cold_start=cold, want_state=AC.BOX, models=models, adaptive_rho=ar)
        return out, out["models"]
    return fn


def port_solve(ar):
    def fn(prob, st, x0, Xref, Uref, state, cold, models):
        return AC.oracle_solve(prob, st, x0, Xref, Uref, state, cold, models, ar)
    return fn


def fixed_plan(solver, x0, Xref, models):
    """stats() of a fixed-rho solve of the same heterogeneous batch (the on-chip kernel without adaptation)"""
    solver.solve(x0, Xref, models=models)
    st = solver.stats()
    assert st["kernel_family"] == abi.KERNEL_GPI
    return st


def expect_adaptive_plan(solver, prob, fixed):
    """The adaptive kernel ran on chip, and its plan counts the staged tables: the fixed plan's shared memory plus the tables
    at the same residency, or fewer instances per CTA."""
    st = solver.stats()
    assert st["kernel_family"] == abi.KERNEL_GPI
    extra = ((prob.nu * prob.nx + prob.nx * prob.nx) * np.dtype(prob.dtype).itemsize + 15) // 16 * 16
    if st["instances_per_cta"] == fixed["instances_per_cta"]:
        assert st["smem_bytes_per_cta"] == fixed["smem_bytes_per_cta"] + extra, (st, fixed, extra)
    else:
        assert st["instances_per_cta"] < fixed["instances_per_cta"], (st, fixed)
    return st


@pytest.mark.parametrize("name", sorted(n for n in AC.make_cases(with_wide=False)))
def test_goldens(name):
    """The fixture cases (closed loops of 4 warm-started steps with the adapted cache carried over) on the GPU: every digest of
    the reference's loop."""
    import test_oracle_adaptive as T

    c, d = T.load_case(name)
    s = BatchedTinySolver(c["prob"], c["st"], device=0)
    fixed = fixed_plan(s, d["x0_seq"][0], c["Xref"], c["models"])
    outs, _ = AC.closed_loop(c["prob"], c["st"], c, gpu_solve(s, c["ar"]), x0_seq=d["x0_seq"])
    expect_adaptive_plan(s, c["prob"], fixed)
    for k, (r, m) in enumerate(outs):
        for key, got, want in zip(KEYS + ["models"], AC.digests(r, m), d["digests"][k]):
            assert got == str(want), f"{name} step {k}: {key}"
    s.close()


GPI_DIMS = [(4, 1), (6, 3), (12, 4), (4, 2), (4, 4), (4, 8), (8, 2), (8, 4), (8, 8), (12, 2), (12, 8), (16, 2), (16, 4), (16, 8)]


@pytest.mark.parametrize("dt", [np.float32, np.float64])
@pytest.mark.parametrize("nx,nu", GPI_DIMS)
def test_every_shape_n50(nx, nu, dt):
    """Every compiled (nx, nu) the on-chip plan covers at N = 50: two warm-started steps vs the restatement.  Wherever the fixed-rho
    on-chip kernel serves the shape, the adaptive one must too."""
    sp = wl.random_lti(nx, nu, 50, seed=1)
    rng = np.random.default_rng(nx * 31 + nu)
    tables = ((0.01 * rng.standard_normal((nu, nx))).astype(dt), (0.01 * rng.standard_normal((nx, nx))).astype(dt))
    inst = wl.random_instances(96, nx, 50, seed=2, dtype=dt)
    c = AC._spec_case(sp, dt, 96, inst, 2, tables, clip=(0.1, 100.0, True), seed=3)
    s = BatchedTinySolver(c["prob"], c["st"], device=0)
    try:
        fixed = fixed_plan(s, c["x0"], c["Xref"], c["models"])
    except TinyMPCError as e:
        assert e.code == abi.ERR_UNSUPPORTED, e
        pytest.skip(f"({nx},{nu}) {np.dtype(dt).name}: no on-chip plan at N = 50, with or without adaptive rho")
    got, _ = AC.closed_loop(c["prob"], c["st"], c, gpu_solve(s, c["ar"]))
    expect_adaptive_plan(s, c["prob"], fixed)
    ref, _ = AC.closed_loop(c["prob"], c["st"], c, port_solve(c["ar"]))
    for k in range(2):
        H.assert_bits_per_instance(dict(got[k][0], models=got[k][1]), dict(ref[k][0], models=ref[k][1]), KEYS + ["models"], f"step {k}")
    s.close()


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_multiwave_device_cold_then_warm(dt):
    """More than 2.5 waves of the persistent kernel (slot refills), device buffers poisoned with NaN bits, cold then warm with
    the adapted models fed back; max_iter 16 (loop index 15 adapts) so that adaptation also lands on the last iteration of the
    capped instances."""
    import torch

    sp = wl.quadrotor(N=50)
    prob = H.problem_from_spec(sp, dt, __import__("oracle.oracle", fromlist=["x"]).port_setup)
    st = abi.Settings()
    C.memmove(C.byref(st), C.byref(sp.settings), C.sizeof(abi.Settings))
    st.max_iter = 16
    s = BatchedTinySolver(prob, st, device=0)
    dK, dP = AC.quad_tables(dt)
    ar = AdaptiveRho(dK, dP, 1.0, 100.0, True)
    B0 = 64
    inst = wl.tracking_instances(B0, N=50, seed=9, dtype=dt)
    fixed = fixed_plan(s, inst["x0"], inst["Xref"], pack_models(prob, B0))
    s.solve(inst["x0"], inst["Xref"], want_state=AC.BOX, adaptive_rho=ar)
    st_ = expect_adaptive_plan(s, prob, fixed)
    B = int(2.6 * torch.cuda.get_device_properties(0).multi_processor_count * st_["instances_per_cta"])
    inst = wl.tracking_instances(B, N=50, seed=10, dtype=dt)
    models = pack_models(prob, B)
    models[:, -1] = (prob.rho * (1.0 + 0.02 * np.random.default_rng(1).uniform(-1, 1, B))).astype(dt)
    state, ref_models = None, models
    tm = torch.as_tensor(models, device="cuda:0").contiguous()
    for step in range(2):
        x0 = inst["x0"] if step == 0 else AC.advance(prob, inst["x0"], ref["u"][:, 0, :])
        batch, out = s.make_device_batch(x0, inst["Xref"], state=state, cold_start=state is None, want_state=AC.BOX)
        # (the oracle updates the state arrays it is given in place: it runs after they are on the device)
        ref, ref_models = AC.oracle_solve(prob, st, x0, inst["Xref"], None, state, state is None, ref_models, ar)
        for key in ("sol_x", "sol_u", "iter", "solved", "residuals"):
            H.poison(out[key])
        if state is None:
            for key in AC.BOX:
                H.poison(out[key])
        s.solve_device_adaptive(batch, tm, ar)
        torch.cuda.synchronize()
        got = {k: out[k].cpu().numpy() for k in KEYS}
        got["models"] = tm.cpu().numpy()
        H.assert_bits_per_instance(got, dict(ref, models=ref_models), KEYS + ["models"], f"step {step}")
        if step == 0:
            H.assert_mixed_termination(ref)
        assert (ref["iter"] == st.max_iter).any() and ref["solved"].any(), step  # capped ones adapt on their last iteration
        state = {k: ref[k] for k in AC.BOX}
    assert np.any(ref_models[:, -1] != models[:, -1])
    s.close()


def test_host_path_chunks(monkeypatch):
    """The host entry point in 7 chunks: models staged in and copied back per chunk."""
    dt = np.float32
    sp = wl.quadrotor(N=50)
    prob = H.problem_from_spec(sp, dt, __import__("oracle.oracle", fromlist=["x"]).port_setup)
    dK, dP = AC.quad_tables(dt)
    ar = AdaptiveRho(dK, dP)
    B = 7 * 512
    inst = wl.tracking_instances(B, N=50, seed=11, dtype=dt)
    models = pack_models(prob, B)
    monkeypatch.setenv("TINYMPC_HOST_CHUNK", "512")
    s = BatchedTinySolver(prob, sp.settings, device=0)
    got = s.solve(inst["x0"], inst["Xref"], want_state=AC.BOX, models=models, adaptive_rho=ar)
    assert s.stats()["kernel_launches"] == 7
    ref, m = AC.oracle_solve(prob, sp.settings, inst["x0"], inst["Xref"], None, None, True, models, ar)
    H.assert_bits_per_instance(got, dict(ref, models=m), KEYS + ["models"], "host chunks")
    s.close()


def test_device_closed_loop():
    """DeviceMPCLoop(adaptive_rho=...): the models stay on the device across steps (one TinySolver per robot)."""
    from tinympc_b200.closed_loop import DeviceMPCLoop

    dt = np.float64
    sp = wl.quadrotor(N=50)
    prob = H.problem_from_spec(sp, dt, __import__("oracle.oracle", fromlist=["x"]).port_setup)
    dK, dP = AC.quad_tables(dt)
    ar = AdaptiveRho(dK, dP)
    inst = wl.tracking_instances(300, N=50, seed=12, dtype=dt)
    s = BatchedTinySolver(prob, sp.settings, device=0)
    loop = DeviceMPCLoop(s, inst["x0"], adaptive_rho=ar)
    x0, state, models = inst["x0"].copy(), None, pack_models(prob, 300)
    for k in range(4):
        Xref = np.ascontiguousarray(np.roll(inst["Xref"], -k, axis=1))
        out = loop.step(Xref)
        ref, models = AC.oracle_solve(prob, sp.settings, x0, Xref, None, state, state is None, models, ar)
        got = {key: out[key].cpu().numpy() for key in AC.OUT + list(loop.fields)}
        got["models"] = loop.models.cpu().numpy()
        H.assert_bits_per_instance(got, dict(ref, models=models), AC.OUT + list(loop.fields) + ["models"], f"step {k}")
        state = {n: ref[n] for n in AC.BOX}
        x0 = AC.advance(prob, x0, np.ascontiguousarray(ref["u"][:, 0, :]))
        assert H.bits_equal(loop.x0.cpu().numpy(), x0)
    s.close()


def test_loud_errors():
    from tinympc_b200._lib import load

    lib = load()
    dt = np.float32
    sp = wl.quadrotor(N=50)
    prob = H.problem_from_spec(sp, dt, __import__("oracle.oracle", fromlist=["x"]).port_setup)
    dK, dP = AC.quad_tables(dt)
    inst = wl.tracking_instances(8, N=50, seed=1, dtype=dt)
    s = BatchedTinySolver(prob, sp.settings, device=0)
    from tinympc_b200.batch import HostBatch

    models = pack_models(prob, 8)
    hb = HostBatch(prob, inst["x0"], inst["Xref"])
    cb = hb.to_c()

    def call(ar_models=models.ctypes.data, io_models=None, reserved=0):
        a = AdaptiveRho(dK, dP).to_c(prob, ar_models)
        a.reserved = reserved
        cb.models = io_models
        return lib.tinympc_b200_solve_adaptive_host(s._h, C.byref(cb), C.byref(a))

    assert call(ar_models=None) == abi.ERR_ARG
    assert call(io_models=models.ctypes.data) == abi.ERR_ARG
    assert call(reserved=1) == abi.ERR_ARG
    for mode, fam in ((abi.MODE_FAST, abi.KERNEL_AUTO), (abi.MODE_STRICT, abi.KERNEL_TPI), (abi.MODE_STRICT, abi.KERNEL_GPS)):
        s.set_mode(mode, fam)
        assert call() == abi.ERR_UNSUPPORTED, (mode, fam)
        assert lib.tinympc_b200_last_error()
    s.set_mode(abi.MODE_STRICT, abi.KERNEL_AUTO)
    assert call() == abi.OK
    s.close()
    # cones: not covered
    rs = wl.rocket(N=20)
    rp = H.problem_from_spec(rs, dt, __import__("oracle.oracle", fromlist=["x"]).port_setup)
    s = BatchedTinySolver(rp, rs.settings, device=0)
    ri = wl.rocket_instances(4, N=20, dtype=dt)
    with pytest.raises(TinyMPCError) as e:
        s.solve(ri["x0"], ri["Xref"], ri["Uref"], adaptive_rho=AdaptiveRho(np.zeros((3, 6)), np.zeros((6, 6))))
    assert e.value.code == abi.ERR_UNSUPPORTED
    s.close()
    # no on-chip plan: a horizon that does not fit in shared memory
    big = wl.quadrotor(N=1000)
    bp = H.problem_from_spec(big, np.float64, __import__("oracle.oracle", fromlist=["x"]).port_setup)
    s = BatchedTinySolver(bp, big.settings, device=0)
    bi = wl.hovering_instances(4, N=1000, dtype=np.float64)
    with pytest.raises(TinyMPCError) as e:
        s.solve(bi["x0"], bi["Xref"], adaptive_rho=AdaptiveRho(*AC.quad_tables(np.float64)))
    assert e.value.code == abi.ERR_UNSUPPORTED
    s.close()


SHIM_LOOP = os.path.join(AC.ROOT, "oracle", "_ref", "shim_tests", "adaptive_loop")


@pytest.mark.parametrize("case", ["track_N50_f64", "track_maxit11_f64"])
def test_shim_closed_loop(case, tmp_path):
    """A reference-style program (tiny_setup, settings->adaptive_rho = 1, tiny_solve in a closed loop; built with the C++ shim)
    against the restatement stepping the same loop: every state array, the solution, iter / solved / residuals, the return
    value and the cache (rho, Kinf, Pinf) the shim writes back into the TinySolver after every step."""
    if not os.path.exists(SHIM_LOOP):
        pytest.skip("shim test program not built (tinympc_b200/shim/Makefile needs Eigen headers)")
    c = dict(AC.make_cases(with_wide=False)[case])
    prob, st, ar = c["prob"], c["st"], c["ar"]
    nx, nu, N = prob.nx, prob.nu, prob.N
    # one robot with a fixed reference window, as a reference program sets it once with tiny_set_x_ref
    c["x0"], c["Xref"], c["models"] = c["x0"][:1], np.ascontiguousarray(c["Xref"][0]), c["models"][:1]
    outs, x0s = AC.closed_loop(prob, st, c, port_solve(ar))
    steps = len(outs)
    f64 = lambda a: np.asarray(a, np.float64).reshape(-1, order="F").tobytes()  # noqa: E731
    head = np.array([nx, nu, N, steps, st.max_iter, st.check_termination, int(ar.enable_clipping)], np.int32).tobytes()
    head += np.array([st.abs_pri_tol, st.abs_dua_tol, ar.rho_min, ar.rho_max], np.float64).tobytes()
    body = c["models"][0].tobytes() + f64(ar.dKinf_drho) + f64(ar.dPinf_drho)
    body += f64(prob.x_min) + f64(prob.x_max) + f64(prob.u_min) + f64(prob.u_max)
    body += c["Xref"].tobytes() + np.ascontiguousarray(np.stack(x0s)[:, 0, :]).tobytes()
    (tmp_path / "in.bin").write_bytes(head + body)
    r = subprocess.run([SHIM_LOOP, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    raw = (tmp_path / "out.bin").read_bytes()
    mb = tinympc_model_blob(nx, nu)
    sizes = [("vnew", nx * N), ("znew", nu * (N - 1)), ("x", nx * N), ("u", nu * (N - 1)), ("v", nx * N), ("z", nu * (N - 1)),
             ("g", nx * N), ("y", nu * (N - 1)), ("iter", 1), ("solved", 1), ("residuals", 4), ("rho", 1), ("Kinf", nu * nx),
             ("Pinf", nx * nx)]
    per = sum(n for _, n in sizes) * 8 + 4
    assert len(raw) == per * steps
    for k, (res, models) in enumerate(outs):
        o, rec = k * per, {}
        for name, n in sizes:
            rec[name] = np.frombuffer(raw, np.float64, n, o)
            o += 8 * n
        rc = int(np.frombuffer(raw, np.int32, 1, o)[0])
        for name in ("vnew", "znew", "x", "u", "v", "z", "g", "y", "residuals"):
            assert H.bits_equal(rec[name], res[name].reshape(-1)), (case, k, name)
        assert int(rec["iter"][0]) == int(res["iter"][0]) and int(rec["solved"][0]) == int(res["solved"][0]), (case, k)
        assert rc == (0 if res["solved"][0] else 1)
        assert H.bits_equal(rec["rho"], models[0, -1:]), (case, k)
        assert H.bits_equal(rec["Kinf"], models[0, mb["Kinf"]:mb["Kinf"] + nu * nx]), (case, k)
        assert H.bits_equal(rec["Pinf"], models[0, mb["Pinf"]:mb["Pinf"] + nx * nx]), (case, k)
    assert outs[-1][1][0, -1] != c["models"][0, -1]  # rho did adapt


def tinympc_model_blob(nx, nu):
    o, out = 0, {}
    for name, n in (("A", nx * nx), ("B", nx * nu), ("f", nx), ("Q", nx), ("R", nu), ("Kinf", nu * nx), ("Pinf", nx * nx)):
        out[name] = o
        o += n
    return out
