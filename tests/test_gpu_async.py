"""Queued use of the asynchronous entry points: sequences of solves, adaptive-rho solves, rollouts, closed-loop steps and host-path
solves enqueued on one handle (or on two handles at once) with no host synchronise and no host read between the calls, each call
held bit for bit to the same call run with a synchronise after every call, and where it is cheap to the CPU oracle.

The handle carries state from one call to the next: the argument buffer of adaptive rho and rollouts with its ring of three
page-locked staging slots, the single-buffered work queue, v-scratch and workspaces, and the wait a solve on another stream makes
for the previous one.  Every sequence starts with a long solve (more than a wave of instances, zero tolerances, so that every
instance runs HEAD_ITERS iterations), and each test asserts that it was still running when the later calls were staged (up to
the call whose staging the library itself makes wait for it: a buffer that grows, or a fourth argument upload): their staging,
buffer growth and work-queue memsets happen behind a running kernel.  Every output buffer is filled with a NaN bit pattern
first.  Each sequence runs once."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest

import adaptive_common as AC
import helpers as H
from oracle import oracle
from tinympc_b200 import abi, workloads as wl
from tinympc_b200._lib import check
from tinympc_b200.closed_loop import DeviceMPCLoop
from tinympc_b200.solver import AdaptiveRho, BatchedTinySolver, pack_models, setup_models

pytestmark = pytest.mark.gpu

NT = os.cpu_count() or 1
DTS = [np.float32, np.float64]
BOX = tuple(H.BOX_STATE)
FIELDS = ("v", "z", "vnew", "znew", "g", "y")
FIELDS_FAST = ("vnew", "znew", "g", "y")
OUTS = ("sol_x", "sol_u", "u0", "iter", "solved", "residuals")
PLAN = ("kernel_family", "lanes_per_instance", "instances_per_cta", "smem_bytes_per_cta", "ctas", "threads_per_cta")
HEAD_ITERS = 2000


def _torch():
    import torch

    return torch


def _st(st, **kw):
    s = abi.Settings.from_buffer_copy(st)
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def _dev(a, dt):
    return _torch().as_tensor(np.ascontiguousarray(a, dtype=dt), device="cuda")


def _shape(prob, n):
    return (prob.N, prob.nx) if abi.STATE_IS_X[n] else (prob.N - 1, prob.nu)


def _quad(dt):
    spec = wl.quadrotor(N=50)
    return H.problem_from_spec(spec, dt, oracle.port_setup), _st(spec.settings, max_iter=15)


def _lti(dt):
    spec = wl.random_lti(8, 4, 30, seed=3)
    return H.problem_from_spec(spec, dt, oracle.port_setup), _st(spec.settings, max_iter=20)


_CAP = {}


def _capacity(prob, st, kernel=abi.KERNEL_GPI):
    """Instances one wave of the persistent kernel holds, from a one-iteration probe solve that fills every SM."""
    torch = _torch()
    key = (prob.nx, prob.nu, prob.N, np.dtype(prob.dtype).name, kernel)
    if key not in _CAP:
        B = 64 * torch.cuda.get_device_properties(0).multi_processor_count
        s = BatchedTinySolver(prob, _st(st, max_iter=1), kernel=kernel)
        batch, _ = s.make_device_batch(np.zeros((B, prob.nx), prob.dtype), np.zeros((prob.N, prob.nx), prob.dtype))
        s.solve_device(batch)
        torch.cuda.synchronize()
        stt = s.stats()
        s.close()
        assert stt["kernel_family"] == kernel, stt
        _CAP[key] = stt["ctas"] * stt["instances_per_cta"]
    return _CAP[key]


# ---------------------------------------------------------------------------------------------------------------------
# calls: inputs are device tensors made before a sequence starts (a host-to-device copy from pageable memory would
# synchronise); in/out arrays (warm state, adapted models) are cloned by each run so that both runs start from the same values
# ---------------------------------------------------------------------------------------------------------------------
def _refs(prob, B, seed, knots=None, per_x=True, uref=False):
    rng = np.random.default_rng(seed)
    knots = prob.N if knots is None else knots
    dt = prob.dtype
    x0 = _dev(rng.standard_normal((B, prob.nx)), dt)
    X = _dev(0.5 * rng.standard_normal((B, knots, prob.nx) if per_x else (knots, prob.nx)), dt)
    U = _dev(0.05 * rng.standard_normal((B, knots - 1, prob.nu) if per_x else (knots - 1, prob.nu)), dt) if uref else None
    return x0, X, U


def _state(prob, B, seed, fields=BOX):
    rng = np.random.default_rng(seed)
    return {n: _dev(0.1 * rng.standard_normal((B,) + _shape(prob, n)), prob.dtype) for n in fields}


def solve_call(prob, st, B, seed, kernel=abi.KERNEL_AUTO, warm=False, per_x=True, uref=False, models=None, **kw):
    x0, X, U = _refs(prob, B, seed, per_x=per_x, uref=uref)
    return dict(kind="solve", st=st, kernel=kernel, x0=x0, Xref=X, Uref=U, state=_state(prob, B, seed + 1) if warm else None,
                fields=BOX, models=models, **kw)


def _head(prob, st, cap, **kw):
    """The long first call of a sequence: 1.5 waves and a ragged remainder, every instance runs HEAD_ITERS iterations."""
    hs = _st(st, max_iter=HEAD_ITERS, abs_pri_tol=0.0, abs_dua_tol=0.0)
    c = solve_call(prob, hs, int(1.5 * cap) + 37, 999, kernel=abi.KERNEL_GPI, head=True, **kw)
    c["fields"] = ()  # no state: the head uses no v-scratch, which the growth tests size themselves
    return c


def _tables(prob, B, seed, per, scale=1.0):
    """Sensitivity tables: the quadrotor's pair (scaled) or a random pair; per instance: [B] random pairs as column-major views
    on the device, which AdaptiveRho passes on without a copy."""
    dt, nx, nu = prob.dtype, prob.nx, prob.nu
    rng = np.random.default_rng(seed)
    if not per:
        if (nx, nu) == (12, 4):
            dK, dP = AC.quad_tables(dt)
            return (scale * dK).astype(dt), (scale * dP).astype(dt)
        return (0.01 * rng.standard_normal((nu, nx))).astype(dt), (0.01 * rng.standard_normal((nx, nx))).astype(dt)
    dK = 0.01 * scale * rng.standard_normal((B, nx, nu))
    dP = 0.01 * scale * rng.standard_normal((B, nx, nx))
    return _dev(dK, dt).transpose(1, 2), _dev(dP, dt).transpose(1, 2)


def adapt_call(prob, st, B, seed, rho_min=1.0, rho_max=100.0, clip=True, per=False, scale=1.0, warm=False, **kw):
    x0, X, _ = _refs(prob, B, seed)
    models = pack_models(prob, B)
    models[:, -1] = (prob.rho * (1.0 + 0.02 * np.random.default_rng(seed + 2).uniform(-1, 1, B))).astype(prob.dtype)
    dK, dP = _tables(prob, B, seed + 3, per, scale)
    return dict(kind="adaptive", st=st, kernel=abi.KERNEL_AUTO, x0=x0, Xref=X, Uref=None, state=_state(prob, B, seed + 1) if warm else None,
                fields=BOX, models=_dev(models, prob.dtype), ar=AdaptiveRho(dK, dP, rho_min, rho_max, clip), **kw)


def roll_call(prob, st, B, T, seed, per_x=True, uref=True, w=False, reset=True, carry=True, warm=False, models=None, **kw):
    x0, X, U = _refs(prob, B, seed, knots=T + prob.N - 1, per_x=per_x, uref=uref)
    fields = FIELDS if carry else FIELDS_FAST
    W = _dev(0.01 * np.random.default_rng(seed + 4).standard_normal((B, T, prob.nx)), prob.dtype) if w else None
    return dict(kind="rollout", st=st, kernel=abi.KERNEL_AUTO, x0=x0, Xref=X, Uref=U, w=W, T=T, reset=reset, carry=carry,
                state=_state(prob, B, seed + 1, fields) if warm else None, fields=fields, models=models, **kw)


def _prime(prob, st, Bmax, kernel=abi.KERNEL_GPI):
    """Calls run (synchronised) before a sequence so that nothing in it grows a buffer: the v-scratch of both on-chip plans for
    Bmax instances, the argument buffer and all three staging slots at their largest (shared tables), the kernel's workspace."""
    calls = [solve_call(prob, st, Bmax, 7, kernel=kernel, warm=True), adapt_call(prob, st, Bmax, 8, warm=True)]
    return calls + [adapt_call(prob, st, 32, 9)] * 2


# ---------------------------------------------------------------------------------------------------------------------
# running a sequence
# ---------------------------------------------------------------------------------------------------------------------
def _enqueue_rollout(solver, c, state, stream):
    torch = _torch()
    p = solver.problem
    B, T = c["x0"].shape[0], c["T"]
    kw = dict(dtype=torch.float32 if p.dtype == np.float32 else torch.float64, device="cuda")
    cold = state is None
    if cold:
        state = {n: H.poison(torch.empty((B,) + _shape(p, n), **kw)) for n in c["fields"]}
    i32 = dict(dtype=torch.int32, device="cuda")
    out = dict(x=torch.empty((B, T + 1, p.nx), **kw), u=torch.empty((B, T, p.nu), **kw), iter=torch.empty((B, T), **i32),
               solved=torch.empty((B, T), **i32), residuals=torch.empty((B, T, 4), **kw), sol_x=torch.empty((B, p.N, p.nx), **kw),
               sol_u=torch.empty((B, p.N - 1, p.nu), **kw))
    for v in out.values():
        H.poison(v)
    b = abi.Batch()
    b.B, b.x0, b.cold_start = B, c["x0"].data_ptr(), int(cold)
    for n, a in state.items():
        setattr(b.state, n, a.data_ptr())
    b.sol_x, b.sol_u = out["sol_x"].data_ptr(), out["sol_u"].data_ptr()
    b.models = None if c["models"] is None else c["models"].data_ptr()
    r = abi.Rollout()
    r.T, r.reset_duals, r.carry_v = T, int(c["reset"]), int(c["carry"])
    r.Xref, r.xref_per_instance = c["Xref"].data_ptr(), int(c["Xref"].dim() == 3)
    r.Uref, r.uref_per_instance = (None, 0) if c["Uref"] is None else (c["Uref"].data_ptr(), int(c["Uref"].dim() == 3))
    r.w = None if c["w"] is None else c["w"].data_ptr()
    r.x_traj, r.u_traj, r.residuals_traj = out["x"].data_ptr(), out["u"].data_ptr(), out["residuals"].data_ptr()
    r.iter_traj, r.solved_traj = out["iter"].data_ptr(), out["solved"].data_ptr()
    check(solver._lib.tinympc_b200_rollout(solver._h, C.byref(b), C.byref(r), C.c_void_p(stream.cuda_stream)))
    return dict(out, state=state, _keep=(b, r))


def _launch(solver, c, stream, outs):
    """Enqueue call c on `stream` with fresh, poisoned outputs; everything it allocates is ordered on `stream`.  A call with
    dep = j starts from call j's warm state (and adapted models): the caller has ordered that dependency with an event."""
    torch = _torch()
    solver.settings = _st(c["st"])
    solver.update_settings()
    solver.set_mode(abi.MODE_STRICT, c["kernel"])
    src = c if c.get("dep") is None else outs[c["dep"]]
    with torch.cuda.stream(stream):
        state = None if src["state"] is None else {n: src["state"][n].clone() for n in c["fields"]}
        if c["kind"] == "rollout":
            return _enqueue_rollout(solver, c, state, stream)
        models = None
        if c["kind"] == "adaptive":
            models = (src["models"] if src.get("models") is not None else c["models"]).clone()
        batch, out = solver.make_device_batch(c["x0"], c["Xref"], c["Uref"], state=state, cold_start=state is None, want_state=c["fields"],
                                              want_u0=True, models=c["models"] if c["kind"] == "solve" else None)
        for k in OUTS + (c["fields"] if state is None else ()):
            H.poison(out[k])
        if c["kind"] == "solve":
            solver.solve_device(batch, stream)
        else:
            solver.solve_device_adaptive(batch, models, c["ar"], stream)
        return dict({k: out[k] for k in OUTS}, state={n: out[n] for n in c["fields"]}, models=models, _keep=batch)


def _numpy(rec):
    d = {}
    for k, v in rec.items():
        if k == "state":
            d.update({"state." + n: a.cpu().numpy() for n, a in v.items()})
        elif not k.startswith("_") and v is not None:
            d[k] = v.cpu().numpy()
    return d


_SIDE = []  # stream 1, one for the whole module: the queued run reuses the blocks torch cached for the synchronised one


def _play(probs, calls, queued, prime=()):
    """Run `calls` on one fresh handle per problem (call key h), on stream 0 (torch's current stream) or stream 1.  queued: no
    host synchronise or read until every call is staged; otherwise a synchronise after every call.  Returns (numpy results,
    stats after each call (synchronised run), stats of each handle at the end, and running[i]: the first call had not finished
    when call i began staging (running[len(calls)]: when the last one had been staged))."""
    torch = _torch()
    if not _SIDE:
        _SIDE.append(torch.cuda.Stream())
    streams = [torch.cuda.current_stream(), _SIDE[0]]
    solvers = [BatchedTinySolver(p, calls[0]["st"]) for p in probs]
    for c in prime:
        _launch(solvers[c.get("h", 0)], c, streams[0], [])
        torch.cuda.synchronize()
    outs, evs, stats, running = [], [], [], [False]
    for i, c in enumerate(calls):
        s = streams[c.get("stream", 0)]
        if c.get("dep") is not None:
            s.wait_event(evs[c["dep"]])  # the caller's own data dependency
        if i:
            running.append(not evs[0].query())
        outs.append(_launch(solvers[c.get("h", 0)], c, s, outs))
        evs.append(torch.cuda.Event())
        evs[-1].record(s)
        if not queued:
            torch.cuda.synchronize()
            stats.append(solvers[c.get("h", 0)].stats())
    running.append(not evs[0].query())
    torch.cuda.synchronize()
    final = [s.stats() for s in solvers]
    res = [_numpy(o) for o in outs]
    for s in solvers:
        s.close()
    return res, stats, final, running


def _run_both(probs, calls, what, prime=(), running_until=None):
    """The sequence synchronised after every call, then queued: every output of every call bit for bit equal, the head still
    running when call `running_until` (default: every call) was staged, the plan of each handle's last call equal.  The
    synchronised run goes first, so that the queued one finds its tensors in torch's cache (no allocation on its way)."""
    ref, stats, _, _ = _play(probs, calls, False, prime)
    got, _, final, running = _play(probs, calls, True, prime)
    for i, c in enumerate(calls):
        assert sorted(got[i]) == sorted(ref[i]), (what, i)
        H.assert_bits_per_instance(got[i], ref[i], sorted(got[i]), f"{what}: call {i} ({c['kind']})")
        if c.get("head"):
            assert (ref[i]["iter"] == HEAD_ITERS).all(), (what, i)
    n = len(calls) if running_until is None else running_until
    assert all(running[1:n + 1]), f"{what}: the first call finished before call {running.index(False, 1)} was staged: {running}"
    for h in range(len(probs)):
        last = max(i for i, c in enumerate(calls) if c.get("h", 0) == h)
        assert {k: final[h][k] for k in PLAN} == {k: stats[last][k] for k in PLAN}, (what, h, final[h], stats[last])
    return got, ref, stats, final


def _oracle_check(prob, c, got, what, n=64):
    """The first n instances of a solve or shared-table adaptive solve without a dependency, against the CPU oracle."""
    sl = slice(0, n)
    np_ = lambda a, per=True: None if a is None else np.ascontiguousarray((a[sl] if per else a).cpu().numpy())  # noqa: E731
    x0, X, U = np_(c["x0"]), np_(c["Xref"], c["Xref"].dim() == 3), None if c["Uref"] is None else np_(c["Uref"], c["Uref"].dim() == 3)
    state = None if c["state"] is None else {k: np_(v).copy() for k, v in c["state"].items()}
    if c["kind"] == "solve":
        o = oracle.solve_batch(prob, c["st"], x0, X, U, state=state, cold_start=state is None, want_state=BOX, impl="port", nthreads=NT)
        ref = {}
    else:
        o, m = AC.oracle_solve(prob, c["st"], x0, X, U, state, state is None, np_(c["models"]), c["ar"], nthreads=NT)
        ref = dict(models=m)
    ref.update({k: o[k] for k in ("sol_x", "sol_u", "iter", "solved", "residuals")}, u0=np.ascontiguousarray(o["u"][:, 0, :]))
    ref.update({"state." + f: o[f] for f in c["fields"]})
    H.assert_bits_per_instance({k: got[k][sl] for k in ref}, ref, sorted(ref), what + " vs oracle")


# ---------------------------------------------------------------------------------------------------------------------
# 1. the argument ring: more staged uploads than staging slots, all queued behind the head
# ---------------------------------------------------------------------------------------------------------------------
# B, rho_min, rho_max, clipping, per-instance tables, table scale, warm start
ADAPT = [(300, 1.0, 100.0, True, False, 1.0, False), (200, 1.0, 100.0, False, False, 0.5, True), (260, 0.5, 50.0, True, True, 1.0, False),
         (128, 4.99, 5.0, True, False, 1.0, True), (333, 1.0, 100.0, False, True, 2.0, True), (96, 2.0, 20.0, True, False, 1.5, False),
         (512, 0.1, 100.0, True, False, 0.8, True), (64, 1.0, 100.0, True, True, 1.0, False)]
# B, T, per-robot references, Uref, disturbance, reset_duals, carry_v, warm start
ROLL = [(400, 5, True, True, False, True, True, False), (256, 1, False, False, True, False, True, False),
        (300, 3, True, False, False, True, False, False), (128, 6, False, True, True, True, True, True),
        (333, 2, True, True, True, False, False, True), (200, 4, False, False, False, False, True, False),
        (96, 7, True, True, True, True, True, False), (512, 2, True, False, False, True, False, True)]


# The fourth argument upload reuses the first one's staging slot, whose copy is queued behind the head: the head is still
# running when that upload begins staging (which then waits for the copy), not after it.
RING = 4


def _adapt_calls(prob, st, variants, seed, **kw):
    return [adapt_call(prob, _st(st, max_iter=16 - i), B, seed + 10 * i, rmin, rmax, clip, per, scale, warm, **kw)
            for i, (B, rmin, rmax, clip, per, scale, warm) in enumerate(variants)]


def _roll_calls(prob, st, variants, seed, **kw):
    return [roll_call(prob, _st(st, max_iter=12 + i), B, T, seed + 10 * i, per_x, uref, w, reset, carry, warm, **kw)
            for i, (B, T, per_x, uref, w, reset, carry, warm) in enumerate(variants)]


@pytest.mark.parametrize("dt", DTS)
def test_adaptive_ring_wraps(dt):
    """Eight adaptive solves behind the head: shared and per-instance tables, clipping on and off, different rho limits, model
    blobs, settings, batch sizes and cold / warm starts; the two shared-table ones of the first wrap against the oracle."""
    prob, st = _quad(dt)
    calls = [_head(prob, st, _capacity(prob, st))] + _adapt_calls(prob, st, ADAPT, 100)
    got, _, _, final = _run_both([prob], calls, f"adaptive ring {dt.__name__}", _prime(prob, st, 512), running_until=RING)
    assert final[0]["kernel_family"] == abi.KERNEL_GPI
    for i in (1, 2):
        _oracle_check(prob, calls[i], got[i], f"adaptive ring call {i}")


@pytest.mark.parametrize("dt", DTS)
def test_rollout_ring_wraps(dt):
    """Eight rollouts behind the head: T from 1 to 7, shared and per-robot references, with and without Uref and disturbance,
    both dual resets, both warm-start modes, cold and warm."""
    prob, st = _quad(dt)
    calls = [_head(prob, st, _capacity(prob, st))] + _roll_calls(prob, st, ROLL, 200)
    _, _, _, final = _run_both([prob], calls, f"rollout ring {dt.__name__}", _prime(prob, st, 512), running_until=RING)
    assert final[0]["kernel_family"] == abi.KERNEL_GPI and final[0]["kernel_launches"] == 1


@pytest.mark.parametrize("dt", DTS)
def test_adaptive_and_rollout_alternate(dt):
    """GpiAdapt and GpiRoll headers take turns in the one argument buffer, eight calls behind the head."""
    prob, st = _quad(dt)
    a, r = _adapt_calls(prob, st, ADAPT[4:], 300), _roll_calls(prob, st, ROLL[4:], 400)
    calls = [_head(prob, st, _capacity(prob, st))] + [c for pair in zip(a, r) for c in pair]
    _run_both([prob], calls, f"adaptive / rollout {dt.__name__}", _prime(prob, st, 512), running_until=RING)


# ---------------------------------------------------------------------------------------------------------------------
# 2. scratch growth behind running kernels
# ---------------------------------------------------------------------------------------------------------------------
FAMILY = {"gpi": abi.KERNEL_GPI, "tpi": abi.KERNEL_TPI, "gps": abi.KERNEL_GPS}


@pytest.mark.parametrize("fam", sorted(FAMILY))
@pytest.mark.parametrize("dt", DTS)
def test_scratch_grows_mid_queue(dt, fam):
    """head, small warm solve, big warm solve, small warm solve on one family; the handle's buffer is sized for the small one
    before the sequence, so the big one grows it while the head and the small one are queued: the v-scratch (GPI), the
    thread-per-instance workspace (a bigger Bpad) or the streamed kernel's workspace (more resident slots: grow and retry)."""
    prob, st = _quad(dt)
    kernel = FAMILY[fam]
    cap = _capacity(prob, st)
    big = {"gpi": int(1.25 * cap) + 37, "tpi": 4000, "gps": 2 * _capacity(prob, st, abi.KERNEL_GPS) + 37}[fam]
    small = solve_call(prob, st, 64, 11, kernel=kernel, warm=True)
    calls = [_head(prob, st, cap), small, solve_call(prob, st, big, 12, kernel=kernel, warm=True),
             solve_call(prob, st, 48, 13, kernel=kernel, warm=True, uref=True)]
    got, _, stats, final = _run_both([prob], calls, f"growth {fam} {dt.__name__}", prime=[small], running_until=2)
    assert [s["kernel_family"] for s in stats[1:]] == [kernel] * 3, stats
    if kernel != abi.KERNEL_GPI:
        assert stats[2]["workspace_bytes"] > stats[1]["workspace_bytes"], (stats[1], stats[2])
    if kernel == abi.KERNEL_TPI:  # the grown workspace stays with the handle
        assert final[0]["workspace_bytes"] == stats[2]["workspace_bytes"], (final, stats[2])
    for i in (1, 3):
        _oracle_check(prob, calls[i], got[i], f"growth {fam} call {i}")


@pytest.mark.parametrize("dt", DTS)
def test_args_buffer_grows_mid_queue(dt):
    """The argument buffer holds a rollout's header when an adaptive solve with shared tables (header + tables) is queued."""
    prob, st = _quad(dt)
    cap = _capacity(prob, st)
    prime = [solve_call(prob, st, 512, 7, kernel=abi.KERNEL_GPI, warm=True)] + [roll_call(prob, st, 32, 1, 8)] * 3
    calls = [_head(prob, st, cap), roll_call(prob, st, 300, 3, 21), adapt_call(prob, st, 256, 22, warm=True),
             roll_call(prob, st, 200, 2, 23, carry=False), adapt_call(prob, st, 128, 24, per=True)]
    got, _, _, _ = _run_both([prob], calls, f"argument growth {dt.__name__}", prime, running_until=2)
    _oracle_check(prob, calls[2], got[2], "argument growth adaptive")


# ---------------------------------------------------------------------------------------------------------------------
# 3. two streams, one handle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fam", sorted(FAMILY))
@pytest.mark.parametrize("dt", DTS)
def test_stream_switch_solves(dt, fam):
    """Solves alone alternate between two streams on one handle, cold and warm, one of them warm-started from an earlier call's
    state behind an event: the work queue, v-scratch and workspace each solve uses are the handle's one copy."""
    prob, st = _quad(dt)
    kernel = FAMILY[fam]
    calls = [_head(prob, st, _capacity(prob, st)),
             solve_call(prob, st, 400, 71, kernel=kernel, stream=1),
             solve_call(prob, st, 300, 72, kernel=kernel, warm=True),
             solve_call(prob, st, 500, 73, kernel=kernel, per_x=False, stream=1),
             solve_call(prob, st, 400, 74, kernel=kernel, uref=True, dep=1),
             solve_call(prob, st, 256, 75, kernel=kernel, warm=True, uref=True, stream=1)]
    got, _, stats, _ = _run_both([prob], calls, f"stream switch solves {fam} {dt.__name__}",
                                 [solve_call(prob, st, 512, 76, kernel=kernel, warm=True)])
    assert [s["kernel_family"] for s in stats[1:]] == [kernel] * 5, stats
    _oracle_check(prob, calls[1], got[1], "stream switch solves call 1")


@pytest.mark.parametrize("fam", ["gpi", "gps"])
@pytest.mark.parametrize("dt", DTS)
def test_stream_switches(dt, fam):
    """Solves (on-chip or streamed family), adaptive solves and rollouts alternate between two streams on one handle.  The calls
    that warm-start from an earlier call's state wait for it with an event; every other ordering is the handle's own."""
    prob, st = _quad(dt)
    kernel = FAMILY[fam]
    calls = [_head(prob, st, _capacity(prob, st)),
             solve_call(prob, st, 400, 31, kernel=kernel, stream=1),
             adapt_call(prob, st, 300, 32),
             roll_call(prob, st, 256, 3, 33, stream=1),
             solve_call(prob, st, 400, 34, kernel=kernel, uref=True, dep=1),
             adapt_call(prob, st, 300, 35, per=True, stream=1, dep=2),
             roll_call(prob, st, 400, 2, 36, dep=4),
             solve_call(prob, st, 200, 37, kernel=kernel, per_x=False, stream=1)]
    prime = _prime(prob, st, 512) + [solve_call(prob, st, 512, 38, kernel=kernel, warm=True)]
    got, _, stats, _ = _run_both([prob], calls, f"streams {fam} {dt.__name__}", prime, running_until=6)  # call 6: the fourth upload
    assert [stats[i]["kernel_family"] for i in (1, 4, 7)] == [kernel] * 3, stats
    _oracle_check(prob, calls[1], got[1], "streams call 1")


# ---------------------------------------------------------------------------------------------------------------------
# 4. two handles at once
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dts", [(np.float32, np.float64), (np.float64, np.float32)], ids=["quad_f32+lti_f64", "quad_f64+lti_f32"])
def test_two_handles_concurrent(dts):
    """(12,4,50) and (8,4,30) of different precision on two streams, their calls interleaved: a head each, multi-wave solves,
    an adaptive solve, a warm start and rollouts."""
    (p0, s0), (p1, s1) = _quad(dts[0]), _lti(dts[1])
    c0, c1 = _capacity(p0, s0), _capacity(p1, s1)
    b0, b1 = int(1.25 * c0) + 37, int(1.25 * c1) + 37
    calls = [_head(p0, s0, c0), _head(p1, s1, c1, h=1, stream=1),
             solve_call(p0, s0, b0, 41), solve_call(p1, s1, b1, 42, h=1, stream=1),
             adapt_call(p0, s0, 300, 43), solve_call(p1, s1, b1, 44, h=1, stream=1, dep=3),
             roll_call(p0, s0, 256, 3, 45), roll_call(p1, s1, 200, 4, 46, h=1, stream=1)]
    prime = [dict(c, h=0) for c in _prime(p0, s0, b0)] + [dict(c, h=1) for c in _prime(p1, s1, b1)]
    got, _, _, _ = _run_both([p0, p1], calls, "two handles", prime)
    _oracle_check(p0, calls[2], got[2], "two handles call 2")
    _oracle_check(p1, calls[3], got[3], "two handles call 3")


# ---------------------------------------------------------------------------------------------------------------------
# 5. the device closed loop, never read until the end
# ---------------------------------------------------------------------------------------------------------------------
LOOP_KEYS = ("u0", "iter", "solved", "residuals", "sol_x", "sol_u")


def _fleet(prob, dt, B):
    spec = wl.quadrotor(N=prob.N)
    M = 6
    A, f = np.stack([spec.A] * M), np.stack([spec.f] * M)
    Bm = np.stack([spec.B * (1.0 + 0.05 * i) for i in range(M)])
    Q = np.stack([spec.Qdiag * (1.0 + 0.2 * i) for i in range(M)])
    R = np.stack([spec.Rdiag * (1.0 + 0.1 * i) for i in range(M)])
    blobs = setup_models(12, 4, A, Bm, f, Q, R, np.array([spec.rho * (1.0 + 0.25 * i) for i in range(M)]), dtype=dt)
    return _dev(blobs[(5 * np.arange(B)) % M], dt)


def _loop_steps(solver, x0, X, U, T, exact, models, sync):
    """T DeviceMPCLoop steps with a sliding window; stream-ordered clones of loop.x0 and of every step's outputs and state."""
    torch = _torch()
    N = solver.problem.N
    loop = DeviceMPCLoop(solver, x0, reset_duals=True, exact_first_residual=exact, models=models)
    per = []
    for t in range(T):
        x = loop.x0.clone()
        out = loop.step(X[:, t:t + N], U[:, t:t + N - 1])
        per.append(dict({k: out[k].clone() for k in LOOP_KEYS + loop.fields}, x=x))
        if sync:
            torch.cuda.synchronize()
    per.append(dict(x=loop.x0.clone()))
    return per, loop.fields


@pytest.mark.parametrize("exact", [True, False], ids=["carry_v", "no_v"])
@pytest.mark.parametrize("fleet", [False, True], ids=["shared", "fleet"])
@pytest.mark.parametrize("dt", DTS)
def test_device_loop_unread(dt, fleet, exact):
    """Head, ten DeviceMPCLoop steps with a sliding window, then a rollout of the same episode on the same handle, all queued:
    every step equals the loop synchronised after every step (and, with one shared model, the oracle stepping the loop on the
    host), the rollout equals the queued steps."""
    torch = _torch()
    prob, st = _quad(dt)
    cap = _capacity(prob, st)
    B, T, N = int(1.25 * cap) + 37, 10, prob.N
    x0, X, U = _refs(prob, B, 51, knots=T + N - 1, uref=True)
    models = _fleet(prob, dt, B) if fleet else None

    def episode(sync):
        """head, T steps, the rollout; sync: a synchronise after each (the same allocations either way, so that the queued run
        finds its tensors in torch's cache)"""
        solver = BatchedTinySolver(prob, st)
        for c in [solve_call(prob, st, B, 52, kernel=abi.KERNEL_GPI, warm=True, models=models)] + [roll_call(prob, st, 32, 1, 53)] * 3:
            _launch(solver, c, torch.cuda.current_stream(), [])  # v-scratch for B, the argument buffer and its staging slots
            torch.cuda.synchronize()
        head = _launch(solver, _head(prob, st, cap), torch.cuda.current_stream(), [])
        ev = torch.cuda.Event()
        ev.record()
        if sync:
            torch.cuda.synchronize()
        solver.settings = _st(st)
        solver.update_settings()
        solver.set_mode(abi.MODE_STRICT, abi.KERNEL_AUTO)
        steps, fields = _loop_steps(solver, x0, X, U, T, exact, models, sync)
        running = [not ev.query()]
        roll = DeviceMPCLoop(solver, x0, reset_duals=True, exact_first_residual=exact, models=models).rollout(X, T, Uref_traj=U)
        running.append(not ev.query())
        torch.cuda.synchronize()
        out = (_numpy(head), [{k: v.cpu().numpy() for k, v in r.items()} for r in steps], {k: v.cpu().numpy() for k, v in roll.items()})
        solver.close()
        return out, running, fields

    (rhead, ref, rres), _, fields = episode(True)
    (head, got, res), running, _ = episode(False)
    assert all(running), f"the head finished before the steps / the rollout were staged: {running}"
    assert (rhead["iter"] == HEAD_ITERS).all()
    what = f"loop {dt.__name__} fleet={fleet} exact={exact}"
    H.assert_bits_per_instance(head, rhead, sorted(rhead), f"{what} head")
    for t in range(T + 1):
        H.assert_bits_per_instance(got[t], ref[t], sorted(ref[t]), f"{what} step {t}")
    H.assert_bits_per_instance(res, rres, sorted(rres), f"{what} rollout, synchronised")
    stepped = dict(x=np.stack([g["x"] for g in got], 1), u=np.stack([g["u0"] for g in got[:T]], 1),
                   **{k: np.stack([g[k] for g in got[:T]], 1) for k in ("iter", "solved", "residuals")})
    H.assert_bits_per_instance(res, stepped, sorted(stepped), f"{what} rollout")
    if not fleet and exact:  # the host oracle stepping the loop, first 64 robots
        n, state = 64, None
        xo = np.ascontiguousarray(x0[:n].cpu().numpy())
        Xn, Un = X[:n].cpu().numpy(), U[:n].cpu().numpy()
        for t in range(T):
            if state is not None:
                state["g"] = np.zeros_like(state["g"])
                state["y"] = np.zeros_like(state["y"])
            o = oracle.solve_batch(prob, st, xo, np.ascontiguousarray(Xn[:, t:t + N]), np.ascontiguousarray(Un[:, t:t + N - 1]),
                                   state=state, cold_start=state is None, want_state=BOX, impl="port", nthreads=NT)
            want = dict({k: o[k] for k in ("iter", "solved", "residuals", "sol_x", "sol_u") + fields}, u0=np.ascontiguousarray(o["u"][:, 0]), x=xo)
            H.assert_bits_per_instance({k: got[t][k][:n] for k in want}, want, sorted(want), f"{what} step {t} vs oracle")
            state = {k: np.array(o[k], copy=True) for k in BOX}
            xo = AC.advance(prob, xo, np.ascontiguousarray(o["u"][:, 0]))
        assert H.bits_equal(got[T]["x"][:n], xo)


# ---------------------------------------------------------------------------------------------------------------------
# 6. the host path between queued device solves
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
def test_host_path_after_queued_solve(dt, monkeypatch):
    """The head queued, then tinympc_b200_solve_host on the same handle in 11 chunks without a synchronise before it, then a
    device solve queued: all three equal their runs alone, the host solve also the oracle."""
    torch = _torch()
    prob, st = _quad(dt)
    monkeypatch.setenv("TINYMPC_HOST_CHUNK", "96")
    cap = _capacity(prob, st)
    hb = 1000
    rng = np.random.default_rng(61)
    hx0 = rng.standard_normal((hb, prob.nx)).astype(dt)
    hX = (0.5 * rng.standard_normal((hb, prob.N, prob.nx))).astype(dt)
    hstate = {n: (0.1 * rng.standard_normal((hb,) + _shape(prob, n))).astype(dt) for n in BOX}
    head, last = _head(prob, st, cap), solve_call(prob, st, 700, 62, warm=True, uref=True)

    def host(solver):
        out = solver.solve(hx0, hX, state={n: a.copy() for n, a in hstate.items()}, cold_start=False, want_state=BOX)
        stt = solver.stats()
        assert stt["kernel_launches"] == 11, stt
        return out

    # alone: each call on a handle of its own, synchronised
    alone = []
    for c in (head, None, last):
        s = BatchedTinySolver(prob, st)
        if c is None:
            alone.append(host(s))
        else:
            alone.append(_numpy(_launch(s, c, torch.cuda.current_stream(), [])))
            torch.cuda.synchronize()
        alone.append(s.stats())
        s.close()
    # queued
    s = BatchedTinySolver(prob, st)
    _launch(s, last, torch.cuda.current_stream(), [])  # the v-scratch of the last call, before the sequence
    torch.cuda.synchronize()
    q0 =_launch(s, head, torch.cuda.current_stream(), [])
    ev = torch.cuda.Event()
    ev.record()
    running = not ev.query()
    s.settings = _st(st)  # the head left its own settings and family on the handle
    s.update_settings()
    s.set_mode(abi.MODE_STRICT, abi.KERNEL_AUTO)
    hq = host(s)
    q2 = _launch(s, last, torch.cuda.current_stream(), [])
    torch.cuda.synchronize()
    final = s.stats()
    s.close()
    assert running, "the head finished before the host path was called"
    H.assert_bits_per_instance(_numpy(q0), alone[0], sorted(alone[0]), "host path: head")
    keys = H.OUT_KEYS + list(BOX)
    H.assert_bits_per_instance(hq, alone[2], keys, "host path: host solve")
    H.assert_bits_per_instance(_numpy(q2), alone[4], sorted(alone[4]), "host path: device solve after it")
    assert {k: final[k] for k in PLAN} == {k: alone[5][k] for k in PLAN}, (final, alone[5])
    o = oracle.solve_batch(prob, st, hx0, hX, None, state={n: a.copy() for n, a in hstate.items()}, cold_start=False, want_state=BOX,
                           impl="port", nthreads=NT)
    H.assert_bits_per_instance(hq, o, keys, "host path vs oracle")
