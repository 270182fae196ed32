"""The reference-compatible C++ shim held to the unmodified reference call for call.  One scripted driver
(tests/shim/shim_script.cpp) is built against the reference (oracle/_ref/shim_tests/script_ref, run on the CPU) and against
the shim (oracle/_ref/shim_tests/script_shim, solves on the GPU); both run the same op streams: closed loops with settings
changed between solves, constraint families switched off and on, bounds / cones / planes re-set mid-run, pokes into the
workspace, a new rho, two interleaved solvers, tiny_solve_batch and one solver per thread.  Every stream first pins the
cache to what the reference's own tiny_setup derives, so both builds solve on the same cache and every dump - the return
code, solution, every slack / dual / family array of work, the residuals, status, iter and the cache - must be equal bit
for bit, and every op must print the same lines.  work->{q, r, p, d} are not compared: they are per-iteration scratch that
each iteration overwrites before reading, and the shim never writes them.  The caches the shim's own tiny_setup /
tiny_precompute_and_set_cache derive are held to the reference's within 1e-9 of each matrix's largest entry."""
import numpy as np
import pytest

import shim_common as S
from oracle import oracle
from tinympc_b200 import workloads as wl

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not (S.have(S.SCRIPT_REF, S.SCRIPT_SHIM) and oracle.ref_available(np.float64)),
                                 reason="scripted shim drivers not built (oracle/Makefile and tinympc_b200/shim/Makefile need a "
                                        "TinyMPC checkout: REF=<path>)")]

TM_DIMS = [(4, 1), (6, 3), (12, 4), (4, 2), (4, 4), (4, 8), (8, 2), (8, 4), (8, 8), (12, 2), (12, 8), (16, 2), (16, 4), (16, 8)]


def compare(script, tmp_path, tag):
    """Both builds on one stream: every record and every op's stdout equal -> the reference's records"""
    ref, ref_out = S.run(S.SCRIPT_REF, script, str(tmp_path), tag + "_ref")
    got, got_out = S.run(S.SCRIPT_SHIM, script, str(tmp_path), tag + "_shim")
    S.assert_same_records(ref, got, tag)
    S.assert_same_stdout(ref_out, got_out, tag)
    return ref, got


def lti(nx, nu, N, seed):
    return S.Model.from_spec(wl.random_lti(nx, nu, N, seed=seed))


def box(s, si, m, xb=3.0, ub=1.0):
    return s.bounds(si, np.full(m.nx, -xb), np.full(m.nx, xb), np.full(m.nu, -ub), np.full(m.nu, ub))


def loop(s, si, steps):
    for _ in range(steps):
        s.solve(si).plant(si)
    return s


def rocket(N):
    sp = wl.rocket(N=N)
    c = sp.constraints
    return S.Model.from_spec(sp), c


def rocket_start(s, si, N, seed):
    m, c = rocket(N)
    inst = wl.rocket_instances(1, N=N, seed=seed)
    s.setup(si, m)
    s.bounds(si, c["x_min"], c["x_max"], c["u_min"], c["u_max"])
    s.cones(si, c["Acx"], c["qcx"], c["cx"], c["Acu"], c["qcu"], c["cu"])
    s.update_settings(si, max_iter=120, abs_pri_tol=1e-2, abs_dua_tol=1e-2, en_state_soc=1, en_input_soc=1)
    s.xref(si, inst["Xref"].T).uref(si, inst["Uref"].T).x0(si, inst["x0"][0])
    return m


def planes_start(s, si, N, seed, tv=False):
    """12-state / 4-input model with static planes (one all-zero padding row per side) or time-varying planes"""
    m = S.Model.from_spec(wl.quadrotor(N=N, hz=50))
    rng = np.random.default_rng(seed)
    s.setup(si, m)
    s.update_settings(si, max_iter=60, abs_pri_tol=1e-2, abs_dua_tol=1e-2, en_state_bound=0, en_input_bound=0)
    if tv:
        s.update_settings(si, en_tv_state_linear=1, en_tv_input_linear=1)
        tv_planes(s, si, m, 0)
    else:
        Ax = np.zeros((4, 12)); Ax[0, 0] = 1.0; Ax[0, 1] = 0.5; Ax[1, 2] = -1.0; Ax[1, 0] = 0.25; Ax[3, 1] = 1.0
        Au = np.zeros((3, 4)); Au[0] = 1.0; Au[2, 1] = -1.0; Au[2, 3] = 0.5
        s.linear(si, Ax, [0.3, -0.2, 0.0, 0.15], Au, [0.4, 1.0, 0.1])  # rows 2 (state) and 1 (input) are padding
        s.update_settings(si, en_state_linear=1, en_input_linear=1)
    s.xref(si, np.zeros((12, N))).x0(si, 0.3 * rng.standard_normal(12))
    return m


def tv_planes(s, si, m, k):
    """examples/quadrotor_tv_linear_constraints.cpp in spirit: two state and one input plane per knot, moving with step k"""
    N = m.N
    Ax = np.zeros((2 * N, 12))
    for i in range(N):
        Ax[2 * i, 0] = 1.0; Ax[2 * i, 1] = 0.1 * (i + k)
        Ax[2 * i + 1, 2] = -1.0; Ax[2 * i + 1, 1] = 0.3
    bx = np.stack([0.2 - 0.01 * k + 0.02 * np.sin(np.arange(N)), 0.1 + 0.02 * np.cos(np.arange(N) + k)])
    Au = np.tile([[1.0, -1.0, 1.0, 0.5]], (N - 1, 1)) * (1.0 + 0.1 * np.arange(N - 1))[:, None]
    bu = 0.3 + 0.02 * k + np.zeros((1, N - 1))
    return s.tv_linear(si, Ax, bx, Au, bu)


# ---- shapes --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("N", [10, 33])
def test_every_compiled_shape_closed_loop(N, tmp_path):
    """Every compiled (nx, nu) in a warm-started closed loop with bounds that bite; steps that converge and steps capped at
    several max_iter values, check_termination 1 to 3.  Also the shim's own tiny_setup cache against the reference's."""
    s = S.Script()
    rng = np.random.default_rng(N)
    for k, (nx, nu) in enumerate(TM_DIMS):
        m = lti(nx, nu, N, seed=k)
        s.setup(0, m)
        box(s, 0, m)
        s.update_settings(0, max_iter=150, abs_pri_tol=1e-2, abs_dua_tol=1e-2, check_termination=1 + k % 3)
        s.xref(0, 0.5 * rng.standard_normal((nx, N))).x0(0, 1.5 * rng.standard_normal(nx))
        loop(s, 0, 2)
        s.update_settings(0, max_iter=4 + k)
        loop(s, 0, 2)
        s.update_settings(0, max_iter=150)
        loop(s, 0, 2)
    ref, _ = compare(s, tmp_path, f"shapes_N{N}")
    t = S.trees(ref)
    iters = [int(r["iter"][0, 0]) for r in t]
    solved = [int(r["solved"][0, 0]) for r in t]
    assert 0 < sum(solved) < len(t) and len(set(iters)) >= 10, (iters, solved)
    assert max(float(np.abs(r["u"]).max()) for r in t) >= 1.0  # the input bound is active


# ---- settings between solves ---------------------------------------------------------------------------------------

def test_settings_changed_between_solves(tmp_path):
    """check_termination 1 / 2 / 3 / 5, tolerances that flip convergence, max_iter 0 / 1 / below check_termination (the tree
    keeps the previous solve's residuals when no check ran), and box, cone and plane families switched off and on again,
    through tiny_update_settings and through direct writes into solver->settings."""
    s = S.Script()
    m = lti(12, 4, 20, seed=7)
    rng = np.random.default_rng(3)
    s.setup(0, m)
    box(s, 0, m)
    s.update_settings(0, max_iter=150, abs_pri_tol=1e-2, abs_dua_tol=1e-2)
    s.xref(0, 0.5 * rng.standard_normal((12, 20))).x0(0, 1.5 * rng.standard_normal(12))
    for c in (1, 2, 3, 5):
        s.update_settings(0, check_termination=c)
        loop(s, 0, 1)
    s.update_settings(0, api=False, abs_pri_tol=0.3, abs_dua_tol=0.3)  # converges at once
    loop(s, 0, 1)
    s.update_settings(0, abs_pri_tol=1e-7, abs_dua_tol=1e-7)  # does not converge
    loop(s, 0, 1)
    s.update_settings(0, abs_pri_tol=1e-2, abs_dua_tol=1e-2)
    no_check = []
    for mi, c in ((0, 1), (1, 2), (2, 3), (1, 1), (2, 5)):  # every one but (1, 1) runs no termination check
        s.update_settings(0, api=False, max_iter=mi, check_termination=c)
        loop(s, 0, 1)
        no_check.append(mi < c)
    s.update_settings(0, max_iter=150, check_termination=1)
    s.update_settings(0, api=False, en_state_bound=0)
    loop(s, 0, 2)
    s.update_settings(0, api=False, en_input_bound=0)
    loop(s, 0, 1)
    s.update_settings(0, en_state_bound=1, en_input_bound=1)
    loop(s, 0, 2)
    # cones and planes on a second solver: switched off for two steps, then on again with the state they left behind
    r = rocket_start(s, 1, 12, seed=4)
    loop(s, 1, 2)
    s.update_settings(1, api=False, en_state_soc=0)
    loop(s, 1, 2)
    s.update_settings(1, en_state_soc=1, en_input_soc=0)
    loop(s, 1, 1)
    s.update_settings(1, en_input_soc=1)
    loop(s, 1, 2)
    planes_start(s, 2, 10, seed=5)
    loop(s, 2, 2)
    s.update_settings(2, en_state_linear=0)
    loop(s, 2, 2)
    s.update_settings(2, api=False, en_state_linear=1, en_input_linear=0)
    loop(s, 2, 1)
    s.update_settings(2, en_input_linear=1)
    loop(s, 2, 2)
    assert r.nx == 6
    ref, _ = compare(s, tmp_path, "settings")
    t0 = [r for r in S.trees(ref) if r["solver"] == 0]
    res = lambda r: np.array([r[f][0, 0] for f in ("primal_residual_state", "dual_residual_state",  # noqa: E731
                                                    "primal_residual_input", "dual_residual_input")])
    k0 = 6  # the five no-check / short solves follow six solves
    for j, nc in enumerate(no_check):
        cur, prev = t0[k0 + j], t0[k0 + j - 1]
        if nc:  # the previous solve's residuals, not zeros
            assert np.array_equal(res(cur), res(prev)) and res(cur).any(), j
    sv = [int(r["solved"][0, 0]) for r in t0[:6]]
    assert sv[4] == 1 and sv[5] == 0, sv


# ---- constraints re-set mid-run ------------------------------------------------------------------------------------

def test_bounds_reset_mid_run(tmp_path):
    """Time-varying bounds re-set every step, bounds at +-0 on some rows and knots, on two shapes (on-chip kernel)."""
    s = S.Script()
    rng = np.random.default_rng(8)
    for si, (nx, nu, N) in enumerate(((8, 4, 15), (16, 2, 12))):
        m = lti(nx, nu, N, seed=20 + si)
        s.setup(si, m)
        s.update_settings(si, max_iter=120, abs_pri_tol=1e-2, abs_dua_tol=1e-2)
        s.xref(si, 0.5 * rng.standard_normal((nx, N))).x0(si, 1.5 * rng.standard_normal(nx))
        for k in range(6):
            xw = 2.0 + 0.5 * np.sin(np.arange(N)[None, :] * 0.7 + k + np.arange(nx)[:, None])
            uw = np.full((nu, N - 1), 0.8 - 0.05 * k)
            xmin, xmax, umin, umax = -xw, xw.copy(), -uw, uw.copy()
            xmin[0, :3] = -0.0; xmax[0, :3] = 0.0  # a state pinned at +-0
            umin[nu - 1, k % (N - 1)] = 0.0; umax[nu - 1, k % (N - 1)] = -0.0
            s.bounds(si, xmin, xmax, umin, umax)
            loop(s, si, 1)
    compare(s, tmp_path, "bounds")


def test_cones_reset_mid_run(tmp_path):
    """Cones re-set with a different mu, start and count: 1 to 4 per side, overlapping starts, input cones on nu = 3 and 4,
    mu from 0.02 to 2 so that the below-cone, in-cone and outside-cone branches of project_soc all occur; nonzero Uref."""
    s = S.Script()
    rocket_start(s, 0, 15, seed=1)
    loop(s, 0, 2)
    s.cones(0, [0, 3, 1], [3, 3, 3], [0.1, 2.0, 0.6], [0, 0], [3, 3], [0.05, 1.5])
    loop(s, 0, 3)
    s.cones(0, [0, 1, 2, 3], [3, 3, 3, 3], [0.3, 0.05, 1.0, 0.2], [0], [3], [0.02])
    loop(s, 0, 3)
    s.cones(0, [3], [3], [0.5], [0], [3], [0.5])  # on the velocity, whose last entry is negative: below the cone at times
    loop(s, 0, 2)
    m = lti(16, 4, 12, seed=9)
    rng = np.random.default_rng(9)
    s.setup(1, m)
    box(s, 1, m, 4.0, 1.5)
    s.update_settings(1, max_iter=100, abs_pri_tol=1e-2, abs_dua_tol=1e-2, en_state_soc=1, en_input_soc=1)
    s.xref(1, 0.5 * rng.standard_normal((16, 12))).uref(1, 0.3 * np.ones((4, 11))).x0(1, rng.standard_normal(16))
    s.cones(1, [0, 5, 13], [3, 3, 3], [0.2, 1.2, 0.05], [1], [3], [0.3])
    loop(s, 1, 3)
    s.cones(1, [0, 4], [3, 3], [0.02, 0.7], [0, 1], [3, 3], [0.4, 0.1])
    loop(s, 1, 3)
    ref, _ = compare(s, tmp_path, "cones")
    # which project_soc branch the last iteration took on the single-cone steps: the slack before projection is the
    # projected slack plus the dual (vcnew + gc), so Z = below (projected to 0), I = inside (unchanged), O = outside
    t0 = [r for r in S.trees(ref) if r["solver"] == 0]
    seen = set()
    for r, start in [(r, 0) for r in t0[:2]] + [(r, 3) for r in t0[-2:]]:
        for v, g, a in ((r["vcnew"], r["gc"], start), (r["zcnew"], r["yc"], 0)):
            for i in range(v.shape[1]):
                b, pre = v[a:a + 3, i], v[a:a + 3, i] + g[a:a + 3, i]
                seen.add("Z" if not b.any() else ("I" if np.array_equal(b, pre) else "O"))
    assert seen == {"Z", "I", "O"}, seen


def test_planes_reset_mid_run(tmp_path):
    """Static planes with several rows and all-zero padding rows, re-set; time-varying planes updated every step; then all
    families together (box, cones, static and time-varying planes) with a nonzero Uref."""
    s = S.Script()
    planes_start(s, 0, 10, seed=2)
    loop(s, 0, 2)
    Ax = np.zeros((3, 12)); Ax[0, 0] = 1.0; Ax[1, 3] = 1.0; Ax[1, 4] = -0.5
    s.linear(0, Ax, [0.1, 0.05, 0.0], np.array([[1.0, 1.0, 1.0, 1.0], [0.0, 0.0, 0.0, 0.0]]), [0.2, 0.5])
    loop(s, 0, 3)
    m = planes_start(s, 1, 12, seed=3, tv=True)
    for k in range(6):
        tv_planes(s, 1, m, k)
        loop(s, 1, 1)
    # everything at once
    m = planes_start(s, 2, 10, seed=4)
    s.update_settings(2, en_state_bound=1, en_input_bound=1, en_state_soc=1, en_input_soc=1, en_tv_state_linear=1,
                      en_tv_input_linear=1, max_iter=80)
    s.bounds(2, np.full((12, 10), -2.0), np.full((12, 10), 2.0), np.full((4, 9), -1.0), np.full((4, 9), 1.0))
    s.cones(2, [0, 6], [3, 3], [0.5, 0.1], [1], [3], [0.8])
    s.uref(2, 0.1 * np.ones((4, 9)))
    for k in range(5):
        tv_planes(s, 2, m, k)
        loop(s, 2, 1)
    compare(s, tmp_path, "planes")


# ---- state and cache pokes -----------------------------------------------------------------------------------------

def test_workspace_and_cache_pokes(tmp_path):
    """Sliding Xref windows through tiny_set_x_ref and through work->Xref, the examples' dual reset, overwritten v / z,
    constraint counts lowered with unchanged matrices (the reference loops to the counts) and raised again, and a mid-run
    tiny_precompute_and_set_cache with a new rho followed by the reference's cache for it."""
    s = S.Script()
    N = 12
    m = lti(12, 4, N, seed=11)
    rng = np.random.default_rng(11)
    traj = rng.standard_normal((12, N + 20)).cumsum(axis=1) * 0.1
    s.setup(0, m)
    box(s, 0, m, 2.5, 0.8)
    Ax = np.zeros((3, 12)); Ax[0, 0] = 1.0; Ax[1, 1] = 1.0; Ax[2, 0] = -1.0; Ax[2, 2] = 1.0
    Au = np.array([[1.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, -1.0]])
    s.linear(0, Ax, [0.2, 0.1, 0.1], Au, [0.3, 0.2])
    s.cones(0, [0, 3], [3, 3], [0.3, 0.2], [0, 1], [3, 3], [0.4, 0.25])
    s.update_settings(0, max_iter=100, abs_pri_tol=1e-2, abs_dua_tol=1e-2, en_state_soc=1, en_input_soc=1, en_state_linear=1,
                      en_input_linear=1)
    s.x0(0, traj[:, 0] + 0.5)
    for k in range(4):  # sliding windows, alternately through the setter and through work->Xref
        w = traj[:, k:k + N]
        (s.xref(0, w) if k % 2 == 0 else s.poke(0, "Xref", w))
        loop(s, 0, 1)
    for f in ("g", "y", "gc", "yc", "gl", "yl"):  # the dual reset of examples/quadrotor_tracking.cpp
        s.poke(0, f, np.zeros((12, N)) if f[0] == "g" else np.zeros((4, N - 1)))
    loop(s, 0, 1)
    s.poke(0, "v", 0.1 * rng.standard_normal((12, N))).poke(0, "z", 0.1 * rng.standard_normal((4, N - 1)))
    s.poke(0, "Uref", 0.05 * np.ones((4, N - 1)))
    loop(s, 0, 2)
    s.poke_counts(0, 1, 1, 1, 1, 0, 0)  # the handle exists: the lower counts must reach it
    loop(s, 0, 2)
    s.poke_counts(0, 2, 2, 3, 2, 0, 0)
    loop(s, 0, 1)
    s.precompute(0, 3.0 * m.rho)  # the shim's own cache (within the precompute bound), then the reference's
    loop(s, 0, 2)
    s.precompute(0, m.rho)
    loop(s, 0, 1)
    compare(s, tmp_path, "pokes")


# ---- two solvers, batch, threads -----------------------------------------------------------------------------------

def test_two_solvers_interleaved(tmp_path):
    """A box solver (on-chip kernel) and a cone solver (streamed kernel) of different shapes, interleaved op by op."""
    s = S.Script()
    m0 = lti(8, 4, 15, seed=13)
    rng = np.random.default_rng(13)
    s.setup(0, m0)
    rocket_start(s, 1, 10, seed=13)
    box(s, 0, m0)
    s.update_settings(0, max_iter=100, abs_pri_tol=1e-2, abs_dua_tol=1e-2)
    s.xref(0, 0.5 * rng.standard_normal((8, 15))).x0(0, 1.5 * rng.standard_normal(8))
    for k in range(8):
        s.solve(0).solve(1).plant(1).plant(0)
        if k == 3:
            s.update_settings(1, max_iter=9)
            s.update_settings(0, check_termination=2)
    compare(s, tmp_path, "two")


def test_solve_batch_matches_cold_reference_solves(tmp_path):
    """tiny_solve_batch (B = 300, an Xref per column, the solver's Uref) against per-column cold reference solves: u0, iter
    and solved bit for bit; the calling solver's tree is left untouched and its next warm solve is unaffected."""
    s = S.Script()
    N, B = 15, 300
    m = lti(12, 4, N, seed=17)
    rng = np.random.default_rng(17)
    s.setup(0, m)
    box(s, 0, m, 3.0, 0.9)
    s.update_settings(0, max_iter=150, abs_pri_tol=1e-2, abs_dua_tol=1e-2)
    s.xref(0, 0.5 * rng.standard_normal((12, N))).uref(0, 0.1 * np.ones((4, N - 1))).x0(0, rng.standard_normal(12))
    loop(s, 0, 2)
    X = 0.5 * rng.standard_normal((B, N, 12))
    s.dump(0).batch(0, 1.5 * rng.standard_normal((12, B)), X.reshape(B, -1).T).dump(0)
    loop(s, 0, 2)
    ref, got = compare(s, tmp_path, "batch")
    b = [r for r in got if r["kind"] == "batch"][0]
    it = b["iter"][:, 0]
    assert len(np.unique(it)) >= 5 and 0 < b["solved"].sum() < B
    dumps = [r for r in got if r["kind"] == "tree" and r["rc"] == -1]
    for f in S.TREE_FIELDS:
        assert np.array_equal(dumps[0][f], dumps[1][f]), f


def thread_scripts():
    """8 independent streams: box loops on the on-chip kernel, cones and planes on the streamed one"""
    out = []
    for k, (nx, nu) in enumerate(((4, 1), (8, 4), (12, 4), (16, 8))):
        s = S.Script()
        m = lti(nx, nu, 20, seed=30 + k)
        rng = np.random.default_rng(30 + k)
        s.setup(0, m)
        box(s, 0, m)
        s.update_settings(0, max_iter=120, abs_pri_tol=1e-2, abs_dua_tol=1e-2, check_termination=1 + k % 2)
        s.xref(0, 0.5 * rng.standard_normal((nx, 20))).x0(0, 1.5 * rng.standard_normal(nx))
        out.append(loop(s, 0, 8))
    for k in range(2):
        s = S.Script()
        rocket_start(s, 0, 12 + 4 * k, seed=40 + k)
        out.append(loop(s, 0, 8))
    for k in range(2):
        s = S.Script()
        m = planes_start(s, 0, 10, seed=50 + k, tv=bool(k))
        for j in range(8):
            if k:
                tv_planes(s, 0, m, j)
            loop(s, 0, 1)
        out.append(s)
    return out


def test_one_solver_per_thread(tmp_path):
    """8 solvers on 8 threads at once (INTEGRATION.md §2: one TinySolver per thread is safe), each stream's records equal to
    the reference running that stream alone."""
    scripts = thread_scripts()
    got = S.run_threads(S.SCRIPT_SHIM, scripts, str(tmp_path), "thr")
    for k, s in enumerate(scripts):
        ref, _ = S.run(S.SCRIPT_REF, s, str(tmp_path), f"thr_ref{k}")
        S.assert_same_records(ref, got[k], f"thread {k}")


# ---- loud errors (the reference has no defined behaviour to compare with) ------------------------------------------

def test_rejected_settings_and_counts_fail_loudly(tmp_path):
    """check_termination = 0 (an integer division by zero in the reference) and a constraint count above the rows of its
    matrix (a read past the matrix there): tiny_solve and tiny_solve_batch return 1, say why, and leave the tree as it was;
    the next valid solve runs as if the failed ones had not happened."""
    s = S.Script()
    m = lti(8, 2, 12, seed=60)
    rng = np.random.default_rng(60)
    s.setup(0, m)
    box(s, 0, m)
    s.xref(0, 0.5 * rng.standard_normal((8, 12))).x0(0, rng.standard_normal(8))
    s.update_settings(0, max_iter=100, abs_pri_tol=1e-2, abs_dua_tol=1e-2)
    loop(s, 0, 1)
    s.dump(0)
    s.update_settings(0, api=False, check_termination=0)
    s.solve(0)
    s.batch(0, rng.standard_normal((8, 4)), 0.5 * rng.standard_normal((8 * 12, 4)))
    s.update_settings(0, check_termination=1, en_state_linear=1)
    s.poke_counts(0, 0, 0, 2, 0, 0, 0)  # two state planes, no rows
    s.solve(0)
    s.poke_counts(0, 0, 0, 0, 0, 0, 0)
    s.update_settings(0, en_state_linear=0)
    s.solve(0)
    recs, ops = S.run(S.SCRIPT_SHIM, s, str(tmp_path), "loud")
    dump, bad_set, bad_batch, bad_cnt, ok = recs[-5:]
    assert bad_set["rc"] == 1 and bad_batch["rc"] == 1 and bad_cnt["rc"] == 1 and ok["rc"] in (0, 1)
    for bad in (bad_set, bad_cnt):
        for f in S.TREE_FIELDS:
            assert np.array_equal(bad[f], dump[f]), f
    printed = ["\n".join(v) for v in ops.values()]
    assert sum("check_termination must be >= 1" in p for p in printed) == 2
    assert sum("numStateLinear" in p for p in printed) == 1
    # the valid solve after them equals the reference's solve from the same tree (the failed ops are absent there)
    t = S.Script()
    t.setup(0, m)
    box(t, 0, m)
    rng = np.random.default_rng(60)
    t.xref(0, 0.5 * rng.standard_normal((8, 12))).x0(0, rng.standard_normal(8))
    t.update_settings(0, max_iter=100, abs_pri_tol=1e-2, abs_dua_tol=1e-2)
    loop(t, 0, 1)
    t.solve(0)
    ref, _ = S.run(S.SCRIPT_REF, t, str(tmp_path), "loud_ref")
    last = S.trees(ref)[-1]
    for f in S.TREE_FIELDS:
        assert S.H.bits_equal(last[f], ok[f]), f
