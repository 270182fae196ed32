"""Routing matrix of per-instance data (models, box bounds, cone coefficients, static hyperplanes): for every case, what the C
ABI returns and, on success, which kernel family ran with how many lanes per instance.

The cases cross five problems (box-only quadrotor at N = 50 and N = 1000, the fp64 conic rocket, the hyperplane quadrotor, the
rocket with cones and hyperplanes), each with its constraint families on and switched off, with per-instance models x bounds
0/1/2 x cones 0/1 x planes 0/1, both modes, every kernel family and four entry points (tinympc_b200_solve, _solve_host,
_solve_adaptive and _rollout).  Every instance brings the problem's own data, so only the routing is under test; the outputs
are held bit for bit by the per-kind test files.  The batch holds every array a problem has whatever its flags say, so a flag
set on a family whose loop does not run is a case of its own.

The expected (return code, last_error) or (kernel_family, lanes_per_instance) of every case are literal, in
tests/golden/per_instance_routing.json; a case id reads problem/settings/entry/mode/family/m<models>b<bounds>c<cones>p<planes>."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import helpers as H
from tinympc_b200 import abi, workloads as wl
from tinympc_b200.solver import BatchedTinySolver, pack_models, setup_problem

pytestmark = pytest.mark.gpu

B = 64
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "per_instance_routing.json")
MODES = {"strict": abi.MODE_STRICT, "fast": abi.MODE_FAST}
FAMILIES = {"auto": abi.KERNEL_AUTO, "gpi": abi.KERNEL_GPI, "gps": abi.KERNEL_GPS, "tpi": abi.KERNEL_TPI}
ENTRIES = ("solve", "host", "adaptive", "rollout")
BOX_OFF = dict(en_state_bound=0, en_input_bound=0)
BOX_ON = dict(en_state_bound=1, en_input_bound=1)
SOC_OFF = dict(en_state_soc=0, en_input_soc=0)
LIN_OFF = dict(en_state_linear=0, en_input_linear=0)


def _rocket_planes(N):
    """the conic rocket with one static state and one input hyperplane"""
    spec = wl.rocket(N=N)
    spec.constraints = dict(spec.constraints, Alin_x=np.array([[1.0, 0.5, 0.0, 0.0, 0.0, 0.0]]), blin_x=np.array([1.0]),
                            Alin_u=np.array([[1.0, 1.0, 0.0]]), blin_u=np.array([4.0]))
    spec.settings.en_state_linear = 1
    spec.settings.en_input_linear = 1
    return spec


# name -> (spec factory, dtype, settings variants)
PROBLEMS = {
    "quad50": (lambda: wl.quadrotor(N=50), np.float32, {"on": {}, "box_off": BOX_OFF}),
    "quad1000": (lambda: wl.quadrotor(N=1000), np.float32, {"on": {}, "box_off": BOX_OFF}),
    "rocket": (lambda: wl.rocket(N=20), np.float64, {"on": {}, "box_off": BOX_OFF, "soc_off": SOC_OFF}),
    "quadplanes": (lambda: H.quad_linear_spec(N=20), np.float32, {"on": {}, "lin_off": LIN_OFF, "box_on": BOX_ON}),
    "rocketplanes": (lambda: _rocket_planes(20), np.float64, {"on": {}, "soc_off": SOC_OFF, "lin_off": LIN_OFF}),
}
DATA = [(m, b, c, p) for m in (0, 1) for b in (0, 1, 2) for c in (0, 1) for p in (0, 1)]


def _cases():
    """every case id; STRICT AUTO solves in full, the rest a fixed sample plus the combinations no per-kind file covers"""
    full, rest = [], []
    for prob in PROBLEMS:
        for sett in PROBLEMS[prob][2]:
            for entry in ENTRIES:
                for mode in MODES:
                    for fam in FAMILIES:
                        for m, b, c, p in DATA:
                            cid = f"{prob}/{sett}/{entry}/{mode}/{fam}/m{m}b{b}c{c}p{p}"
                            (full if (entry, mode, fam) == ("solve", "strict", "auto") else rest).append(cid)
    must = [cid for cid in rest if _matters(cid)]
    pick = np.random.default_rng(2026).choice(len(rest), 150, replace=False)
    return full + sorted(set(must) | {rest[i] for i in pick}, key=rest.index)


def _matters(cid):
    """a flag set on a family whose loop does not run, with per-instance bounds, adaptive rho, a rollout or FAST; models +
    bounds + cones with a loop switched off"""
    prob, sett, entry, mode, fam, d = cid.split("/")
    m, b, c, p = (int(d[i]) for i in (1, 3, 5, 7))
    if fam != "auto":
        return False
    idle = (c and (prob in ("quad50", "quad1000", "quadplanes") or sett == "soc_off")) or \
           (p and (prob in ("quad50", "quad1000", "rocket") or sett == "lin_off"))
    if idle and mode == "strict":
        return (b and entry in ("solve", "host")) or (not m and not b and entry in ("adaptive", "rollout"))
    if idle:
        return not m and entry == "solve"
    return bool(m and b == 1 and c and not p and sett != "on" and entry == "solve" and mode == "strict")


def _abi_data(prob):
    """every per-instance array of the problem in ABI layout, each instance holding the problem's own values"""
    dt, nx, nu, N = prob.dtype, prob.nx, prob.nu, prob.N
    rep = lambda a: np.ascontiguousarray(np.broadcast_to(np.asarray(a, dt), (B,) + np.shape(a)))  # noqa: E731

    def box(a, n, k, lim):
        a = np.full((n, k), lim) if a is None else np.asarray(a).reshape(n, k)
        return rep(a[:, 0]), rep(a.T)

    d = {"models": pack_models(prob, B)}
    for key, a, n, k, lim in (("x_min", prob.x_min, nx, N, -10.0), ("x_max", prob.x_max, nx, N, 10.0),
                              ("u_min", prob.u_min, nu, N - 1, -10.0), ("u_max", prob.u_max, nu, N - 1, 10.0)):
        d[key + "/1"], d[key + "/2"] = box(a, n, k, lim)
    if len(prob.cx):
        d["cone_x_mu"] = rep(prob.cx)
    if len(prob.cu):
        d["cone_u_mu"] = rep(prob.cu)
    for side in ("x", "u"):
        A = getattr(prob, "Alin_" + side)
        if A is not None:
            d["Alin_" + side] = rep(np.asarray(A).T)  # [nx][n]: each instance's n x nx matrix column-major
            d["blin_" + side] = rep(np.asarray(getattr(prob, "blin_" + side)).reshape(-1))
    return d


class _Problem:
    """one handle per problem and settings variant, with every buffer its cases need on the host and on the device"""

    def __init__(self, name, sett):
        import torch

        spec_fn, dt, variants = PROBLEMS[name]
        spec = spec_fn()
        self.prob = setup_problem(spec, dt)
        st = abi.Settings.from_buffer_copy(spec.settings)
        st.max_iter = 2
        for k, v in variants[sett].items():
            setattr(st, k, v)
        self.s = BatchedTinySolver(self.prob, st)
        p = self.prob
        rng = np.random.default_rng(7)
        self.host = dict(_abi_data(p), x0=(0.1 * rng.standard_normal((B, p.nx))).astype(dt), Xref=np.zeros((p.N, p.nx), dt),
                         sol_x=np.zeros((B, p.N, p.nx), dt), sol_u=np.zeros((B, p.N - 1, p.nu), dt),
                         iter=np.zeros(B, np.int32), solved=np.zeros(B, np.int32), residuals=np.zeros((B, 4), dt),
                         dK=np.zeros((p.nu, p.nx), dt), dP=np.zeros((p.nx, p.nx), dt))
        for n in ("vnew", "znew", "g", "y"):
            self.host[n] = np.zeros((B, p.N, p.nx) if abi.STATE_IS_X[n] else (B, p.N - 1, p.nu), dt)
        for n, shape, t in (("x_traj", (B, 2, p.nx), dt), ("u_traj", (B, 1, p.nu), dt), ("res_traj", (B, 1, 4), dt),
                            ("iter_traj", (B, 1), np.int32), ("solved_traj", (B, 1), np.int32)):
            self.host[n] = np.zeros(shape, t)
        self.dev = {k: torch.as_tensor(v, device="cuda") for k, v in self.host.items()}

    def run(self, entry, mode, fam, m, b, c, p):
        import torch

        s = self.s
        s.set_mode(MODES[mode], FAMILIES[fam])
        on_host = entry == "host"
        ptr = (lambda k: self.host[k].ctypes.data) if on_host else (lambda k: self.dev[k].data_ptr())
        io = abi.Batch()
        io.B, io.x0, io.cold_start = B, ptr("x0"), 1
        io.sol_x, io.sol_u = ptr("sol_x"), ptr("sol_u")
        if entry != "rollout":
            io.Xref, io.iter, io.solved, io.residuals = ptr("Xref"), ptr("iter"), ptr("solved"), ptr("residuals")
        for n in ("vnew", "znew", "g", "y"):
            setattr(io.state, n, ptr(n))
        io.models = ptr("models") if m else None
        io.bounds_per_instance = b
        for k in ("x_min", "x_max", "u_min", "u_max"):
            setattr(io, k, ptr(f"{k}/{b or 1}"))
        io.cones_per_instance = c
        io.planes_per_instance = p
        for k in ("cone_x_mu", "cone_u_mu", "Alin_x", "blin_x", "Alin_u", "blin_u"):
            setattr(io, k, ptr(k) if k in self.host else None)
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        if entry == "solve":
            rc = s._lib.tinympc_b200_solve(s._h, C.byref(io), stream)
        elif entry == "host":
            rc = s._lib.tinympc_b200_solve_host(s._h, C.byref(io))
        elif entry == "adaptive":
            ar = abi.AdaptiveRho()
            ar.rho_min, ar.rho_max, ar.enable_clipping = 1.0, 100.0, 1
            ar.models = self.dev["models"].data_ptr()
            ar.dKinf_drho, ar.dPinf_drho = self.host["dK"].ctypes.data, self.host["dP"].ctypes.data
            rc = s._lib.tinympc_b200_solve_adaptive(s._h, C.byref(io), C.byref(ar), stream)
        else:
            ro = abi.Rollout()
            ro.T, ro.Xref, ro.xref_per_instance = 1, self.dev["Xref"].data_ptr(), 0
            ro.x_traj, ro.u_traj, ro.residuals_traj = ptr("x_traj"), ptr("u_traj"), ptr("res_traj")
            ro.iter_traj, ro.solved_traj = ptr("iter_traj"), ptr("solved_traj")
            rc = s._lib.tinympc_b200_rollout(s._h, C.byref(io), C.byref(ro), stream)
        torch.cuda.synchronize()
        if rc != abi.OK:
            return [rc, s._lib.tinympc_b200_last_error().decode()]
        st = s.stats()
        return [rc, st["kernel_family"], st["lanes_per_instance"]]


def observe(cases):
    """case id -> observed result, one handle per problem and settings variant"""
    out, handles = {}, {}
    for cid in cases:
        prob, sett, entry, mode, fam, d = cid.split("/")
        if (prob, sett) not in handles:
            handles[(prob, sett)] = _Problem(prob, sett)
        out[cid] = handles[(prob, sett)].run(entry, mode, fam, *(int(d[i]) for i in (1, 3, 5, 7)))
    for h in handles.values():
        h.s.close()
    return out


def test_routing_matrix():
    with open(GOLDEN) as f:
        want = json.load(f)
    cases = _cases()
    assert sorted(cases) == sorted(want), "the case list and the expectations differ"
    got = observe(cases)
    bad = {cid: (got[cid], want[cid]) for cid in cases if got[cid] != want[cid]}
    assert not bad, f"{len(bad)} of {len(cases)} cases differ (got, want): " + json.dumps(dict(list(bad.items())[:20]), indent=1)
