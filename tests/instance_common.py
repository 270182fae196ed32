"""Per-instance data of a batch (tinympc_batch_t's bounds_per_instance, cones_per_instance and planes_per_instance) for the
tests: palettes of bound sets, cone coefficients and plane sets dealt to the instances of a batch, the oracle run once per
distinct (model, arrays) over the instances that use them, and the solve paths and scenarios the GPU suites share.

Instance b of a solve with per-instance data computes what one TinySolver computes after tiny_set_bound_constraints,
tiny_set_cone_constraints or tiny_set_linear_constraints got that instance's arrays; everything else (the cone structure,
the row counts, the settings) is the problem's.  The oracle's problem takes the arrays of one such solver, so a batch whose
instances use K distinct sets is checked with K oracle runs, not B.

On the GPU, outputs and, on cold starts, the requested state arrays are filled with a NaN bit pattern before each solve
(H.poison), so an element a solve never writes cannot match an oracle value by accident."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import helpers as H
from adaptive_common import advance
from oracle import oracle
from tinympc_b200 import abi
from tinympc_b200.batch import BOUND_NAMES, KINDS, PLANE_NAMES, HostBatch
from tinympc_b200.problem import MPCProblem
from tinympc_b200.solver import AdaptiveRho, pack_models, unpack_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NT = os.cpu_count() or 1
OUTS = ("sol_x", "sol_u", "iter", "solved", "residuals", "u0")
DIMS = [(4, 1), (6, 3), (12, 4), (4, 2), (4, 4), (4, 8), (8, 2), (8, 4), (8, 8), (12, 2), (12, 8), (16, 2), (16, 4), (16, 8)]
PLAN = ("kernel_family", "lanes_per_instance", "instances_per_cta", "threads_per_cta", "ctas")


# the last tinympc_batch_t field before each kind's fields, and the reserved field after its mode: each kind was appended to
# the layout before it, so every earlier offset stayed where it was
BEFORE = dict(bounds="models", cones="reserved2", planes="reserved3")
RESERVED = dict(bounds="reserved2", cones="reserved3", planes="reserved4")


def assert_batch_fields_match_header(kind):
    """the ctypes mirror of a kind's tinympc_batch_t fields (batch.KINDS: its arrays and mode, then its reserved field) has the
    header's offsets, comes after the fields before it, and a zero-initialised batch holds no pointer and mode 0 (the
    handle's own data)"""
    spec = KINDS[kind]
    fields = [BEFORE[kind], *spec.fields.values(), spec.mode_field, RESERVED[kind]]
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"tinympc_b200.h\"\nint main(void){\n"
    src += '  printf("%zu\\n", sizeof(tinympc_batch_t));\n'
    src += "".join(f'  printf("%zu\\n", offsetof(tinympc_batch_t, {n}));\n' for n in fields)
    src += "  return 0; }\n"
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "probe.c")
        open(c, "w").write(src)
        exe = os.path.join(td, "probe")
        subprocess.check_call(["/usr/bin/gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = list(map(int, subprocess.check_output([exe], text=True).split()))
    assert out[0] == C.sizeof(abi.Batch)
    assert out[1:] == [getattr(abi.Batch, n).offset for n in fields]
    before = getattr(abi.Batch, BEFORE[kind])
    assert getattr(abi.Batch, fields[1]).offset >= before.offset + before.size
    b = abi.Batch()
    assert getattr(b, spec.mode_field) == 0 and getattr(b, RESERVED[kind]) == 0
    assert all(getattr(b, f) is None for f in spec.fields.values())


# ---------------------------------------------------------------------------------------------------------------------
# palettes and the batch arrays
# ---------------------------------------------------------------------------------------------------------------------
def deal(B, K, stride=7):
    """set of every instance: neighbouring instances (and so neighbouring slots and the refills of a slot) get different
    sets.  stride and K are coprime, so every set is used."""
    assert np.gcd(stride, K) == 1
    return (np.arange(B) * stride) % K


def palette(prob, K, layout, seed, scale=1.0, tight=0.0, zeros=False):
    """K bound sets around the problem's own bounds, in the per-instance layout: layout 1 gives x [nx] / u [nu], layout 2
    x [N, nx] / u [N-1, nu] columns that vary with k and between sets.  Each set scales the problem's column 0 by a factor in
    [scale * (1 - tight), scale], so small factors bite.  zeros: every third row of each set's bounds at -0 / +0 (mins / maxes),
    where slacks land on them."""
    rng = np.random.default_rng(seed)
    dt = prob.dtype
    N = prob.N
    out = []
    for s in range(K):
        d = {}
        for side, n, kn in (("x", prob.nx, N), ("u", prob.nu, N - 1)):
            lo0, hi0 = getattr(prob, side + "_min"), getattr(prob, side + "_max")
            lo0 = np.full(n, -5.0) if lo0 is None else np.asarray(lo0, np.float64)[:, 0]
            hi0 = np.full(n, 5.0) if hi0 is None else np.asarray(hi0, np.float64)[:, 0]
            f = scale * (1.0 - tight * rng.random(n))
            lo, hi = lo0 * f, hi0 * f
            if layout == 2:
                wob = 1.0 + 0.3 * np.sin(0.37 * np.arange(kn)[:, None] + 1.3 * s + np.arange(n)[None, :])
                lo, hi = lo[None, :] * wob, hi[None, :] * wob
            if zeros:
                lo[..., s % 3::3] = -0.0
                hi[..., (s + 1) % 3::3] = 0.0
            d[side + "_min"] = np.ascontiguousarray(lo, dtype=dt)
            d[side + "_max"] = np.ascontiguousarray(hi, dtype=dt)
        out.append(d)
    return out


def equal_palette(prob, layout):
    """one bound set equal to the problem's own bounds (layout 1: column 0, which is every column of a constant box)"""
    d = {}
    for k in BOUND_NAMES:
        a = np.asarray(getattr(prob, k))
        d[k] = np.ascontiguousarray(a[:, 0] if layout == 1 else a.T, dtype=prob.dtype)
    return [d]


def batch_bounds(pal, which):
    """the per-instance arrays of a batch whose instance b uses bound set which[b]: [B, n] or [B, N, n]"""
    return {k: np.ascontiguousarray(np.stack([pal[w][k] for w in which])) for k in pal[0]}


def thrust_palette(prob, K, layout, seed):
    """K rockets' thrust limits (the problem's u bounds scaled by 0.6 .. 1.0) and the problem's state bounds"""
    pal = palette(prob, K, layout, seed, scale=1.0, tight=0.4)
    for d in pal:
        for k in ("x_min", "x_max"):
            a = np.asarray(getattr(prob, k))
            d[k] = np.ascontiguousarray(a[:, 0] if layout == 1 else a.T, dtype=prob.dtype)
    return pal


def mu_palette(prob, K, seed, scale=(0.6, 1.0), extra=()):
    """K mu sets: the problem's cx / cu times a factor from U(scale) per set and cone, rounded to the problem dtype.  extra:
    further sets given as (x_mu, u_mu) pairs of plain numbers (e.g. 0.3 and 0.55, which float cannot represent)."""
    rng = np.random.default_rng(seed)
    dt = prob.dtype
    cx, cu = np.asarray(prob.cx, np.float64), np.asarray(prob.cu, np.float64)
    out = [dict(x_mu=(cx * rng.uniform(*scale, size=cx.size)).astype(dt), u_mu=(cu * rng.uniform(*scale, size=cu.size)).astype(dt))
           for _ in range(K)]
    for xm, um in extra:
        out.append(dict(x_mu=np.full(cx.size, xm, dtype=dt), u_mu=np.full(cu.size, um, dtype=dt)))
    return out


def batch_cones(pal, which, sides=("x_mu", "u_mu")):
    """the per-instance arrays of a batch whose instance b uses mu set which[b]: x_mu [B, ncx], u_mu [B, ncu]"""
    return {k: np.ascontiguousarray(np.stack([pal[w][k] for w in which])) for k in sides}


def plane_palette(prob, K, seed, tilt=0.25, shift=(-0.3, 0.1), pad=0):
    """K plane sets around the problem's own static hyperplanes: every non-zero coefficient of row i scaled by a factor from
    U(1 - tilt, 1 + tilt), every offset moved by U(shift), rounded to the problem dtype.  pad: the last `pad` rows of every
    side are a = 0, b = 0 (a robot with fewer planes)."""
    rng = np.random.default_rng(seed)
    dt = prob.dtype
    out = []
    for _ in range(K):
        s = {}
        for side in ("x", "u"):
            A = getattr(prob, "Alin_" + side)
            if A is None:
                continue
            A = np.asarray(A, np.float64) * rng.uniform(1.0 - tilt, 1.0 + tilt, size=A.shape)
            b = np.asarray(getattr(prob, "blin_" + side), np.float64).reshape(-1) + rng.uniform(*shift, size=A.shape[0])
            if pad:
                A[-pad:] = 0.0
                b[-pad:] = 0.0
            s["Alin_" + side], s["blin_" + side] = A.astype(dt), b.astype(dt)
        out.append(s)
    return out


def own_planes(prob):
    """the problem's own plane set"""
    return {k: np.asarray(getattr(prob, k)).reshape(-1) if k.startswith("blin") else np.asarray(getattr(prob, k))
            for k in PLANE_NAMES if getattr(prob, k) is not None}


def batch_planes(pal, which, sides=("x", "u")):
    """the per-instance arrays of a batch whose instance b uses plane set which[b], rows as users write them:
    Alin_x [B, nlx, nx], blin_x [B, nlx], Alin_u [B, nlu, nu], blin_u [B, nlu]"""
    keys = [k for k in PLANE_NAMES if k[-1] in sides and k in pal[0]]
    return {k: np.ascontiguousarray(np.stack([pal[w][k] for w in which])) for k in keys}


# ---------------------------------------------------------------------------------------------------------------------
# the oracle once per distinct (model, arrays)
# ---------------------------------------------------------------------------------------------------------------------
def with_model(prob, blob):
    """prob with the model, cache and rho of one per-instance blob"""
    kw = {k: getattr(prob, k) for k in prob.__dataclass_fields__}
    m = unpack_model(np.asarray(blob), prob.nx, prob.nu)
    kw.update({k: m[k] for k in ("A", "B", "f", "Q", "R", "Kinf", "Pinf", "Quu_inv", "AmBKt", "APf", "BPf")}, rho=m["rho"])
    return MPCProblem(**kw)


def with_instance(prob, kind, arrays):
    """prob with one instance's arrays of a kind (keyed as users pass them to solve(), one instance's row each) in place of its
    own: the problem of one TinySolver.  bounds: the four bounds are replaced together, an absent one unset, a horizon taken
    as [n, N]; cones (x_mu -> cx, u_mu -> cu) and planes: an absent side keeps the problem's."""
    kw = {k: getattr(prob, k) for k in prob.__dataclass_fields__}
    if kind == "bounds":
        kw.update(dict.fromkeys(BOUND_NAMES))
    for k, v in arrays.items():
        if v is not None:
            v = np.asarray(v)
            kw[dict(x_mu="cx", u_mu="cu").get(k, k)] = v.T if kind == "bounds" else v
    return MPCProblem(**kw)


def grouped_oracle(prob, st, models=None, model_of=None, *, bounds=None, cones=None, planes=None, impl="port", nthreads=8):
    """run(x0, Xref, Uref, state, cold, want) -> the oracle's result for the whole batch, one oracle run per distinct
    (model, bound set, mu set, plane set) over the instances that use it.  bounds / cones / planes: the batch's per-instance
    arrays as users pass them to solve(); models / model_of: per-instance models (blob palette and the blob of every
    instance)."""
    kinds = {kind: {k: np.asarray(a) for k, a in arrays.items() if a is not None}
             for kind, arrays in dict(bounds=bounds, cones=cones, planes=planes).items() if arrays is not None}
    given = [a for arrays in kinds.values() for a in arrays.values()]
    B = len(given[0])
    mo = np.zeros(B, np.int64) if model_of is None else np.asarray(model_of, np.int64)
    rows = np.concatenate([np.ascontiguousarray(a).reshape(B, -1).view(np.uint8) for a in [mo] + given], axis=1)
    # each instance's bytes as one opaque record: np.unique(axis=0) would sort a record field per byte, minutes for horizons
    _, key = np.unique(rows.view(np.dtype((np.void, rows.shape[1]))).reshape(-1), return_inverse=True)
    key = key.reshape(-1)
    probs = {}
    for g in np.unique(key):
        b = int(np.flatnonzero(key == g)[0])
        p = prob if models is None else with_model(prob, models[mo[b]])
        for kind, arrays in kinds.items():
            p = with_instance(p, kind, {k: a[b] for k, a in arrays.items()})
        probs[g] = p

    def run(x0, Xref, Uref, state, cold, want):
        out = {}
        for g, p in probs.items():
            idx = np.flatnonzero(key == g)
            sub = None if state is None else {n: np.array(a[idx], copy=True) for n, a in state.items()}
            xr = Xref[idx] if Xref.ndim == 3 else Xref
            ur = None if Uref is None else (Uref[idx] if Uref.ndim == 3 else Uref)
            o = oracle.solve_batch(p, st, x0[idx], xr, ur, state=sub, cold_start=cold, want_state=tuple(want), impl=impl,
                                   nthreads=nthreads)
            for k, v in o.items():
                if v is not None:
                    out.setdefault(k, np.empty((len(x0),) + v.shape[1:], v.dtype))[idx] = v
        return out
    return run


def assert_one_run_per_set(monkeypatch, prob, st, x0, Xref, Uref, which, **kinds):
    """the batch's arrays (kinds), dealt by `which` from sets of which set 0 is the problem's own, are solved with one oracle
    run per set, and the instances of set 0 get the shared result"""
    calls = []
    real = oracle.solve_batch

    def counting(*a, **k):
        calls.append(len(a[2]))
        return real(*a, **k)

    monkeypatch.setattr(oracle, "solve_batch", counting)
    got = grouped_oracle(prob, st, nthreads=2, **kinds)(x0, Xref, Uref, None, True, ())
    monkeypatch.undo()
    assert sorted(calls) == [int(np.sum(which == w)) for w in np.unique(which)], calls
    ref = oracle.solve_batch(prob, st, x0, Xref, Uref, cold_start=True, nthreads=2)
    for k in H.OUT_KEYS:
        assert H.bits_equal(got[k][which == 0], ref[k][which == 0]), k


# ---------------------------------------------------------------------------------------------------------------------
# what the projections did
# ---------------------------------------------------------------------------------------------------------------------
def soc_branches(s, starts, mu):
    """which branch of project_soc (admm.cpp:39-60) produced each cone of the final slacks s [B, K, n] (vcnew or zcnew): per
    instance, flags (below: the slack is zero; inside: strictly inside the cone; projected: on its surface, not zero), for the
    cones starting at `starts` with mu [B, ncones].  The surface test uses mu narrowed to float, as the projection does."""
    B = s.shape[0]
    below = np.zeros(B, bool)
    inside = np.zeros(B, bool)
    proj = np.zeros(B, bool)
    for c, st0 in enumerate(starts):
        v = s[:, :, st0:st0 + 3].astype(np.float64)
        m = mu[:, c].astype(np.float32).astype(np.float64)[:, None]
        nrm = np.hypot(v[..., 0], v[..., 1])
        zero = np.all(v == 0, axis=-1)
        tol = 1e-4 * np.maximum(1.0, np.abs(m * v[..., 2]))
        on = ~zero & (np.abs(nrm - m * v[..., 2]) <= tol)
        ins = ~zero & (nrm < m * v[..., 2] - tol)
        below |= zero.any(axis=1)
        inside |= ins.any(axis=1)
        proj |= on.any(axis=1)
    return below, inside, proj


def active_rows(planes, x, u):
    """per instance: does some static hyperplane row hold with equality-or-beyond at some knot, i.e. is a projection active?
    x [B, N, nx] / u [B, N-1, nu]: the slacks the planes produced (vlnew / zlnew).  A row is active where a.s >= b - tol."""
    B = len(next(iter(planes.values())))
    act = np.zeros(B, bool)
    for side, s in (("x", x), ("u", u)):
        A, b = planes.get("Alin_" + side), planes.get("blin_" + side)
        if A is None or s is None:
            continue
        cv = np.einsum("bin,bkn->bki", A.astype(np.float64), s.astype(np.float64))  # [B, K, rows]
        nz = np.any(A != 0, axis=2)[:, None, :]
        tol = 1e-5 * np.maximum(1.0, np.abs(b))[:, None, :]
        act |= np.any(nz & (np.abs(cv - b[:, None, :].astype(np.float64)) <= tol), axis=(1, 2))
    return act


# ---------------------------------------------------------------------------------------------------------------------
# the GPU solve paths; kinds: any of bounds= / cones= / planes=, the batch's per-instance arrays
# ---------------------------------------------------------------------------------------------------------------------
def settings(spec, **kw):
    st = abi.Settings.from_buffer_copy(spec.settings)
    for k, v in kw.items():
        setattr(st, k, v)
    return st


def check(got, o, want, what):
    """every output, u0 and the requested state of a solve bit for bit against an oracle result"""
    ref = {k: o[k] for k in H.OUT_KEYS + list(want)}
    ref["u0"] = np.ascontiguousarray(o["u"][:, 0, :])
    H.assert_bits_per_instance(got, ref, H.OUT_KEYS + list(want) + ["u0"], what)


def device(solver, x0, Xref, Uref, state, cold, want, models=None, **kinds):
    """tinympc_b200_solve on tensors from make_device_batch -> (numpy results, stats)"""
    import torch

    batch, out = solver.make_device_batch(x0, Xref, Uref, state=state, cold_start=cold, want_state=tuple(want), want_u0=True,
                                          models=models, **kinds)
    for k in OUTS:
        H.poison(out[k])
    if cold:
        for n in want:
            H.poison(out[n])
    solver.solve_device(batch)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items() if v is not None}, solver.stats()


def _pinned(a, keep):
    import torch

    t = torch.empty(a.nbytes, dtype=torch.uint8, pin_memory=True)
    keep.append(t)
    p = t.numpy().view(a.dtype).reshape(a.shape)
    p[...] = a
    return p


def host(solver, x0, Xref, Uref, state, cold, want, models=None, pin=False, **kinds):
    """tinympc_b200_solve_host on a HostBatch (u0 requested too); pin: every caller buffer page-locked"""
    p = solver.problem
    state = None if state is None else {n: np.array(a, copy=True) for n, a in state.items()}
    hb = HostBatch(p, x0, Xref, Uref, state=state, cold_start=cold, want_state=tuple(want), models=models, **kinds)
    hb.u0 = np.empty((hb.B, p.nu), p.dtype)
    keep = []
    if pin:
        for n in ("x0", "Xref", "Uref", "sol_x", "sol_u", "iter", "solved", "residuals", "u0", "models"):
            if getattr(hb, n) is not None:
                setattr(hb, n, _pinned(getattr(hb, n), keep))
        hb.state = {n: _pinned(a, keep) for n, a in hb.state.items()}
        for kind in kinds:
            setattr(hb, kind, {n: _pinned(a, keep) for n, a in getattr(hb, kind).items()})
    for k in OUTS:
        H.poison(getattr(hb, k))
    if cold:
        for n in want:
            H.poison(hb.state[n])
    cb = hb.to_c()
    cb.u0 = hb.u0.ctypes.data
    solver.solve_prepared(hb, cb)
    return {k: np.array(v, copy=True) for k, v in dict(hb.result(), u0=hb.u0).items() if v is not None}, solver.stats()


def warm_inputs(x0, res, seed, want):
    """the next MPC step: perturbed measurements, the returned state, duals reset on every third instance"""
    rng = np.random.default_rng(seed)
    x0b = (x0 + 0.02 * rng.standard_normal(x0.shape)).astype(x0.dtype)
    state = {n: np.array(res[n], copy=True) for n in want}
    for n in ("g", "y", "gl", "yl", "gl_tv", "yl_tv", "gc", "yc"):
        if n in state:
            state[n][::3] = 0
    return x0b, state


def capacity(solver, arrays_fn, models=None, per_sm=256):
    """instances one wave of the solver's persistent kernel holds (ctas x instances_per_cta), from a one-iteration probe solve
    of per_sm instances per SM that fills every SM; arrays_fn(B) -> the probe's per-instance arrays ({kind: arrays})"""
    import torch

    p = solver.problem
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    B = per_sm * sm
    mi = solver.settings.max_iter
    solver.update_settings(max_iter=1)
    m = None if models is None else models[np.zeros(B, int)]
    batch, _ = solver.make_device_batch(np.zeros((B, p.nx), p.dtype), np.zeros((p.N, p.nx), p.dtype), cold_start=True,
                                        models=m, **arrays_fn(B))
    solver.solve_device(batch)
    torch.cuda.synchronize()
    solver.update_settings(max_iter=mi)
    stt = solver.stats()
    assert stt["ctas"] == sm, stt
    return stt["ctas"] * stt["instances_per_cta"]


def cold_warm(solver, inst, what, want, family=abi.KERNEL_GPS, models=None, model_of=None, mult=None, **kinds):
    """cold solve, then a warm step from the returned state with the duals reset on every third instance; every instance vs
    the grouped oracle; the plan is `family` in one launch, with at least `mult` waves when given.  Returns the two oracle
    results and the stats of the cold solve."""
    port = grouped_oracle(solver.problem, solver.settings, models, model_of, nthreads=NT, **kinds)
    m = None if models is None else models[model_of]
    x0, Xref, Uref = inst["x0"], inst["Xref"], inst.get("Uref")
    o1 = port(x0, Xref, Uref, None, True, want)
    g1, st1 = device(solver, x0, Xref, Uref, None, True, want, models=m, **kinds)
    assert st1["kernel_family"] == family and st1["kernel_launches"] == 1, st1
    if mult:
        assert len(x0) >= mult * st1["ctas"] * st1["instances_per_cta"], (len(x0), st1)
    check(g1, o1, want, what + " cold")
    x0b, state = warm_inputs(x0, o1, seed=len(x0), want=want)
    o2 = port(x0b, Xref, Uref, state, False, want)
    g2, st2 = device(solver, x0b, Xref, Uref, state, False, want, models=m, **kinds)
    assert st2["kernel_family"] == family, st2
    check(g2, o2, want, what + " warm")
    return o1, o2, st1


def plan(stt):
    return {k: stt[k] for k in PLAN}


def shared_plan(solver, inst, want, models=None):
    """the launch statistics of the same batch without per-instance data"""
    device(solver, inst["x0"], inst["Xref"], inst.get("Uref"), None, True, want, models=models)
    return solver.stats()


def same_plan(shared, stt, table_bytes=0):
    """per-instance data kept the shared solve's plan (lanes, instances per lane group, warps, CTAs); shared memory grew by
    table_bytes per instance of a CTA"""
    assert plan(stt) == plan(shared), (stt, shared)
    assert stt["smem_bytes_per_cta"] - shared["smem_bytes_per_cta"] == stt["instances_per_cta"] * table_bytes, (stt, shared)


def one_per_group(stt):
    """the streamed kernel ran a one-instance-per-lane-group variant"""
    assert stt["kernel_family"] == abi.KERNEL_GPS, stt
    assert stt["instances_per_cta"] == stt["threads_per_cta"] // stt["lanes_per_instance"], stt


def two_per_group(stt):
    """the streamed kernel kept two instances per lane group"""
    assert stt["kernel_family"] == abi.KERNEL_GPS, stt
    assert stt["instances_per_cta"] == 2 * (stt["threads_per_cta"] // stt["lanes_per_instance"]), stt


# ---------------------------------------------------------------------------------------------------------------------
# scenarios every kind runs; each kind's suite brings its problem, instances and arrays
# ---------------------------------------------------------------------------------------------------------------------
HOST_B = 11 * 96 - 40  # the host path in 11 chunks of 96


def host_path_chunks(solver, inst, want, pin, monkeypatch, models=None, model_of=None, **kinds):
    """HOST_B instances through tinympc_b200_solve_host in 11 chunks, cold then warm, against the grouped oracle"""
    monkeypatch.setenv("TINYMPC_HOST_CHUNK", "96")
    port = grouped_oracle(solver.problem, solver.settings, models, model_of, nthreads=NT, **kinds)
    m = None if models is None else models[model_of]
    x0, Xref, Uref = inst["x0"], inst["Xref"], inst.get("Uref")
    o1 = port(x0, Xref, Uref, None, True, want)
    g1, stt = host(solver, x0, Xref, Uref, None, True, want, models=m, pin=pin, **kinds)
    assert stt["kernel_launches"] == 11, stt
    check(g1, o1, want, "host cold")
    x0b, state = warm_inputs(x0, o1, seed=32, want=want)
    o2 = port(x0b, Xref, Uref, state, False, want)
    g2, stt = host(solver, x0b, Xref, Uref, state, False, want, models=m, pin=pin, **kinds)
    check(g2, o2, want, "host warm")


def closed_loop(solver, inst, kind, arrays, step2, steps, want=None, roll=False, extra_state=(), models=None, model_of=None):
    """`steps` DeviceMPCLoop steps with the duals reset, the kind's arrays overridden by step2 in step 2, against the oracle
    stepping the same loop on the host (the oracle asked for `want`, the loop's fields when None); roll: the reference window
    moves by one knot every step.  loop.x0 bit-equal to the host loop's plant; rollouts refused."""
    from tinympc_b200.closed_loop import DeviceMPCLoop

    prob, st = solver.problem, solver.settings
    loop = DeviceMPCLoop(solver, inst["x0"], reset_duals=True, extra_state=extra_state, models=None if models is None else models[model_of],
                         **{kind: arrays})
    want = loop.fields if want is None else want
    Uref = inst.get("Uref")
    x0 = inst["x0"].copy()
    state = None
    for k in range(steps):
        Xref = np.ascontiguousarray(np.roll(inst["Xref"], -k, axis=1)) if roll else inst["Xref"]
        out = loop.step(Xref, Uref, **{kind: step2 if k == 2 else None})
        if state is not None:
            state["g"] = np.zeros_like(state["g"])
            state["y"] = np.zeros_like(state["y"])
        o = grouped_oracle(prob, st, models, model_of, nthreads=NT, **{kind: step2 if k == 2 else arrays})(
            x0, Xref, Uref, state, state is None, want)
        got = {key: out[key].cpu().numpy() for key in H.OUT_KEYS + list(loop.fields) + ["u0"]}
        check(got, o, loop.fields, f"closed loop step {k}")
        state = {n: o[n] for n in want}
        u0 = o["u"][:, 0, :]
        if models is None:
            x0 = advance(prob, x0, u0)
        else:
            nxt = np.empty_like(x0)
            for m in range(len(models)):
                idx = np.flatnonzero(model_of == m)
                nxt[idx] = advance(with_model(prob, models[m]), x0[idx], u0[idx])
            x0 = nxt
        assert H.bits_equal(loop.x0.cpu().numpy(), x0), ("advance", k)
    with pytest.raises(ValueError):
        loop.rollout(inst["Xref"], 3)


def queued_solves(solver, inst, want, kind, batches):
    """one cold device solve per entry of batches (the kind's arrays, moved to the device first) queued back to back on one
    handle, against the same solves each synchronised, and against the grouped oracle"""
    import torch

    dev = torch.device("cuda", 0)
    on_dev = [{k: torch.as_tensor(v, device=dev) for k, v in arrays.items()} for arrays in batches]
    x0, Xref, Uref = inst["x0"], inst["Xref"], inst.get("Uref")

    def run(sync):
        res = []
        for arrays in on_dev:
            batch, out = solver.make_device_batch(x0, Xref, Uref, cold_start=True, want_state=want, want_u0=True, **{kind: arrays})
            for k in OUTS + want:
                H.poison(out[k])
            solver.solve_device(batch)
            if sync:
                torch.cuda.synchronize()
            res.append((batch, out))
        torch.cuda.synchronize()
        return [{k: v.cpu().numpy() for k, v in out.items() if v is not None} for _, out in res]

    queued, synced = run(False), run(True)
    for q, y, arrays in zip(queued, synced, batches):
        H.assert_bits_per_instance(q, y, list(y), "queued vs synchronised")
        o = grouped_oracle(solver.problem, solver.settings, nthreads=NT, **{kind: arrays})(x0, Xref, Uref, None, True, want)
        check(q, o, want, "queued vs oracle")


def solve_rc(solver, batch):
    """tinympc_b200_solve's return code for a prepared batch, the device synchronised"""
    import torch

    r = solver._lib.tinympc_b200_solve(solver._h, C.byref(batch), None)
    torch.cuda.synchronize()
    return r


def assert_refused(solver, batch, Xref, adaptive_word):
    """per-instance data runs in STRICT mode on the lane-group kernels only: FAST mode and an explicit thread per instance are
    refused, and so are adaptive rho (last_error naming adaptive_word) and rollouts"""
    import torch

    lib, B, prob = solver._lib, batch.B, solver.problem
    solver.set_mode(abi.MODE_FAST)
    assert solve_rc(solver, batch) == abi.ERR_UNSUPPORTED and b"STRICT" in lib.tinympc_b200_last_error()
    solver.set_mode(abi.MODE_STRICT, abi.KERNEL_TPI)
    assert solve_rc(solver, batch) == abi.ERR_UNSUPPORTED and b"thread per instance" in lib.tinympc_b200_last_error()
    solver.set_mode(abi.MODE_STRICT, abi.KERNEL_AUTO)
    models = torch.as_tensor(pack_models(prob, B), device="cuda")
    dK, dP = np.zeros((prob.nu, prob.nx), prob.dtype), np.zeros((prob.nx, prob.nx), prob.dtype)
    ar = AdaptiveRho(dK, dP).to_c(prob, models.data_ptr(), B, models.device)
    assert lib.tinympc_b200_solve_adaptive(solver._h, C.byref(batch), C.byref(ar), None) == abi.ERR_UNSUPPORTED
    assert adaptive_word in lib.tinympc_b200_last_error()
    rb = abi.Batch.from_buffer_copy(batch)
    rb.Xref = rb.Uref = rb.iter = rb.solved = rb.residuals = rb.u0 = None
    rb.sol_x = rb.sol_u = None
    r = abi.Rollout()
    X = torch.as_tensor(np.ascontiguousarray(Xref if Xref.ndim == 2 else Xref[0]), device="cuda")
    r.T, r.Xref = 1, X.data_ptr()
    assert lib.tinympc_b200_rollout(solver._h, C.byref(rb), C.byref(r), None) == abi.ERR_UNSUPPORTED
    assert b"rollout" in lib.tinympc_b200_last_error()


def assert_python_rejects(solver, inst, kind, bad):
    """every malformed arrays dict of `bad` raises ValueError from make_device_batch and from solve"""
    for arrays in bad:
        with pytest.raises(ValueError):
            solver.make_device_batch(inst["x0"], inst["Xref"], cold_start=True, **{kind: arrays})
        with pytest.raises(ValueError):
            solver.solve(inst["x0"], inst["Xref"], **{kind: arrays})
