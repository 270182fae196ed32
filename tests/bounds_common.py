"""Per-instance box bounds (tinympc_batch_t.bounds_per_instance) for the tests: bound palettes dealt to the instances of a batch,
and the oracle run once per bound set (and model) over the instances that use it.

Instance b of a solve with per-instance bounds computes what one TinySolver whose tiny_set_bound_constraints was called with
that instance's x_min, x_max, u_min, u_max computes.  The oracle's problem takes the bounds of one such solver, so a batch whose
instances use K bound sets is checked with K oracle runs, not B."""
import numpy as np

from oracle import oracle
from tinympc_b200.batch import BOUND_NAMES
from tinympc_b200.problem import MPCProblem
from tinympc_b200.solver import unpack_model


def deal(B, K, stride=7):
    """bound set of every instance: neighbouring instances (and so neighbouring slots and the refills of a slot) get different
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


def with_bounds(prob, bset):
    """prob with its box bounds replaced by one bound set (the bounds of one TinySolver)"""
    kw = {k: getattr(prob, k) for k in prob.__dataclass_fields__}
    for k in BOUND_NAMES:
        v = bset.get(k)
        kw[k] = None if v is None else (v if v.ndim == 1 else v.T)
    return MPCProblem(**kw)


def with_model(prob, blob):
    """prob with the model, cache and rho of one per-instance blob"""
    kw = {k: getattr(prob, k) for k in prob.__dataclass_fields__}
    m = unpack_model(np.asarray(blob), prob.nx, prob.nu)
    kw.update({k: m[k] for k in ("A", "B", "f", "Q", "R", "Kinf", "Pinf", "Quu_inv", "AmBKt", "APf", "BPf")}, rho=m["rho"])
    return MPCProblem(**kw)


def grouped_oracle(prob, st, pal, which, models=None, model_of=None, impl="port", nthreads=8):
    """run(x0, Xref, Uref, state, cold, want) -> the oracle's result for the whole batch, one oracle run per (model, bound set)
    over the instances that use it.  models / model_of: per-instance models (blob palette and the blob of every instance)."""
    which = np.asarray(which)
    mo = np.zeros_like(which) if model_of is None else np.asarray(model_of)
    key = mo * len(pal) + which
    probs = {}
    for g in np.unique(key):
        p = prob if models is None else with_model(prob, models[g // len(pal)])
        probs[g] = with_bounds(p, pal[g % len(pal)])

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
