"""Per-instance cone coefficients (tinympc_batch_t.cones_per_instance) for the tests: mu palettes dealt to the instances of a
batch, and the oracle run once per distinct mu set (and model, and bound set) over the instances that use it.

Instance b of a solve with per-instance cones computes what one TinySolver whose tiny_set_cone_constraints got that
instance's cx / cu computes; the cone structure (Acx, qcx, Acu, qcu) is the problem's.  The oracle's problem takes the mu of
one such solver, so a batch whose instances use K mu sets is checked with K oracle runs, not B."""
import numpy as np

from bounds_common import with_bounds, with_model
from oracle import oracle
from tinympc_b200.problem import MPCProblem


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


def with_cones(prob, x_mu=None, u_mu=None):
    """prob with its cone coefficients replaced by one mu set (the cx / cu of one TinySolver); None keeps the problem's"""
    kw = {k: getattr(prob, k) for k in prob.__dataclass_fields__}
    if x_mu is not None:
        kw["cx"] = np.asarray(x_mu)
    if u_mu is not None:
        kw["cu"] = np.asarray(u_mu)
    return MPCProblem(**kw)


def grouped_oracle(prob, st, cones, models=None, model_of=None, bpal=None, bwhich=None, impl="port", nthreads=8):
    """run(x0, Xref, Uref, state, cold, want) -> the oracle's result for the whole batch, one oracle run per distinct
    (mu set, model, bound set) over the instances that use it.  cones: the batch's per-instance arrays (x_mu [B, ncx] and / or
    u_mu [B, ncu]; an absent side keeps the problem's mu).  models / model_of: per-instance models (blob palette and the blob
    of every instance); bpal / bwhich: per-instance bounds (bound palette and the set of every instance)."""
    xm, um = cones.get("x_mu"), cones.get("u_mu")
    B = len(xm if xm is not None else um)
    rows = [np.asarray(a).reshape(B, -1).view(np.uint8) for a in (xm, um) if a is not None]
    _, cid = np.unique(np.concatenate(rows, axis=1), axis=0, return_inverse=True)
    mo = np.zeros(B, np.int64) if model_of is None else np.asarray(model_of)
    bw = np.zeros(B, np.int64) if bwhich is None else np.asarray(bwhich)
    _, key = np.unique(np.stack([cid.reshape(-1), mo, bw], axis=1), axis=0, return_inverse=True)
    key = key.reshape(-1)
    probs = {}
    for g in np.unique(key):
        b = int(np.flatnonzero(key == g)[0])
        p = prob if models is None else with_model(prob, models[mo[b]])
        p = p if bpal is None else with_bounds(p, bpal[bw[b]])
        probs[g] = with_cones(p, None if xm is None else xm[b], None if um is None else um[b])

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
