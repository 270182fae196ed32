"""Per-instance static hyperplanes (tinympc_batch_t.planes_per_instance) for the tests: plane-set palettes dealt to the
instances of a batch, and the oracle run once per distinct plane set (and model) over the instances that use it.

Instance b of a solve with per-instance planes computes what one TinySolver whose tiny_set_linear_constraints got that
instance's Alin_x, blin_x, Alin_u, blin_u computes; the row counts and the settings are the problem's.  The oracle's problem
takes the planes of one such solver, so a batch whose instances use K plane sets is checked with K oracle runs, not B."""
import numpy as np

from bounds_common import with_model
from oracle import oracle
from tinympc_b200.batch import PLANE_NAMES
from tinympc_b200.problem import MPCProblem


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


def with_planes(prob, pset):
    """prob with its static hyperplanes replaced by one plane set (the planes of one TinySolver); an absent side keeps the
    problem's"""
    kw = {k: getattr(prob, k) for k in prob.__dataclass_fields__}
    for k in PLANE_NAMES:
        if pset.get(k) is not None:
            kw[k] = np.asarray(pset[k])
    return MPCProblem(**kw)


def grouped_oracle(prob, st, planes, models=None, model_of=None, impl="port", nthreads=8):
    """run(x0, Xref, Uref, state, cold, want) -> the oracle's result for the whole batch, one oracle run per distinct
    (plane set, model) over the instances that use it.  planes: the batch's per-instance arrays as in batch_planes (an absent
    side keeps the problem's planes); models / model_of: per-instance models (blob palette and the blob of every instance)."""
    given = [k for k in PLANE_NAMES if planes.get(k) is not None]
    B = len(planes[given[0]])
    rows = [np.asarray(planes[k]).reshape(B, -1).view(np.uint8) for k in given]
    _, pid = np.unique(np.concatenate(rows, axis=1), axis=0, return_inverse=True)
    mo = np.zeros(B, np.int64) if model_of is None else np.asarray(model_of)
    _, key = np.unique(np.stack([pid.reshape(-1), mo], axis=1), axis=0, return_inverse=True)
    key = key.reshape(-1)
    probs = {}
    for g in np.unique(key):
        b = int(np.flatnonzero(key == g)[0])
        p = prob if models is None else with_model(prob, models[mo[b]])
        probs[g] = with_planes(p, {k: planes[k][b] for k in given})

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
