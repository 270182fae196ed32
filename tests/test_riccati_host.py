"""The host Riccati precompute, pinned bit for bit: SHA-256 digests of what tinympc_b200_precompute_cache,
tinympc_b200_precompute_cache_batch and tinympc_b200_precompute_sensitivity_batch return, for fp32 and fp64, every compiled
(nx, nu), two shapes no kernel is compiled for, a singular model and the fp32 quadrotor that runs all 1000 sweeps.  The
digests are stored in tests/golden/riccati_host_digests.json; any change to the operation sequence of the recursion shows
up here, without a GPU.  Regenerate (only when the arithmetic is meant to change) with

    python tests/test_riccati_host.py
"""
import hashlib
import json
import os
import sys

import numpy as np

if __name__ == "__main__":
    sys.path[:0] = [os.path.dirname(os.path.dirname(os.path.abspath(__file__))), os.path.dirname(os.path.abspath(__file__))]

import sensitivity_common as SC
from tinympc_b200 import workloads as wl
from tinympc_b200._lib import TinyMPCError
from tinympc_b200.solver import precompute_cache, setup_models, setup_problem, setup_sensitivity

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "riccati_host_digests.json")
# every compiled (nx, nu) (csrc/launch.h: TM_DIMS) and two that only the host routine serves
SHAPES = [(4, 1), (6, 3), (12, 4), (4, 2), (4, 4), (4, 8), (8, 2), (8, 4), (8, 8), (12, 2), (12, 8), (16, 2), (16, 4), (16, 8),
          (3, 1), (20, 6)]
DTYPES = {"f32": np.float32, "f64": np.float64}


def _digest(*arrays):
    """SHA-256 of the arrays' bytes in order, every NaN replaced by the one canonical quiet NaN"""
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        if a.dtype.kind == "f":
            a = np.where(np.isnan(a), np.array(np.nan, a.dtype), a)
        h.update(str(a.dtype).encode() + str(a.shape).encode())
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def _single(nx, nu, A, B, f, Qdiag, Rdiag, rho, dt):
    rho = dt(rho)
    Qw, Rw = (np.asarray(Qdiag, dt) + rho).astype(dt), (np.asarray(Rdiag, dt) + rho).astype(dt)
    out, sweeps = precompute_cache(nx, nu, rho, A, B, f, Qw, Rw, dt)
    return _digest(*out.values(), np.array([sweeps]))


def _batches(nx, nu, args, dt):
    """digests of the batched cache and sensitivity calls, each the same with 1 and with 8 threads"""
    d = {}
    for name, fn in (("cache_batch", setup_models), ("sensitivity_batch", setup_sensitivity)):
        runs = []
        for nthreads in (1, 8):
            try:
                r = fn(nx, nu, *args, dtype=dt, nthreads=nthreads)
                runs.append(_digest(*(r if isinstance(r, tuple) else (r,))))
            except TinyMPCError as e:
                runs.append(str(e))
        assert runs[0] == runs[1], (name, nx, nu, dt)
        d[name] = runs[0]
    return d


def digests():
    out = {}
    for tag, dt in DTYPES.items():
        for nx, nu in SHAPES:
            sp = wl.random_lti(nx, nu, 10, seed=11)
            key = f"{tag}_{nx}_{nu}"
            out[f"{key}_cache"] = _single(nx, nu, sp.A, sp.B, sp.f, sp.Qdiag, sp.Rdiag, 0.5 + 0.1 * nx, dt)
            for k, v in _batches(nx, nu, SC.lti_batch(nx, nu, 19, seed=nx * 100 + nu), dt).items():
                out[f"{key}_{k}"] = v
        # one singular model among nine: the batch calls name it, the single call refuses it as a bad argument
        args = SC.lti_batch(4, 2, 9, seed=5, singular_at=6)
        for k, v in _batches(4, 2, args, dt).items():
            out[f"{tag}_singular_{k}"] = v
        try:
            _single(4, 2, *(a[6] for a in args), dt)
            out[f"{tag}_singular_cache"] = "no error"
        except TinyMPCError as e:
            out[f"{tag}_singular_cache"] = str(e)
        # the quadrotor: in fp32 its stop test never passes, so the recursion runs all 1000 sweeps
        q = wl.quadrotor(N=10)
        out[f"{tag}_quadrotor_cache"] = _single(12, 4, q.A, q.B, q.f, q.Qdiag, q.Rdiag, q.rho, dt)
        out[f"{tag}_quadrotor_sweeps"] = setup_problem(q, dt).riccati_sweeps
        qb = tuple(np.repeat(np.asarray(a, np.float64)[None], 4, 0) for a in (q.A, np.reshape(q.B, (12, 4)), q.f, q.Qdiag, q.Rdiag))
        for k, v in _batches(12, 4, qb + (np.array([q.rho, 0.5 * q.rho, 2 * q.rho, q.rho + 1]),), dt).items():
            out[f"{tag}_quadrotor_{k}"] = v
    return out


def test_host_precompute_bits_unchanged():
    with open(FIXTURE) as fh:
        want = json.load(fh)
    got = digests()
    assert want["f32_quadrotor_sweeps"] == 1000
    assert sorted(got) == sorted(want)
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, bad


if __name__ == "__main__":
    with open(FIXTURE, "w") as fh:
        json.dump(digests(), fh, indent=1, sort_keys=True)
        fh.write("\n")
