"""Shared helpers of the scripted shim tests (tests/shim/shim_script.cpp): an op-stream writer, the parser of what the
driver dumps, and the comparisons.  The driver is built twice from one source, against the unmodified reference
(oracle/_ref/shim_tests/script_ref, CPU) and against the shim (oracle/_ref/shim_tests/script_shim, GPU); the op codes,
the POKE_FIELDS order and the record layouts below mirror that file."""
from __future__ import annotations

import os
import subprocess

import numpy as np

import helpers as H
from oracle import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT_DIR = os.path.join(ROOT, "oracle", "_ref", "shim_tests")
SCRIPT_REF = os.path.join(SCRIPT_DIR, "script_ref")
SCRIPT_SHIM = os.path.join(SCRIPT_DIR, "script_shim")

OPS = dict(setup=1, set_cache=2, bounds=3, cones=4, linear=5, tv_linear=6, x0=7, xref=8, uref=9, update_settings=10,
           poke_settings=11, poke_work=12, poke_counts=13, precompute=14, solve=15, plant=16, batch=17, dump=18)
POKE_FIELDS = ["Xref", "Uref", "x_min", "x_max", "u_min", "u_max", "x", "u", "v", "z", "vnew", "znew", "g", "y", "gc", "yc",
               "gl", "yl", "gl_tv", "yl_tv"]
SETTING_NAMES = ["abs_pri_tol", "abs_dua_tol", "max_iter", "check_termination", "en_state_bound", "en_input_bound",
                 "en_state_soc", "en_input_soc", "en_state_linear", "en_input_linear", "en_tv_state_linear",
                 "en_tv_input_linear"]
DEFAULT_SETTINGS = dict(abs_pri_tol=1e-3, abs_dua_tol=1e-3, max_iter=1000, check_termination=1, en_state_bound=1,
                        en_input_bound=1, en_state_soc=0, en_input_soc=0, en_state_linear=0, en_input_linear=0,
                        en_tv_state_linear=0, en_tv_input_linear=0)  # tiny_api_constants.hpp
# record kinds and their matrices, in the order the driver writes them.  work->{q, r, p, d} are not dumped: they are
# per-iteration scratch that every iteration overwrites before reading, and the shim never writes them.
CACHE_FIELDS = ["rho", "Kinf", "Pinf", "Quu_inv", "AmBKt", "APf", "BPf"]
TREE_FIELDS = (["iter", "solved", "sol_x", "sol_u", "x", "u", "v", "vnew", "z", "znew", "g", "y", "vcnew", "zcnew", "gc", "yc",
                "vlnew", "zlnew", "gl", "yl", "vlnew_tv", "zlnew_tv", "gl_tv", "yl_tv", "vc", "zc", "vl", "zl", "vl_tv", "zl_tv",
                "Kinf", "Pinf", "primal_residual_state", "dual_residual_state", "primal_residual_input",
                "dual_residual_input", "status", "work_iter", "rho"])
BATCH_FIELDS = ["u0", "iter", "solved"]
KINDS = {1: ("cache", CACHE_FIELDS), 2: ("tree", TREE_FIELDS), 3: ("batch", BATCH_FIELDS)}


def have(*paths):
    return all(os.path.exists(p) for p in paths)


class Model:
    """What tiny_setup takes: dynamics, the user's Q and R diagonals (without rho) and rho."""

    def __init__(self, nx, nu, N, A, B, f, Qdiag, Rdiag, rho):
        self.nx, self.nu, self.N = nx, nu, N
        self.A, self.B = np.asarray(A, np.float64), np.asarray(B, np.float64).reshape(nx, nu)
        self.f, self.Qdiag, self.Rdiag, self.rho = np.asarray(f, np.float64), np.asarray(Qdiag, np.float64), \
            np.asarray(Rdiag, np.float64), float(rho)

    @staticmethod
    def from_spec(spec, N=None):
        return Model(spec.nx, spec.nu, N or spec.N, spec.A, spec.B, spec.f, spec.Qdiag, spec.Rdiag, spec.rho)

    def ref_cache(self, rho=None):
        """The cache the reference's own tiny_setup derives (rho: a new rho, as tiny_precompute_and_set_cache takes it)."""
        return oracle.ref_setup(self.nx, self.nu, self.N, self.rho if rho is None else rho, self.A, self.B, self.f,
                                self.Qdiag, self.Rdiag)


def _mat(a):
    a = np.asarray(a, np.float64)
    if a.ndim == 0:
        a = a.reshape(1, 1)
    elif a.ndim == 1:
        a = a.reshape(-1, 1)
    return np.array(a.shape, np.int32).tobytes() + a.tobytes(order="F")


def _ivec(a):
    a = np.asarray(a, np.int32).reshape(-1)
    return np.int32(len(a)).tobytes() + a.tobytes()


class Script:
    """An op stream for the driver.  Every method appends one op on solver slot `si` (0..3)."""

    def __init__(self):
        self.parts = []
        self.nops = 0
        self.models = {}
        self.settings = {}

    def _op(self, name, si, *payload):
        self.parts.append(np.array([OPS[name], si], np.int32).tobytes() + b"".join(payload))
        self.nops += 1
        return self

    def bytes(self):
        return b"".join(self.parts)

    def setup(self, si, m: Model, pin=True):
        """tiny_setup, then (pin) the cache the reference's tiny_setup derives, so that both builds solve on the same cache."""
        self.models[si] = m
        self.settings[si] = dict(DEFAULT_SETTINGS)
        self._op("setup", si, np.array([m.nx, m.nu, m.N], np.int32).tobytes(), np.float64(m.rho).tobytes(), _mat(m.A),
                 _mat(m.B), _mat(m.f), _mat(np.diag(m.Qdiag)), _mat(np.diag(m.Rdiag)))
        if pin:
            self.set_cache(si, m.ref_cache())
        return self

    def set_cache(self, si, p):
        return self._op("set_cache", si, np.float64(p.rho).tobytes(), _mat(p.Kinf), _mat(p.Pinf), _mat(p.Quu_inv),
                        _mat(p.AmBKt), _mat(p.APf), _mat(p.BPf))

    def precompute(self, si, rho, pin=True):
        """tiny_precompute_and_set_cache with a new rho (the model's own Q, R), then (pin) the reference's cache for it."""
        m = self.models[si]
        self._op("precompute", si, np.float64(rho).tobytes(), _mat(np.diag(m.Qdiag)), _mat(np.diag(m.Rdiag)))
        if pin:
            self.set_cache(si, m.ref_cache(rho))
        return self

    def bounds(self, si, x_min, x_max, u_min, u_max):
        m = self.models[si]
        full = lambda v, n, k: np.broadcast_to(np.asarray(v, np.float64).reshape(n, -1), (n, k))  # noqa: E731
        return self._op("bounds", si, _mat(full(x_min, m.nx, m.N)), _mat(full(x_max, m.nx, m.N)),
                        _mat(full(u_min, m.nu, m.N - 1)), _mat(full(u_max, m.nu, m.N - 1)))

    def cones(self, si, Acx=(), qcx=(), cx=(), Acu=(), qcu=(), cu=()):
        return self._op("cones", si, _ivec(Acx), _ivec(qcx), _mat(np.asarray(cx, np.float64).reshape(-1, 1)), _ivec(Acu),
                        _ivec(qcu), _mat(np.asarray(cu, np.float64).reshape(-1, 1)))

    def linear(self, si, Alin_x, blin_x, Alin_u, blin_u):
        m = self.models[si]
        return self._op("linear", si, _mat(np.reshape(Alin_x, (-1, m.nx))), _mat(np.reshape(blin_x, (-1, 1))),
                        _mat(np.reshape(Alin_u, (-1, m.nu))), _mat(np.reshape(blin_u, (-1, 1))))

    def tv_linear(self, si, tvAx, tvbx, tvAu, tvbu):
        return self._op("tv_linear", si, _mat(tvAx), _mat(tvbx), _mat(tvAu), _mat(tvbu))

    def x0(self, si, x0):
        return self._op("x0", si, _mat(np.reshape(x0, (-1, 1))))

    def xref(self, si, Xref):
        """Xref as nx x N"""
        return self._op("xref", si, _mat(Xref))

    def uref(self, si, Uref):
        return self._op("uref", si, _mat(Uref))

    def update_settings(self, si, api=True, **kw):
        """tiny_update_settings (api) or direct writes into solver->settings (not api) of the whole settings block, with
        `kw` changed from the slot's current settings."""
        unknown = set(kw) - set(SETTING_NAMES)
        assert not unknown, unknown
        st = self.settings[si]
        st.update(kw)
        payload = np.array([st["abs_pri_tol"], st["abs_dua_tol"]], np.float64).tobytes()
        payload += np.array([st[n] for n in SETTING_NAMES[2:]], np.int32).tobytes()
        return self._op("update_settings" if api else "poke_settings", si, payload)

    def poke(self, si, name, value):
        return self._op("poke_work", si, np.int32(POKE_FIELDS.index(name)).tobytes(), _mat(value))

    def poke_counts(self, si, ncx, ncu, nlx, nlu, ntx, ntu):
        return self._op("poke_counts", si, np.array([ncx, ncu, nlx, nlu, ntx, ntu], np.int32).tobytes())

    def solve(self, si):
        return self._op("solve", si)

    def plant(self, si):
        return self._op("plant", si)

    def batch(self, si, x0, Xref):
        """tiny_solve_batch: x0 nx x B, Xref (nx*N) x B"""
        return self._op("batch", si, _mat(x0), _mat(Xref))

    def dump(self, si):
        return self._op("dump", si)


def parse(raw: bytes):
    """-> list of records: dict(kind, op, solver, rc, <field>: array) with every matrix in its (rows, cols) shape."""
    recs, o = [], 0
    while o < len(raw):
        kind, op, si, rc, nm = (int(v) for v in np.frombuffer(raw, np.int32, 5, o))
        o += 20
        name, fields = KINDS[kind]
        assert nm == len(fields), (kind, nm)
        rec = dict(kind=name, op=op, solver=si, rc=rc)
        for f in fields:
            r, c = (int(v) for v in np.frombuffer(raw, np.int32, 2, o))
            o += 8
            rec[f] = np.frombuffer(raw, np.float64, r * c, o).reshape((r, c), order="F")
            o += 8 * r * c
        recs.append(rec)
    return recs


def split_ops(stdout: str):
    """stdout grouped by op: op index -> the lines printed while that op ran (the driver prints a marker before each)"""
    out, cur = {}, None
    for ln in stdout.splitlines():
        if ln.startswith("## op "):
            cur = int(ln.split()[2])
            out[cur] = []
        elif cur is not None:
            out[cur].append(ln)
    return out


def run(binary, script: Script, tmp, tag):
    """Run one op stream -> (records, stdout by op)"""
    pin, pout = os.path.join(tmp, f"{tag}.in"), os.path.join(tmp, f"{tag}.out")
    with open(pin, "wb") as fh:
        fh.write(script.bytes())
    r = subprocess.run([binary, pin, pout], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (tag, r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    with open(pout, "rb") as fh:
        recs = parse(fh.read())
    ops = split_ops(r.stdout)
    assert sorted(ops) == list(range(script.nops)), (tag, len(ops), script.nops)
    return recs, ops


def run_threads(binary, scripts, tmp, tag):
    """Run several op streams at once, one thread per stream -> [records of each stream]"""
    args = []
    for k, s in enumerate(scripts):
        pin, pout = os.path.join(tmp, f"{tag}{k}.in"), os.path.join(tmp, f"{tag}{k}.out")
        with open(pin, "wb") as fh:
            fh.write(s.bytes())
        args += [pin, pout]
    r = subprocess.run([binary, "--threads"] + args, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (tag, r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    out = []
    for k in range(len(scripts)):
        with open(args[2 * k + 1], "rb") as fh:
            out.append(parse(fh.read()))
    return out


def cache_close(ref, got, rtol=1e-9):
    """fp64 cache agreement: every matrix within rtol of its largest entry (the bound of the device precompute test)"""
    for f in CACHE_FIELDS:
        a, b = ref[f], got[f]
        if a.shape != b.shape:
            return f
        scale = max(float(np.max(np.abs(a))), 1e-300)
        if float(np.max(np.abs(a - b), initial=0.0)) > rtol * scale:
            return f
    return None


def assert_same_records(ref, got, what):
    """Trees and batch results bit for bit, caches within the precompute bound, and the same rc everywhere."""
    assert len(ref) == len(got), (what, len(ref), len(got))
    for a, b in zip(ref, got):
        where = (what, a["kind"], "op", a["op"], "solver", a["solver"])
        assert (a["kind"], a["op"], a["solver"]) == (b["kind"], b["op"], b["solver"]), (where, b["kind"], b["op"])
        assert a["rc"] == b["rc"], (where, "rc", a["rc"], b["rc"])
        if a["kind"] == "cache":
            bad = cache_close(a, b)
            assert bad is None, (where, bad)
            continue
        for f in KINDS[{"tree": 2, "batch": 3}[a["kind"]]][1]:
            if not H.bits_equal(a[f], b[f]):
                d = np.abs(a[f] - b[f]) if a[f].shape == b[f].shape else None
                raise AssertionError(f"{where}: {f} differs (shapes {a[f].shape} / {b[f].shape}, max |diff| "
                                     f"{None if d is None else float(np.nanmax(d))})")


def assert_same_stdout(ref_ops, got_ops, what):
    for k in sorted(ref_ops):
        assert ref_ops[k] == got_ops.get(k), (what, "stdout of op", k, ref_ops[k][:5], (got_ops.get(k) or [])[:5])
    assert sorted(ref_ops) == sorted(got_ops), what


def trees(recs):
    return [r for r in recs if r["kind"] == "tree"]
