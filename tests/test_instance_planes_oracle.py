"""CPU checks of per-instance static hyperplanes (tinympc_batch_t.planes_per_instance): the ctypes mirror of the new batch
fields matches the header, and the helper the GPU tests compare against (planes_common.grouped_oracle) equals the unmodified
reference run once per instance, each with its own tiny_set_linear_constraints, bit for bit."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import helpers as H
import planes_common as PC
from oracle import oracle
from tinympc_b200 import abi, workloads as wl
from tinympc_b200.batch import planes_abi, planes_check

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FIELDS = ["Alin_x", "blin_x", "Alin_u", "blin_u", "planes_per_instance", "reserved4"]


def test_batch_planes_fields_match_header():
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"tinympc_b200.h\"\nint main(void){\n"
    src += '  printf("%zu\\n", sizeof(tinympc_batch_t));\n'
    src += "".join(f'  printf("%zu\\n", offsetof(tinympc_batch_t, {n}));\n' for n in FIELDS)
    src += "  return 0; }\n"
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "probe.c")
        open(c, "w").write(src)
        exe = os.path.join(td, "probe")
        subprocess.check_call(["/usr/bin/gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = list(map(int, subprocess.check_output([exe], text=True).split()))
    assert out[0] == C.sizeof(abi.Batch)
    assert out[1:] == [getattr(abi.Batch, n).offset for n in FIELDS]
    # the new fields come after every field of the previous layout
    assert abi.Batch.Alin_x.offset >= abi.Batch.reserved3.offset + 4
    b = abi.Batch()
    assert b.planes_per_instance == 0 and b.reserved4 == 0  # a zero-initialised batch: the handle's hyperplanes
    assert b.Alin_x is None and b.blin_x is None and b.Alin_u is None and b.blin_u is None


def test_planes_check_and_layout():
    B, nlx, nlu, nx, nu = 3, 2, 1, 12, 4
    dt = np.float32
    good = dict(Alin_x=np.zeros((B, nlx, nx), dt), blin_x=np.zeros((B, nlx), dt), Alin_u=np.zeros((B, nlu, nu), dt),
                blin_u=np.zeros((B, nlu), dt))
    planes_check(good, B, nlx, nlu, nx, nu, dt)
    planes_check({k: good[k] for k in ("Alin_x", "blin_x")}, B, nlx, nlu, nx, nu, dt)
    for bad in ({"Alin_x": good["Alin_x"]}, {"A": 1}, {}, dict(good, blin_u=np.zeros((B, 2), dt)),
                dict(good, Alin_x=good["Alin_x"].astype(np.float64)), dict(good, Alin_x=np.zeros((B, nx, nlx), dt))):
        with pytest.raises(ValueError):
            planes_check(bad, B, nlx, nlu, nx, nu, dt)
    # each instance's matrix goes column-major: element (row i, column j) of instance b at b*nx*nlx + j*nlx + i
    A = np.arange(B * nlx * nx, dtype=dt).reshape(B, nlx, nx)
    flat = np.ascontiguousarray(planes_abi(dict(Alin_x=A, blin_x=good["blin_x"]))["Alin_x"]).reshape(-1)
    b, i, j = 2, 1, 5
    assert flat[b * nx * nlx + j * nlx + i] == A[b, i, j]


OUT = H.OUT_KEYS + H.LIN_STATE


def _quad(dt, N=12):
    spec = H.quad_linear_spec(N=N)
    return spec, H.problem_from_spec(spec, dt, oracle.ref_setup)


def _instances(spec, B, dt, seed=4):
    inst = wl.tracking_instances(B, N=spec.N, seed=seed, dtype=dt, jitter=0.3)
    return inst["x0"], inst["Xref"]


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_plane_helper_equals_reference_per_instance(dt):
    """16 quadrotors with 12 distinct plane sets (both sides): the helper (the C restatement once per plane set) against the
    compiled reference once per instance with its own tiny_set_linear_constraints, cold, then warm from the cold result."""
    if not oracle.ref_available(dt):
        pytest.skip("the compiled reference (oracle/_ref, made by build() from the TinyMPC checkout) is not present")
    spec, prob = _quad(dt)
    st = spec.settings
    B = 16
    x0, Xref = _instances(spec, B, dt)
    pal = PC.plane_palette(prob, 12, seed=2)
    which = (np.arange(B) * 5) % 12
    planes = PC.batch_planes(pal, which)
    helper = PC.grouped_oracle(prob, st, planes, nthreads=4)

    def reference(x0_, state, cold):
        outs = []
        for b in range(B):
            p = PC.with_planes(prob, {k: v[b] for k, v in planes.items()})
            sub = None if state is None else {n: np.array(a[b:b + 1], copy=True) for n, a in state.items()}
            outs.append(oracle.solve_batch(p, st, x0_[b:b + 1], Xref[b:b + 1], None, state=sub, cold_start=cold,
                                           want_state=tuple(H.LIN_STATE), impl="reference"))
        return {k: np.concatenate([o[k] for o in outs]) for k in OUT}

    h1 = helper(x0, Xref, None, None, True, H.LIN_STATE)
    r1 = reference(x0, None, True)
    H.assert_bits_per_instance(h1, r1, OUT, "cold")
    # the planes bite: most instances end with a slack on one of their planes
    act = PC.active_rows(planes, h1["vlnew"], h1["zlnew"])
    assert act.sum() >= (3 * B) // 4, act
    # and they matter: the same batch with the problem's own planes differs for at least half of the instances
    shared = oracle.solve_batch(prob, st, x0, Xref, None, cold_start=True, nthreads=4)
    differ = [not np.array_equal(shared["sol_u"][b], h1["sol_u"][b]) for b in range(B)]
    assert sum(differ) >= B // 2, differ
    state = {n: h1[n] for n in H.LIN_STATE}
    x0w = np.ascontiguousarray(h1["x"][:, 1, :])
    h2 = helper(x0w, Xref, None, state, False, H.LIN_STATE)
    r2 = reference(x0w, state, False)
    H.assert_bits_per_instance(h2, r2, OUT, "warm")


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_padding_rows_are_inert(dt):
    """a robot with fewer planes pads its rows with a = 0, b = 0: the padded solve equals the solve without the row, bit for
    bit (a.z = 0 > 0 is false, so the row never projects)"""
    spec, prob = _quad(dt)
    spec0 = H.quad_linear_spec(N=spec.N)
    st = spec.settings
    B = 8
    x0, Xref = _instances(spec, B, dt)
    pset = PC.plane_palette(prob, 1, seed=7)[0]
    # the problem with one extra state row and one extra input row, which this robot pads with zeros
    cons = dict(spec0.constraints)
    cons["Alin_x"] = np.vstack([pset["Alin_x"], np.zeros((1, prob.nx))])
    cons["blin_x"] = np.concatenate([pset["blin_x"], [0.0]])
    cons["Alin_u"] = np.vstack([pset["Alin_u"], np.zeros((1, prob.nu))])
    cons["blin_u"] = np.concatenate([pset["blin_u"], [0.0]])
    spec0.constraints = cons
    padded = H.problem_from_spec(spec0, dt, oracle.port_setup)
    plain = PC.with_planes(padded, pset)
    assert padded.Alin_x.shape[0] == plain.Alin_x.shape[0] + 1
    a = oracle.solve_batch(padded, st, x0, Xref, None, cold_start=True, want_state=tuple(H.LIN_STATE), nthreads=4)
    b = oracle.solve_batch(plain, st, x0, Xref, None, cold_start=True, want_state=tuple(H.LIN_STATE), nthreads=4)
    for k in OUT:
        assert H.bits_equal(a[k], b[k]), k


def test_plane_helper_groups_by_distinct_set(monkeypatch):
    """a batch dealt 3 plane sets is solved with 3 oracle runs, and a set equal to the problem's gives the shared result"""
    dt = np.float64
    spec = H.quad_linear_spec(N=10)
    prob = H.problem_from_spec(spec, dt, oracle.port_setup)
    st = spec.settings
    B = 9
    x0, Xref = _instances(spec, B, dt, seed=1)
    pal = [PC.own_planes(prob)] + PC.plane_palette(prob, 2, seed=9)
    which = np.arange(B) % 3
    planes = PC.batch_planes(pal, which)
    calls = []
    real = oracle.solve_batch

    def counting(*a, **k):
        calls.append(len(a[2]))
        return real(*a, **k)

    monkeypatch.setattr(oracle, "solve_batch", counting)
    got = PC.grouped_oracle(prob, st, planes, nthreads=2)(x0, Xref, None, None, True, ())
    monkeypatch.undo()
    assert sorted(calls) == [3, 3, 3]
    ref = oracle.solve_batch(prob, st, x0, Xref, None, cold_start=True, nthreads=2)
    for k in H.OUT_KEYS:
        assert H.bits_equal(got[k][which == 0], ref[k][which == 0]), k


def test_plane_fleet_is_seeded_and_keeps_structure():
    spec = H.quad_linear_spec(N=10)
    a = wl.plane_fleet(spec, 16, seed=3)
    b = wl.plane_fleet(spec, 16, seed=3)
    assert sorted(a) == ["Alin_u", "Alin_x", "blin_u", "blin_x"]
    for k in a:
        assert np.array_equal(a[k], b[k])
    Ax = np.asarray(spec.constraints["Alin_x"])
    assert a["Alin_x"].shape == (16,) + Ax.shape and a["blin_u"].shape == (16, 1)
    assert np.array_equal(a["Alin_x"] != 0, np.broadcast_to(Ax != 0, a["Alin_x"].shape))  # zero coefficients stay zero
    assert not np.array_equal(a["blin_x"][0], a["blin_x"][1])
    assert wl.plane_fleet(wl.quadrotor(N=10), 4) == {}  # a spec without hyperplanes
