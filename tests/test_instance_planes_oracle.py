"""CPU checks of per-instance static hyperplanes (tinympc_batch_t.planes_per_instance): the ctypes mirror of the batch fields
matches the header, the check and layout of the arrays, and the grouped helper the GPU tests compare against
(instance_common.grouped_oracle) equals the unmodified reference run once per instance, each with its own
tiny_set_linear_constraints, bit for bit."""
import numpy as np
import pytest

import helpers as H
import instance_common as IC
from oracle import oracle
from tinympc_b200 import workloads as wl
from tinympc_b200.batch import planes_abi, planes_check


def test_batch_planes_fields_match_header():
    IC.assert_batch_fields_match_header("planes")


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
    pal = IC.plane_palette(prob, 12, seed=2)
    which = (np.arange(B) * 5) % 12
    planes = IC.batch_planes(pal, which)
    helper = IC.grouped_oracle(prob, st, planes=planes, nthreads=4)

    def reference(x0_, state, cold):
        outs = []
        for b in range(B):
            p = IC.with_instance(prob, "planes", {k: v[b] for k, v in planes.items()})
            sub = None if state is None else {n: np.array(a[b:b + 1], copy=True) for n, a in state.items()}
            outs.append(oracle.solve_batch(p, st, x0_[b:b + 1], Xref[b:b + 1], None, state=sub, cold_start=cold,
                                           want_state=tuple(H.LIN_STATE), impl="reference"))
        return {k: np.concatenate([o[k] for o in outs]) for k in OUT}

    h1 = helper(x0, Xref, None, None, True, H.LIN_STATE)
    r1 = reference(x0, None, True)
    H.assert_bits_per_instance(h1, r1, OUT, "cold")
    # the planes bite: most instances end with a slack on one of their planes
    act = IC.active_rows(planes, h1["vlnew"], h1["zlnew"])
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
    pset = IC.plane_palette(prob, 1, seed=7)[0]
    # the problem with one extra state row and one extra input row, which this robot pads with zeros
    cons = dict(spec0.constraints)
    cons["Alin_x"] = np.vstack([pset["Alin_x"], np.zeros((1, prob.nx))])
    cons["blin_x"] = np.concatenate([pset["blin_x"], [0.0]])
    cons["Alin_u"] = np.vstack([pset["Alin_u"], np.zeros((1, prob.nu))])
    cons["blin_u"] = np.concatenate([pset["blin_u"], [0.0]])
    spec0.constraints = cons
    padded = H.problem_from_spec(spec0, dt, oracle.port_setup)
    plain = IC.with_instance(padded, "planes", pset)
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
    pal = [IC.own_planes(prob)] + IC.plane_palette(prob, 2, seed=9)
    which = np.arange(B) % 3
    IC.assert_one_run_per_set(monkeypatch, prob, st, x0, Xref, None, which, planes=IC.batch_planes(pal, which))


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
