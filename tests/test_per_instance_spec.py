"""CPU checks of the per-instance data spec (tinympc_b200.batch.KINDS, per_instance) through HostBatch: the accepted inputs of
box bounds, cone coefficients and static hyperplanes, the mode each sets in the batch, the ABI layout of their arrays, and
a ValueError naming the kind for every malformed input."""
import numpy as np
import pytest

import helpers as H
from oracle import oracle
from tinympc_b200 import abi, workloads as wl
from tinympc_b200.batch import KINDS, HostBatch

B = 3


def _bounds():
    prob = H.problem_from_spec(wl.quadrotor(N=10), np.float32, oracle.port_setup)
    dt, nx, nu, N = prob.dtype, prob.nx, prob.nu, prob.N
    good = dict(x_min=np.full((B, nx), -1, dt), x_max=np.full((B, nx), 1, dt), u_min=np.full((B, nu), -1, dt),
                u_max=np.full((B, nu), 1, dt))
    horizon = dict(x_min=np.full((B, N, nx), -1, dt), x_max=np.full((B, N, nx), 1, dt), u_min=np.full((B, N - 1, nu), -1, dt),
                   u_max=np.full((B, N - 1, nu), 1, dt))
    bad = [dict(good, x_min=good["x_min"][:, :5]), dict(good, x_min=good["x_min"].astype(np.float64)), {"x_min": good["x_min"]},
           dict(good, u_min=horizon["u_min"]), dict(good, q=good["x_min"]), {}]
    return prob, [(good, 1), (horizon, 2), ({k: good[k] for k in ("x_min", "x_max")}, 1)], bad


def _cones():
    prob = H.problem_from_spec(wl.rocket(N=10), np.float64, oracle.port_setup)
    dt = prob.dtype
    good = dict(x_mu=np.full((B, len(prob.Acx)), 0.5, dt), u_mu=np.full((B, len(prob.Acu)), 0.5, dt))
    bad = [dict(good, x_mu=good["x_mu"][:, :0]), dict(good, u_mu=good["u_mu"][:-1]), dict(good, x_mu=good["x_mu"].astype(np.float32)),
           dict(good, x_mu=good["x_mu"][:, :, None]), dict(good, mu=good["x_mu"]), {}]
    return prob, [(good, 1), ({"u_mu": good["u_mu"]}, 1)], bad


def _planes():
    prob = H.problem_from_spec(H.quad_linear_spec(N=10), np.float32, oracle.port_setup)
    dt, nx, nu = prob.dtype, prob.nx, prob.nu
    nlx, nlu = prob.Alin_x.shape[0], prob.Alin_u.shape[0]
    good = dict(Alin_x=np.zeros((B, nlx, nx), dt), blin_x=np.zeros((B, nlx), dt), Alin_u=np.zeros((B, nlu, nu), dt),
                blin_u=np.zeros((B, nlu), dt))
    bad = [dict(good, Alin_x=good["Alin_x"][:, :, :-1]), dict(good, blin_u=good["blin_u"][:-1]),
           dict(good, Alin_x=good["Alin_x"].astype(np.float64)), {"Alin_x": good["Alin_x"]}, dict(good, A=good["Alin_x"]), {},
           {"A": 1}, dict(good, blin_u=np.zeros((B, 2), dt)), dict(good, Alin_x=np.zeros((B, nx, nlx), dt))]
    return prob, [(good, 1), ({k: good[k] for k in ("Alin_x", "blin_x")}, 1)], bad


@pytest.mark.parametrize("kind", ["bounds", "cones", "planes"])
def test_check_and_layout(kind):
    prob, goods, bad = dict(bounds=_bounds, cones=_cones, planes=_planes)[kind]()
    spec = KINDS[kind]
    x0, Xref = np.zeros((B, prob.nx), prob.dtype), np.zeros((prob.N, prob.nx), prob.dtype)
    for arrays, mode in goods:
        hb = HostBatch(prob, x0, Xref, **{kind: arrays})
        b = hb.to_c()
        assert getattr(b, spec.mode_field) == mode
        assert sorted(getattr(hb, kind)) == sorted(spec.fields[k] for k in arrays)
        for k in spec.fields.values():
            a = getattr(hb, kind).get(k)
            assert getattr(b, k) == (None if a is None else a.ctypes.data)
    assert getattr(HostBatch(prob, x0, Xref).to_c(), spec.mode_field) == 0
    for arrays in bad:
        with pytest.raises(ValueError, match=kind):
            HostBatch(prob, x0, Xref, **{kind: arrays})
    if kind == "planes":  # each instance's matrix goes column-major: element (row i, column j) of instance b at b*nx*nlx + j*nlx + i
        nx, nlx = prob.nx, prob.Alin_x.shape[0]
        A = np.arange(B * nlx * nx, dtype=prob.dtype).reshape(B, nlx, nx)
        hb = HostBatch(prob, x0, Xref, planes=dict(Alin_x=A, blin_x=goods[0][0]["blin_x"]))
        flat = hb.planes["Alin_x"].reshape(-1)
        b, i, j = 2, 1, 5
        assert flat[b * nx * nlx + j * nlx + i] == A[b, i, j]
        assert abi.Batch.from_buffer_copy(hb.to_c()).Alin_x == hb.planes["Alin_x"].ctypes.data
