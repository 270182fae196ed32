"""CPU-side checks of closed loops against plants of their own: workloads.plant_fleet, the plant records DeviceMPCLoop packs
(the A | B | f prefix of a model blob), their input checks, and tinympc_b200_advance_plant's refusal of null arguments.  The
extended tinympc_rollout_t is covered by test_rollout_abi.py's layout check through the ctypes mirror."""
import numpy as np
import pytest
import torch

from tinympc_b200 import _lib, abi, workloads as wl
from tinympc_b200.closed_loop import pack_plant
from tinympc_b200.solver import setup_models


def test_plant_fleet_shapes_and_masses():
    spec = wl.quadrotor(N=50)
    B = 1000
    pl = wl.plant_fleet(spec, B, seed=3, mass_spread=0.2)
    assert pl["A"].shape == (B, 12, 12) and pl["B"].shape == (B, 12, 4) and pl["f"].shape == (B, 12) and pl["m"].shape == (B,)
    assert all(pl[k].dtype == np.float64 for k in ("A", "B", "f", "m"))
    assert (pl["m"] >= 0.8).all() and (pl["m"] <= 1.2).all() and pl["m"].std() > 0.05
    assert np.array_equal(pl["A"], np.broadcast_to(spec.A, (B, 12, 12)))
    assert np.array_equal(pl["B"], spec.B[None] / pl["m"][:, None, None])
    assert np.array_equal(pl["f"], np.broadcast_to(spec.f, (B, 12)))  # no drift
    windy = wl.plant_fleet(spec, B, seed=3, mass_spread=0.2, drift=0.01)
    assert np.array_equal(windy["m"], pl["m"]) and np.array_equal(windy["B"], pl["B"])
    d = windy["f"] - spec.f[None]
    assert 0.008 < d.std() < 0.012 and np.abs(d.mean()) < 0.002
    assert np.array_equal(wl.plant_fleet(spec, B, seed=3)["m"], pl["m"])
    assert not np.array_equal(wl.plant_fleet(spec, B, seed=4)["m"], pl["m"])


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_plant_records_are_the_model_blob_prefix(dt):
    """pack_plant's records equal the A | B | f pieces that setup_models writes at the start of every model blob."""
    nx, nu, B = 8, 4, 5
    spec = wl.random_lti(nx, nu, 10, seed=2)
    rng = np.random.default_rng(1)
    A = spec.A[None] * (1.0 + 0.05 * rng.standard_normal((B, nx, nx)))
    Bm = spec.B[None] * (1.0 + 0.05 * rng.standard_normal((B, nx, nu)))
    f = 0.1 * rng.standard_normal((B, nx))
    blobs = setup_models(nx, nu, A, Bm, f, np.stack([spec.Qdiag] * B), np.stack([spec.Rdiag] * B), np.full(B, spec.rho), dtype=dt)
    tdt = torch.float32 if dt == np.float32 else torch.float64
    rec, per = pack_plant(dict(A=A, B=Bm, f=f), nx, nu, B, tdt)
    n = nx * nx + nx * nu + nx
    assert per and rec.shape == (B, n) and rec.is_contiguous()
    assert np.array_equal(rec.numpy().view(np.uint8), np.ascontiguousarray(blobs[:, :n]).view(np.uint8))
    one, per1 = pack_plant(dict(A=A[2], B=Bm[2], f=f[2]), nx, nu, B, tdt)
    assert not per1 and one.shape == (n,)
    assert np.array_equal(one.numpy().view(np.uint8), np.ascontiguousarray(blobs[2, :n]).view(np.uint8))


def test_plant_records_reject_bad_input():
    nx, nu, B = 4, 2, 3
    good = dict(A=np.eye(nx), B=np.ones((nx, nu)), f=np.zeros(nx))
    for bad in (dict(A=good["A"], B=good["B"]),                       # f missing
                dict(good, f=None),                                    # f missing
                dict(good, A=np.eye(nx + 1)),                          # shape
                dict(good, A=np.stack([np.eye(nx)] * B)),              # per robot A with shared B, f
                dict(good, B=np.ones((B + 1, nx, nu))),                # leading dimension
                dict(good, B=np.ones((nx, nu), np.int32)),             # dtype
                [good["A"], good["B"], good["f"]]):                    # not a dict
        with pytest.raises(ValueError):
            pack_plant(bad, nx, nu, B, torch.float64)


def test_advance_plant_refuses_null_arguments():
    lib = _lib.load()
    assert lib.tinympc_b200_advance_plant(None, 1, None, None, 1, None, 0, None) == abi.ERR_ARG
    assert b"null" in lib.tinympc_b200_last_error()
