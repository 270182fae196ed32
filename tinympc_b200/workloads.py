"""Workload definitions = the reference's examples restated as data + seeded instance generators.

These are the five BASELINE.json configs (SURVEY.md §8d):
  C1 cartpole            examples/cartpole_example.cpp:32-70
  C2 quadrotor hovering  examples/quadrotor_hovering.cpp:18-66 with N=50
  C3 quadrotor tracking  examples/quadrotor_tracking.cpp:33-106 with N=50, per-instance reference windows
  C4 rocket landing      examples/rocket_landing_mpc.cpp:46-135 with N=100, cones enabled
  C5 random LTI sweep    (no reference example; generator defined in SURVEY §8d)
Numeric tables come from tinympc_b200/data/*.npz (written by tools/extract_problem_data.py).
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field

import numpy as np

from . import abi
from .problem import default_settings

_DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data")


@dataclass
class ModelSpec:
    """User-level arguments of tiny_setup (tiny_api.hpp:10-12) + constraint setters + settings."""
    name: str
    nx: int
    nu: int
    N: int
    rho: float
    A: np.ndarray
    B: np.ndarray
    f: np.ndarray
    Qdiag: np.ndarray
    Rdiag: np.ndarray
    constraints: dict = field(default_factory=dict)  # kwargs of MPCProblem (x_min, ..., Acx, ...)
    settings: abi.Settings = field(default_factory=default_settings)


def _load(name):
    return np.load(os.path.join(_DATA, name))


def cartpole(N=10) -> ModelSpec:
    A = np.array([[1.0, 0.01, 0.0, 0.0], [0.0, 1.0, 0.039, 0.0], [0.0, 0.0, 1.002, 0.01], [0.0, 0.0, 0.458, 1.002]])
    B = np.array([[0.0], [0.02], [0.0], [0.067]])
    s = default_settings()
    s.max_iter = 100  # cartpole_example.cpp:58
    big = 1e17  # :45-48
    return ModelSpec("cartpole", 4, 1, N, 1.0, A, B, np.zeros(4), np.array([10.0, 1.0, 10.0, 1.0]), np.array([1.0]),
                     dict(x_min=np.full(4, -big), x_max=np.full(4, big), u_min=np.full(1, -big), u_max=np.full(1, big)), s)


def quadrotor(N=50, hz=20) -> ModelSpec:
    d = _load(f"quadrotor_{hz}hz.npz")
    s = default_settings()
    s.max_iter = 100  # quadrotor_hovering.cpp:54
    return ModelSpec(f"quadrotor_{hz}hz", 12, 4, N, float(d["rho"]), d["A"], d["B"], d["f"], d["Q"], d["R"],
                     dict(x_min=np.full(12, -5.0), x_max=np.full(12, 5.0), u_min=np.full(4, -0.5), u_max=np.full(4, 0.5)), s)


def rocket(N=100, cones=True) -> ModelSpec:
    d = _load("rocket_20hz.npz")
    s = default_settings()
    s.max_iter = 100  # rocket_landing_mpc.cpp:97
    s.abs_pri_tol = 2e-3  # :98
    if cones:  # the shipped example never flips these (SURVEY A.3-4); BASELINE config 4 asks for the conic path
        s.en_state_soc = 1
        s.en_input_soc = 1
    cons = dict(
        x_min=np.array([-5.0, -5.0, -0.5, -10.0, -10.0, -20.0]), x_max=np.array([5.0, 5.0, 100.0, 10.0, 10.0, 20.0]),
        u_min=np.full(3, -10.0), u_max=np.full(3, 105.0),
        # the example calls tiny_set_cone_constraints(solver, Acu,qcu,cu, Acx,qcx,cx) (:94) and the DEFINITION
        # binds the first triple to the STATE cones (tiny_api.cpp:176-178): state mu = 0.25, input mu = 0.5.
        Acx=[0], qcx=[3], cx=[0.25], Acu=[0], qcu=[3], cu=[0.5],
    )
    return ModelSpec("rocket_20hz", 6, 3, N, float(d["rho"]), d["A"], d["B"], d["f"], d["Q"], d["R"], cons, s)


def rocket_fleet(B, N=100, seed=0, mass_spread=0.2) -> dict:
    """A fleet of B rockets of different masses: the 20 Hz rocket's model with instance b's input matrix scaled by 1/m_b,
    m_b = 1 + mass_spread * U(-1, 1) (the thrust acts on a heavier or lighter vehicle; gravity in f does not depend on
    the mass).  -> per-instance A [B,nx,nx], B [B,nx,nu], f [B,nx], Qdiag [B,nx], Rdiag [B,nu], rho [B] (the arguments
    of solver.setup_models), the masses m, and the shared spec (constraints, settings) of rocket(N)."""
    spec = rocket(N=N)
    rng = np.random.default_rng(seed)
    m = 1.0 + mass_spread * rng.uniform(-1.0, 1.0, size=B)
    tile = lambda a: np.tile(np.asarray(a, dtype=np.float64)[None], (B,) + (1,) * np.ndim(a))  # noqa: E731
    return dict(A=tile(spec.A), B=tile(spec.B) / m[:, None, None], f=tile(spec.f), Qdiag=tile(spec.Qdiag),
                Rdiag=tile(spec.Rdiag), rho=np.full(B, spec.rho), m=m, spec=spec)


def plant_fleet(spec: ModelSpec, B, seed=0, mass_spread=0.2, drift=0.0) -> dict:
    """The real robots behind one controller: robot b's plant is the spec's model with its input matrix scaled by 1/m_b,
    m_b = 1 + mass_spread * U(-1, 1) (the convention of rocket_fleet), and its f plus a constant drift drift * N(0, 1) per state
    (a steady wind).  -> dict(A [B,nx,nx], B [B,nx,nu], f [B,nx], m [B]) in float64, the `plant=` argument of DeviceMPCLoop."""
    rng = np.random.default_rng(seed)
    m = 1.0 + mass_spread * rng.uniform(-1.0, 1.0, size=B)
    A = np.tile(np.asarray(spec.A, dtype=np.float64)[None], (B, 1, 1))
    Bm = np.asarray(spec.B, dtype=np.float64)[None] / m[:, None, None]
    f = np.asarray(spec.f, dtype=np.float64).reshape(1, -1) + drift * rng.standard_normal((B, spec.nx))
    return dict(A=A, B=Bm, f=f, m=m)


def cone_fleet(spec: ModelSpec, B, seed=0, scale=(0.6, 1.0), dtype=np.float64) -> dict:
    """Per-robot cone coefficients for a fleet of B robots of `spec` (e.g. rocket(), or rocket_fleet's spec): robot b's mu
    of every state and input cone is the spec's cx / cu times its own factor drawn from U(scale), e.g. a tighter glide
    slope and thrust-vector cone per rocket, or a friction coefficient per legged robot.  -> dict(x_mu [B, ncx],
    u_mu [B, ncu]) of `dtype`, the `cones=` argument of BatchedTinySolver.solve / make_device_batch / DeviceMPCLoop."""
    rng = np.random.default_rng(seed)
    cx = np.asarray(spec.constraints.get("cx", []), dtype=np.float64)
    cu = np.asarray(spec.constraints.get("cu", []), dtype=np.float64)
    lo, hi = scale
    x_mu = cx[None, :] * rng.uniform(lo, hi, size=(B, cx.size))
    u_mu = cu[None, :] * rng.uniform(lo, hi, size=(B, cu.size))
    return dict(x_mu=x_mu.astype(dtype), u_mu=u_mu.astype(dtype))


def plane_fleet(spec: ModelSpec, B, seed=0, tilt=0.25, shift=(-0.3, 0.1), dtype=np.float64) -> dict:
    """Per-robot static hyperplanes for a fleet of B robots of `spec` (a spec with Alin_x / blin_x and / or Alin_u / blin_u
    constraints): robot b's row i is the spec's row i with every non-zero coefficient scaled by its own factor from
    U(1 - tilt, 1 + tilt) and its offset moved by U(shift), e.g. a separating half-space per robot from the obstacle that
    robot sees.  The default shift tightens most rows, so most robots meet an active row.  -> dict(Alin_x [B, nlx, nx],
    blin_x [B, nlx], Alin_u [B, nlu, nu], blin_u [B, nlu]) of `dtype` (the sides the spec has), the `planes=` argument of
    BatchedTinySolver.solve / make_device_batch / DeviceMPCLoop."""
    rng = np.random.default_rng(seed)
    out = {}
    for side in ("x", "u"):
        A = spec.constraints.get("Alin_" + side)
        if A is None:
            continue
        A = np.asarray(A, dtype=np.float64)
        b = np.asarray(spec.constraints["blin_" + side], dtype=np.float64).reshape(-1)
        out["Alin_" + side] = (A[None] * rng.uniform(1.0 - tilt, 1.0 + tilt, size=(B,) + A.shape)).astype(dtype)
        out["blin_" + side] = (b[None] + rng.uniform(*shift, size=(B, b.size))).astype(dtype)
    return out


def random_lti(nx, nu, N, seed=0) -> ModelSpec:
    """SURVEY §8d C5 generator: A = I + 0.05 G rescaled to spectral radius 1, B ~ N(0, 0.1^2)."""
    rng = np.random.default_rng(1000003 * seed + 7919 * nx + 104729 * nu)
    A = np.eye(nx) + 0.05 * rng.standard_normal((nx, nx))
    A = A / np.max(np.abs(np.linalg.eigvals(A)))
    B = 0.1 * rng.standard_normal((nx, nu))
    Q = rng.uniform(1.0, 10.0, nx)
    R = rng.uniform(0.1, 1.0, nu)
    s = default_settings()
    s.max_iter = 50
    return ModelSpec(f"lti_{nx}_{nu}", nx, nu, N, 1.0, A, B, np.zeros(nx), Q, R,
                     dict(x_min=np.full(nx, -10.0), x_max=np.full(nx, 10.0), u_min=np.full(nu, -1.0), u_max=np.full(nu, 1.0)), s)


# ---- instance generators (inputs of one batched tiny_solve) ----------------------------------------------

def hovering_instances(B, N=50, dtype=np.float32):
    """C2: B identical instances, x0 / Xref of quadrotor_hovering.cpp:61-66; Xref shared by the batch."""
    x0 = np.array([0, 1, 0, 0.2, 0, 0, 0.1, 0, 0, 0, 0, 0], dtype=dtype)
    xref = np.zeros(12, dtype=dtype)
    xref[2] = 2.0
    return dict(x0=np.tile(x0, (B, 1)), Xref=np.tile(xref, (N, 1)), Uref=None)


def tracking_instances(B, N=50, seed=0, dtype=np.float32, jitter=0.05):
    """C3: instance b tracks a window of examples/trajectory_data/quadrotor_20hz_y_axis_line.hpp starting at a
    random offset; x0 = first reference point + N(0, jitter^2) on the position states."""
    traj = _load("quadrotor_20hz_y_axis_line.npz")["Xref"]  # (301, 12)
    rng = np.random.default_rng(seed)
    off = rng.integers(0, traj.shape[0] - N + 1, size=B)
    idx = off[:, None] + np.arange(N)[None, :]
    Xref = traj[idx].astype(dtype)  # (B, N, 12)
    x0 = Xref[:, 0, :].copy()
    x0[:, :3] += (jitter * rng.standard_normal((B, 3))).astype(dtype)
    return dict(x0=x0, Xref=Xref, Uref=None)


def rocket_instances(B, N=100, seed=0, dtype=np.float64, spread=0.1, step=0, per_instance_refs=False):
    """C4: x0 = 1.1*xinit*(1 +- spread) per instance, Xref = linear interpolation to the origin over NTOTAL=100
    (rocket_landing_mpc.cpp:104-135), Uref[2] = 10.  per_instance_refs: every instance sits at its own closed-loop step
    (uniform in 0..20, the `k` of rocket_landing_mpc.cpp:131-135) and gets its own Xref window and Uref copy
    ([B][N][nx] / [B][N-1][nu], the 14 440 B/instance case of SURVEY §8d)."""
    xinit = np.array([4, 2, 20, -3, 2, -4.5], dtype=np.float64)
    rng = np.random.default_rng(seed)
    x0 = 1.1 * xinit[None, :] * (1.0 + spread * rng.uniform(-1, 1, size=(B, 6)))
    ntotal = 100
    Uref = np.zeros((N - 1, 3))
    Uref[:, 2] = 10.0
    if per_instance_refs:
        steps = rng.integers(0, 21, size=B)
        k = (np.arange(N)[None, :] + steps[:, None])[:, :, None]  # (B, N, 1)
        Xref = xinit[None, None, :] + (0.0 - xinit[None, None, :]) * k / (ntotal - 1)
        Uref = np.broadcast_to(Uref[None], (B, N - 1, 3))
        return dict(x0=x0.astype(dtype), Xref=np.ascontiguousarray(Xref, dtype=dtype), Uref=np.ascontiguousarray(Uref, dtype=dtype))
    k = (np.arange(N) + step)[:, None]
    Xref = xinit[None, :] + (0.0 - xinit[None, :]) * k / (ntotal - 1)
    return dict(x0=x0.astype(dtype), Xref=Xref.astype(dtype), Uref=Uref.astype(dtype))


def random_instances(B, nx, N, seed=0, dtype=np.float32):
    rng = np.random.default_rng(seed)
    return dict(x0=rng.standard_normal((B, nx)).astype(dtype), Xref=np.zeros((N, nx), dtype=dtype), Uref=None)
