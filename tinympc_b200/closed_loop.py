"""Device-resident closed-loop MPC (SURVEY.md §8f-1): thousands of simulated plants stepping without host round trips.

Mirrors the loop of the reference's examples (examples/quadrotor_tracking.cpp:77-106):

    tiny_set_x0(solver, x0); work->Xref = window(k); [work->y = 0; work->g = 0;] tiny_solve(solver);
    x0 = Adyn * x0 + Bdyn * work->u.col(0)

with the whole TinyWorkspace state of every instance kept on the GPU between steps (warm start) and the plant
update done by tinympc_b200_advance() (tinympc_b200_advance_models() for a fleet with per-instance models,
tinympc_b200_advance_plant() for plants that are not the controller's model).  torch only owns the device buffers.
"""
from __future__ import annotations

import ctypes as C

from . import abi
from ._lib import check
from .batch import KINDS, per_instance, problem_dims
from .solver import AdaptiveRho, BatchedTinySolver, pack_models

# box-constrained warm start: slacks + duals (+ the previous-iteration slacks v, z, which only feed the dual residual of
# the next solve's first iteration; drop them with exact_first_residual=False for ~30 % more steps per second)
# Cones / hyperplanes: pass extra_state=("x", "u", <the family's slack / dual fields>), e.g. ("x", "u", "vcnew", "zcnew", "gc", "yc") —
# solve() re-initialises those slacks from the previous rollout work->x / work->u (admm.cpp:352-376).
WARM_FIELDS = ("v", "z", "vnew", "znew", "g", "y")
WARM_FIELDS_FAST = ("vnew", "znew", "g", "y")


def pack_plant(plant: dict, nx: int, nu: int, B: int, dtype, device="cpu"):
    """plant = dict(A [nx, nx], B [nx, nu], f [nx]) for one plant shared by every robot, or the same with a leading B for one
    plant per robot (other keys are ignored) -> (records, per_instance): the plant records A | B | f, each column-major (the
    first pieces of a model blob), as one contiguous torch tensor [nx*nx + nx*nu + nx] or [B, ...] of `dtype` on `device`."""
    import torch

    if not isinstance(plant, dict):
        raise ValueError("plant must be a dict with the keys A, B and f")
    missing = [k for k in ("A", "B", "f") if plant.get(k) is None]
    if missing:
        raise ValueError(f"plant: {', '.join(missing)} missing (A, B and f are required)")
    arrs = {}
    for k in ("A", "B", "f"):
        a = torch.as_tensor(plant[k], device=device)
        if not a.is_floating_point():
            raise ValueError(f"plant: {k} must be a floating-point array, not {a.dtype}")
        arrs[k] = a.to(dtype)
    per = arrs["A"].dim() == 3
    lead = (B,) if per else ()
    for k, shape in (("A", (nx, nx)), ("B", (nx, nu)), ("f", (nx,))):
        if tuple(arrs[k].shape) != lead + shape:
            raise ValueError(f"plant: A, B, f must be [{nx}, {nx}], [{nx}, {nu}], [{nx}] (one plant) or the same with a leading "
                             f"{B} (one per robot); {k} is {list(arrs[k].shape)}")
    cm = lambda a: a.transpose(-1, -2).reshape(lead + (-1,))  # noqa: E731
    return torch.cat([cm(arrs["A"]), cm(arrs["B"]), arrs["f"]], dim=-1).contiguous(), per


class DeviceMPCLoop:
    def __init__(self, solver: BatchedTinySolver, x0, reset_duals: bool = False, extra_state=(), exact_first_residual: bool = True,
                 adaptive_rho: AdaptiveRho | None = None, models=None, bounds: dict | None = None, cones: dict | None = None,
                 planes: dict | None = None, plant: dict | None = None):
        """models ([B, blob], tinympc_batch_t.models, e.g. from setup_models): a heterogeneous fleet, one model, cache and rho
        per plant.  Every step solves with them and advances plant b with its own A, B, f (tinympc_b200_advance_models).
        adaptive_rho: every plant adapts its own rho / Kinf / Pinf, kept on the device across steps in self.models
        (starting from `models` or the problem's own cache), as one TinySolver per robot would; with `models`, give it
        per-instance tables (solver.setup_sensitivity_device), which stay on the GPU with the models.
        bounds: per-instance box bounds of every plant (a dict as in BatchedTinySolver.solve), kept on the device across steps
        in self.bounds; step(..., bounds=...) replaces them for one step (a moving corridor).
        cones: per-instance cone coefficients of every plant (a dict as in BatchedTinySolver.solve), kept on the device across
        steps in self.cones; step(..., cones=...) replaces them for one step.
        planes: per-instance static hyperplanes of every plant (a dict as in BatchedTinySolver.solve), converted to the ABI's
        column-major layout once and kept on the device across steps in self.planes; step(..., planes=...) replaces them for one
        step (a moving obstacle's fresh half-space).
        plant: the real robots the controller drives, dict(A=, B=, f=) for one plant shared by the batch or the same with a
        leading B for one per robot (e.g. workloads.plant_fleet), packed once into plant records on the device (self.plant).
        Every step advances the plants with them (tinympc_b200_advance_plant) instead of the controller's model."""
        import torch

        self.solver = solver
        self.reset_duals = reset_duals
        self.fields = tuple(WARM_FIELDS if exact_first_residual else WARM_FIELDS_FAST) + tuple(extra_state)
        p = solver.problem
        self._tdt = torch.float32 if p.dtype.__name__ == "float32" else torch.float64
        self.dev = torch.device("cuda", solver.device)
        self.x0 = torch.as_tensor(x0, dtype=self._tdt, device=self.dev).reshape(-1, p.nx).contiguous().clone()
        self.B = self.x0.shape[0]
        self.state = None
        self.out = None
        self._first = True
        self.want_solution = True  # also return solution->x / solution->u (= vnew / znew) every step
        self.adaptive_rho = adaptive_rho
        if adaptive_rho is not None and adaptive_rho.per_instance:
            # per-instance tables live on the GPU across steps, in the column-major storage the solve reads (no copy per step)
            cm = lambda a: torch.as_tensor(a, device=self.dev).to(self._tdt).transpose(1, 2).contiguous().transpose(1, 2)  # noqa: E731
            self.adaptive_rho = AdaptiveRho(cm(adaptive_rho.dKinf_drho), cm(adaptive_rho.dPinf_drho), adaptive_rho.rho_min,
                                            adaptive_rho.rho_max, adaptive_rho.enable_clipping)
        for kind, arrays in dict(bounds=bounds, cones=cones, planes=planes).items():
            setattr(self, kind, None if arrays is None else self._device(kind, arrays))
        self.plant, self.plant_per_instance = None, False
        if plant is not None:
            self.plant, self.plant_per_instance = pack_plant(plant, p.nx, p.nu, self.B, self._tdt, self.dev)
        self.models = None
        if adaptive_rho is not None or models is not None:
            m = pack_models(p, self.B) if models is None else models
            self.models = torch.as_tensor(m, dtype=self._tdt, device=self.dev).reshape(self.B, -1).contiguous().clone()

    def _device(self, kind, arrays):
        """one kind's per-instance arrays checked, each kept on the device in ABI layout (contiguous) and handed on as its view
        in the user's layout, which make_device_batch uses in place"""
        import torch

        p = self.solver.problem
        per_instance(kind, arrays, self.B, problem_dims(p), p.dtype)
        to_abi = KINDS[kind].to_abi
        return {k: to_abi(k, to_abi(k, torch.as_tensor(v, device=self.dev)).contiguous()) for k, v in arrays.items() if v is not None}

    def _noise(self, noise, shape, what):
        import torch

        n = torch.as_tensor(noise, device=self.dev)
        if not n.is_floating_point():
            raise ValueError(f"{what}: noise must be a floating-point array, not {n.dtype}")
        if tuple(n.shape) != shape:
            raise ValueError(f"{what}: noise must be {list(shape)}")
        return n.to(self._tdt).contiguous()

    def step(self, Xref, Uref=None, stream=None, bounds=None, cones=None, planes=None, noise=None):
        """One MPC step for every instance: solve (warm-started), then advance the plants.  Returns the output dict
        (device tensors: sol_x, sol_u, iter, solved, residuals and the state fields).  bounds: per-instance box bounds for this
        step only, in place of the loop's; cones: per-instance cone coefficients for this step only, likewise; planes:
        per-instance static hyperplanes for this step only, likewise.  noise ([B, nx]): measurement noise; the solve starts
        from x0 + noise and the plants advance from the true x0."""
        import torch

        s = self.solver
        st = stream if stream is not None else torch.cuda.current_stream(s.device)
        x_meas = self.x0
        if noise is not None:
            n = self._noise(noise, (self.B, s.problem.nx), "step")
            with torch.cuda.stream(st):
                x_meas = self.x0 + n
        if self.state is not None and self.reset_duals:
            self.state["g"].zero_()
            self.state["y"].zero_()
        het = self.models is not None and self.adaptive_rho is None
        batch, out = s.make_device_batch(x_meas, Xref, Uref, state=self.state, cold_start=self._first, want_state=self.fields,
                                         want_u0=True, want_solution=self.want_solution, models=self.models if het else None,
                                         **{kind: getattr(self, kind) if over is None else over
                                            for kind, over in dict(bounds=bounds, cones=cones, planes=planes).items()})
        if self.adaptive_rho is None:
            s.solve_device(batch, stream)
        else:
            s.solve_device_adaptive(batch, self.models, self.adaptive_rho, stream)
        self.state = {n: out[n] for n in self.fields}
        self.out = out
        self._first = False
        x0p, u0p = C.c_void_p(self.x0.data_ptr()), C.c_void_p(out["u0"].data_ptr())
        if self.plant is not None:
            check(s._lib.tinympc_b200_advance_plant(s._h, self.B, x0p, u0p, s.problem.nu, C.c_void_p(self.plant.data_ptr()),
                                                    int(self.plant_per_instance), C.c_void_p(st.cuda_stream)))
        elif self.models is None:
            check(s._lib.tinympc_b200_advance(s._h, self.B, x0p, u0p, s.problem.nu, C.c_void_p(st.cuda_stream)))
        else:
            check(s._lib.tinympc_b200_advance_models(s._h, self.B, x0p, u0p, s.problem.nu, C.c_void_p(self.models.data_ptr()),
                                                     C.c_void_p(st.cuda_stream)))
        return out

    def rollout(self, Xref_traj, T: int, Uref_traj=None, w=None, stream=None, noise=None):
        """T steps in one launch (tinympc_b200_rollout): bit-identical to
            for t in range(T): self.step(Xref_traj[..., t:t+N, :], Uref_traj[..., t:t+N-1, :], noise=noise[:, t]); self.x0 += w[:, t]
        with the warm state kept on chip between steps, against the loop's plants.  Xref_traj: [B, >= T+N-1, nx] or
        [>= T+N-1, nx]; Uref_traj: [B, >= T+N-2, nu] or [>= T+N-2, nu] or None; w, noise: [B, T, nx] or None.  Returns device
        tensors with a step axis: x [B, T+1, nx] (the true plant state before every step and after the last), u [B, T, nu],
        iter / solved [B, T], residuals [B, T, 4].  Leaves x0, state and out as the T steps would.  Box constraints only,
        without adaptive rho (the on-chip kernel's rollout variant)."""
        import torch

        if self.adaptive_rho is not None:
            raise ValueError("rollout: adaptive rho is not available in a rollout; use step()")
        for kind in KINDS:
            if getattr(self, kind) is not None:
                raise ValueError(f"rollout: per-instance {kind} are not available in a rollout; use step()")
        if len(self.fields) != len(WARM_FIELDS if "v" in self.fields else WARM_FIELDS_FAST):
            raise ValueError("rollout: covers box constraints only (no extra_state); use step()")
        T = int(T)
        if T < 0:
            raise ValueError("rollout: T must be >= 0")
        s, p = self.solver, self.solver.problem
        B, N = self.B, p.N
        st = stream if stream is not None else torch.cuda.current_stream(s.device)

        def traj(a, knots, width, name):
            a = torch.as_tensor(a, device=self.dev).to(self._tdt)
            if a.dim() not in (2, 3) or a.shape[-2] < knots or a.shape[-1] != width or (a.dim() == 3 and a.shape[0] != B):
                raise ValueError(f"rollout: {name} must be [{B}, >= {knots}, {width}] or [>= {knots}, {width}]")
            return a[..., :knots, :].contiguous()

        X = traj(Xref_traj, T + N - 1, p.nx, "Xref_traj")
        U = None if Uref_traj is None else traj(Uref_traj, T + N - 2, p.nu, "Uref_traj")
        W = None
        if w is not None:
            W = torch.as_tensor(w, device=self.dev).to(self._tdt).contiguous()
            if tuple(W.shape) != (B, T, p.nx):
                raise ValueError(f"rollout: w must be [{B}, {T}, {p.nx}]")
        Nz = None if noise is None else self._noise(noise, (B, T, p.nx), "rollout")
        if self.state is not None and self.reset_duals:
            self.state["g"].zero_()
            self.state["y"].zero_()
        kw = dict(dtype=self._tdt, device=self.dev)
        state = self.state
        if state is None:
            state = {n: torch.zeros((B, N, p.nx) if abi.STATE_IS_X[n] else (B, N - 1, p.nu), **kw) for n in self.fields}
        het = self.models is not None
        res = dict(x=torch.empty((B, T + 1, p.nx), **kw), u=torch.empty((B, T, p.nu), **kw),
                   iter=torch.empty((B, T), dtype=torch.int32, device=self.dev),
                   solved=torch.empty((B, T), dtype=torch.int32, device=self.dev), residuals=torch.empty((B, T, 4), **kw))
        sol_x = torch.empty((B, N, p.nx), **kw) if self.want_solution else None
        sol_u = torch.empty((B, N - 1, p.nu), **kw) if self.want_solution else None
        b = abi.Batch()
        b.B, b.x0, b.cold_start = B, self.x0.data_ptr(), int(self._first)
        for n, a in state.items():
            setattr(b.state, n, a.data_ptr())
        b.sol_x = None if sol_x is None else sol_x.data_ptr()
        b.sol_u = None if sol_u is None else sol_u.data_ptr()
        b.models = self.models.data_ptr() if het else None
        r = abi.Rollout()
        r.T, r.reset_duals, r.carry_v = T, int(self.reset_duals), int("v" in self.fields)
        r.Xref, r.xref_per_instance = X.data_ptr(), int(X.dim() == 3)
        r.Uref, r.uref_per_instance = (None, 0) if U is None else (U.data_ptr(), int(U.dim() == 3))
        r.w = None if W is None else W.data_ptr()
        r.plant = None if self.plant is None else self.plant.data_ptr()
        r.plant_per_instance = int(self.plant_per_instance)
        r.noise = None if Nz is None else Nz.data_ptr()
        r.x_traj, r.u_traj, r.residuals_traj = res["x"].data_ptr(), res["u"].data_ptr(), res["residuals"].data_ptr()
        r.iter_traj, r.solved_traj = res["iter"].data_ptr(), res["solved"].data_ptr()
        check(s._lib.tinympc_b200_rollout(s._h, C.byref(b), C.byref(r), C.c_void_p(st.cuda_stream)))
        self._roll_inputs = (X, U, W, Nz)  # read by the launch on `stream`
        if T == 0:
            res["x"] = self.x0.clone().reshape(B, 1, p.nx)
            return res
        self.state = state
        self.out = dict(sol_x=sol_x, sol_u=sol_u, u0=res["u"][:, -1], iter=res["iter"][:, -1], solved=res["solved"][:, -1],
                        residuals=res["residuals"][:, -1], **state)
        self._first = False
        with torch.cuda.stream(st):
            self.x0.copy_(res["x"][:, -1])
        return res
