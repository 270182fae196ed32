"""Device-resident closed-loop MPC (SURVEY.md §8f-1): thousands of simulated plants stepping without host round trips.

Mirrors the loop of the reference's examples (examples/quadrotor_tracking.cpp:77-106):

    tiny_set_x0(solver, x0); work->Xref = window(k); [work->y = 0; work->g = 0;] tiny_solve(solver);
    x0 = Adyn * x0 + Bdyn * work->u.col(0)

with the whole TinyWorkspace state of every instance kept on the GPU between steps (warm start) and the plant
update done by tinympc_b200_advance().  torch only owns the device buffers.
"""
from __future__ import annotations

import ctypes as C

from . import abi
from ._lib import check
from .solver import AdaptiveRho, BatchedTinySolver, pack_models

# box-constrained warm start: slacks + duals (+ the previous-iteration slacks v, z, which only feed the dual residual of
# the next solve's first iteration; drop them with exact_first_residual=False for ~30 % more steps per second)
# Cones / hyperplanes: pass extra_state=("x", "u", <the family's slack / dual fields>), e.g. ("x", "u", "vcnew", "zcnew", "gc", "yc") —
# solve() re-initialises those slacks from the previous rollout work->x / work->u (admm.cpp:352-376).
WARM_FIELDS = ("v", "z", "vnew", "znew", "g", "y")
WARM_FIELDS_FAST = ("vnew", "znew", "g", "y")


class DeviceMPCLoop:
    def __init__(self, solver: BatchedTinySolver, x0, reset_duals: bool = False, extra_state=(), exact_first_residual: bool = True,
                 adaptive_rho: AdaptiveRho | None = None, models=None):
        """adaptive_rho: every plant adapts its own rho / Kinf / Pinf, kept on the device across steps in self.models
        ([B, blob], starting from `models` or the problem's own cache), as one TinySolver per robot would."""
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
        self.models = None
        if adaptive_rho is not None:
            m = pack_models(p, self.B) if models is None else models
            self.models = torch.as_tensor(m, dtype=self._tdt, device=self.dev).reshape(self.B, -1).contiguous().clone()

    def step(self, Xref, Uref=None, stream=None):
        """One MPC step for every instance: solve (warm-started), then advance the plants.  Returns the output dict
        (device tensors: sol_x, sol_u, iter, solved, residuals and the state fields)."""
        import torch

        s = self.solver
        if self.state is not None and self.reset_duals:
            self.state["g"].zero_()
            self.state["y"].zero_()
        batch, out = s.make_device_batch(self.x0, Xref, Uref, state=self.state, cold_start=self._first, want_state=self.fields,
                                         want_u0=True, want_solution=self.want_solution)
        if self.adaptive_rho is None:
            s.solve_device(batch, stream)
        else:
            s.solve_device_adaptive(batch, self.models, self.adaptive_rho, stream)
        self.state = {n: out[n] for n in self.fields}
        self.out = out
        self._first = False
        st = stream if stream is not None else torch.cuda.current_stream(s.device)
        check(s._lib.tinympc_b200_advance(s._h, self.B, C.c_void_p(self.x0.data_ptr()), C.c_void_p(out["u0"].data_ptr()),
                                          s.problem.nu, C.c_void_p(st.cuda_stream)))
        return out
