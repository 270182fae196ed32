#!/usr/bin/env python3
"""Closed-loop episodes of T steps: DeviceMPCLoop.step called T times against one DeviceMPCLoop.rollout (tinympc_b200_rollout),
alternating in one process, on three workloads:

  C3 fp32   65 536 quadrotors (12,4), N = 50, per-robot sliding reference, duals reset, work->v / z carried, to convergence
  C3 fp64   the same in fp64
  fleet     C3 fp32 with six quadrotor models (input gain and weights varied) dealt to the robots with a stride of five

Per repetition: one timed step episode (and, when the planner puts the step off chip, one with the on-chip family forced), one
timed rollout (CUDA events around the whole episode, after a synchronise), and one
untimed step episode that reads stats() after every step for the kernel time and keeps every per-step output.  The rollout's
outputs (x, u, iter, solved, residuals per step; final state, x0, sol_x, sol_u) are compared bit for bit with that episode's.
Reports the median over the repetitions of milliseconds per step, and kernel time from stats().  Prints one JSON line with the
card's name and power limit.

    python tools/rollout_bench.py [--T 50] [--batch 65536] [--reps 5] [--warmup 1]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tinympc_b200 import abi, workloads as wl  # noqa: E402
from tinympc_b200.closed_loop import DeviceMPCLoop  # noqa: E402
from tinympc_b200.solver import BatchedTinySolver, setup_models, setup_problem  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def fleet_models(spec, dt, M=6):
    A = np.stack([spec.A] * M)
    Bm = np.stack([spec.B * (1.0 + 0.05 * i) for i in range(M)])
    f = np.stack([spec.f] * M)
    Q = np.stack([spec.Qdiag * (1.0 + 0.2 * i) for i in range(M)])
    R = np.stack([spec.Rdiag * (1.0 + 0.1 * i) for i in range(M)])
    return setup_models(12, 4, A, Bm, f, Q, R, np.array([spec.rho] * M), dtype=dt)


def episode_steps(solver, x0, X, T, models, timed):
    """T calls of DeviceMPCLoop.step -> (ms, kernel ms (None when timed), outputs)"""
    N = solver.problem.N
    loop = DeviceMPCLoop(solver, x0, reset_duals=True, models=models)
    per = {k: [] for k in ("x", "u", "iter", "solved", "residuals")}
    kms = 0.0
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(T):
        if not timed:
            per["x"].append(loop.x0.clone())
        out = loop.step(X[:, t:t + N])
        if not timed:
            kms += solver.stats()["kernel_ms"]
            for k, o in (("u", "u0"), ("iter", "iter"), ("solved", "solved"), ("residuals", "residuals")):
                per[k].append(out[o])
    e1.record()
    torch.cuda.synchronize()
    if timed:
        return e0.elapsed_time(e1), None, None, solver.stats()
    per["x"].append(loop.x0.clone())
    res = {k: torch.stack(v, 1) for k, v in per.items()}
    res.update({n: loop.state[n] for n in loop.fields})
    res.update(sol_x=loop.out["sol_x"], sol_u=loop.out["sol_u"], x0=loop.x0)
    return None, kms, res, None


def episode_rollout(solver, x0, X, T, models):
    loop = DeviceMPCLoop(solver, x0, reset_duals=True, models=models)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    res = loop.rollout(X, T)
    e1.record()
    torch.cuda.synchronize()
    st = solver.stats()
    res = dict(res)
    res.update({n: loop.state[n] for n in loop.fields})
    res.update(sol_x=loop.out["sol_x"], sol_u=loop.out["sol_u"], x0=loop.x0)
    return e0.elapsed_time(e1), st["kernel_ms"], res, st


def plan(st):
    return dict(family=st["kernel_family"], lanes_per_instance=st["lanes_per_instance"], warps_per_cta=st["threads_per_cta"] // 32,
                instances_per_cta=st["instances_per_cta"], ctas=st["ctas"])


def run(name, dt, B, T, reps, warmup, fleet):
    spec = wl.quadrotor(N=50)
    prob = setup_problem(spec, dt)
    solver = BatchedTinySolver(prob, spec.settings, device=0)
    inst = wl.tracking_instances(B, N=T + 49, seed=0, dtype=dt)
    x0 = torch.as_tensor(inst["x0"], device="cuda:0")
    X = torch.as_tensor(inst["Xref"], device="cuda:0")
    models = None
    if fleet:
        models = torch.as_tensor(fleet_models(spec, dt)[(5 * np.arange(B)) % 6], device="cuda:0").contiguous()
    # the planner sends some big batches off chip (thread per instance); the rollout only exists on chip, so the step loop is
    # also timed with the on-chip family forced, which separates the rollout's own effect from the family choice
    gpi = BatchedTinySolver(prob, spec.settings, device=0, kernel=abi.KERNEL_GPI)
    ms_step, ms_gpi, ms_roll, k_step, k_roll, equal = [], [], [], [], [], True
    iters = None
    for r in range(warmup + reps):
        t_step, _, _, st_step = episode_steps(solver, x0, X, T, models, timed=True)
        t_gpi = episode_steps(gpi, x0, X, T, models, timed=True)[0] if st_step["kernel_family"] != abi.KERNEL_GPI else t_step
        t_roll, kr, got, st_roll = episode_rollout(solver, x0, X, T, models)
        _, ks, ref, _ = episode_steps(solver, x0, X, T, models, timed=False)
        for k, v in ref.items():
            same = torch.equal(got[k].contiguous().view(torch.uint8), v.contiguous().view(torch.uint8))
            equal = equal and same
        iters = float(ref["iter"].double().mean().item())
        if r >= warmup:
            ms_step.append(t_step / T)
            ms_gpi.append(t_gpi / T)
            ms_roll.append(t_roll / T)
            k_step.append(ks / T)
            k_roll.append(kr / T)
    solver.close()
    gpi.close()
    med = lambda v: float(np.median(v))  # noqa: E731
    return dict(workload=name, batch=B, T=T, reps=reps, mean_iters_per_step=iters, bit_identical=equal,
                step_ms_per_step=med(ms_step), rollout_ms_per_step=med(ms_roll), speedup=med(ms_step) / med(ms_roll),
                step_on_chip_ms_per_step=med(ms_gpi), step_ms_range=[min(ms_step), max(ms_step)], rollout_ms_range=[min(ms_roll), max(ms_roll)],
                step_kernel_ms_per_step=med(k_step), rollout_kernel_ms_per_step=med(k_roll),
                step_plan=plan(st_step), rollout_plan=plan(st_roll))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=50)
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    res = {"card": card(), "results": [
        run("C3 tracking fp32", np.float32, a.batch, a.T, a.reps, a.warmup, False),
        run("C3 tracking fp64", np.float64, a.batch, a.T, a.reps, a.warmup, False),
        run("C3 tracking fp32, 6-model fleet", np.float32, a.batch, a.T, a.reps, a.warmup, True)]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
