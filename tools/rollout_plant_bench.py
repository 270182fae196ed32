#!/usr/bin/env python3
"""What a plant of its own costs a closed-loop rollout: C3 fp32 (65 536 quadrotors (12,4), N = 50, per-robot sliding references,
duals reset, work->v / z carried, default settings) for T = 50 steps, four ways, alternating in one process:

  plain        DeviceMPCLoop.rollout against the controller's own model (the GPI_ROLLOUT kernel)
  plant        the same against a per-robot plant fleet (workloads.plant_fleet, masses +-20 %, a steady drift; GPI_PLANT)
  plant+noise  the same with measurement noise on every step's state
  steps        DeviceMPCLoop.step x T with the same plants and noise (tinympc_b200_advance_plant between solves)

Each is timed with CUDA events around the whole episode after a synchronise; the median of --reps repetitions after --warmup
is reported in milliseconds per step.  The noisy rollout's outputs (x, u, iter, solved, residuals per step; final state, x0,
sol_x, sol_u) are compared bit for bit with the step loop's of the same repetition.  Prints one JSON line with the card's name
and power limit.

    python tools/rollout_plant_bench.py [--T 50] [--batch 65536] [--reps 5] [--warmup 1]
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

from tinympc_b200 import workloads as wl  # noqa: E402
from tinympc_b200.closed_loop import DeviceMPCLoop  # noqa: E402
from tinympc_b200.solver import BatchedTinySolver, setup_problem  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def finish(loop, res):
    res = dict(res)
    res.update({n: loop.state[n] for n in loop.fields})
    res.update(sol_x=loop.out["sol_x"], sol_u=loop.out["sol_u"], x0=loop.x0)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=50)
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    B, T, dt = a.batch, a.T, np.float32
    spec = wl.quadrotor(N=50)
    N = spec.N
    solver = BatchedTinySolver(setup_problem(spec, dt), spec.settings, device=0)
    inst = wl.tracking_instances(B, N=T + N - 1, seed=0, dtype=dt)
    x0 = torch.as_tensor(inst["x0"], device="cuda:0")
    X = torch.as_tensor(inst["Xref"], device="cuda:0")
    plant = wl.plant_fleet(spec, B, seed=1, mass_spread=0.2, drift=0.002)
    noise = torch.as_tensor((0.01 * np.random.default_rng(2).standard_normal((B, T, spec.nx))).astype(dt), device="cuda:0")

    def rollout(pl, nz):
        loop = DeviceMPCLoop(solver, x0, reset_duals=True, plant=pl)
        ms, res = timed(lambda: loop.rollout(X, T, noise=nz))
        return ms, finish(loop, res), solver.stats()

    def steps():
        loop = DeviceMPCLoop(solver, x0, reset_duals=True, plant=plant)
        per = {k: [] for k in ("x", "u", "iter", "solved", "residuals")}

        def run():
            for t in range(T):
                per["x"].append(loop.x0.clone())
                out = loop.step(X[:, t:t + N], noise=noise[:, t])
                for k, o in (("u", "u0"), ("iter", "iter"), ("solved", "solved"), ("residuals", "residuals")):
                    per[k].append(out[o])
            per["x"].append(loop.x0.clone())

        ms, _ = timed(run)
        return ms, finish(loop, {k: torch.stack(v, 1) for k, v in per.items()})

    ms = {k: [] for k in ("plain", "plant", "plant+noise", "steps")}
    equal, iters, plans = True, {}, {}
    for r in range(a.warmup + a.reps):
        t_plain, plain, plans["plain"] = rollout(None, None)
        t_plant, own, plans["plant"] = rollout(plant, None)
        t_noise, got, plans["plant+noise"] = rollout(plant, noise)
        t_steps, ref = steps()
        for k, v in ref.items():
            equal = equal and torch.equal(got[k].contiguous().view(torch.uint8), v.contiguous().view(torch.uint8))
        for k, res in (("plain", plain), ("plant", own), ("plant+noise", got), ("steps", ref)):
            iters[k] = float(res["iter"].double().mean().item())
        if r >= a.warmup:
            for k, t in (("plain", t_plain), ("plant", t_plant), ("plant+noise", t_noise), ("steps", t_steps)):
                ms[k].append(t / T)
    solver.close()
    med = {k: float(np.median(v)) for k, v in ms.items()}
    keys = ("kernel_family", "lanes_per_instance", "instances_per_cta", "ctas", "threads_per_cta")
    print(json.dumps({"card": card(), "batch": B, "T": T, "reps": a.reps, "mean_iters_per_step": iters,
                      "noisy_rollout_equals_steps": equal, "ms_per_step": med,
                      "ms_per_step_range": {k: [min(v), max(v)] for k, v in ms.items()},
                      "plans": {k: {q: p[q] for q in keys} for k, p in plans.items()},
                      "plant_record_bytes_per_robot_step": (spec.nx * spec.nx + spec.nx * spec.nu + spec.nx) * 4}))


if __name__ == "__main__":
    main()
