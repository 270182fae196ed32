#!/usr/bin/env python3
"""Device time of one batched solve with the handle's box bounds and with per-instance bounds (tinympc_batch_t.bounds_per_instance).

  C3  65 536 fp32 quadrotors, tracking, N = 50, to convergence, on the on-chip kernel:
        shared      the handle's bounds (the fp32 min / max clamp: no bound is a signed zero)
        l1_equal    layout 1, every instance's column equal to the handle's
        l1_fleet    layout 1, a fleet: every robot's thrust and state limits scaled by its own factor in [0.6, 1]
        l2_equal    layout 2, every instance's horizon equal to the handle's (the per-knot reload on the handle's numbers)
  C4  16 384 fp64 rockets, cones, N = 100, per-instance references, to convergence, on the streamed kernel:
        shared      the handle's bounds (two instances per lane group)
        l1_fleet    layout 1, per-robot thrust limits scaled by [0.6, 1] (one instance per lane group)

The arms of a workload alternate step by step in one process; every step flushes L2 (256 MiB write) and is timed with CUDA events
around tinympc_b200_solve; median of --steps after --warmup rounds.  The equal-bounds arms must return the shared arm's outputs
bit for bit.  The card's name, power limit and SM clock are read in the same run.  Prints one JSON line.

    python tools/instance_bounds_bench.py [--steps 10] [--warmup 3]
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
from tinympc_b200.solver import BatchedTinySolver, setup_problem  # noqa: E402

FAMILY = {abi.KERNEL_GPI: "GPI", abi.KERNEL_GPS: "GPS", abi.KERNEL_TPI: "TPI"}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit, smax, sm = [s.strip() for s in out.split(",")]
        return dict(name=name, power_limit=limit, sm_clock_max=smax, sm_clock_idle=sm)
    except Exception as e:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(0), power_limit=f"not read ({e})")


def equal(prob, B, layout):
    out = {}
    for k in ("x_min", "x_max", "u_min", "u_max"):
        a = np.asarray(getattr(prob, k))
        col = a[:, 0] if layout == 1 else a.T
        out[k] = torch.as_tensor(np.ascontiguousarray(np.broadcast_to(col, (B,) + col.shape)), device="cuda:0")
    return out


def fleet(prob, B, sides, seed):
    """layout 1: the handle's column 0 scaled per robot by a factor in [0.6, 1] on the given sides"""
    rng = np.random.default_rng(seed)
    out = {}
    for side in ("x", "u"):
        f = (0.6 + 0.4 * rng.random((B, 1))) if side in sides else np.ones((B, 1))
        for k in (side + "_min", side + "_max"):
            out[k] = torch.as_tensor((np.asarray(getattr(prob, k))[:, 0][None, :] * f).astype(prob.dtype), device="cuda:0")
    return out


def run(s, inst, arms, steps, warmup):
    """arms: name -> bounds dict or None; alternated step by step"""
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")
    ms = {a: [] for a in arms}
    last, plan = {}, {}
    for k in range(warmup + steps):
        for a, bnd in arms.items():
            batch, res = s.make_device_batch(inst["x0"], inst["Xref"], inst.get("Uref"), cold_start=True, bounds=bnd)
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            s.solve_device(batch)
            e1.record()
            torch.cuda.synchronize()
            if k >= warmup:
                ms[a].append(e0.elapsed_time(e1))
            last[a] = res
            st = s.stats()
            plan[a] = dict(family=FAMILY[st["kernel_family"]], lanes_per_instance=st["lanes_per_instance"],
                           instances_per_cta=st["instances_per_cta"], ctas=st["ctas"])
    B = inst["x0"].shape[0]
    out = {}
    for a in arms:
        med = float(np.median(ms[a]))
        out[a] = dict(ms_median=med, ms_min=float(np.min(ms[a])), ms_max=float(np.max(ms[a])), instances_per_s=B / (med * 1e-3),
                      mean_iters=float(last[a]["iter"].float().mean().item()), plan=plan[a])
    for a in arms:
        if a.endswith("equal"):
            for k in ("sol_x", "sol_u", "iter", "residuals"):
                assert torch.equal(last[a][k].view(torch.uint8), last["shared"][k].view(torch.uint8)), (a, k)
    return out


def c3(steps, warmup, B=65536):
    spec = wl.quadrotor(N=50)
    prob = setup_problem(spec, np.float32)
    s = BatchedTinySolver(prob, spec.settings, device=0)
    inst = wl.tracking_instances(B, N=50, seed=0, dtype=np.float32)
    arms = dict(shared=None, l1_equal=equal(prob, B, 1), l1_fleet=fleet(prob, B, "xu", 1), l2_equal=equal(prob, B, 2))
    out = dict(workload=f"quadrotor tracking, fp32, N=50, {B} instances, to convergence", **run(s, inst, arms, steps, warmup))
    s.close()
    return out


def c4(steps, warmup, B=16384):
    spec = wl.rocket(N=100)
    prob = setup_problem(spec, np.float64)
    s = BatchedTinySolver(prob, spec.settings, device=0)
    inst = wl.rocket_instances(B, N=100, seed=0, dtype=np.float64, per_instance_refs=True)
    arms = dict(shared=None, l1_fleet=fleet(prob, B, "u", 2))
    out = dict(workload=f"rocket landing, cones, fp64, N=100, per-instance refs, {B} instances, to convergence",
               **run(s, inst, arms, steps, warmup))
    s.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps(dict(gpu=card(), C3=c3(a.steps, a.warmup), C4=c4(a.steps, a.warmup))))


if __name__ == "__main__":
    main()
