#!/usr/bin/env python3
"""Device time of one batched solve with the handle's cone coefficients and with per-instance ones
(tinympc_batch_t.cones_per_instance).

  C4  16 384 fp64 rockets, cones, N = 100, per-instance references, to convergence, on the streamed kernel:
        shared        the handle's mu (two instances per lane group)
        equal         per-instance mu, every instance's equal to the handle's
        fleet         per-robot mu: every state and input cone's mu scaled by the robot's own factor in [0.6, 1]
                      (workloads.cone_fleet)
        models        per-robot masses (workloads.rocket_fleet), the handle's mu (one instance per lane group)
        fleet_models  per-robot masses and per-robot mu

The arms alternate step by step in one process; every step flushes L2 (256 MiB write) and is timed with CUDA events around
tinympc_b200_solve; median of --steps after --warmup rounds.  The equal arm must return the shared arm's outputs bit for bit.
The card's name, power limit and SM clock are read in the same run.  Prints one JSON line with every arm's plan (lanes per
instance, instances per lane group, warps and CTAs).

    python tools/instance_cones_bench.py [--steps 10] [--warmup 3]
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
from tinympc_b200.solver import BatchedTinySolver, setup_models, setup_problem  # noqa: E402

FAMILY = {abi.KERNEL_GPI: "GPI", abi.KERNEL_GPS: "GPS", abi.KERNEL_TPI: "TPI"}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit, smax, sm = [s.strip() for s in out.split(",")]
        return dict(name=name, power_limit=limit, sm_clock_max=smax, sm_clock_idle=sm)
    except Exception as e:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(0), power_limit=f"not read ({e})")


def run(s, inst, arms, steps, warmup):
    """arms: name -> (models tensor or None, cones dict or None); alternated step by step"""
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")
    ms = {a: [] for a in arms}
    last, plan = {}, {}
    for k in range(warmup + steps):
        for a, (models, cones) in arms.items():
            batch, res = s.make_device_batch(inst["x0"], inst["Xref"], inst.get("Uref"), cold_start=True, models=models, cones=cones)
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
            groups = st["threads_per_cta"] // st["lanes_per_instance"]
            plan[a] = dict(family=FAMILY[st["kernel_family"]], lanes_per_instance=st["lanes_per_instance"],
                           instances_per_group=st["instances_per_cta"] // groups, warps=st["threads_per_cta"] // 32, ctas=st["ctas"],
                           instances_per_cta=st["instances_per_cta"], smem_bytes_per_cta=st["smem_bytes_per_cta"])
    B = inst["x0"].shape[0]
    out = {}
    for a in arms:
        med = float(np.median(ms[a]))
        out[a] = dict(ms_median=med, ms_min=float(np.min(ms[a])), ms_max=float(np.max(ms[a])), instances_per_s=B / (med * 1e-3),
                      mean_iters=float(last[a]["iter"].float().mean().item()), plan=plan[a])
    for k in ("sol_x", "sol_u", "iter", "residuals"):
        assert torch.equal(last["equal"][k].view(torch.uint8), last["shared"][k].view(torch.uint8)), ("equal", k)
    base = out["shared"]["ms_median"]
    for a in arms:
        out[a]["vs_shared"] = out[a]["ms_median"] / base
    return out


def c4(steps, warmup, B=16384):
    spec = wl.rocket(N=100)
    prob = setup_problem(spec, np.float64)
    s = BatchedTinySolver(prob, spec.settings, device=0)
    inst = wl.rocket_instances(B, N=100, seed=0, dtype=np.float64, per_instance_refs=True)
    dev = torch.device("cuda", 0)
    t = lambda d: {k: torch.as_tensor(v, device=dev) for k, v in d.items()}  # noqa: E731
    equal = t(dict(x_mu=np.tile(prob.cx, (B, 1)), u_mu=np.tile(prob.cu, (B, 1))))
    fleet = t(wl.cone_fleet(spec, B, seed=1, scale=(0.6, 1.0)))
    f = wl.rocket_fleet(B, N=100, seed=2)
    models = torch.as_tensor(setup_models(6, 3, f["A"], f["B"], f["f"], f["Qdiag"], f["Rdiag"], f["rho"], dtype=np.float64), device=dev)
    arms = dict(shared=(None, None), equal=(None, equal), fleet=(None, fleet), models=(models, None), fleet_models=(models, fleet))
    out = dict(workload=f"rocket landing, cones, fp64, N=100, per-instance refs, {B} instances, to convergence",
               **run(s, inst, arms, steps, warmup))
    s.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps(dict(gpu=card(), C4=c4(a.steps, a.warmup))))


if __name__ == "__main__":
    main()
