#!/usr/bin/env python3
"""Device time of one batched solve with the handle's static hyperplanes and with per-instance ones
(tinympc_batch_t.planes_per_instance), on the streamed kernel.

  quad    65 536 fp32 hyperplane quadrotors (two state planes, one input plane), N = 50, per-instance references, fixed
          work (zero tolerances, 50 iterations)
  rocket  16 384 fp64 rockets with their cones plus a state plane (a lateral corridor) and an input plane, N = 100,
          per-instance references, to convergence
for each:
  shared  the handle's planes
  equal   per-instance planes, every instance's equal to the handle's
  fleet   per-robot planes (workloads.plane_fleet)

The arms alternate step by step in one process; every step flushes L2 (256 MiB write) and is timed with CUDA events around
tinympc_b200_solve; median of --steps after --warmup rounds.  The equal arm must return the shared arm's outputs bit for bit.
The card's name, power limit and SM clock are read in the same run.  Prints one JSON line with every arm's plan (lanes per
instance, instances per lane group, warps and CTAs).

    python tools/instance_planes_bench.py [--steps 10] [--warmup 3]
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


def run(s, inst, arms, steps, warmup):
    """arms: name -> planes dict or None; alternated step by step"""
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")
    ms = {a: [] for a in arms}
    last, plan = {}, {}
    for k in range(warmup + steps):
        for a, planes in arms.items():
            batch, res = s.make_device_batch(inst["x0"], inst["Xref"], inst.get("Uref"), cold_start=True, planes=planes)
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


def _arms(spec, prob, B):
    dev = torch.device("cuda", 0)
    t = lambda d: {k: torch.as_tensor(v, device=dev) for k, v in d.items()}  # noqa: E731
    own = {k: np.asarray(getattr(prob, k)) for k in ("Alin_x", "blin_x", "Alin_u", "blin_u")}
    equal = t({k: np.repeat((v if k[0] == "A" else v.reshape(-1))[None], B, axis=0) for k, v in own.items()})
    fleet = t(wl.plane_fleet(spec, B, seed=1, dtype=prob.dtype))
    return dict(shared=None, equal=equal, fleet=fleet)


def quad(steps, warmup, B=65536, N=50):
    spec = wl.quadrotor(N=N, hz=50)
    s_ = abi.Settings.from_buffer_copy(spec.settings)
    s_.en_state_bound = s_.en_input_bound = 0
    s_.en_state_linear = s_.en_input_linear = 1
    s_.max_iter, s_.abs_pri_tol, s_.abs_dua_tol = 50, 0.0, 0.0
    Ax = np.zeros((2, 12)); Ax[0, 0] = 1.0; Ax[0, 1] = 0.5; Ax[1, 2] = -1.0; Ax[1, 0] = 0.25  # noqa: E702
    spec.constraints = dict(Alin_x=Ax, blin_x=np.array([0.3, -0.2]), Alin_u=np.array([[1.0, 1.0, 1.0, 1.0]]), blin_u=np.array([0.4]))
    spec.settings = s_
    prob = setup_problem(spec, np.float32)
    s = BatchedTinySolver(prob, s_, device=0)
    inst = wl.tracking_instances(B, N=N, seed=0, dtype=np.float32, jitter=0.3)
    out = dict(workload=f"hyperplane quadrotor, fp32, N={N}, per-instance refs, {B} instances, 50 iterations (fixed work)",
               **run(s, inst, _arms(spec, prob, B), steps, warmup))
    s.close()
    return out


def rocket(steps, warmup, B=16384):
    spec = wl.rocket(N=100)
    spec.constraints = dict(spec.constraints, Alin_x=np.array([[1.0, 0.5, 0.0, 0.0, 0.0, 0.0]]), blin_x=np.array([1.0]),
                            Alin_u=np.array([[1.0, 1.0, 0.0]]), blin_u=np.array([4.0]))
    spec.settings.en_state_linear = spec.settings.en_input_linear = 1
    prob = setup_problem(spec, np.float64)
    s = BatchedTinySolver(prob, spec.settings, device=0)
    inst = wl.rocket_instances(B, N=100, seed=0, dtype=np.float64, per_instance_refs=True)
    out = dict(workload=f"rocket landing, cones + hyperplanes, fp64, N=100, per-instance refs, {B} instances, to convergence",
               **run(s, inst, _arms(spec, prob, B), steps, warmup))
    s.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps(dict(gpu=card(), quad=quad(a.steps, a.warmup), rocket=rocket(a.steps, a.warmup))))


if __name__ == "__main__":
    main()
