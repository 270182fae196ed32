#!/usr/bin/env python3
"""Device time of one batched solve on the streamed lane-group kernel (GPS) with a shared model and with per-instance models
(tinympc_batch_t.models, the kernel's one-instance-per-lane-group variant).

  C4   rocket landing with cones, fp64, N = 100, per-instance references, 16 384 instances, 100 iterations (tolerances 0, so
       every instance does the same work whatever its model):
         shared     the handle's model (two instances per lane group, as bench.py runs C4)
         identical  pack_models blobs: the per-instance-model variant on the shared model's numbers
         fleet      workloads.rocket_fleet: every rocket has its own mass (input matrix scaled by 1/m)
  box  quadrotor tracking, box constraints, fp64, N = 200 (no on-chip plan for this horizon), 16 384 instances, 50 iterations:
       shared model vs a fleet tuned per robot (rho, state weights); the plan that ran is printed and must be GPS.

Times tinympc_b200_solve with CUDA events around each step and a 256 MiB L2 flush before it; median of --steps after --warmup.
The card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/het_streamed_bench.py [--steps 10] [--warmup 3] [--batch 16384]
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
from tinympc_b200.solver import BatchedTinySolver, pack_models, setup_problem  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return dict(name=name, power_limit=limit)
    except Exception as e:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(0), power_limit=f"not read ({e})")


def settings(spec, max_iter):
    st = abi.Settings.from_buffer_copy(spec.settings)
    st.abs_pri_tol = st.abs_dua_tol = 0.0
    st.max_iter = max_iter
    return st


def time_solve(s, inst, models, steps, warmup):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")
    ms = []
    for k in range(warmup + steps):
        batch, res = s.make_device_batch(inst["x0"], inst["Xref"], inst.get("Uref"), cold_start=True, want_residuals=False,
                                         models=models)
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        s.solve_device(batch)
        e1.record()
        torch.cuda.synchronize()
        if k >= warmup:
            ms.append(e0.elapsed_time(e1))
    st = s.stats()
    B = inst["x0"].shape[0]
    return dict(ms_median=float(np.median(ms)), ms_min=float(np.min(ms)), instances_per_s=B / (float(np.median(ms)) * 1e-3),
                mean_iters=float(res["iter"].float().mean().item()),
                plan=dict(family={abi.KERNEL_GPI: "GPI", abi.KERNEL_GPS: "GPS", abi.KERNEL_TPI: "TPI"}[st["kernel_family"]],
                          lanes_per_instance=st["lanes_per_instance"], warps_per_cta=st["threads_per_cta"] // 32,
                          instances_per_cta=st["instances_per_cta"], ctas=st["ctas"], smem_bytes_per_cta=st["smem_bytes_per_cta"],
                          workspace_bytes=st["workspace_bytes"]))


def fleet_models(s, fl):
    return s.setup_models_device(fl["A"], fl["B"], fl["f"], fl["Qdiag"], fl["Rdiag"], fl["rho"])


def c4(B, steps, warmup):
    spec = wl.rocket(N=100)
    prob = setup_problem(spec, np.float64)
    s = BatchedTinySolver(prob, settings(spec, 100), device=0)
    inst = wl.rocket_instances(B, N=100, seed=0, dtype=np.float64, per_instance_refs=True)
    out = dict(workload=f"rocket landing, cones, fp64, N=100, per-instance refs, {B} instances, 100 iterations")
    out["shared"] = time_solve(s, inst, None, steps, warmup)
    out["identical"] = time_solve(s, inst, torch.as_tensor(pack_models(prob, B), device="cuda:0"), steps, warmup)
    out["fleet"] = time_solve(s, inst, fleet_models(s, wl.rocket_fleet(B, N=100, seed=1, mass_spread=0.3)), steps, warmup)
    s.close()
    for k in ("shared", "identical", "fleet"):
        assert out[k]["plan"]["family"] == "GPS", out[k]
    return out


def box_off_chip(B, steps, warmup):
    N = 200
    spec = wl.quadrotor(N=N)
    prob = setup_problem(spec, np.float64)
    s = BatchedTinySolver(prob, settings(spec, 50), device=0)
    inst = wl.tracking_instances(B, N=N, seed=0, dtype=np.float64)
    t = lambda a: np.tile(np.asarray(a, np.float64)[None], (B,) + (1,) * np.ndim(a))  # noqa: E731
    k = np.arange(B) % 6
    models = s.setup_models_device(t(spec.A), t(spec.B), t(spec.f), t(spec.Qdiag) * (1.0 + 0.25 * k)[:, None], t(spec.Rdiag),
                                   spec.rho * (0.6 + 0.2 * k))
    out = dict(workload=f"quadrotor tracking, box, fp64, N={N} (no on-chip plan), {B} instances, 50 iterations")
    out["shared"] = time_solve(s, inst, None, steps, warmup)
    out["fleet"] = time_solve(s, inst, models, steps, warmup)
    s.close()
    assert out["fleet"]["plan"]["family"] == "GPS", out["fleet"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16384)
    a = ap.parse_args()
    res = dict(gpu=card(), C4=c4(a.batch, a.steps, a.warmup), box_off_chip=box_off_chip(a.batch, a.steps, a.warmup))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
