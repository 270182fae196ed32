#!/usr/bin/env python3
"""BASELINE config 5: synthetic random-LTI sweep nx x nu x N, fp32, fixed work (max_iter=50, tolerances 0) -> roofline
table (ADMM iterations/s, algorithmic HBM bytes vs peak, fp32-pipe fraction), plus configs 3 and 4 at full size.
Writes a markdown table to stdout; one GPU.  B per GPU = 2^20 / 8 = 131072 (the 8-GPU share of the config)."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402

from tinympc_b200 import abi, workloads as wl  # noqa: E402
from tinympc_b200.solver import BatchedTinySolver, setup_problem  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--B", type=int, default=131072)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--quick", action="store_true")
a = ap.parse_args()
peaks = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "MEASURED_PEAKS.json")
HBM = float(json.load(open(peaks))["hbm_gbs"]) if os.path.exists(peaks) else 3350.0  # H100 SXM data sheet


def run(spec, dt, inst, kernel, mode, reps):
    prob = setup_problem(spec, dt)
    s = BatchedTinySolver(prob, spec.settings, device=0, mode=mode, kernel=kernel)
    batch, out = s.make_device_batch(inst["x0"], inst["Xref"], inst.get("Uref"), cold_start=True)
    ms = []
    for _ in range(reps + 1):
        s.solve_device(batch)
        torch.cuda.synchronize()
        ms.append(s.stats()["kernel_ms"])
    st = s.stats()
    iters = int(out["iter"].sum().item())
    solved = int(out["solved"].sum().item())
    s.close()
    return min(ms[1:]), iters, solved, st


def bytes_inst(nx, nu, N, es, per_inst_ref):
    nN, mN = nx * N, nu * (N - 1)
    return es * nx + es * (nN + mN) * (1 if per_inst_ref else 0) + es * (nN + mN) + 4 * es + 8


def flops_iter(nx, nu, N):
    return (N - 1) * (4 * nx * nx + 8 * nx * nu + 2 * nu * nu + 5 * nx + 4 * nu) + 2 * nx * nx + 15 * (nx * N + nu * (N - 1))


print("| workload | nx | nu | N | B | dtype | kernel | mode | ms | instances/s | ADMM it/s | solved | alg. GB/s | HBM frac | fp32/64 TFLOP/s |")
print("|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|")


def row(name, spec, dt, inst, B, kernel, kname, mode, mname, per_inst_ref):
    try:
        ms, iters, solved, st = run(spec, dt, inst, kernel, mode, a.reps)
    except Exception as e:  # unsupported combination (e.g. GPI does not fit): report, do not hide
        print(f"| {name} | {spec.nx} | {spec.nu} | {spec.N} | {B} | {np.dtype(dt).name} | {kname} | {mname} | n/a ({str(e)[:60]}) | | | | | | |")
        return
    es = np.dtype(dt).itemsize
    gbs = B * bytes_inst(spec.nx, spec.nu, spec.N, es, per_inst_ref) / (ms * 1e-3) / 1e9
    tf = iters * flops_iter(spec.nx, spec.nu, spec.N) / (ms * 1e-3) / 1e12
    lanes, ipc = st["lanes_per_instance"], st["instances_per_cta"]
    fam = {1: "tpi", 2: f"gpi L={lanes} {ipc}/SM", 4: f"gps L={lanes} {ipc}/SM"}[st["kernel_family"]]
    print(f"| {name} | {spec.nx} | {spec.nu} | {spec.N} | {B} | {np.dtype(dt).name} | {fam} | {mname} | {ms:.3f} | {B / ms * 1e3:.3e} | "
          f"{iters / ms * 1e3:.3e} | {solved / B:.2f} | {gbs:.1f} | {gbs / HBM:.5f} | {tf:.2f} |", flush=True)


S, F = abi.MODE_STRICT, abi.MODE_FAST
# configs 2, 3, 4 at full size
spec = wl.quadrotor(N=50)
row("C2 hovering", spec, np.float32, wl.hovering_instances(65536, N=50), 65536, abi.KERNEL_GPI, "gpi", S, "strict", False)
row("C2 hovering", spec, np.float32, wl.hovering_instances(65536, N=50), 65536, abi.KERNEL_TPI, "tpi", S, "strict", False)
row("C2 hovering", spec, np.float32, wl.hovering_instances(65536, N=50), 65536, abi.KERNEL_GPI, "gpi", F, "fast", False)
row("C3 tracking", spec, np.float32, wl.tracking_instances(65536, N=50, seed=0), 65536, abi.KERNEL_GPI, "gpi", S, "strict", True)
row("C3 tracking", spec, np.float32, wl.tracking_instances(65536, N=50, seed=0), 65536, abi.KERNEL_TPI, "tpi", S, "strict", True)
spec = wl.rocket(N=100)
row("C4 rocket+SOC", spec, np.float64, wl.rocket_instances(16384, N=100, seed=0), 16384, abi.KERNEL_AUTO, "auto", S, "strict", False)
row("C4 rocket+SOC", spec, np.float64, wl.rocket_instances(16384, N=100, seed=0), 16384, abi.KERNEL_TPI, "tpi", S, "strict", False)
# config 5 sweep (fixed work)
for nx in (4, 8, 12, 16):
    for nu in (2, 4, 8):
        for N in ((10, 50, 100) if not a.quick else (50,)):
            spec = wl.random_lti(nx, nu, N, seed=1)
            spec.settings.abs_pri_tol = 0.0
            spec.settings.abs_dua_tol = 0.0
            spec.settings.max_iter = 50
            inst = wl.random_instances(a.B, nx, N, seed=2)
            row("C5 LTI fixed-work", spec, np.float32, inst, a.B, abi.KERNEL_AUTO, "auto", S, "strict", False)
            if N == 100 and nu != 2:  # the AUTO rule's evidence: both families on the long horizons
                row("C5 (forced tpi)", spec, np.float32, inst, a.B, abi.KERNEL_TPI, "tpi", S, "strict", False)
