#!/usr/bin/env python3
"""Batch-size sweep of the device-resident solve on BASELINE configs 2 and 4 (AUTO family, STRICT): from one instance (latency)
to a million (throughput).  Markdown to stdout.  usage: python tools/batch_sweep.py [--reps n]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402

from tinympc_b200 import abi, workloads as wl  # noqa: E402
from tinympc_b200.solver import BatchedTinySolver, setup_problem  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--only", default="", help="c2 | c4")
ap.add_argument("--max-b", type=int, default=1 << 30)
a = ap.parse_args()
NAMES = {1: "tpi", 2: "gpi", 4: "gps"}
print("| config | B | family | plan | ms per solve | instances/s | ADMM it/s | us per instance-iteration |")
print("|---|---|---|---|---|---|---|---|")
for cfg, sizes in (("C2 quadrotor hovering fp32 N=50, 100 it", [1, 64, 1024, 4096, 16384, 65536, 262144, 1048576]),
                   ("C4 rocket + cones fp64 N=100, 100 it", [1, 64, 1024, 4096, 16384, 65536, 131072])):
    if a.only and not cfg.lower().startswith(a.only):
        continue
    for B in sizes:
        if B > a.max_b:
            continue
        if cfg.startswith("C2"):
            spec, dt = wl.quadrotor(N=50), np.float32
            inst = wl.hovering_instances(B, N=50, dtype=dt)
        else:
            spec, dt = wl.rocket(N=100), np.float64
            inst = wl.rocket_instances(B, N=100, seed=0, dtype=dt)
        s = BatchedTinySolver(setup_problem(spec, dt), spec.settings, device=0, kernel=abi.KERNEL_AUTO)
        batch, out = s.make_device_batch(inst["x0"], inst["Xref"], inst.get("Uref"), cold_start=True)
        ms = []
        for _ in range(a.reps + 1):
            s.solve_device(batch)
            torch.cuda.synchronize()
            ms.append(s.stats()["kernel_ms"])
        st = s.stats()
        best = min(ms[1:])
        iters = int(out["iter"].sum().item())
        plan = f"L={st['lanes_per_instance']} x{st['ctas']} CTAs"
        print(f"| {cfg} | {B} | {NAMES[st['kernel_family']]} | {plan} | {best:.3f} | {B / best * 1e3:.3e} | {iters / best * 1e3:.3e} | "
              f"{best * 1e3 / iters:.4f} |", flush=True)
        s.close()
        del batch, out
        torch.cuda.empty_cache()
