#!/usr/bin/env python3
"""Evidence for the AUTO kernel-family rule: the same fixed-work batch on each family (on-chip lane groups `gpi`, streamed
lane groups `gps`, thread per instance `tpi`) for the shapes where on-chip residency is low (long horizons, wide inputs,
fp64).  One line per (shape, family); markdown to stdout.  usage: python tools/auto_rule_sweep.py [--B n] [--reps n]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402

from tinympc_b200 import abi, workloads as wl  # noqa: E402
from tinympc_b200._lib import TinyMPCError  # noqa: E402
from tinympc_b200.solver import BatchedTinySolver, setup_problem  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--B", type=int, default=131072)
ap.add_argument("--reps", type=int, default=2)
ap.add_argument("--only", default="", help="f64_12_4: just the fp64 (12,4,50) big-batch row on the on-chip kernel (ncu capture)")
a = ap.parse_args()
FAM = {"gpi": abi.KERNEL_GPI, "gps": abi.KERNEL_GPS, "tpi": abi.KERNEL_TPI, "auto": abi.KERNEL_AUTO}
NAMES = {1: "tpi", 2: "gpi", 4: "gps"}
shapes = [(np.float32, 4, 8, 100), (np.float32, 8, 8, 100), (np.float32, 12, 4, 100), (np.float32, 12, 8, 100), (np.float32, 16, 4, 100),
          (np.float32, 16, 8, 100), (np.float32, 12, 8, 50), (np.float32, 16, 8, 50), (np.float32, 12, 4, 50),
          (np.float64, 12, 4, 50), (np.float64, 6, 3, 100), (np.float64, 4, 2, 100), (np.float64, 4, 4, 100), (np.float64, 4, 2, 50),
          (np.float64, 16, 8, 50),
          # small batches (one thread per instance cannot fill the GPU)
          (np.float64, 12, 4, 50, 4096), (np.float32, 12, 8, 100, 4096), (np.float32, 16, 4, 100, 8192), (np.float64, 8, 4, 50, 16384)]
if a.only == "f64_12_4":
    shapes = [(np.float64, 12, 4, 50)]
print("| dtype | nx | nu | N | B | family asked | ran | plan | ms | ADMM it/s |")
print("|---|---|---|---|---|---|---|---|---|---|")
for shp in shapes:
    dt, nx, nu, N = shp[:4]
    B = shp[4] if len(shp) > 4 else (a.B if dt == np.float32 else a.B // 2)
    spec = wl.random_lti(nx, nu, N, seed=1)
    spec.settings.abs_pri_tol = 0.0
    spec.settings.abs_dua_tol = 0.0
    spec.settings.max_iter = 50
    prob = setup_problem(spec, dt)
    inst = wl.random_instances(B, nx, N, seed=2, dtype=dt)
    for fam in (("gpi",) if a.only else ("auto", "gpi", "gps", "tpi")):
        try:
            s = BatchedTinySolver(prob, spec.settings, device=0, kernel=FAM[fam])
            batch, out = s.make_device_batch(inst["x0"], inst["Xref"], None, cold_start=True)
            ms = []
            for _ in range(a.reps + 1):
                s.solve_device(batch)
                torch.cuda.synchronize()
                ms.append(s.stats()["kernel_ms"])
            st = s.stats()
            best = min(ms[1:])
            plan = f"L={st['lanes_per_instance']} {st['instances_per_cta']}/CTA x{st['ctas']}"
            print(f"| {np.dtype(dt).name} | {nx} | {nu} | {N} | {B} | {fam} | {NAMES[st['kernel_family']]} | {plan} | {best:.3f} | "
                  f"{int(out['iter'].sum().item()) / best * 1e3:.3e} |", flush=True)
            s.close()
            del batch, out
            torch.cuda.empty_cache()
        except TinyMPCError as e:
            print(f"| {np.dtype(dt).name} | {nx} | {nu} | {N} | {B} | {fam} | n/a | {str(e)[:50]} | | |", flush=True)
