#!/usr/bin/env python3
"""Device time of one batched solve with and without adaptive rho, on the quadrotor shapes of bench.py:
C2 (hovering, fp32, 65 536 instances, max_iter 100) and C3 (tracking to convergence, fp32, 65 536 instances).

Times the device entry points (tinympc_b200_solve / tinympc_b200_solve_adaptive) with CUDA events around each step and a
256 MiB L2 flush between steps, as bench.py does; every step is a cold start from the same models.  The CPU figure for the same
work is taken on a --cpu-sample of the batch with every host thread: the plain-C restatement of the adaptive solve
(tests/adaptive/adaptive_oracle.c), which is bit-identical to the reference's adaptive loop, and, where the TinyMPC checkout
(TINYMPC_REFERENCE) is present, the reference's own compiled stage functions (tests/adaptive/ref_adaptive_driver.cpp, one
thread: the driver is sequential).  Prints one JSON line.

    python tools/adaptive_rho_bench.py [--steps 10] [--warmup 3] [--batch 65536] [--cpu-sample 4096]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from tinympc_b200 import workloads as wl  # noqa: E402
from tinympc_b200.solver import AdaptiveRho, BatchedTinySolver, pack_models, setup_problem  # noqa: E402


def cpu_figure(prob, settings, ar, inst, sample):
    """instances/s of the CPU checkers on the first `sample` instances (cold start, same settings)"""
    import time

    import adaptive_common as AC

    x0, Xref = inst["x0"][:sample], inst["Xref"] if inst["Xref"].ndim == 2 else inst["Xref"][:sample]
    models = pack_models(prob, sample)
    out = {}
    t0 = time.perf_counter()
    AC.oracle_solve(prob, settings, x0, Xref, None, None, True, models, ar, nthreads=os.cpu_count() or 1)
    out["restatement"] = dict(instances_per_s=sample / (time.perf_counter() - t0), threads=os.cpu_count() or 1, instances=sample)
    ref = os.environ.get("TINYMPC_REFERENCE", "/root/reference")
    if os.path.exists(os.path.join(ref, "src", "tinympc", "admm.cpp")):
        import tempfile

        sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
        import make_golden_adaptive as MG

        n = min(sample, 256)
        with tempfile.TemporaryDirectory() as td:
            lib = MG.build_ref(td, prob.dtype)
            t0 = time.perf_counter()
            AC.oracle_solve(prob, settings, x0[:n], Xref if Xref.ndim == 2 else Xref[:n], None, None, True, models[:n], ar, lib=lib,
                            fn="tinympc_ref_solve_adaptive")
            out["reference_driver"] = dict(instances_per_s=n / (time.perf_counter() - t0), threads=1, instances=n,
                                           note="includes one tiny_setup per instance: the driver builds a TinySolver per instance "
                                                "so that no adapted cache leaks into the next one")
    return out


def run(name, inst, steps, warmup, cpu_sample):
    spec = wl.quadrotor(N=50)
    prob = setup_problem(spec, np.float32)
    tables = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "reference",
                                  "sensitivity_tables.npz"))
    ar = AdaptiveRho(tables["t0"].astype(np.float32), tables["t1"].astype(np.float32))
    s = BatchedTinySolver(prob, spec.settings, device=0)
    B = inst["x0"].shape[0]
    models = torch.as_tensor(pack_models(prob, B), device="cuda:0").contiguous()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")
    out = {}
    for adaptive in (False, True):
        ms, iters = [], 0
        for k in range(warmup + steps):
            batch, res = s.make_device_batch(inst["x0"], inst["Xref"], cold_start=True, want_residuals=False)
            m = models.clone() if adaptive else None
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            if adaptive:
                s.solve_device_adaptive(batch, m, ar)
            else:
                s.solve_device(batch)
            e1.record()
            torch.cuda.synchronize()
            if k >= warmup:
                ms.append(e0.elapsed_time(e1))
            iters = int(res["iter"].sum().item())
        st = s.stats()
        out["adaptive" if adaptive else "fixed"] = dict(
            ms_median=float(np.median(ms)), ms_min=float(np.min(ms)), mean_iters=iters / B,
            plan=dict(lanes_per_instance=st["lanes_per_instance"], warps_per_cta=st["threads_per_cta"] // 32,
                      instances_per_cta=st["instances_per_cta"], ctas=st["ctas"], smem_bytes_per_cta=st["smem_bytes_per_cta"]))
    s.close()
    out["workload"] = name
    if cpu_sample:
        out["cpu_adaptive"] = cpu_figure(prob, spec.settings, ar, inst, min(cpu_sample, B))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--cpu-sample", type=int, default=4096, help="instances for the CPU figure (0: skip it)")
    a = ap.parse_args()
    B = a.batch
    res = {"gpu": torch.cuda.get_device_name(0), "batch": B,
           "C2": run("quadrotor hovering N=50 fp32, max_iter 100", wl.hovering_instances(B, N=50, dtype=np.float32), a.steps, a.warmup,
                 a.cpu_sample),
           "C3": run("quadrotor tracking N=50 fp32, to convergence", wl.tracking_instances(B, N=50, seed=0, dtype=np.float32), a.steps,
                     a.warmup, a.cpu_sample)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
