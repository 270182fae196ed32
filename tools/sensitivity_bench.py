#!/usr/bin/env python3
"""Device time of the batched sensitivity precompute next to the cache precompute, and of the adaptive solve with
per-instance tables next to the shared-table one.

Part 1: tinympc_b200_precompute_sensitivity_batch_device and tinympc_b200_precompute_cache_batch_device for --models
differently tuned quadrotors (rho and state weights vary per model), fp32 and fp64, CUDA events around each call, the two
calls alternating.  Part 2: tinympc_b200_solve_adaptive on the C3 shape of tools/adaptive_rho_bench.py (quadrotor tracking
N=50 fp32, to convergence, cold start from the same models, 256 MiB L2 flush between steps) with one shared table pair and with
that pair repeated per instance, alternating; the two give bit-identical results, so the difference is the table reads.
Prints one JSON line with the card's name and power limit.  Needs a GPU: there is no CPU path.

    python tools/sensitivity_bench.py [--steps 10] [--warmup 3] [--models 65536] [--batch 65536]
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
from tinympc_b200.solver import AdaptiveRho, BatchedTinySolver, pack_models, setup_problem  # noqa: E402


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def precompute(dt, M, steps, warmup):
    sp = wl.quadrotor(N=50)
    s = BatchedTinySolver(setup_problem(sp, dt), sp.settings, device=0)
    tdt = torch.float32 if dt == np.float32 else torch.float64
    rng = np.random.default_rng(0)
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a), device="cuda:0").to(tdt)  # noqa: E731
    A, Bm, f = (t(np.broadcast_to(a, (M,) + np.shape(a))) for a in (sp.A, np.reshape(sp.B, (sp.nx, sp.nu)), sp.f))
    Q, R = t(sp.Qdiag[None] * rng.uniform(0.5, 2.0, (M, 1))), t(np.broadcast_to(sp.Rdiag, (M, sp.nu)))
    rho = t(sp.rho * rng.uniform(0.5, 2.0, M))
    ms = {"cache": [], "sensitivity": []}
    for k in range(warmup + steps):
        a = timed(lambda: s.setup_models_device(A, Bm, f, Q, R, rho))
        b = timed(lambda: s.setup_sensitivity_device(A, Bm, f, Q, R, rho))
        if k >= warmup:
            ms["cache"].append(a)
            ms["sensitivity"].append(b)
    _, _, sweeps = s.setup_sensitivity_device(A, Bm, f, Q, R, rho, want_sweeps=True)
    s.close()
    # the timings include the wrapper's input transposes and output allocation, the same for both calls
    return dict(models=M, mean_sweeps=float(sweeps.float().mean().item()), singular=int((sweeps < 0).sum().item()),
                **{k + "_ms_median": float(np.median(v)) for k, v in ms.items()}, **{k + "_ms_min": float(np.min(v)) for k, v in ms.items()})


def adaptive(B, steps, warmup):
    sp = wl.quadrotor(N=50)
    prob = setup_problem(sp, np.float32)
    s = BatchedTinySolver(prob, sp.settings, device=0)
    inst = wl.tracking_instances(B, N=50, seed=0, dtype=np.float32)
    dK, dP = s.setup_sensitivity_device(sp.A[None], np.reshape(sp.B, (1, sp.nx, sp.nu)), sp.f[None], sp.Qdiag[None], sp.Rdiag[None], [sp.rho])
    ars = {"shared_tables": AdaptiveRho(dK[0].cpu().numpy(), dP[0].cpu().numpy()),
           "per_instance_tables": AdaptiveRho(dK.transpose(1, 2).repeat(B, 1, 1).transpose(1, 2), dP.transpose(1, 2).repeat(B, 1, 1).transpose(1, 2))}
    models = torch.as_tensor(pack_models(prob, B), device="cuda:0").contiguous()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")
    ms, iters, blobs = {k: [] for k in ars}, {}, {}
    for k in range(warmup + steps):
        for name, ar in ars.items():
            batch, res = s.make_device_batch(inst["x0"], inst["Xref"], cold_start=True, want_residuals=False)
            m = models.clone()
            flush.zero_()
            v = timed(lambda: s.solve_device_adaptive(batch, m, ar))
            if k >= warmup:
                ms[name].append(v)
            iters[name], blobs[name] = int(res["iter"].sum().item()) / B, m
    st = s.stats()
    s.close()
    return dict(batch=B, workload="quadrotor tracking N=50 fp32, to convergence, tables of this model from the device call",
                same_bits=bool(torch.equal(blobs["shared_tables"].view(torch.int32), blobs["per_instance_tables"].view(torch.int32))),
                instances_per_cta=st["instances_per_cta"], smem_bytes_per_cta=st["smem_bytes_per_cta"],
                **{k: dict(ms_median=float(np.median(v)), ms_min=float(np.min(v)), mean_iters=iters[k]) for k, v in ms.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--models", type=int, default=65536)
    ap.add_argument("--batch", type=int, default=65536)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sensitivity_bench.py measures on a GPU; none is available")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi.stdout.strip(),
           "precompute_fp32": precompute(np.float32, a.models, a.steps, a.warmup),
           "precompute_fp64": precompute(np.float64, a.models, a.steps, a.warmup),
           "adaptive_C3": adaptive(a.batch, a.steps, a.warmup)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
