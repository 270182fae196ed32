"""FAST-mode accuracy report (needs a GPU): for each case of tests/test_gpu_fast.py, the worst ratio of FAST's error against
the fp64 restatement to what the FAST rule allows (tests/fast_common.py: <= 1 passes; fp32: C32 x the pinned fp32 oracle's
error + a few ulps, fp64: 1e-10 relative), per kernel family and solve (cold / warm / warm at max_iter = 1), and, run to
convergence, how many instances' iteration counts differ from the pinned oracle.

    python tools/fast_accuracy_report.py [--quick]

Prints a table; writes nothing.  A case outside the rule prints FAIL with the message instead of a ratio.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

import fast_common as F  # noqa: E402
import helpers as H  # noqa: E402
import test_gpu_fast as G  # noqa: E402
from tinympc_b200 import workloads as wl  # noqa: E402
from tinympc_b200.solver import setup_problem  # noqa: E402


def _row(name, fn):
    try:
        res = fn()
    except AssertionError as e:
        print(f"{name:34s} FAIL {str(e)[:160]}")
        return
    per_kernel = {}
    for (kernel, label), r in res.items():
        k, w = max(r.items(), key=lambda kv: kv[1])
        if w >= per_kernel.get(kernel, (0.0,))[0]:
            per_kernel[kernel] = (w, f"{label}: {k}")
    print(f"{name:34s} " + "  ".join(f"{k}={w:.3f} ({where})" for k, (w, where) in per_kernel.items()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="three shapes instead of every compiled one")
    a = ap.parse_args()
    import torch

    p = torch.cuda.get_device_properties(0)
    print(f"device: {p.name}")
    print(f"rule: fp32 C32={F.C32} ULPS32={F.ULPS32}; fp64 {F.REL64} relative; {F.FIXED_ITERS} iterations, tolerances 0")
    print("worst FAST error / allowed, per kernel family (case, dtype)")
    dims = [(6, 3), (12, 4), (16, 8)] if a.quick else G.ALL_DIMS
    for tag, dt in G.DT.items():
        for nx, nu in dims:
            def box(nx=nx, nu=nu, dt=dt):
                spec, inst, want = F.lti_case(nx, nu, 50, G.B_RAGGED, dt)
                return G._fixed_work_case(setup_problem(spec, dt), spec.settings, inst, want, ["tpi", "gpi", "gps"], "box")
            _row(f"box ({nx},{nu}) {tag}", box)

        def track(dt=dt):
            spec = wl.quadrotor(N=50)
            return G._fixed_work_case(setup_problem(spec, dt), spec.settings, F.tracking(77, 50, dt, seed=3), H.BOX_STATE,
                                      ["tpi", "gpi", "gps"], "track")
        _row(f"quad tracking {tag}", track)
        for case in F.FAMILY_CASES:
            def fam(case=case, dt=dt):
                spec, inst, want = F.family_case(case, 53, dt)
                return G._fixed_work_case(setup_problem(spec, dt), spec.settings, inst, want, ["tpi", "gps"], case)
            _row(f"{case} {tag}", fam)
        for mask in (0, 1, 6, 7):
            def het(mask=mask, dt=dt):
                sp, blobs, probs, model, inst, want, kernel = G._gps_het_case(mask, dt)
                return G._fixed_work_case(probs, sp.settings, inst, want, [kernel], "het", model=model, models=blobs[model])
            _row(f"gps per-instance mask {mask} {tag}", het)
    print("\nto convergence (default tolerances, B = 301): instances whose iter differs from the pinned oracle")
    for case, (tag, kernels) in G.CONVERGED.items():
        dt = G.DT[tag]
        if case.startswith("box"):
            spec, inst = wl.quadrotor(N=50), wl.tracking_instances(301, N=50, seed=5, dtype=dt)
        else:
            spec, inst, _ = F.family_case(case.rsplit("_", 1)[0], 301, dt)
        prob = setup_problem(spec, dt)
        pin, o64 = F.oracle_pair(prob, spec.settings)(inst["x0"], inst["Xref"], inst.get("Uref"), None, True, ())
        for kernel in kernels:
            solver = G._solver(prob, spec.settings, kernel)
            g, _ = G._device(solver, spec.settings, inst["x0"], inst, None, True, (), None)
            shifted = g["iter"] != pin["iter"]
            print(f"{case:14s} [{kernel}] {int(shifted.sum()):4d} / {len(shifted)}  shifts "
                  f"{sorted(set((g['iter'][shifted] - pin['iter'][shifted]).tolist()))}  mean iter fast {g['iter'].mean():.2f} "
                  f"pinned {pin['iter'].mean():.2f}")
            solver.close()


if __name__ == "__main__":
    np.set_printoptions(linewidth=200)
    main()
