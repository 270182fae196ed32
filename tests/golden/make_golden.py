#!/usr/bin/env python3
"""Generate the golden fixtures from the UNMODIFIED reference (needs the compiled reference under oracle/_ref,
see oracle/Makefile: make -C oracle REF=<TinyMPC checkout>, and for the example outputs the binaries the shim Makefile
builds from the same checkout).

    python tests/golden/make_golden.py

For each parity case (tests/helpers.py:make_cases) this runs the reference — compiled with the pinned flags
into oracle/_ref/libtinympc_ref_{f64,f32}.so by oracle/Makefile — through a warm-started closed loop and stores,
per case, one compressed .npz with
  * the complete problem (model, the cache the reference's tiny_setup computed, bounds, cones, hyperplanes),
  * the settings, the inputs of every step (x0 sequence, Xref, Uref),
  * the reference's outputs of every step (solution, iter, solved, residuals, and every state array).
The fixtures pin the oracle restatement (tests/test_oracle_golden.py, runs anywhere) and the CUDA path
(tests/test_gpu_parity.py) to the reference bit-for-bit without the reference being present.

tests/golden/reference/ holds what the other reference comparisons check against:
  * lti_sweep_{f32,f64}.npz   the randomised (nx, nu) sweep of tests/test_oracle_vs_reference.py (the cache tiny_setup
                              derives, x0 sequence and the SHA-256 digest of every output array of every step),
  * precompute_{f32,f64}.npz  the cache tiny_setup derives for the models of the device-precompute test,
  * sensitivity_tables.npz    tiny_initialize_sensitivity_matrices' tables,
  * examples.json             per example program of the reference: how many lines its stdout has, how many of them are
                              result lines (helpers.example_key_lines) and the SHA-256 digest of those.
"""
import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import helpers as H  # noqa: E402
from oracle import oracle  # noqa: E402
from tinympc_b200 import abi  # noqa: E402

PROBLEM_FIELDS = ["A", "B", "f", "Q", "R", "Kinf", "Pinf", "Quu_inv", "AmBKt", "APf", "BPf", "x_min", "x_max", "u_min",
                  "u_max", "Acx", "qcx", "cx", "Acu", "qcu", "cu", "Alin_x", "blin_x", "Alin_u", "blin_u", "tv_Alin_x",
                  "tv_blin_x", "tv_Alin_u", "tv_blin_u"]


def save_problem(out, prefix, prob):
    for f in PROBLEM_FIELDS:
        v = getattr(prob, f)
        if v is not None:
            out[prefix + "prob_" + f] = v


def ref_fn(prob, settings, x0, Xref, Uref, state, cold, want):
    return oracle.solve_batch(prob, settings, x0, Xref, Uref, state=state, cold_start=cold, want_state=want, impl="reference")


def make_reference_checks():
    os.makedirs(H.REFERENCE_DIR, exist_ok=True)
    for dt in (np.float32, np.float64):
        tag = "f32" if dt == np.float32 else "f64"
        out = {}
        for n, (nx, nu, N, spec, inst) in enumerate(H.lti_sweep_cases(dt)):
            prob = H.problem_from_spec(spec, dt, oracle.ref_setup)
            res, x0s = H.closed_loop(prob, spec.settings, inst, 3, False, H.BOX_STATE, ref_fn)
            for f in H.CACHE_FIELDS:
                out[f"d{n}_{f}"] = getattr(prob, f)
            out[f"d{n}_x0_seq"] = np.stack(x0s)
            out[f"d{n}_digests"] = np.array([[H.digest(r[key]) for key in H.OUT_KEYS + H.BOX_STATE] for r in res])
        path = os.path.join(H.REFERENCE_DIR, f"lti_sweep_{tag}.npz")
        np.savez_compressed(path, **out)
        print(f"{path}: {os.path.getsize(path)} bytes")
        out = {}
        for n, (nx, nu, spec) in enumerate(H.precompute_models()):
            prob = H.problem_from_spec(spec, dt, oracle.ref_setup)
            for f in H.CACHE_FIELDS:
                out[f"m{n}_{f}"] = getattr(prob, f)
        path = os.path.join(H.REFERENCE_DIR, f"precompute_{tag}.npz")
        np.savez_compressed(path, **out)
        print(f"{path}: {os.path.getsize(path)} bytes")
    import ctypes as C
    shapes = [(4, 12), (12, 12), (4, 4), (12, 12)]
    ref = [np.zeros(s, np.float64, order="F") for s in shapes]
    assert oracle.ref_lib(np.float64).tinympc_ref_sensitivity_tables(*[C.c_void_p(a.ctypes.data) for a in ref]) == 0
    np.savez_compressed(os.path.join(H.REFERENCE_DIR, "sensitivity_tables.npz"), **{f"t{i}": a for i, a in enumerate(ref)})
    make_example_digests()


def make_example_digests():
    exdir = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "examples_ref")
    ex = {}
    for name in sorted(os.listdir(exdir)):
        r = subprocess.run([os.path.join(exdir, name)], capture_output=True, text=True, timeout=600, cwd=exdir, check=True)
        key = H.example_key_lines(r.stdout.splitlines())
        ex[name] = {"lines": len(key), "sha256": H.text_digest(key), "stdout_lines": len(r.stdout.splitlines())}
    with open(os.path.join(H.REFERENCE_DIR, "examples.json"), "w") as fh:
        json.dump(ex, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print(ex)


def main():
    make_reference_checks()
    cases = H.make_cases()
    for name in sorted(cases):
        c = cases[name]
        prob = H.problem_from_spec(c["spec"], c["dtype"], oracle.ref_setup)
        st = c["spec"].settings

        def fn(prob, settings, x0, Xref, Uref, state, cold, want):
            return oracle.solve_batch(prob, settings, x0, Xref, Uref, state=state, cold_start=cold, want_state=want,
                                      impl="reference")

        res, x0s = H.closed_loop(prob, st, c["inst"], c["steps"], c["reset_duals"], c["state"], fn)
        out = dict(nx=prob.nx, nu=prob.nu, N=prob.N, rho=prob.rho, dtype=np.dtype(prob.dtype).name, steps=c["steps"],
                   reset_duals=int(c["reset_duals"]), state_names=np.array(c["state"]))
        save_problem(out, "", prob)
        for n, _ in abi.Settings._fields_:
            out["set_" + n] = getattr(st, n)
        out["Xref"] = np.asarray(c["inst"]["Xref"], dtype=prob.dtype)
        if c["inst"].get("Uref") is not None:
            out["Uref"] = np.asarray(c["inst"]["Uref"], dtype=prob.dtype)
        out["x0_seq"] = np.stack(x0s)
        for k, r in enumerate(res):
            for key in H.OUT_KEYS + c["state"]:
                out[f"step{k}_{key}"] = r[key]
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **out)
        print(f"{name}: {os.path.getsize(path)} bytes, iters step0 {res[0]['iter'].tolist()}")


if __name__ == "__main__":
    main()
