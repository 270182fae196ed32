#!/usr/bin/env python3
"""Generate the adaptive-rho fixtures tests/golden/adaptive/adaptive_<case>.npz from the UNMODIFIED reference.

    python tests/golden/make_golden_adaptive.py            (TINYMPC_REFERENCE: the TinyMPC checkout, default /root/reference)

tests/adaptive/ref_adaptive_driver.cpp is compiled with the reference's own sources and the pinned parity flags
(-O3 -DNDEBUG -DEIGEN_DONT_VECTORIZE -ffp-contract=off, as oracle/Makefile builds the reference) into a temporary directory;
the fp32 build compiles a scratch copy of the sources with `typedef float tinytype`.  For every case of
tests/adaptive_common.make_cases it runs the warm-started closed loop and stores the inputs (x0 of every step, the starting
model blobs, tables and settings) and the SHA-256 digest of every output, state array and adapted model blob of every step.
The other fixtures are not touched.
"""
import ctypes as C
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import adaptive_common as AC  # noqa: E402
from tinympc_b200 import abi  # noqa: E402

REF = os.environ.get("TINYMPC_REFERENCE", "/root/reference")
PIN = ["-O3", "-DNDEBUG", "-DEIGEN_DONT_VECTORIZE", "-ffp-contract=off"]


def build_ref(td, dt):
    src = os.path.join(REF, "src", "tinympc")
    if dt == np.float32:
        scratch = os.path.join(td, "f32src")
        os.makedirs(scratch)
        for n in ("admm.cpp", "admm.hpp", "tiny_api.cpp", "tiny_api.hpp", "tiny_api_constants.hpp", "rho_benchmark.cpp",
                  "rho_benchmark.hpp"):
            shutil.copy(os.path.join(src, n), scratch)
        t = open(os.path.join(src, "types.hpp")).read()
        assert "typedef double tinytype;" in t
        open(os.path.join(scratch, "types.hpp"), "w").write(t.replace("typedef double tinytype;", "typedef float tinytype;"))
        src = scratch
    so = os.path.join(td, f"libref_adaptive_{np.dtype(dt).name}.so")
    subprocess.check_call(["g++", "-std=c++17", "-shared", "-fPIC", "-w", *PIN, "-I", os.path.join(AC.ROOT, "include"), "-I", src,
                           "-I", os.path.join(REF, "include", "Eigen"), "-o", so, os.path.join(AC.ADIR, "ref_adaptive_driver.cpp"),
                           os.path.join(src, "admm.cpp"), os.path.join(src, "tiny_api.cpp"), os.path.join(src, "rho_benchmark.cpp")])
    lib = C.CDLL(so)
    lib.tinympc_ref_solve_adaptive.restype = C.c_int
    return lib


def main():
    with tempfile.TemporaryDirectory() as td:
        libs = {dt: build_ref(td, dt) for dt in (np.float32, np.float64)}
        for name, c in sorted(AC.make_cases().items()):
            prob, st, ar = c["prob"], c["st"], c["ar"]
            lib = libs[prob.dtype]

            def solve(prob, st, x0, Xref, Uref, state, cold, models):
                return AC.oracle_solve(prob, st, x0, Xref, Uref, state, cold, models, ar, lib=lib, fn="tinympc_ref_solve_adaptive")

            outs, x0s = AC.closed_loop(prob, st, c, solve)
            d = dict(x0_seq=np.stack(x0s), models=c["models"], dKinf=np.asarray(ar.dKinf_drho), dPinf=np.asarray(ar.dPinf_drho),
                     rho_min=ar.rho_min, rho_max=ar.rho_max, clip=int(ar.enable_clipping),
                     digests=np.array([AC.digests(r, m) for r, m in outs]),
                     iters=np.stack([r["iter"] for r, _ in outs]), solved=np.stack([r["solved"] for r, _ in outs]),
                     rho=np.stack([m[:, -1] for _, m in outs]))
            for n, _ in abi.Settings._fields_:
                d["set_" + n] = getattr(st, n)
            path = os.path.join(AC.GOLDEN, f"adaptive_{name}.npz")
            np.savez_compressed(path, **d)
            print(f"{path}: {os.path.getsize(path)} bytes; iters step0 {outs[0][0]['iter'].tolist()[:8]} "
                  f"rho {outs[-1][1][:3, -1].tolist()}")


if __name__ == "__main__":
    main()
