#!/usr/bin/env python3
"""Extract the numeric problem/trajectory tables of the reference examples into .npz fixtures.

Needs a TinyMPC checkout, named by TINYMPC_REFERENCE:
    python tools/extract_problem_data.py
Reads   $TINYMPC_REFERENCE/examples/problem_data/*.hpp and examples/trajectory_data/*.hpp  (numbers only)
Writes  tinympc_b200/data/{quadrotor_20hz,quadrotor_50hz,rocket_20hz}.npz  and quadrotor_20hz_y_axis_line.npz

The .npz files hold INPUT DATA (A, B, f, Q, R, rho and a reference trajectory), i.e. the workload
definitions SURVEY.md §2 #9 marks "as fixtures"; no reference code is copied.  Literals with an `f` suffix
(rocket_landing_params_20hz.hpp:7-29) are rounded to float32 first and then widened, as the C++ compiler
does when it initialises a `double tinytype` array from them (SURVEY A.3-9).
"""
import os
import re
import sys

import numpy as np

REF = os.environ["TINYMPC_REFERENCE"]
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tinympc_b200", "data")


def parse_arrays(path):
    txt = open(path).read()
    txt = re.sub(r"//.*", "", txt)
    out = {}
    for m in re.finditer(r"tinytype\s+(\w+)\s*(?:\[[^\]]*\])?\s*=\s*\{([^}]*)\}\s*;", txt, re.S):
        name, body = m.group(1), m.group(2)
        vals = []
        for tok in body.replace("\n", " ").split(","):
            tok = tok.strip()
            if not tok:
                continue
            if tok.endswith("f"):
                vals.append(float(np.float32(float(tok[:-1]))))
            else:
                vals.append(float(tok))
        out[name] = np.array(vals, dtype=np.float64)
    m = re.search(r"tinytype\s+rho_value\s*=\s*([0-9.eE+-]+)f?\s*;", txt)
    if m:
        out["rho_value"] = float(m.group(1))
    return out


def model(path, nx, nu, has_f):
    a = parse_arrays(path)
    d = dict(
        A=a["Adyn_data"].reshape(nx, nx),  # headers are row-major (Map<..., RowMajor>, quadrotor_hovering.cpp:33)
        B=a["Bdyn_data"].reshape(nx, nu),
        f=a["fdyn_data"] if has_f else np.zeros(nx),
        Q=a["Q_data"],
        R=a["R_data"],
        rho=np.float64(a["rho_value"]),
    )
    return d


def main():
    if not os.path.isdir(REF):
        sys.exit(f"{REF} not present; the committed .npz files are the fixtures")
    os.makedirs(OUT, exist_ok=True)
    pd = os.path.join(REF, "examples", "problem_data")
    np.savez(os.path.join(OUT, "quadrotor_20hz.npz"), **model(os.path.join(pd, "quadrotor_20hz_params.hpp"), 12, 4, False))
    np.savez(os.path.join(OUT, "quadrotor_50hz.npz"), **model(os.path.join(pd, "quadrotor_50hz_params.hpp"), 12, 4, False))
    np.savez(os.path.join(OUT, "rocket_20hz.npz"), **model(os.path.join(pd, "rocket_landing_params_20hz.hpp"), 6, 3, True))
    tr = parse_arrays(os.path.join(REF, "examples", "trajectory_data", "quadrotor_20hz_y_axis_line.hpp"))
    X = tr["Xref_data"].reshape(-1, 12)  # time-major: Xref_data[k*12+i]  (quadrotor_tracking.cpp:65)
    np.savez(os.path.join(OUT, "quadrotor_20hz_y_axis_line.npz"), Xref=X)
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()
