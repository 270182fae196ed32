"""Adaptive rho on the CPU: the C restatement (tests/adaptive/adaptive_oracle.c) against the unmodified reference's adaptive
loop (tests/adaptive/ref_adaptive_driver.cpp, whose outputs tests/golden/adaptive/*.npz store), bit for bit, on every output,
state array and adapted model blob of every step of warm-started closed loops.  The cases cover fp32 and fp64, all three
column-block regimes of Eigen's GEMV (one block, 16-column and 4-column blocks), clipping on / off / binding, max_iter 6 and
11 (adaptation on the last iteration) and instances that converge on an adaptation iteration."""
import os

import numpy as np
import pytest

import adaptive_common as AC
from tinympc_b200.solver import AdaptiveRho

CASES = AC.make_cases()


def load_case(name):
    c = dict(CASES[name])
    d = np.load(os.path.join(AC.GOLDEN, f"adaptive_{name}.npz"))
    st = c["st"]
    for n, _ in type(st)._fields_:
        assert getattr(st, n) == d["set_" + n], (name, n)
    c["models"] = d["models"]
    c["ar"] = AdaptiveRho(d["dKinf"], d["dPinf"], float(d["rho_min"]), float(d["rho_max"]), bool(d["clip"]))
    return c, d


def port_solve(ar):
    def fn(prob, st, x0, Xref, Uref, state, cold, models):
        return AC.oracle_solve(prob, st, x0, Xref, Uref, state, cold, models, ar)
    return fn


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_matches_reference_adaptive_loop(name):
    c, d = load_case(name)
    outs, _ = AC.closed_loop(c["prob"], c["st"], c, port_solve(c["ar"]), x0_seq=d["x0_seq"])
    keys = AC.OUT + AC.BOX + ["models"]
    for k, (r, m) in enumerate(outs):
        for key, got, want in zip(keys, AC.digests(r, m), d["digests"][k]):
            assert got == str(want), f"{name} step {k}: {key} differs from the reference"


def test_fixture_coverage():
    """The fixtures exercise what they are meant to: adapted rho moves, the clip binds, adaptation happens on the last
    iteration, and some instances converge exactly on an adaptation iteration."""
    moved = binds = conv_on_adapt = 0
    for name in CASES:
        d = np.load(os.path.join(AC.GOLDEN, f"adaptive_{name}.npz"))
        rho = d["rho"]
        moved += int(np.any(rho != d["models"][:, -1]))
        if "clipbind" in name:
            assert np.all(rho == rho.dtype.type(float(d["rho_min"])))
            binds += 1
        if "maxit" in name:
            assert np.any(d["iters"] == int(d["set_max_iter"]))
        conv_on_adapt += int(np.sum(d["solved"].astype(bool) & (d["iters"] > 1) & ((d["iters"] - 1) % 5 == 0)))
    assert moved >= 10 and binds == 2 and conv_on_adapt >= 4, (moved, binds, conv_on_adapt)
