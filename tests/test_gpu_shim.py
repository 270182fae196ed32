"""Drop-in check of the reference-compatible C++ front end (tinympc_b200/shim): the reference's OWN example programs
(examples/*.cpp, compiled unmodified together with the shim by tinympc_b200/shim/Makefile into oracle/_ref/examples_shim;
at run time they load only libtinympc_b200.so) run on the GPU and must print the
same closed-loop results as the unmodified reference (CPU, pinned flags): every "tracking error" value, every iteration
count, every "Solver converged" line, and as many lines in all.  The reference's output is stored as line counts and a
digest of the result lines (tests/golden/reference/examples.json).  The example binaries are built where the TinyMPC
checkout (its examples and its Eigen headers) is available; without them the test skips."""
import json
import os
import subprocess

import pytest

import helpers as H

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM = os.path.join(ROOT, "oracle", "_ref", "examples_shim")
EXAMPLES = ["cartpole_example", "quadrotor_hovering", "quadrotor_tracking", "rocket_landing_mpc",
            "quadrotor_linear_constraints", "quadrotor_tv_linear_constraints"]


def _run(path):
    r = subprocess.run([path], capture_output=True, text=True, timeout=600, cwd=os.path.dirname(path))
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout.splitlines()


@pytest.mark.parametrize("name", EXAMPLES)
def test_reference_example_prints_identical_results_through_the_shim(name):
    if not os.path.exists(os.path.join(SHIM, name)):
        pytest.skip("example binaries not built (tinympc_b200/shim/Makefile needs a TinyMPC checkout: REF=<path>)")
    ref = json.load(open(os.path.join(H.REFERENCE_DIR, "examples.json")))[name]
    out = _run(os.path.join(SHIM, name))
    key = H.example_key_lines(out)
    assert ref["lines"] > 10
    assert len(out) == ref["stdout_lines"]
    assert len(key) == ref["lines"]
    assert H.text_digest(key) == ref["sha256"]
