"""The C++ shim's adaptive-rho guard (no GPU needed): with settings->adaptive_rho set and sensitivity tables that do not have
the solver's shape (tiny_initialize_sensitivity_matrices always fills the reference's 4 x 12 / 12 x 12 quadrotor tables),
tiny_solve prints the reason and returns 1 instead of solving.  The program is built with the shim by
tinympc_b200/shim/Makefile (tests/adaptive/shim_adaptive_loop.cpp)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROG = os.path.join(ROOT, "oracle", "_ref", "shim_tests", "adaptive_loop")


@pytest.mark.skipif(not os.path.exists(PROG), reason="shim test program not built (tinympc_b200/shim/Makefile needs Eigen headers)")
def test_shim_refuses_tables_of_another_shape():
    r = subprocess.run([PROG, "--bad-tables"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "settings->adaptive_rho needs cache->dKinf_drho (2 x 4)" in r.stdout
    assert "tiny_solve returned 1" in r.stdout
