"""CPU checks of per-instance box bounds (tinympc_batch_t.bounds_per_instance): the ctypes mirror of the new batch fields
matches the header, and the palette helper the GPU tests compare against (bounds_common.grouped_oracle) equals the unmodified
reference run once per instance, each with its own tiny_set_bound_constraints, bit for bit."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import bounds_common as BC
import helpers as H
from oracle import oracle
from tinympc_b200 import abi, workloads as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FIELDS = ["models", "x_min", "x_max", "u_min", "u_max", "bounds_per_instance", "reserved2"]


def test_batch_bounds_fields_match_header():
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"tinympc_b200.h\"\nint main(void){\n"
    src += '  printf("%zu\\n", sizeof(tinympc_batch_t));\n'
    src += "".join(f'  printf("%zu\\n", offsetof(tinympc_batch_t, {n}));\n' for n in FIELDS)
    src += "  return 0; }\n"
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "probe.c")
        open(c, "w").write(src)
        exe = os.path.join(td, "probe")
        subprocess.check_call(["/usr/bin/gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = list(map(int, subprocess.check_output([exe], text=True).split()))
    assert out[0] == C.sizeof(abi.Batch)
    assert out[1:] == [getattr(abi.Batch, n).offset for n in FIELDS]
    assert abi.Batch().bounds_per_instance == 0 and abi.Batch().reserved2 == 0  # a zero-initialised batch: the handle's bounds


OUT = H.OUT_KEYS + H.BOX_STATE


@pytest.mark.parametrize("layout", [1, 2])
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_palette_helper_equals_reference_per_instance(dt, layout):
    """12 instances with 12 distinct bound sets (tight ones that bite, and +-0 bounds where slacks land): the helper (the C
    restatement once per bound set) against the compiled reference once per instance, cold, then warm from the cold result."""
    if not oracle.ref_available(dt):
        pytest.skip("the compiled reference (oracle/_ref, made by build() from the TinyMPC checkout) is not present")
    spec = wl.quadrotor(N=20)
    prob = oracle.ref_setup(spec.nx, spec.nu, spec.N, spec.rho, spec.A, spec.B, spec.f, spec.Qdiag, spec.Rdiag, dtype=dt,
                            **spec.constraints)
    st = spec.settings
    st.max_iter = 40
    inst = wl.tracking_instances(12, N=spec.N, seed=11, dtype=dt)
    x0, Xref = inst["x0"], inst["Xref"]
    pal = BC.palette(prob, 6, layout, seed=3, scale=0.5, tight=0.9) + BC.palette(prob, 6, layout, seed=4, scale=0.3, zeros=True)
    which = BC.deal(12, 12, stride=5)
    helper = BC.grouped_oracle(prob, st, pal, which, nthreads=4)

    def reference(x0_, state, cold):
        outs = []
        for b in range(12):
            p = BC.with_bounds(prob, pal[which[b]])
            sub = None if state is None else {n: np.array(a[b:b + 1], copy=True) for n, a in state.items()}
            xr = Xref[b:b + 1] if Xref.ndim == 3 else Xref
            outs.append(oracle.solve_batch(p, st, x0_[b:b + 1], xr, None, state=sub, cold_start=cold,
                                           want_state=tuple(H.BOX_STATE), impl="reference"))
        return {k: np.concatenate([o[k] for o in outs]) for k in OUT}

    h1 = helper(x0, Xref, None, None, True, H.BOX_STATE)
    r1 = reference(x0, None, True)
    H.assert_bits_per_instance(h1, r1, OUT, f"cold, layout {layout}")
    # the bounds bite: most instances have an input slack on a bound of their own
    bite = [np.any((h1["znew"][b] == pal[which[b]]["u_max"]) | (h1["znew"][b] == pal[which[b]]["u_min"])) for b in range(12)]
    assert sum(bite) >= 6, bite
    state = {n: h1[n] for n in H.BOX_STATE}
    x0w = np.ascontiguousarray(h1["x"][:, 1, :])
    h2 = helper(x0w, Xref, None, state, False, H.BOX_STATE)
    r2 = reference(x0w, state, False)
    H.assert_bits_per_instance(h2, r2, OUT, f"warm, layout {layout}")
    zs = pal[6]["u_min"]
    assert np.signbit(zs).any() and (zs == 0).any()
