"""CPU checks of per-instance box bounds (tinympc_batch_t.bounds_per_instance): the ctypes mirror of the batch fields matches
the header, and the grouped helper the GPU tests compare against (instance_common.grouped_oracle) equals the unmodified
reference run once per instance, each with its own tiny_set_bound_constraints, bit for bit."""
import numpy as np
import pytest

import helpers as H
import instance_common as IC
from oracle import oracle
from tinympc_b200 import workloads as wl


def test_batch_bounds_fields_match_header():
    IC.assert_batch_fields_match_header("bounds")


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
    pal = IC.palette(prob, 6, layout, seed=3, scale=0.5, tight=0.9) + IC.palette(prob, 6, layout, seed=4, scale=0.3, zeros=True)
    which = IC.deal(12, 12, stride=5)
    helper = IC.grouped_oracle(prob, st, bounds=IC.batch_bounds(pal, which), nthreads=4)

    def reference(x0_, state, cold):
        outs = []
        for b in range(12):
            p = IC.with_instance(prob, "bounds", pal[which[b]])
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
