"""CPU checks of per-instance cone coefficients (tinympc_batch_t.cones_per_instance): the ctypes mirror of the batch fields
matches the header, and the grouped helper the GPU tests compare against (instance_common.grouped_oracle) equals the
unmodified reference run once per instance, each with its own tiny_set_cone_constraints, bit for bit."""
import numpy as np
import pytest

import helpers as H
import instance_common as IC
from oracle import oracle
from tinympc_b200 import workloads as wl


def test_batch_cones_fields_match_header():
    IC.assert_batch_fields_match_header("cones")


OUT = H.OUT_KEYS + H.SOC_STATE


def _rocket(dt, N=20):
    spec = wl.rocket(N=N)
    prob = oracle.ref_setup(spec.nx, spec.nu, spec.N, spec.rho, spec.A, spec.B, spec.f, spec.Qdiag, spec.Rdiag, dtype=dt,
                            **spec.constraints)
    return spec, prob


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_cone_helper_equals_reference_per_instance(dt):
    """16 rockets with 16 distinct mu sets (wide ones whose cones hold the slack inside, or send it to the apex, and narrow
    ones that project it onto the surface; fp64 also 0.3 / 0.55, which float cannot represent): the helper (the C restatement
    once per mu set) against the compiled reference once per instance, cold, then warm from the cold result."""
    if not oracle.ref_available(dt):
        pytest.skip("the compiled reference (oracle/_ref, made by build() from the TinyMPC checkout) is not present")
    spec, prob = _rocket(dt)
    st = spec.settings
    st.max_iter = 40
    B = 16
    inst = wl.rocket_instances(B, N=spec.N, seed=5, dtype=dt, per_instance_refs=True)
    x0, Xref, Uref = inst["x0"], inst["Xref"], inst["Uref"]
    x0[::3, 2] = -np.abs(x0[::3, 2]) - 1.0  # below the landing plane: the state cone's apex branch
    extra = [(0.3, 0.55), (0.55, 0.3)] if dt == np.float64 else [(0.3, 0.55)]
    pal = IC.mu_palette(prob, 8, seed=2, scale=(0.2, 1.0)) + IC.mu_palette(prob, 8 - len(extra), seed=3, scale=(2.0, 12.0), extra=extra)
    which = (np.arange(B) * 5) % B
    cones = IC.batch_cones(pal, which)
    if dt == np.float64:
        assert np.any(cones["x_mu"] == 0.3) and np.float64(np.float32(0.3)) != 0.3
    helper = IC.grouped_oracle(prob, st, cones=cones, nthreads=4)

    def reference(x0_, state, cold):
        outs = []
        for b in range(B):
            p = IC.with_instance(prob, "cones", {k: a[b] for k, a in cones.items()})
            sub = None if state is None else {n: np.array(a[b:b + 1], copy=True) for n, a in state.items()}
            outs.append(oracle.solve_batch(p, st, x0_[b:b + 1], Xref[b:b + 1], Uref[b:b + 1], state=sub, cold_start=cold,
                                           want_state=tuple(H.SOC_STATE), impl="reference"))
        return {k: np.concatenate([o[k] for o in outs]) for k in OUT}

    h1 = helper(x0, Xref, Uref, None, True, H.SOC_STATE)
    r1 = reference(x0, None, True)
    H.assert_bits_per_instance(h1, r1, OUT, "cold")
    # the projections bite: instances land in each of project_soc's three branches, on the state or the input side
    bx = IC.soc_branches(h1["vcnew"], prob.Acx, cones["x_mu"])
    bu = IC.soc_branches(h1["zcnew"], prob.Acu, cones["u_mu"])
    counts = [int(np.sum(a | b)) for a, b in zip(bx, bu)]
    assert all(c >= 2 for c in counts), f"instances per branch (below, inside, projected): {counts}"
    # the coefficients matter: the same batch with the problem's own mu differs for most instances
    shared = IC.grouped_oracle(prob, st, cones={"x_mu": np.tile(prob.cx, (B, 1)), "u_mu": np.tile(prob.cu, (B, 1))}, nthreads=4)
    s1 = shared(x0, Xref, Uref, None, True, H.SOC_STATE)
    differ = [not np.array_equal(s1["sol_u"][b], h1["sol_u"][b]) for b in range(B)]
    assert sum(differ) >= B // 2, differ
    state = {n: h1[n] for n in H.SOC_STATE}
    x0w = np.ascontiguousarray(h1["x"][:, 1, :])
    h2 = helper(x0w, Xref, Uref, state, False, H.SOC_STATE)
    r2 = reference(x0w, state, False)
    H.assert_bits_per_instance(h2, r2, OUT, "warm")


def test_cone_helper_groups_by_distinct_mu(monkeypatch):
    """a batch dealt 3 mu sets is solved with 3 oracle runs, and a mu set equal to the problem's gives the shared result"""
    dt = np.float64
    spec = wl.rocket(N=10)
    prob = oracle.port_setup(spec.nx, spec.nu, spec.N, spec.rho, spec.A, spec.B, spec.f, spec.Qdiag, spec.Rdiag, dtype=dt,
                             **spec.constraints)
    st = spec.settings
    st.max_iter = 20
    B = 9
    inst = wl.rocket_instances(B, N=spec.N, seed=1, dtype=dt)
    pal = [dict(x_mu=prob.cx.copy(), u_mu=prob.cu.copy())] + IC.mu_palette(prob, 2, seed=9)
    which = np.arange(B) % 3
    IC.assert_one_run_per_set(monkeypatch, prob, st, inst["x0"], inst["Xref"], inst["Uref"], which, cones=IC.batch_cones(pal, which))
