"""The C restatement (oracle/tinympc_oracle.c) against the unmodified reference compiled with the pinned flags: its
precompute, and a randomised sweep of warm-started closed loops over the compiled (nx, nu) pairs, bit for bit.  The
reference's outputs are stored under tests/golden (tests/golden/make_golden.py), so these checks run anywhere; the
parity cases themselves are replayed by tests/test_oracle_golden.py."""
import os

import numpy as np
import pytest

import helpers as H
from oracle import oracle


def _solve(impl):
    def fn(prob, settings, x0, Xref, Uref, state, cold, want):
        return oracle.solve_batch(prob, settings, x0, Xref, Uref, state=state, cold_start=cold, want_state=want, impl=impl)
    return fn


def test_precompute_port_close_to_reference():
    """The restated precompute vs the cache the reference's tiny_setup derived (stored with the golden cases)."""
    cases = H.make_cases()
    for name in ("cartpole_f64", "quad_hover_N10_f64", "rocket_soc_N10_f64", "lti_8_2_f64"):
        pr = H.load_golden(name)[0]
        pp = H.problem_from_spec(cases[name]["spec"], np.float64, oracle.port_setup)
        for f in ("Kinf", "Pinf", "Quu_inv", "AmBKt", "APf", "BPf", "Q", "R"):
            a, b = getattr(pr, f), getattr(pp, f)
            assert np.allclose(a, b, rtol=1e-9, atol=1e-9 * max(1.0, np.abs(a).max())), (name, f)


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_port_bit_identical_to_reference_random_lti_sweep(dt):
    """Randomised sweep over the compiled (nx, nu) pairs and short horizons (BASELINE config 5's generator): warm-started
    three-step loops with active box bounds, restatement vs the unmodified reference (its cache, measured states and the
    digest of every output array stored in tests/golden/reference), bit for bit."""
    tag = "f32" if dt == np.float32 else "f64"
    d = np.load(os.path.join(H.REFERENCE_DIR, f"lti_sweep_{tag}.npz"))
    for n, (nx, nu, N, sp, inst) in enumerate(H.lti_sweep_cases(dt)):
        prob = H.problem_from_spec(sp, dt, oracle.port_setup)
        for f in H.CACHE_FIELDS:
            setattr(prob, f, d[f"d{n}_{f}"])
        port, _ = H.closed_loop(prob, sp.settings, inst, 3, False, H.BOX_STATE, _solve("port"), x0_seq=d[f"d{n}_x0_seq"])
        for k, p in enumerate(port):
            for key, want in zip(H.OUT_KEYS + H.BOX_STATE, d[f"d{n}_digests"][k]):
                assert H.digest(p[key]) == str(want), f"({nx},{nu},{N}) step {k}: {key} differs"
