"""CPU checks of the SLAM-landmark members of out-of-state plane updates (use_plane_constraint_slamu, UpdaterMSCKF.cpp:231-254, 454-560):
the oracle's row of a feature without measurements (get_feature_jacobian_full, UpdaterHelper.cpp:313-315), which the GPU tests take as the
member row, against central differences of its residual; and the adapter's wiring of the members."""
import os
import re

import numpy as np
import pytest

from ov_plane_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("do_fej", [0, 1])
def test_member_row_against_central_differences(do_fej):
    import oracle_backend
    S = synth.make_scenario("tiny_planes", seed=0)
    S.options["do_fej"] = do_fej
    orc = oracle_backend.OracleContext(S.options)
    synth.load_scenario_into(orc, S)
    rng = np.random.RandomState(4)
    sig_c = 0.01
    for _ in range(5):
        cp = rng.randn(3)
        cp *= (1.0 + rng.rand()) / np.linalg.norm(cp)
        p = rng.randn(3) * 2.0
        pf, cpf = (p + 1e-3 * rng.randn(3), cp + 1e-3 * rng.randn(3)) if do_fej else (p, cp)

        def row(p_, cp_):  # residual = -w (n^T p - d); with do_fej the Jacobians are taken at the first estimates
            return orc.feature_jacobian_full([], np.zeros((0, 2)), p_, pf if do_fej else p_, 7, cp_, cpf if do_fej else cp_, 1.0, sig_c)

        Hf, Hx, r, xo = row(p, cp)
        assert Hf.shape == (1, 6) and Hx.shape == (1, 0) and r.shape == (1,) and xo == []
        # the Jacobians are those of the measurement h = n^T p - d (res = -w h), at the linearisation point
        lp, lcp = (pf, cpf) if do_fej else (p, cp)
        h = lambda p_, cp_: -row(p_, cp_)[2][0]
        eps = 1e-6
        num_f = np.array([(h(lp + eps * e, lcp) - h(lp - eps * e, lcp)) / (2 * eps) for e in np.eye(3)])
        num_cp = np.array([(h(lp, lcp + eps * e) - h(lp, lcp - eps * e)) / (2 * eps) for e in np.eye(3)])
        assert np.allclose(Hf[0, :3], num_f, rtol=1e-7, atol=1e-6)
        assert np.allclose(Hf[0, 3:], num_cp, rtol=1e-7, atol=1e-6)
        d = np.linalg.norm(cp)
        assert np.isclose(r[0], -(cp / d @ p - d) / sig_c, rtol=1e-13)  # the residual is always at the current value
    orc.close()


def test_adapter_passes_the_members():
    """UpdaterMSCKF::update enters the plane stage on msckf || slamu (:199), takes the landmark positions from the device into the plane
    hypothesis and refinement, and calls the update with the members."""
    src = open(os.path.join(ROOT, "adapter", "UpdaterMSCKFB200.cpp")).read()
    assert re.search(r"use_plane_constraint\s*&&\s*\(state->_options\.use_plane_constraint_msckf\s*\|\|\s*state->_options\.use_plane_constraint_slamu\)", src)
    assert "ovp_var_get(state->ctx, ovp_slam_handle(" in src
    assert "ovp_msckf_update_landmarks(" in src and "ovp_msckf_update(" not in src
