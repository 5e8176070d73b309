"""FeatureInitializer::single_triangulation + single_gaussnewton on the device (ovp_triangulate_features) against the oracle's
independent restatement of the same published algorithm (ov_core is not part of the reference tree: parity unpinned), and against
the simulated truth."""
import numpy as np
import pytest

from conftest import make_pair
from ov_plane_b200 import synth, vio_sim

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["cfg1_euroc_n96", "cfg2_n256_f200", "cfg3_n512_f600_p8"])
def test_triangulation_matches_the_oracle(name, chi2_table):
    S = synth.make_scenario(name, seed=1)
    ctx, orc, chg, cho = make_pair(S, chi2_table)
    cam = S.intr_value
    uvn = np.array([vio_sim.undistort(cam, uv.astype(np.float64)) for uv in S.uv], dtype=np.float32)  # Feature::uvs_norm
    # one degenerate track: identical bearings (no parallax).  A point behind the cameras, a far point and every other rejection rule,
    # on both sides of its threshold, are in tests/test_gpu_triangulation_reference.py
    uvn = uvn.copy()
    a, b = S.meas_offset[0], S.meas_offset[1]
    uvn[a:b] = uvn[a]
    pg, sg = ctx.triangulate_features(S.meas_offset, np.asarray(chg, dtype=np.int32)[S.meas_clone_idx], uvn)
    po, so = orc.triangulate_features(S.meas_offset, np.asarray(cho, dtype=np.int32)[S.meas_clone_idx], uvn)
    assert np.array_equal(sg, so), np.nonzero(sg != so)
    ok = so == 1
    d = np.abs(pg[ok] - po[ok]).max()
    err_truth = np.linalg.norm(pg[ok] - S.pf_true[ok], axis=1)
    print(name, "triangulated %d of %d, max |gpu - oracle| %.2e m, median / max distance to the simulated truth %.3f / %.3f m" % (
        ok.sum(), S.F, d, np.median(err_truth), err_truth.max()))
    assert ok.sum() > 0.8 * S.F and sg[0] == 0
    assert d < 5e-5          # both run LM on SINGLE-precision residuals (ov_core: uvs_norm and the predicted z are floats): one float ulp of the
                             # reprojection (6e-8) moves a point at 3-5 m depth seen over a 0.4 m baseline by ~1e-6 .. 1e-5 m
    assert np.median(err_truth) < 0.5
