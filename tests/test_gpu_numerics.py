"""Numerical hardening of the measurement compression (Cholesky of the stacked Gram matrix, DESIGN.md §4) and regression tests
for the plan / graph / handle-table lifetime issues found in round 1 (ADVICE.md)."""
import numpy as np
import pytest

from conftest import make_pair
from ov_plane_b200 import api, synth
from test_gpu_parity import relerr, compare_states, oracle_msckf_update, _check_msckf

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["cfg2_n256_f200", "small_planes"])
def test_rank_tolerance_sweep(name, chi2_table):
    """The zero-pivot rule separates gauge directions (pivot / original diagonal ~ 1e-16..1e-14 after cancellation) from the
    weakest observable direction (>= 1e-12 on every scenario): the posterior must not depend on where the threshold sits."""
    S = synth.make_scenario(name, seed=0)
    errs = []
    for tol in (1e-9, 1e-10, 1e-11, 1e-12, 1e-13):
        ctx, orc, chg, cho = make_pair(S, chi2_table)
        ctx.set_rank_tolerance(tol)
        g = ctx.msckf_update(synth.feature_batch(S, chg), 1.0, 1.0)
        o = oracle_msckf_update(orc, synth.feature_batch(S, cho), 1.0, 1.0)
        errs.append(_check_msckf(S, ctx, orc, chg, cho, g, o, chi_tol=1e-6))
        ctx.close()
    print(name, "cov rel err over tol 1e-9..1e-13:", ["%.1e" % e for e in errs])


@pytest.mark.parametrize("sigma_px,name,over", [(0.3, "cfg2_n256_f200", dict(calib_intr=1)), (0.1, "cfg1_euroc_n96", {}),
                                                (0.3, "small_planes", {})])
def test_compression_stress_scenarios(sigma_px, name, over, chi2_table):
    """Sharper pixel noise (larger whitened Jacobians, smaller posteriors => stronger cancellation in P - K M^T) and intrinsics
    calibration on: the Cholesky-QR path must still meet the north-star tolerance against the Givens oracle."""
    S = synth.make_scenario(name, seed=2, sigma_px=sigma_px, **over)
    ctx, orc, chg, cho = make_pair(S, chi2_table)
    g = ctx.msckf_update(synth.feature_batch(S, chg), sigma_px, 1.0)
    o = oracle_msckf_update(orc, synth.feature_batch(S, cho), sigma_px, 1.0)
    e = _check_msckf(S, ctx, orc, chg, cho, g, o, chi_tol=1e-6)
    print(name, "sigma_px", sigma_px, "cov rel err %.2e" % e, "accepted", int((g["feat_status"] == 1).sum()), "of", S.F)


@pytest.mark.parametrize("cond", [1e3, 1e5, 1e6])
def test_compress_ill_conditioned(cond, chi2_table):
    """measurement_compress_inplace on a stack with column scales spread over `cond`: the quantities the posterior depends on
    (R^T R, R^T z, |z|^2) agree with the Givens oracle to round-off; R itself loses cond * eps, as any Q-less QR does."""
    S = synth.make_scenario("tiny_points", seed=0)
    ctx, orc, chg, cho = make_pair(S, chi2_table)
    rng = np.random.RandomState(3)
    rows, cx = 400, 48
    Q1, _ = np.linalg.qr(rng.randn(rows, cx))
    Q2, _ = np.linalg.qr(rng.randn(cx, cx))
    Hx = (Q1 * np.logspace(0, -np.log10(cond), cx)) @ Q2.T * 100.0
    res = rng.randn(rows)
    gR, gz = ctx.measurement_compress_inplace(Hx, res)
    oR, oz = orc.measurement_compress_inplace(Hx, res)
    G = Hx.T @ Hx
    e_g = np.abs(gR.T @ gR - G).max() / np.abs(G).max()
    e_o = np.abs(oR.T @ oR - G).max() / np.abs(G).max()
    e_z = relerr(gR.T @ gz, Hx.T @ res)
    print("cond %.0e: |R^T R - H^T H| / |H^T H|  gpu %.1e  oracle %.1e;  R^T z rel err %.1e" % (cond, e_g, e_o, e_z))
    assert e_g < 1e-13 and e_z < 1e-11
    # |z|^2 (what a stacked chi2 sees of the residual): the component along a direction with relative singular value s carries a
    # relative error ~ eps / s^2 when R comes from the Gram matrix (Householder / Givens: eps / s) - bounded accordingly
    e_zz = abs(gz @ gz - oz @ oz) / (oz @ oz)
    print("          |z|^2 rel diff vs oracle %.1e (bound %.1e)" % (e_zz, max(1e-12, 10 * cond ** 2 * 2.3e-16)))
    assert e_zz < max(1e-12, 10 * cond ** 2 * 2.3e-16)


def test_graph_replay_sees_new_plane_estimates(chi2_table):
    """Same batch layout, different out-of-state plane estimates on every call: a replayed CUDA graph must linearise around the
    plane_cp of THIS call (ADVICE r1: by-value kernel arguments were baked into the captured graph)."""
    S = synth.make_scenario("small_planes", seed=0)
    planes = synth.drop_planes_from_state(S)
    ids = np.array([p[0] for p in planes], dtype=np.int64)
    cp0 = np.ascontiguousarray([p[1] for p in planes], dtype=np.float64)
    ctx = api.Context(S.options, device=0, max_state=S.N + 64, max_meas_rows=60000)
    ctx.set_chi2_table(chi2_table)
    chg = synth.load_scenario_into(ctx, S)
    ctx.snapshot()
    rng = np.random.RandomState(0)
    for it in range(5):  # call 1 eager, call 2 captures, calls 3.. replay
        cp = cp0 + (0.0 if it < 2 else 2e-3 * rng.randn(*cp0.shape))
        b = synth.feature_batch(S, chg)
        b["plane_ids"], b["plane_cp"] = ids, cp
        ctx.restore()
        g = ctx.msckf_update(b, 1.0, 1.0)
        P = ctx.cov()
        fresh = api.Context(S.options, device=0, max_state=S.N + 64, max_meas_rows=60000)
        fresh.set_chi2_table(chi2_table)
        chf = synth.load_scenario_into(fresh, S)
        bf = synth.feature_batch(S, chf)
        bf["plane_ids"], bf["plane_cp"] = ids, cp
        gf = fresh.msckf_update(bf, 1.0, 1.0)
        assert np.array_equal(g["plane_status"], gf["plane_status"]) and np.array_equal(g["feat_status"], gf["feat_status"])
        assert np.allclose(g["plane_chi2"], gf["plane_chi2"], rtol=1e-9, equal_nan=True), (it, g["plane_chi2"], gf["plane_chi2"])
        assert relerr(P, fresh.cov()) < 1e-10, it
        fresh.close()


def test_chi2_table_swap_invalidates_the_plan(chi2_table):
    S = synth.make_scenario("tiny_planes", seed=0)
    ctx, orc, chg, cho = make_pair(S, chi2_table)
    ctx.snapshot()
    for _ in range(3):
        ctx.restore()
        g0 = ctx.msckf_update(synth.feature_batch(S, chg), 1.0, 1.0)
    assert (g0["feat_status"] == 1).any()
    ctx.set_chi2_table(chi2_table * 1e-3)  # every gate must now fail, through the same (formerly captured) plan
    ctx.restore()
    g1 = ctx.msckf_update(synth.feature_batch(S, chg), 1.0, 1.0)
    assert not (g1["feat_status"] == 1).any() and not (g1["plane_status"] == 1).any()
    ctx.set_chi2_table(chi2_table)
    ctx.restore()
    g2 = ctx.msckf_update(synth.feature_batch(S, chg), 1.0, 1.0)
    assert np.array_equal(g2["feat_status"], g0["feat_status"]) and np.array_equal(g2["plane_status"], g0["plane_status"])


def test_snapshot_survives_stage_growth_and_use_graphs_setting(chi2_table):
    """ADVICE r1: growing the host staging buffer used to free the snapshot buffers, the profiling events and the prepared batch."""
    S = synth.make_scenario("cfg3_n512_f600_p8", seed=0)
    ctx = api.Context(S.options, device=0, max_state=576, max_meas_rows=40000)
    ctx.set_chi2_table(chi2_table)
    chg = synth.load_scenario_into(ctx, S)
    ctx.set_use_graphs(False)
    ctx.get_marginal_covariance([ctx.handle_calib()])  # first (small) staging allocation
    ctx.snapshot()
    P0 = ctx.cov()
    M = ctx.get_marginal_covariance(chg)  # 456 x 456 doubles: the staging buffer grows AFTER the snapshot
    assert M.shape == (6 * len(chg), 6 * len(chg))
    rng = np.random.RandomState(1)
    hg = [ctx.handle_calib(), ctx.handle_intrinsics()] + chg[:6]
    H, res = rng.randn(40, 14 + 36) * 30, rng.randn(40)
    ctx.ekf_update(hg, H, res)
    assert relerr(ctx.cov(), P0) > 1e-6
    ctx.restore()
    assert np.array_equal(ctx.cov(), P0)
    ctx.snapshot()
    ctx.restore()
    assert np.array_equal(ctx.cov(), P0)
    # ... and a batch prepared before the growth is still launchable
    ctx.set_use_graphs(True)
    ctx.msckf_prepare(synth.feature_batch(S, chg), 1.0, 1.0)
    ctx.get_marginal_covariance(chg + [ctx.handle_calib()])
    ctx.msckf_launch()
    r = ctx.msckf_finish()
    assert (r["feat_status"] >= 0).all()


def test_handle_table_stays_bounded_over_a_long_run(chi2_table):
    """300 frames of augment_clone + marginalize(oldest): handles are recycled (the table must not grow by one slot per frame)
    and the covariance keeps matching the oracle."""
    S = synth.make_scenario("tiny_points", seed=1)
    ctx, orc, chg, cho = make_pair(S, chi2_table)
    t = S.timestamp
    w = np.array([0.01, -0.02, 0.03])
    seen = set(chg)
    for k in range(300):
        t += 0.05
        hg, ho = ctx.augment_clone(t, w), orc.augment_clone(t, w)
        seen.add(hg)
        chg.append(hg)
        cho.append(ho)
        ctx.marginalize(chg.pop(0))
        orc.marginalize(cho.pop(0))
    assert ctx.cov_rows() == orc.cov_rows()
    assert max(seen) < len(chg) + 80 + 8, "handle table grew to %d slots for %d live clones" % (max(seen) + 1, len(chg))
    compare_states(ctx, orc, S, chg, cho, 1e-9)


@pytest.mark.parametrize("name", ["cfg1_euroc_n96", "small_planes", "cfg3_n512_f600_p8"])
def test_block_sparse_gram_equals_dense_stacked_path(name, chi2_table):
    """The warp-per-feature path (G = D - Y^T Y, never materialising the stacked Jacobian, msckf_warp.inc) against the dense stacked
    path (feature_kernel + SYRK over all projected rows; the ovp_debug_force_dense_features hook of libovp_debug.so): same gates, chi2
    and posterior."""
    S = synth.make_scenario(name, seed=0)
    out = {}
    for dense in (0, 1):
        ctx = api.Context(S.options, device=0, max_state=max(128, S.N + 64), max_meas_rows=60000, debug=True)
        ctx._ck(ctx.lib.ovp_debug_force_dense_features(ctx.h, dense))
        ctx.set_chi2_table(chi2_table)
        ch = synth.load_scenario_into(ctx, S)
        r = ctx.msckf_update(synth.feature_batch(S, ch), 1.0, 1.0)
        out[dense] = (r, ctx.cov(), ctx.launch_count())
        ctx.close()
    (r0, P0, l0), (r1, P1, l1) = out[0], out[1]
    assert np.array_equal(r0["feat_status"], r1["feat_status"]) and np.array_equal(r0["plane_status"], r1["plane_status"])
    m = (r0["feat_status"] == 0) | (r0["feat_status"] == 1)
    e_chi = np.abs(r0["feat_chi2"][m] / r1["feat_chi2"][m] - 1).max() if m.any() else 0.0
    e = relerr(P0, P1)
    print(name, "block-sparse vs dense: cov rel diff %.2e, per-feature chi2 max rel diff %.2e, launches %d vs %d" % (e, e_chi, l0, l1))
    assert e < 1e-7 and e_chi < 1e-6
