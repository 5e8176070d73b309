"""The triangulation modes of ovp_set_triangulation_mode (FeatureInitializerOptions::triangulate_1d / refine_features) against the
long-double reference (tests/triangulation_1d_reference.py): ovp_triangulate_features in all four modes on a threshold pair on either side
of every rule of each mode, collinear rays, clones observed twice, degenerate tracks, track lengths 2 .. 100 and batches of 1, 63, 64, 65
and 2000 features, under the defaults and a non-default option set; {0, 1} against a context that never set a mode, bit for bit; the
setter's refusals and clearing; and ovp_plane_init_tracks and ovp_slam_delayed_init_tracks in the 1-D modes."""
import numpy as np
import pytest

import feature_jacobian_reference as fjr
import triangulation_1d_reference as t1
import triangulation_reference as tr
from conftest import make_pair
from test_cpu_slam_init_tracks import plane_gate
from ov_plane_b200 import api, synth
from ov_plane_b200 import slam_init_chain as sic

pytestmark = pytest.mark.gpu

MODES = sorted(t1.MODES)


@pytest.fixture(scope="module")
def setup():
    tr.require_long_double()
    S = tr.scenario()
    ctx = api.Context(S.options, device=0, max_state=S.N + 64, max_meas_rows=4096)
    ch = synth.load_scenario_into(ctx, S)
    base = tr.Context(ctx, ch, S.intr_value[0])
    ctxs = {mode: t1.ModeContext(base, mode) for mode in MODES}
    pool = tr.random_cases(base, 2000, 11)
    pairs = {(mode, o): t1.threshold_pairs(ctxs[mode], tr.OPTION_SETS[o]) for mode in MODES for o in tr.OPTION_SETS}
    yield ctx, base, ctxs, pool, pairs
    ctx.close()


def _run(ctx, mode, cases, opt):
    ctx.set_triangulation_mode(*t1.MODES[mode])
    try:
        return ctx.triangulate_features(*tr.flatten(cases), options=opt)
    finally:
        ctx.set_triangulation_mode(None)


def _check(ref, cases, opt, st, pf, label):
    """statuses equal on every decided feature, positions within the reference's bound, zero positions where it fails; returns
    (undecided, worst |dp| / bound)"""
    undecided, worst = 0, 0.0
    for i, c in enumerate(cases):
        if st[i] == 0:
            assert not pf[i].any(), (label, i, c["name"])
        res = ref.run(c, opt)
        if not res["decided"]:
            undecided += 1
            continue
        assert st[i] == res["status"], (label, i, c["name"], res["reason"], st[i])
        if res["status"] == 1:
            q = float(np.abs(pf[i] - np.asarray(res["p_FinG"], np.float64)).max()) / res["p_bound"]
            assert q <= 1.0, (label, i, c["name"], q)
            worst = max(worst, q)
    return undecided, worst


@pytest.mark.parametrize("opt_name", sorted(tr.OPTION_SETS))
@pytest.mark.parametrize("mode", MODES)
def test_modes_match_the_reference(setup, mode, opt_name):
    ctx, base, ctxs, pool, pairs = setup
    opt, ref = tr.OPTION_SETS[opt_name], ctxs[mode]
    planted = pairs[(mode, opt_name)] + t1.collinear_cases(base) + t1.clone_twice_cases(base) + tr.degenerate_cases(base)
    assert all(ref.run(c, opt)["decided"] for c in pairs[(mode, opt_name)])
    pf, st = _run(ctx, mode, planted, opt)
    und, worst = _check(ref, planted, opt, st, pf, "%s %s" % (mode, opt_name))
    rules = sorted({(c["rule"], c["side"], int(st[i])) for i, c in enumerate(planted) if "rule" in c})
    print("\n%s %s: rules (rule, side, gpu status) %s; planted %d, undecided %d, worst |dp| / bound %.2e" % (mode, opt_name, rules, len(planted),
                                                                                                          und, worst))
    assert und == 0
    for F in (1, 63, 64, 65, len(pool)):
        pf, st = _run(ctx, mode, pool[:F], opt)
        und, worst = _check(ref, pool[:F], opt, st, pf, "%s %s F=%d" % (mode, opt_name, F))
        print("%s %s: F = %d, %d triangulated, %d undecided, worst |dp| / bound %.2e" % (mode, opt_name, F, int(st.sum()), und, worst))
        assert und <= 0.3 * F + 1
    assert {len(c["track"]) for c in pool} >= {2, 3, 16, 32, 33, 64, 100}


def test_baseline_only_rejection_passes_unrefined(setup):
    """the outside case of the refined baseline pair, which only the baseline rule rejects, is triangulated unrefined"""
    ctx, base, ctxs, _, pairs = setup
    for opt_name, opt in tr.OPTION_SETS.items():
        out = [c for c in pairs[("3d_refine", opt_name)] if c["rule"] == "baseline" and c["side"] == "out"]
        assert out and base.run(out[0], opt)["reason"] == "baseline"
        _, st = _run(ctx, "3d_refine", out, opt)
        assert st[0] == 0
        pf, st = _run(ctx, "3d_linear", out, opt)
        res = ctxs["3d_linear"].run(out[0], opt)
        assert res["decided"] and res["status"] == 1 and st[0] == 1
        assert float(np.abs(pf[0] - np.asarray(res["p_FinG"], np.float64)).max()) <= res["p_bound"]


def test_default_mode_is_bit_identical_to_no_mode(setup):
    ctx, base, ctxs, pool, pairs = setup
    cases = pool[:300] + pairs[("3d_refine", "defaults")]
    out = []
    for mode in (None, (0, 1), (False, True), None):
        if mode is None:
            ctx.set_triangulation_mode(None)
        else:
            ctx.set_triangulation_mode(*mode)
        n, tb = ctx.launch_count(), ctx.transfer_bytes()
        pf, st = ctx.triangulate_features(*tr.flatten(cases))
        out.append((pf.tobytes(), st.tobytes(), ctx.launch_count() - n, tuple(b - a for a, b in zip(tb, ctx.transfer_bytes()))))
    ctx.set_triangulation_mode(None)
    assert out[0] == out[1] == out[2] == out[3]
    S = tr.scenario()
    fresh = api.Context(S.options, device=0, max_state=S.N + 64, max_meas_rows=4096)
    try:
        ch = synth.load_scenario_into(fresh, S)
        assert list(ch) == base.handles
        pf, st = fresh.triangulate_features(*tr.flatten(cases))
        assert pf.tobytes() == out[0][0] and st.tobytes() == out[0][1]
    finally:
        fresh.close()


def test_setter_refusals_keep_the_mode_and_clearing_restores_the_defaults(setup):
    ctx, base, ctxs, pool, _ = setup
    cases = pool[:200]
    flat = tr.flatten(cases)
    ref = {}
    for mode in MODES:
        ctx.set_triangulation_mode(*t1.MODES[mode])
        ref[mode] = ctx.triangulate_features(*flat)
    assert not np.array_equal(ref["1d_linear"][0], ref["3d_refine"][0])
    ctx.set_triangulation_mode(True, False)
    for bad in ((2, 1), (0, 2), (-1, 1), (1, -1)):
        n = ctx.launch_count()
        with pytest.raises(api.OvpError) as e:
            ctx.set_triangulation_mode(*bad)
        assert e.value.status == 1 and ctx.launch_count() == n  # OVP_ERR_BAD_ARGS
        pf, st = ctx.triangulate_features(*flat)
        assert pf.tobytes() == ref["1d_linear"][0].tobytes() and st.tobytes() == ref["1d_linear"][1].tobytes()
    ctx.set_triangulation_mode(None)
    pf, st = ctx.triangulate_features(*flat)
    assert pf.tobytes() == ref["3d_refine"][0].tobytes() and st.tobytes() == ref["3d_refine"][1].tobytes()


@pytest.mark.parametrize("mode", ["1d_linear", "1d_refine"])
def test_plane_init_tracks_in_1d_modes(setup, mode):
    """the threshold pairs of the mode (those with distinct clones) on a plane that is not in the state, RANSAC held off by its inlier
    minimum: feature status -2 exactly where the reference rejects, the others' positions within its bound"""
    ctx, base, ctxs, _, pairs = setup
    opt = tr.NON_DEFAULT
    cases = [x for x in pairs[(mode, "non_default")] if len(set(x["track"])) == len(x["track"]) and len(x["track"]) <= 37]
    assert {x["rule"] for x in cases} >= {"lin1_min", "lin1_max"}
    mo, mc, uvn = tr.flatten(cases)
    F = len(cases)
    t = dict(meas_offset=mo, meas_clone=mc, uv_norm=uvn, uv=uvn * 458.0 + 300.0, featid=np.arange(1, F + 1, dtype=np.int64),
             planeid=np.full(F, 7, dtype=np.int64))
    ctx.set_triangulation_mode(*t1.MODES[mode])
    try:
        out = ctx.plane_init_tracks(t, plane_init_min_feat=10 ** 6, tri_options=opt)
    finally:
        ctx.set_triangulation_mode(None)
    for i, case in enumerate(cases):
        res = ctxs[mode].run(case, opt)
        assert res["decided"]
        assert (out["feat_status"][i] == -2) == (res["status"] == 0), (mode, case["rule"], case["side"], out["feat_status"][i])
        if res["status"] == 1:
            assert float(np.abs(out["p_FinG"][i] - np.asarray(res["p_FinG"], np.float64)).max()) <= res["p_bound"]
    print("%s: %d threshold cases through plane_init_tracks, statuses %s" % (mode, F, list(out["feat_status"])))


@pytest.mark.parametrize("mode", ["1d_linear", "1d_refine"])
def test_slam_delayed_init_tracks_in_1d_modes(mode, chi2_table):
    """ANCHORED_MSCKF_INVERSE_DEPTH landmarks from tracks: -2 where the reference's mode rejects, the first estimate's get_xyz against the
    mode's p_FinA; unrefined, the first two components are the anchor measurement's normalised coordinates"""
    S, mk, _ = sic.tracks_scene(seed=1)
    ctx, orc, ch, _ = make_pair(S, plane_gate(chi2_table))
    orc.close()
    t = mk(ch)
    rep = 4
    ctx.set_landmark_options(rep, rep)
    ctx.set_triangulation_mode(*t1.MODES[mode])
    poses = tr.camera_poses(ctx, sorted({int(h) for h in t["meas_clone"]}))  # before any initialisation moves the clones
    r = ctx.slam_delayed_init_tracks(t, 1.0, 1.0, use_plane_constraint=False)
    n, n_rej, worst = 0, 0, 0.0
    for f in range(len(t["featid"])):
        a, e = int(t["meas_offset"][f]), int(t["meas_offset"][f + 1])
        if e - a < 2:
            continue
        cl = [int(x) for x in t["meas_clone"][a:e]]
        res = t1.triangulate(np.array([poses[x][0] for x in cl]), np.array([poses[x][1] for x in cl]), t["uv_norm"][a:e], tr.DEFAULTS, mode)
        if not res["decided"]:
            continue
        assert (r["feat_status"][f] == -2) == (res["status"] == 0), (f, res["reason"], r["feat_status"][f])
        n_rej += res["status"] == 0
        h = int(r["new_handles"][f])
        if h < 0:
            continue
        fe = ctx.var_get(h)[1][:3]
        got = fjr.get_xyz(rep, fjr.ld(fe))
        err = float(np.abs(np.asarray(got - res["p_FinA"], dtype=np.float64)).max())
        bound = res["p_bound"] + 64 * np.finfo(np.float64).eps * float(np.abs(np.asarray(res["p_FinA"], dtype=np.float64)).max())
        assert err <= bound, (f, err, bound)
        worst = max(worst, err / bound)
        if mode == "1d_linear":
            uvA = t["uv_norm"][e - 1].astype(np.float64)
            assert np.all(np.abs(fe[:2] - uvA) <= 8 * np.finfo(np.float64).eps * np.maximum(np.abs(uvA), 1.0)), (f, fe[:2], uvA)
        n += 1
    print("%s: %d landmarks, %d rejected by the triangulation; first estimate vs the reference's p_FinA: worst error / bound %.2e" % (mode, n, n_rej,
                                                                                                                                worst))
    assert n >= 10
    ctx.close()
