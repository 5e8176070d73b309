"""ovp_triangulate_features and the triangulation stage of ovp_plane_init_tracks against the long-double reference
(tests/triangulation_reference.py) on generated tracks: one pair per rejection rule on either side of its threshold, degenerate tracks,
every exit of the LM loop, track lengths 2 .. 100 and batches of 1, 63, 64, 65 and 2000 features, under the defaults and a non-default
option set; and the refusal of malformed track offsets."""
import numpy as np
import pytest

import triangulation_reference as tr
from ov_plane_b200 import api, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def setup():
    tr.require_long_double()
    S = tr.scenario()
    ctx = api.Context(S.options, device=0, max_state=S.N + 64, max_meas_rows=4096)
    ch = synth.load_scenario_into(ctx, S)
    ref = tr.Context(ctx, ch, S.intr_value[0])
    yield ctx, ref, tr.case_sets(ref), ch
    ctx.close()


def _check(ref, cases, opt, st, pf, label, table=None):
    """statuses equal on every decided feature, positions within the reference's bound; returns (undecided, worst |dp| / bound)"""
    undecided, worst = 0, 0.0
    for i, c in enumerate(cases):
        res = ref.run(c, opt)
        if not res["decided"]:
            undecided += 1
            continue
        assert st[i] == res["status"], (label, i, c["name"], res["reason"], st[i])
        q = 0.0
        if res["status"] == 1:
            q = float(np.abs(pf[i] - np.asarray(res["p_FinG"], np.float64)).max()) / res["p_bound"]
            assert q <= 1.0, (label, i, c["name"], q)
            worst = max(worst, q)
        if table is not None and "rule" in c:
            table.append("  %-9s %-3s margin %+.2e (bound %.1e)  reference %d  gpu %d  |dp| / bound %.2e" % (
                c["rule"], c["side"], c["margin"], c["bound"], res["status"], st[i], q))
    return undecided, worst


@pytest.mark.parametrize("opt_name", ["defaults", "non_default"])
def test_triangulation_matches_the_reference(setup, opt_name):
    ctx, ref, cs, _ = setup
    c = cs[opt_name]
    opt = c["opt"]
    planted = c["pairs"] + c["degenerate"] + list(c["lm"].values())
    for case in c["pairs"]:
        assert ref.run(case, opt)["decided"], case["rule"]
    mo, mc, uvn = tr.flatten(planted)
    pf, st = ctx.triangulate_features(mo, mc, uvn, options=opt)
    table = []
    und, worst = _check(ref, planted, opt, st, pf, opt_name, table)
    print("\n%s: threshold pairs" % opt_name)
    print("\n".join(table))
    print("%s: planted cases %d, undecided %d, worst |dp| / bound %.2e" % (opt_name, len(planted), und, worst))
    assert und == 0
    # the noisy pool in batches straddling the 64-thread block, then whole
    pool = c["random"]
    for F in (1, 63, 64, 65, len(pool)):
        mo, mc, uvn = tr.flatten(pool[:F])
        pf, st = ctx.triangulate_features(mo, mc, uvn, options=opt)
        und, worst = _check(ref, pool[:F], opt, st, pf, "%s F=%d" % (opt_name, F))
        print("%s: F = %d, %d triangulated, %d undecided excluded, worst |dp| / bound %.2e" % (opt_name, F, int(st.sum()), und, worst))
        assert und <= 0.3 * F + 1  # noisy features whose float32 residuals sit on a rounding boundary within the bound


@pytest.mark.parametrize("opt_name", sorted(tr.LM_OPTION_SETS))
def test_lm_exits_match_the_reference(setup, opt_name):
    ctx, ref, cs, _ = setup
    c = cs[opt_name]
    cases = list(c["lm"].values())
    assert cases
    mo, mc, uvn = tr.flatten(cases)
    pf, st = ctx.triangulate_features(mo, mc, uvn, options=c["opt"])
    und, worst = _check(ref, cases, c["opt"], st, pf, opt_name)
    print("%s: paths %s, worst |dp| / bound %.2e" % (opt_name, sorted(c["lm"]), worst))
    assert und == 0


@pytest.mark.parametrize("opt_name", ["defaults", "non_default"])
def test_plane_init_tracks_triangulates_with_the_given_options(setup, opt_name):
    """the threshold pairs (those with distinct clones, as plane_init_tracks requires) on a plane that is not in the state, RANSAC held
    off by its inlier minimum: feature status -2 exactly where the reference rejects, the others' positions within its bound"""
    ctx, ref, cs, _ = setup
    c = cs[opt_name]
    opt = c["opt"]
    cases = [x for x in c["pairs"] if len(set(x["track"])) == len(x["track"]) and len(x["track"]) <= 37]
    assert {x["rule"] for x in cases} >= {"lin_min", "lin_max", "fin_max", "baseline"}
    mo, mc, uvn = tr.flatten(cases)
    F = len(cases)
    t = dict(meas_offset=mo, meas_clone=mc, uv_norm=uvn, uv=uvn * 458.0 + 300.0, featid=np.arange(1, F + 1, dtype=np.int64),
             planeid=np.full(F, 7, dtype=np.int64))
    launches = ctx.launch_count()
    out = ctx.plane_init_tracks(t, plane_init_min_feat=10 ** 6, tri_options=opt)
    assert ctx.launch_count() > launches
    assert list(out["plane_ids"]) in ([7], [])
    for i, case in enumerate(cases):
        res = ref.run(case, opt)
        assert (out["feat_status"][i] == -2) == (res["status"] == 0), (opt_name, case["rule"], case["side"], out["feat_status"][i])
        if res["status"] == 1:
            assert float(np.abs(out["p_FinG"][i] - np.asarray(res["p_FinG"], np.float64)).max()) <= res["p_bound"]
    print("%s: %d threshold cases through plane_init_tracks, statuses %s" % (opt_name, F, list(out["feat_status"])))


def test_malformed_offsets_are_refused(setup):
    ctx, ref, cs, ch = setup
    good = cs["defaults"]["pairs"][:4]
    mo, mc, uvn = tr.flatten(good)
    for bad in ([1] + list(mo[1:]), [0, mo[2], mo[1]] + list(mo[3:]), list(mo[:-2]) + [mo[-1] + 5, mo[-1]]):
        bad = np.asarray(bad, dtype=np.int32)
        n = ctx.launch_count()
        with pytest.raises(api.OvpError) as e:
            ctx.triangulate_features(bad, mc, uvn)
        assert e.value.status == 1  # OVP_ERR_BAD_ARGS
        assert "meas_offset" in str(e.value)
        assert ctx.launch_count() == n
    pf, st = ctx.triangulate_features(mo, mc, uvn)
    for i, c in enumerate(good):
        res = ref.run(c, tr.DEFAULTS)
        assert st[i] == res["status"]
