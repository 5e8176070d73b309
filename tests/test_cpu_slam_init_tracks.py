"""UpdaterSLAM::delayed_init's orchestration on the CPU oracle: the C++ composition (tests/oracle_slam_init.cpp) against the oracle's stages
chained by hand from Python (ov_plane_b200.slam_init_chain), on scenes with every hazard, and the rule that a refinement candidate is refined
before its triangulation is judged."""
import numpy as np
import pytest

import oracle_backend
import oracle_slam_init as osi
from ov_plane_b200 import synth
from ov_plane_b200 import slam_init_chain as sic


def plane_gate(chi2):
    """The chi2 table with a near-zero quantile at every dof 3 (mod 6): the plane-constrained attempt of a track with an odd number m of
    measurements (3m rows) is rejected, its retry without the plane (2m rows, even) and every attempt of an even track keep the real quantiles.
    The scenes' cameras see the planes mostly along their normals, so a point refined onto its plane stays consistent with its rays and the
    real gate does not reject the plane; this table makes the chi2 fallback (status 3) happen on a known set of features."""
    q = np.array(chi2, dtype=np.float64, copy=True)
    q[3::6] = 1e-9
    return q


def _oracle(S, chi2):
    orc = oracle_backend.OracleContext(S.options)
    orc.set_chi2_table(plane_gate(chi2))
    return orc, synth.load_scenario_into(orc, S)


def _run(S, mk, chi2, which, preset0=(), tri=None, **kw):
    orc, ch = _oracle(S, chi2)
    t = mk(ch)
    for k in preset0:  # _features_SLAM_to_PLANE = 0 from an earlier failure
        osi.set_slam_plane_of(orc, t["featid"][k], 0)
    if which == "composed":
        r = osi.slam_delayed_init_tracks(orc, t, S.options["sigma_constraint"], tri=tri, **kw)
    else:
        r = sic.chain(orc, t, S.options["sigma_constraint"], tri=tri, plane_of=lambda f: osi.slam_plane_of(orc, f),
                      set_plane_of=lambda f, p: osi.set_slam_plane_of(orc, f, p), **kw)
    r["s2p"] = np.array([osi.slam_plane_of(orc, f) for f in t["featid"]])
    r["P"] = orc.cov()
    r["values"] = [orc.var_get(h) for h in orc.variable_order()]
    return r, t


def _assert_equal(a, b):
    for k in ("feat_status", "plane_status", "new_handles", "p_FinG", "s2p", "P"):
        assert np.array_equal(a[k], b[k]), k
    assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(a["values"], b["values"]))


SWITCHES = {"default": {}, "refine_off": dict(use_refine_plane_feat=False), "plane_off": dict(use_plane_constraint=False)}


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("switch", sorted(SWITCHES))
def test_composition_equals_the_chained_stages(seed, switch, chi2_table):
    S, mk, hz = sic.tracks_scene(seed=seed)
    pre = [int(np.nonzero(mk(np.zeros(64, dtype=np.int32))["planeid"] == 1)[0][-1])]  # the last plane 1 feature: failed on its plane before
    a, t = _run(S, mk, chi2_table, "composed", preset0=pre, **SWITCHES[switch])
    b, _ = _run(S, mk, chi2_table, "chain", preset0=pre, **SWITCHES[switch])
    _assert_equal(a, b)
    fs, ps = a["feat_status"], a["plane_status"]
    assert fs[hz["single"]] == -1 and fs[hz["far_free"]] == -2 and fs[hz["far_cand"]] == -2 and fs[hz["outlier"]] == 0
    assert (fs == 1).sum() > 10 and (a["new_handles"] >= 0).sum() == ((fs == 1) | (fs == 3)).sum()
    assert ps[pre[0]] == -1 and a["s2p"][pre[0]] == 0  # not a candidate; initialised without its plane
    assert (ps[t["planeid"] == 4] == -1).all() and (ps[t["planeid"] == 0] == -1).all()  # plane not in the state / no plane
    assert (a["p_FinG"][hz["single"]] == 0).all()
    # plane_gate: the features that try their plane first fall back to status 3 exactly when their track is odd
    with_plane = {"default": ps == 1, "refine_off": np.isin(t["planeid"], (1, 2, 3)) & (np.arange(len(fs)) != pre[0]),
                  "plane_off": np.zeros(len(fs), dtype=bool)}[switch] & (fs != -2)
    assert np.array_equal(fs == 3, with_plane & (np.diff(t["meas_offset"]) % 2 == 1))
    assert (fs == 3).any() == (switch != "plane_off")
    if switch == "default":
        assert ps[hz["far_cand"]] == 0  # refined although its triangulation failed
        assert (ps == 1).any() and (ps == 0).sum() > 1
        assert a["s2p"][hz["far_cand"]] == -1  # a failed refinement of a failed triangulation leaves the entry alone
        for f in np.nonzero((ps == 0) & (fs >= 0))[0]:
            assert a["s2p"][f] == 0
    else:
        assert (ps == -1).all()


def test_refinement_comes_before_the_triangulation_verdict(chi2_table):
    """A candidate whose triangulation failed is still refined, and a successful refinement leaves _features_SLAM_to_PLANE pointing at the
    plane (UpdaterSLAM.cpp:147-193).  The oracle's own triangulation is fed back with one refined-onto-its-plane candidate marked failed."""
    S, mk, hz = sic.tracks_scene(seed=0)
    orc, ch = _oracle(S, chi2_table)
    t = mk(ch)
    cnt = np.diff(t["meas_offset"])
    trk = [f for f in range(len(cnt)) if cnt[f] >= 2]
    sel = np.concatenate([np.arange(t["meas_offset"][f], t["meas_offset"][f + 1]) for f in trk])
    p, st = orc.triangulate_features(np.concatenate([[0], np.cumsum(cnt[trk])]).astype(np.int32), t["meas_clone"][sel], t["uv_norm"][sel])
    ref, _ = _run(S, mk, chi2_table, "composed", tri=(p, st))
    f = int(np.nonzero(ref["plane_status"] == 1)[0][0])
    st = st.copy()
    st[trk.index(f)] = 0
    a, _ = _run(S, mk, chi2_table, "composed", tri=(p, st))
    b, _ = _run(S, mk, chi2_table, "chain", tri=(p, st))
    _assert_equal(a, b)
    assert a["feat_status"][f] == -2 and a["plane_status"][f] == 1 and a["s2p"][f] == t["planeid"][f] and a["new_handles"][f] == -1
    assert np.array_equal(a["p_FinG"][f], ref["p_FinG"][f])  # the refined position stays in the Feature


def test_fallback_position_and_the_refined_position(chi2_table):
    """p_FinG out: the refined position of every refined feature, the triangulated one where the refinement failed.  The landmark of a
    refined feature initialised with its plane starts at the refined position; one initialised only after the chi2 test rejected its plane
    (status 3) and one whose refinement failed start at the triangulated position."""
    S, mk, hz = sic.tracks_scene(seed=1)
    orc, ch = _oracle(S, chi2_table)
    t = mk(ch)
    a = osi.slam_delayed_init_tracks(orc, t, S.options["sigma_constraint"])
    orc2, ch2 = _oracle(S, chi2_table)
    cnt = np.diff(t["meas_offset"])
    trk = [f for f in range(len(cnt)) if cnt[f] >= 2]
    sel = np.concatenate([np.arange(t["meas_offset"][f], t["meas_offset"][f + 1]) for f in trk])
    p, st = orc2.triangulate_features(np.concatenate([[0], np.cumsum(cnt[trk])]).astype(np.int32), t["meas_clone"][sel], t["uv_norm"][sel])
    n = {1: 0, 3: 0, "fail": 0}
    for k, f in enumerate(trk):
        if a["feat_status"][f] not in (1, 3):
            continue
        v, fej = orc.var_get(int(a["new_handles"][f]))
        if a["plane_status"][f] == 0:
            n["fail"] += 1
            assert np.array_equal(a["p_FinG"][f], p[k]) and np.array_equal(fej, p[k])
        elif a["plane_status"][f] == 1:
            n[int(a["feat_status"][f])] += 1
            assert not np.array_equal(a["p_FinG"][f], p[k])  # the Feature keeps the refined position, for status 3 as well
            assert np.array_equal(fej, a["p_FinG"][f] if a["feat_status"][f] == 1 else p[k])  # a status-3 landmark starts at the triangulation
    assert n[1] > 0 and n[3] > 0 and n["fail"] > 0, n
