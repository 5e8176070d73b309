"""ovp_plane_init_tracks (UpdaterPlane::init_vio_plane end to end on raw tracks) on the device: orchestration parity against the oracle's
stages chained in the reference's order (fed the device's triangulation), bit-identity with the four existing entry points chained by hand,
the host<->device traffic of the composed call, an end-to-end comparison against the oracle's own triangulation, refusals and the empty call."""
import ctypes as C

import numpy as np
import pytest

import oracle_plane_init
from conftest import make_pair
from test_cpu_plane_init_tracks import CHI2_SCENE
from ov_plane_b200 import api, synth
from ov_plane_b200 import plane_init_chain as pic

pytestmark = pytest.mark.gpu

CAP = 15  # small_planes puts ~20 features on each plane: every plane is over the cap and keeps its 16 shortest tracks
HAZARDS = dict(name="small_planes", px_noise=0.1, keep_in_state=(4,), off_plane=((1, 0.03), (2, 0.045)), ransac_fail_plane=50, n_single=3, n_far=1)


def _candidates(be, t):
    mo, pid = np.asarray(t["meas_offset"]), np.asarray(t["planeid"])
    return [f for f in range(len(mo) - 1) if pid[f] != 0 and be.plane_handle(int(pid[f])) < 0 and mo[f + 1] - mo[f] >= 2]


def _tri_of(ctx, t, cand):
    cnt = np.diff(t["meas_offset"])
    offs = np.concatenate([[0], np.cumsum(cnt[cand])]).astype(np.int32)
    sel = np.concatenate([np.arange(t["meas_offset"][f], t["meas_offset"][f + 1]) for f in cand])
    return ctx.triangulate_features(offs, t["meas_clone"][sel], t["uv_norm"][sel])


def _state(be):
    order = be.variable_order()
    return be.cov(), [be.var_get(h) for h in order], order


SCENES = {"hazards_s0": (dict(HAZARDS, seed=0), 1.0), "hazards_s2": (dict(HAZARDS, seed=2), 1.0), "chi2_reject": CHI2_SCENE}


@pytest.mark.parametrize("scene", sorted(SCENES))
def test_orchestration_matches_the_oracle_fed_the_device_triangulation(scene, chi2_table):
    kw, c2 = SCENES[scene]
    S, mk = pic.tracks_scene(**kw)
    S.options["const_init_chi2"] = c2
    ctx, orc, chg, cho = make_pair(S, chi2_table)
    assert np.array_equal(np.asarray(chg), np.asarray(cho))
    t = mk(chg)
    cand = _candidates(ctx, t)
    tri = _tri_of(ctx, t, cand)
    n0 = ctx.cov_rows()
    g = ctx.plane_init_tracks(t, max_msckf_plane=CAP)
    o = oracle_plane_init.plane_init_tracks(orc, mk(cho), S.options["sigma_constraint"], max_msckf_plane=CAP, tri=tri)
    o["stages"] = oracle_plane_init.stages_of(o, t["planeid"])
    print("%s: planes %s status gpu %s oracle %s" % (scene, g["plane_ids"], g["plane_status"], o["plane_status"]))
    # the scene covers: ties over more than 16 valid features, planes over the cap, RANSAC and refinement failures, one-measurement tracks,
    # a triangulation failure, an in-state plane and off-plane features, a plane that initialises
    fs = o["feat_status"]
    assert len(cand) > 16 and len(set(np.diff(t["meas_offset"])[cand])) < len(cand) // 2
    assert all(len(st["grouped"]) == CAP + 1 for p, st in o["stages"].items() if p != 50)
    assert (o["plane_status"] == -2).any() and (o["plane_status"] == -3).any() and (o["plane_status"] == 1).any()
    if scene == "chi2_reject":  # a chi2-rejected plane, then one initialised at the posterior of that attempt
        assert list(o["plane_status"]) == [0, -3, 1, -2]
    assert (fs == -1).sum() == 3 and (fs == -2).any() and (fs == 0).sum() > 0 and (fs == 2).any() and (fs == 1).any()
    for k in ("feat_status", "plane_ids", "plane_status", "new_handles"):
        assert np.array_equal(g[k], o[k]), (k, g[k], o[k])
    assert np.abs(g["cp"] - o["cp"]).max() < 1e-7
    assert np.abs(g["p_FinG"] - o["p_FinG"]).max() < 1e-7
    n_init = int((g["plane_status"] == 1).sum())
    assert ctx.cov_rows() == n0 + 3 * n_init == orc.cov_rows()
    Pg, Po = ctx.cov(), orc.cov()
    assert np.linalg.norm(Pg - Po) / np.linalg.norm(Po) < 1e-6
    for h in g["new_handles"][g["new_handles"] >= 0]:
        vg, vo = ctx.var_get(int(h)), orc.var_get(int(h))
        assert np.abs(vg[0] - vo[0]).max() < 1e-6 and np.abs(vg[1] - vo[1]).max() < 1e-6
    # the per-stage feature sets: the device's stages chained by hand against the oracle's
    ctx2, _, ch2, _ = make_pair(S, chi2_table)
    h = pic.chain(ctx2, mk(ch2), S.options["sigma_constraint"], max_msckf_plane=CAP)
    for p in o["stages"]:
        for k in ("grouped", "ransac", "refined"):
            assert o["stages"][p][k] == set(h["stages"][p].get(k, ())), (p, k)
    ctx.close()
    ctx2.close()


def test_composed_call_equals_the_hand_chain_bit_for_bit_and_moves_less(chi2_table):
    S, mk = pic.tracks_scene(seed=2, **HAZARDS)
    a, _, cha, _ = make_pair(S, chi2_table)
    b, _, chb, _ = make_pair(S, chi2_table)
    ta, tb = mk(cha), mk(chb)
    ha0, da0 = a.transfer_bytes()
    hb0, db0 = b.transfer_bytes()
    ra = a.plane_init_tracks(ta, max_msckf_plane=CAP)
    rb = pic.chain(b, tb, S.options["sigma_constraint"], max_msckf_plane=CAP)
    ha, da = a.transfer_bytes()
    hb, db = b.transfer_bytes()
    for k in ("feat_status", "plane_ids", "plane_status", "new_handles", "cp", "p_FinG"):
        assert np.array_equal(ra[k], rb[k]), k
    Pa, va, oa = _state(a)
    Pb, vb, ob = _state(b)
    assert oa == ob and np.array_equal(Pa, Pb)
    assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(va, vb))
    F, P = len(ta["featid"]), len(ra["plane_ids"])
    h2d_c, h2d_h, d2h_c, d2h_h = ha - ha0, hb - hb0, da - da0, db - db0
    print("host->device bytes: composed %d, hand chain %d; device->host: composed %d, hand chain %d (F=%d, planes=%d)" % (
        h2d_c, h2d_h, d2h_c, d2h_h, F, P))
    assert h2d_c < h2d_h
    # statuses and inlier flags of three stages (4 B each per feature), the positions (24 B per feature), per plane the RANSAC / refinement
    # statuses and the refined plane; plus the initialisation stage, which reads back a chi2 and status words per plane
    assert d2h_c <= 64 * F + 1024 * P, d2h_c
    a.close()
    b.close()


def test_end_to_end_against_the_oracle_triangulation(chi2_table):
    """Device triangulation differs from the oracle's by up to 5e-5 m (test_gpu_triangulation.py).  The scene is checked to keep every point
    more than 1e-3 m away from RANSAC's 0.05 m inlier distance to the winning plane in the oracle's run, so the final inlier sets cannot flip.
    The check does not cover the other 199 hypotheses, whose inlier counts could in principle differ and change the winning draw; the
    statuses are therefore asserted equal first, and a flip would fail there rather than pass unnoticed.  With equal decisions, the refinement
    starts from points 5e-5 m apart and converges to the same optimum within its tolerances, so the posteriors agree to 1e-5 relative."""
    S, mk = pic.tracks_scene(name="small_planes", seed=3, px_noise=0.1, keep_in_state=(4,))
    ctx, orc, chg, cho = make_pair(S, chi2_table)
    o = pic.chain(orc, mk(cho), S.options["sigma_constraint"], max_msckf_plane=CAP)  # the oracle's stages, with its own triangulation
    for p, st in o["stages"].items():
        if "abcd" in st:
            d = np.abs(o["p_FinG"][st["grouped"]] @ st["abcd"][:3] + st["abcd"][3])
            assert np.abs(d - 0.05).min() > 1e-3, p
    g = ctx.plane_init_tracks(mk(chg), max_msckf_plane=CAP)
    for k in ("feat_status", "plane_ids", "plane_status", "new_handles"):
        assert np.array_equal(g[k], o[k]), k
    assert (g["plane_status"] == 1).sum() >= 2
    assert np.abs(g["cp"] - o["cp"]).max() < 1e-4
    Pg, Po = ctx.cov(), orc.cov()
    rel = np.linalg.norm(Pg - Po) / np.linalg.norm(Po)
    print("posterior covariance rel. difference %.2e" % rel)
    assert rel < 1e-5
    ctx.close()


def _raw_call(ctx, t, opt, F):
    """ovp_plane_init_tracks through ctypes, so that the tracks / options may be NULL"""
    fs, pf, npl = np.zeros(F, dtype=np.int32), np.zeros((F, 3)), C.c_int(0)
    pids, ps, nh, cp = np.zeros(len(fs), dtype=np.int64), np.zeros(len(fs), dtype=np.int32), np.zeros(len(fs), dtype=np.int32), np.zeros((len(fs), 3))
    return ctx.lib.ovp_plane_init_tracks(ctx.h, t, opt, fs.ctypes.data, pf.ctypes.data, C.byref(npl), pids.ctypes.data, ps.ctypes.data, nh.ctypes.data,
                                         cp.ctypes.data)


def test_refusals_launch_nothing_and_leave_the_state_as_it_was(chi2_table):
    S, mk = pic.tracks_scene(seed=2, **HAZARDS)
    ctx, _, ch, _ = make_pair(S, chi2_table)
    t = mk(ch)
    cand = _candidates(ctx, t)
    f0 = cand[0]
    a0 = int(t["meas_offset"][f0])

    def variant(**kw):
        v = {k: np.array(x, copy=True) for k, x in t.items()}
        v.update(kw)
        return v
    bad_clone = variant()
    bad_clone["meas_clone"][a0] = ctx.handle_imu()
    dup = variant()
    dup["featid"][cand[1]] = dup["featid"][f0]
    # one candidate with 38 measurements (one above the plane-system limit)
    cnt = np.diff(t["meas_offset"])
    m_long = 38
    mc_f = np.resize(t["meas_clone"][a0:a0 + cnt[f0]], m_long)
    uv_f = np.resize(t["uv"][a0:a0 + cnt[f0]], (m_long, 2))
    uvn_f = np.resize(t["uv_norm"][a0:a0 + cnt[f0]], (m_long, 2))
    sl = slice(a0, a0 + cnt[f0])
    long = variant(meas_offset=np.concatenate([t["meas_offset"][:f0 + 1], t["meas_offset"][f0 + 1:] + (m_long - cnt[f0])]).astype(np.int32),
                   meas_clone=np.concatenate([t["meas_clone"][:sl.start], mc_f, t["meas_clone"][sl.stop:]]).astype(np.int32),
                   uv=np.concatenate([t["uv"][:sl.start], uv_f, t["uv"][sl.stop:]]).astype(np.float32),
                   uv_norm=np.concatenate([t["uv_norm"][:sl.start], uvn_f, t["uv_norm"][sl.stop:]]).astype(np.float32))
    cases = [(bad_clone, {}, api.OvpError, 1), (dup, {}, api.OvpError, 1), (long, {}, api.OvpError, 7), (t, dict(max_msckf_plane=5000), api.OvpError, 7),
             (t, dict(shuffle_kind=3), api.OvpError, 1)]
    P0, v0, o0 = _state(ctx)
    l0 = ctx.launch_count()
    for tr, kw, exc, code in cases:
        with pytest.raises(exc) as ei:
            ctx.plane_init_tracks(tr, **dict(dict(max_msckf_plane=CAP), **kw))
        assert ei.value.status == code, (ei.value, code)
    # null pointers: the tracks, the options, an output
    tt = api.FeatureTracks(len(t["featid"]), t["meas_offset"].ctypes.data, t["meas_clone"].ctypes.data, t["uv"].ctypes.data, None,
                           t["featid"].ctypes.data, t["planeid"].ctypes.data)
    oo = api.PlaneInitOptions(1.0, CAP, 8, 200.0, 0, None)
    F = len(t["featid"])
    assert _raw_call(ctx, None, C.byref(oo), F) == 1
    assert _raw_call(ctx, C.byref(tt), C.byref(oo), F) == 1  # uv_norm is NULL
    assert _raw_call(ctx, C.byref(tt), None, F) == 1
    assert ctx.launch_count() == l0
    P1, v1, o1 = _state(ctx)
    assert o1 == o0 and np.array_equal(P1, P0)
    assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(v0, v1))
    ctx.close()


def test_nothing_to_do_launches_nothing(chi2_table):
    S, mk = pic.tracks_scene(seed=2, **HAZARDS)
    ctx, _, ch, _ = make_pair(S, chi2_table)
    t = mk(ch)
    P0, v0, o0 = _state(ctx)
    l0 = ctx.launch_count()
    for planeid in (np.zeros_like(t["planeid"]), np.where(t["planeid"] != 0, 4, 0)):  # no plane at all; only the in-state plane
        r = ctx.plane_init_tracks(dict(t, planeid=planeid), max_msckf_plane=CAP)
        assert len(r["plane_ids"]) == 0 and (r["feat_status"] == 0).all()
    empty = dict(meas_offset=np.zeros(1, dtype=np.int32), meas_clone=np.zeros(0, dtype=np.int32), uv=np.zeros((0, 2), dtype=np.float32),
                 uv_norm=np.zeros((0, 2), dtype=np.float32), featid=np.zeros(0, dtype=np.int64), planeid=np.zeros(0, dtype=np.int64))
    assert len(ctx.plane_init_tracks(empty)["plane_ids"]) == 0
    assert ctx.launch_count() == l0
    P1, v1, o1 = _state(ctx)
    assert o1 == o0 and np.array_equal(P1, P0)
    assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(v0, v1))
    ctx.close()
