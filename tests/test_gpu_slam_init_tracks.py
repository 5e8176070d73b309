"""ovp_slam_delayed_init_tracks (UpdaterSLAM::delayed_init end to end on raw tracks) on the device: parity with the oracle's stages composed in
the reference's order (fed the device's triangulation), bit-identity with the three existing entry points chained by hand and the host->device
traffic saved, an end-to-end comparison against the oracle's own triangulation, refusals, the empty call and a state-capacity refusal."""
import ctypes as C

import numpy as np
import pytest

import oracle_slam_init as osi
from conftest import make_pair
from test_cpu_slam_init_tracks import plane_gate
from ov_plane_b200 import api
from ov_plane_b200 import slam_init_chain as sic

pytestmark = pytest.mark.gpu

SWITCHES = {"default": {}, "refine_off": dict(use_refine_plane_feat=False), "plane_off": dict(use_plane_constraint=False)}


def _state(be):
    order = be.variable_order()
    return be.cov(), [be.var_get(h) for h in order], order


def _tri_of(ctx, t):
    cnt = np.diff(t["meas_offset"])
    trk = [f for f in range(len(cnt)) if cnt[f] >= 2]
    sel = np.concatenate([np.arange(t["meas_offset"][f], t["meas_offset"][f + 1]) for f in trk])
    return ctx.triangulate_features(np.concatenate([[0], np.cumsum(cnt[trk])]).astype(np.int32), t["meas_clone"][sel], t["uv_norm"][sel])


def _preset_failed(be, t, k, sigma_constraint):
    """_features_SLAM_to_PLANE[featid of k] = 0 without a landmark, as an earlier delayed_init leaves a feature that failed with and without its
    plane: ovp_slam_delayed_init on its track with a 40 px outlier"""
    a, b = int(t["meas_offset"][k]), int(t["meas_offset"][k + 1])
    uv = np.array(t["uv"][a:b])
    uv[-1] += 40.0
    p, st = be.triangulate_features(np.array([0, b - a], dtype=np.int32), t["meas_clone"][a:b], t["uv_norm"][a:b])
    assert st[0]
    r = be.slam_delayed_init(dict(F=1, meas_offset=np.array([0, b - a], dtype=np.int32), meas_clone=np.ascontiguousarray(t["meas_clone"][a:b]), uv=uv,
                                  p_FinG=p, p_FinG_original=p, featid=t["featid"][[k]], planeid=t["planeid"][[k]]), 1.0, 1.0)
    assert r["feat_status"][0] == 0


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("switch", sorted(SWITCHES))
def test_matches_the_oracle_fed_the_device_triangulation(seed, switch, chi2_table):
    S, mk, hz = sic.tracks_scene(seed=seed)
    ctx, orc, chg, cho = make_pair(S, plane_gate(chi2_table))
    tg, to = mk(chg), mk(cho)
    pre = int(np.nonzero(tg["planeid"] == 1)[0][-1])
    _preset_failed(ctx, tg, pre, S.options["sigma_constraint"])
    _preset_failed(orc, to, pre, S.options["sigma_constraint"])
    tri = _tri_of(ctx, tg)
    n0 = ctx.cov_rows()
    g = ctx.slam_delayed_init_tracks(tg, **SWITCHES[switch])
    o = osi.slam_delayed_init_tracks(orc, to, S.options["sigma_constraint"], tri=tri, **SWITCHES[switch])
    fs, ps = o["feat_status"], o["plane_status"]
    print("%s/%d: feat_status %s plane_status %s" % (switch, seed, fs.tolist(), ps.tolist()))
    assert fs[hz["single"]] == -1 and fs[hz["far_free"]] == -2 and fs[hz["far_cand"]] == -2 and fs[hz["outlier"]] == 0 and (fs == 1).sum() > 10
    if switch == "default":
        assert ps[hz["far_cand"]] == 0 and (ps == 1).any() and ((ps == 0) & (fs == 1)).any() and ps[pre] == -1
        assert ((fs == 3) & (ps == 1)).any()  # refined, rejected with the plane by plane_gate, initialised without it
    assert (fs == 3).any() == (switch != "plane_off")
    for k in ("feat_status", "plane_status", "new_handles"):
        assert np.array_equal(g[k], o[k]), (k, g[k], o[k])
    assert np.abs(g["p_FinG"] - o["p_FinG"]).max() < 1e-7
    # status 3: the Feature keeps the position the refinement gave it, the landmark starts at the device's triangulation
    trk = [f for f in range(len(fs)) if tg["meas_offset"][f + 1] - tg["meas_offset"][f] >= 2]
    for f in np.nonzero(g["feat_status"] == 3)[0]:
        p_tri = tri[0][trk.index(f)]
        _, fej = ctx.var_get(int(g["new_handles"][f]))
        assert np.array_equal(fej, p_tri), f
        assert np.array_equal(g["p_FinG"][f], p_tri) == (g["plane_status"][f] != 1), f
    for f in list(tg["featid"]) + [S.slam[0][0]]:
        assert ctx.slam_plane_of(f) == osi.slam_plane_of(orc, f), f
    n_new = int((g["new_handles"] >= 0).sum())
    assert ctx.cov_rows() == n0 + 3 * n_new == orc.cov_rows()
    Pg, Po = ctx.cov(), orc.cov()
    assert np.linalg.norm(Pg - Po) / np.linalg.norm(Po) < 1e-6
    for h in g["new_handles"][g["new_handles"] >= 0]:
        vg, vo = ctx.var_get(int(h)), orc.var_get(int(h))
        assert np.abs(vg[0] - vo[0]).max() < 1e-6 and np.abs(vg[1] - vo[1]).max() < 1e-6
    ctx.close()


@pytest.mark.parametrize("switch", sorted(SWITCHES))
def test_composed_call_equals_the_hand_chain_bit_for_bit_and_moves_less(switch, chi2_table):
    S, mk, hz = sic.tracks_scene(seed=1)
    a, _, cha, _ = make_pair(S, plane_gate(chi2_table))
    b, _, chb, _ = make_pair(S, plane_gate(chi2_table))
    ta, tb = mk(cha), mk(chb)
    ha0, da0 = a.transfer_bytes()
    hb0, db0 = b.transfer_bytes()
    ra = a.slam_delayed_init_tracks(ta, **SWITCHES[switch])
    rb = sic.chain(b, tb, S.options["sigma_constraint"], **SWITCHES[switch])
    ha, da = a.transfer_bytes()
    hb, db = b.transfer_bytes()
    for k in ("feat_status", "plane_status", "new_handles", "p_FinG"):
        assert np.array_equal(ra[k], rb[k]), k
    assert (ra["feat_status"] == 3).any() == (switch != "plane_off")
    Pa, va, oa = _state(a)
    Pb, vb, ob = _state(b)
    assert oa == ob and np.array_equal(Pa, Pb)
    assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(va, vb))
    print("%s: host->device bytes composed %d, hand chain %d; device->host composed %d, hand chain %d" % (switch, ha - ha0, hb - hb0, da - da0,
                                                                                                          db - db0))
    assert ha - ha0 < hb - hb0
    a.close()
    b.close()


def test_end_to_end_against_the_oracle_triangulation(chi2_table):
    """Device triangulation differs from the oracle's by up to 5e-5 m (test_gpu_triangulation.py); the decisions are asserted equal first, then
    the posteriors, which start from points that far apart"""
    S, mk, hz = sic.tracks_scene(seed=2)
    ctx, orc, chg, cho = make_pair(S, plane_gate(chi2_table))
    g = ctx.slam_delayed_init_tracks(mk(chg))
    o = osi.slam_delayed_init_tracks(orc, mk(cho), S.options["sigma_constraint"])
    for k in ("feat_status", "plane_status", "new_handles"):
        assert np.array_equal(g[k], o[k]), k
    assert np.abs(g["p_FinG"] - o["p_FinG"]).max() < 1e-3
    Pg, Po = ctx.cov(), orc.cov()
    rel = np.linalg.norm(Pg - Po) / np.linalg.norm(Po)
    print("posterior covariance rel. difference %.2e" % rel)
    assert rel < 1e-5
    ctx.close()


def _raw_call(ctx, t, opt, F):
    """ovp_slam_delayed_init_tracks through ctypes, so that the tracks / options / outputs may be NULL"""
    fs, ps, pf, nh = np.zeros(F, dtype=np.int32), np.zeros(F, dtype=np.int32), np.zeros((F, 3)), np.zeros(F, dtype=np.int32)
    return ctx.lib.ovp_slam_delayed_init_tracks(ctx.h, t, opt, fs.ctypes.data, ps.ctypes.data, pf.ctypes.data, nh.ctypes.data)


def _variant(t, **kw):
    v = {k: np.array(x, copy=True) for k, x in t.items()}
    v.update(kw)
    return v


def _with_track(t, f, clones, uv, uvn):
    """t with feature f's track replaced"""
    mo = t["meas_offset"]
    a, b = int(mo[f]), int(mo[f + 1])
    d = len(clones) - (b - a)
    return _variant(t, meas_offset=np.concatenate([mo[:f + 1], mo[f + 1:] + d]).astype(np.int32),
                    meas_clone=np.concatenate([t["meas_clone"][:a], clones, t["meas_clone"][b:]]).astype(np.int32),
                    uv=np.concatenate([t["uv"][:a], uv, t["uv"][b:]]).astype(np.float32),
                    uv_norm=np.concatenate([t["uv_norm"][:a], uvn, t["uv_norm"][b:]]).astype(np.float32))


def test_refusals_launch_nothing_and_leave_the_state_as_it_was(chi2_table):
    S, mk, hz = sic.tracks_scene(seed=0)
    ctx, _, ch, _ = make_pair(S, chi2_table)
    t = mk(ch)
    f0 = 2 if hz["far_cand"] != 2 else 3
    a0, n0 = int(t["meas_offset"][f0]), int(t["meas_offset"][f0 + 1] - t["meas_offset"][f0])
    bad_clone = _variant(t)
    bad_clone["meas_clone"][a0] = ctx.handle_imu()
    twice = _variant(t)
    twice["meas_clone"][a0 + 1] = twice["meas_clone"][a0]
    dup = _variant(t)
    dup["featid"][f0 + 1] = dup["featid"][f0]
    landmark = _variant(t)
    landmark["featid"][f0] = S.slam[0][0]  # already a SLAM landmark
    aruco = _variant(t)
    aruco["featid"][f0] = 7
    offset0 = _variant(t, meas_offset=t["meas_offset"] + 1)
    decreasing = _variant(t)
    decreasing["meas_offset"][f0 + 1] = decreasing["meas_offset"][f0] - 1
    m_long = 65  # one above OVP_SLAM_INIT_MAX_TRACK
    long = _with_track(t, f0, np.resize(t["meas_clone"][a0:a0 + n0], m_long), np.resize(t["uv"][a0:a0 + n0], (m_long, 2)),
                       np.resize(t["uv_norm"][a0:a0 + n0], (m_long, 2)))
    cases = [(bad_clone, {}, 1), (twice, {}, 1), (dup, {}, 1), (landmark, {}, 6), (aruco, {}, 1), (offset0, {}, 1), (decreasing, {}, 1), (long, {}, 7),
             (t, dict(sigma_pix=0.0), 1)]
    P0, v0, o0 = _state(ctx)
    l0, b0 = ctx.launch_count(), ctx.transfer_bytes()
    for tr, kw, code in cases:
        with pytest.raises(api.OvpError) as ei:
            ctx.slam_delayed_init_tracks(tr, **kw)
        assert ei.value.status == code, (ei.value, code)
    F = len(t["featid"])
    tt = api.FeatureTracks(F, t["meas_offset"].ctypes.data, t["meas_clone"].ctypes.data, t["uv"].ctypes.data, None, t["featid"].ctypes.data,
                           t["planeid"].ctypes.data)
    oo = api.SlamInitOptions(1.0, 1.0, 1, 1, None)
    assert _raw_call(ctx, None, C.byref(oo), F) == 1
    assert _raw_call(ctx, C.byref(tt), C.byref(oo), F) == 1  # uv_norm is NULL
    assert _raw_call(ctx, C.byref(tt), None, F) == 1
    assert ctx.launch_count() == l0 and ctx.transfer_bytes() == b0
    # a chi2 table too short for the rows of the longest track (3 per measurement with its plane)
    mmax = int(np.diff(t["meas_offset"]).max())
    ctx.set_chi2_table(chi2_table[:3 * mmax - 1])
    l1, b1 = ctx.launch_count(), ctx.transfer_bytes()
    with pytest.raises(api.OvpError) as ei:
        ctx.slam_delayed_init_tracks(t)
    assert ei.value.status == 1 and "chi2" in str(ei.value)
    assert ctx.launch_count() == l1 and ctx.transfer_bytes() == b1
    P1, v1, o1 = _state(ctx)
    assert o1 == o0 and np.array_equal(P1, P0)
    assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(v0, v1))
    assert all(ctx.slam_plane_of(f) == -1 for f in t["featid"])
    ctx.close()


def test_nothing_to_do_launches_nothing(chi2_table):
    S, mk, hz = sic.tracks_scene(seed=0)
    ctx, _, ch, _ = make_pair(S, chi2_table)
    t = mk(ch)
    P0, v0, o0 = _state(ctx)
    l0, b0 = ctx.launch_count(), ctx.transfer_bytes()
    empty = dict(meas_offset=np.zeros(1, dtype=np.int32), meas_clone=np.zeros(0, dtype=np.int32), uv=np.zeros((0, 2), dtype=np.float32),
                 uv_norm=np.zeros((0, 2), dtype=np.float32), featid=np.zeros(0, dtype=np.int64), planeid=np.zeros(0, dtype=np.int64))
    assert len(ctx.slam_delayed_init_tracks(empty)["feat_status"]) == 0
    k = hz["single"]
    one = dict(meas_offset=np.array([0, 1], dtype=np.int32), meas_clone=t["meas_clone"][t["meas_offset"][k]:t["meas_offset"][k] + 1],
               uv=t["uv"][t["meas_offset"][k]:t["meas_offset"][k] + 1], uv_norm=t["uv_norm"][t["meas_offset"][k]:t["meas_offset"][k] + 1],
               featid=t["featid"][[k]], planeid=t["planeid"][[k]])
    r = ctx.slam_delayed_init_tracks(one)
    assert list(r["feat_status"]) == [-1] and list(r["new_handles"]) == [-1]
    assert ctx.launch_count() == l0 and ctx.transfer_bytes() == b0
    P1, v1, o1 = _state(ctx)
    assert o1 == o0 and np.array_equal(P1, P0)
    ctx.close()


def test_state_capacity_refusal_keeps_the_earlier_landmarks(chi2_table):
    """A state with room for two more landmarks: the third initialisation is refused with OVP_ERR_CAPACITY, after the launches; the two
    landmarks before it stay, as they would with ovp_slam_delayed_init"""
    S, mk, hz = sic.tracks_scene(seed=1)
    ctx, _, ch, _ = make_pair(S, chi2_table, max_state=S.N + 6)
    nmax = (S.N + 6 + 63) // 64 * 64
    pad = (nmax - S.N - 6) // 3  # fill the rest of the rounded-up capacity with landmarks of the caller's own
    for i in range(pad):
        ctx.add_slam_raw(10 ** 9 + i, np.array([1.0, 2.0, 3.0 + i]), np.array([1.0, 2.0, 3.0 + i]))
    room = nmax - ctx.cov_rows()
    assert 6 <= room < 9
    t = mk(ch)
    with pytest.raises(api.OvpError) as ei:
        ctx.slam_delayed_init_tracks(t)
    assert ei.value.status == 7, ei.value
    made = [f for f in t["featid"] if ctx.slam_handle(f) >= 0]
    assert len(made) == 2 and ctx.cov_rows() == nmax - room + 6
    ctx.close()
