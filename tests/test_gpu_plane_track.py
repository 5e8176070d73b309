"""The device plane tracker (ovp_plane_track_*) against tests/plane_track_reference.py and the reference's own CDT
(oracle/_ref/libref_cdt.so): the mesh triangle for triangle, then frame sequences of RoomSimulator tracks, refusals and bookkeeping."""
import ctypes as C
import math
import os
import sys
from fractions import Fraction

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import plane_track_reference as ref  # noqa: E402
from ov_plane_b200 import api, jpl, vio_sim  # noqa: E402

pytestmark = pytest.mark.gpu

EUROC = dict(max_tri_side_px=400, max_norm_count=12, max_norm_avg_max=20.0, max_norm_avg_var=15.0, max_norm_deg=10.0, max_dist_between_z=0.05,
             max_pairwise_px=300, min_norms=5, check_old_feats=1, filter_num_feat=8, filter_z_thresh=1.5, feat_init_min_obs=2, min_dist=0.10,
             max_dist=20.0, max_cond_number=20000.0)
RPNG = dict(EUROC, max_tri_side_px=300, max_norm_avg_max=15.0, max_norm_deg=7.0, max_dist_between_z=0.10, max_pairwise_px=200)
CALIB = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])


def make_ctx(debug=True):
    return api.Context(vio_sim.state_options(), device=0, max_state=128, max_meas_rows=512, debug=debug)


def rot_quat(R):
    return jpl.rot_2_quat(R)


# ---- the mesh against CDT -----------------------------------------------------------------------------------------------------------
def mesh_of(uv, seed=0):
    """run two frames whose features all triangulate (two camera positions, points at 3-6 m), with uv as the second frame's pixels"""
    rng = np.random.RandomState(seed)
    n = len(uv)
    P = np.c_[rng.uniform(-2, 2, n), rng.uniform(-2, 2, n), rng.uniform(3, 6, n)]
    ctx = make_ctx(debug=False)
    ctx.plane_track_set_options(dict(api.PLANE_TRACK_DEFAULTS, feat_init_min_obs=2, max_cond_number=1e15, min_dist=0.01, max_dist=1e3))
    fid = np.arange(1, n + 1)
    for px in (0.0, 0.5):
        uvn = ((P[:, :2] - [px, 0.0]) / P[:, 2:3]).astype(np.float32)
        pose = np.r_[0, 0, 0, 1, px, 0, 0]
        ctx.plane_track_frame(pose, CALIB, fid, uv, uvn)
    tri, nrm = ctx.plane_track_mesh()
    ctx.close()
    return tri, nrm


def orient(a, b, c):
    a, b, c = [tuple(Fraction(float(x)) for x in p) for p in (a, b, c)]
    return (a[0] - c[0]) * (b[1] - c[1]) - (a[1] - c[1]) * (b[0] - c[0])


def incircle(a, b, c, d):
    a, b, c, d = [tuple(Fraction(float(x)) for x in p) for p in (a, b, c, d)]
    m = [[p[0] - d[0], p[1] - d[1]] for p in (a, b, c)]
    m = [[x, y, x * x + y * y] for x, y in m]
    return (m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0])
            + m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]))


@pytest.mark.parametrize("n", [3, 4, 200, 2048])
def test_mesh_equals_cdt_random(n):
    rng = np.random.RandomState(n)
    uv = np.c_[rng.uniform(0, 752, n), rng.uniform(0, 480, n)].astype(np.float32)
    tri, _ = mesh_of(uv)
    want = ref.cdt_triangulate(uv)
    assert len(want) > 0
    assert np.array_equal(tri, want)


def test_mesh_equals_cdt_nearly_collinear():
    rng = np.random.RandomState(5)
    x = np.sort(rng.uniform(0, 700, 150))
    uv = np.c_[x, 200 + 0.3 * x + rng.uniform(-0.05, 0.05, 150)].astype(np.float32)
    rng.shuffle(uv)
    tri, _ = mesh_of(uv)
    assert np.array_equal(tri, ref.cdt_triangulate(uv))


def test_mesh_all_collinear_has_no_triangles():
    x = np.arange(1, 40, dtype=np.float32) * 7.0
    uv = np.c_[x, 2 * x].astype(np.float32)
    tri, _ = mesh_of(uv)
    assert len(ref.cdt_triangulate(uv)) == 0 and len(tri) == 0


def test_mesh_lattice_is_delaunay_with_cdt_count():
    """integer lattices put points exactly on edges, where CDT's walk picks one of the two triangles by its own path: the mesh has CDT's
    triangle count and every circumcircle is empty under the exact predicate (DESIGN.md)"""
    g = np.array([(20.0 * i + 5, 20.0 * j + 7) for i in range(8) for j in range(8)], dtype=np.float32)
    rng = np.random.RandomState(1)
    rng.shuffle(g)
    tri, _ = mesh_of(g)
    want = ref.cdt_triangulate(g)
    assert len(tri) == len(want)
    for t in tri:
        a, b, c = g[t[0]], g[t[1]], g[t[2]]
        assert orient(a, b, c) > 0
        for k in range(len(g)):
            if k not in t:
                assert incircle(a, b, c, g[k]) <= 0


# ---- sequences against the restatement ------------------------------------------------------------------------------------------------
def sequence(sim_seed, n_frames, n_feats=200):
    """(pose7, featid, uv, uv_norm) per frame of a RoomSimulator run: noisy float pixels, truth poses perturbed"""
    sim = vio_sim.RoomSimulator(seed=sim_seed, n_feats=n_feats, sigma_px=0.3, plane_frac=0.9)
    rng = np.random.RandomState(100 + sim_seed)
    fx, fy, cx, cy = sim.cam[:4]
    out = []
    for k in range(n_frames):
        t = 0.1 * k
        obs = sim.camera_frame(t)
        R_GtoI, p = sim.pose(t)
        R_GtoI = jpl.exp_so3(rng.normal(0, 2e-3, 3)) @ R_GtoI
        p = p + rng.normal(0, 5e-3, 3)
        fid = np.array(sorted(obs), dtype=np.int64)
        rng.shuffle(fid)  # the tracker's order is not the id order
        uv = np.array([obs[f][0] for f in fid], dtype=np.float32).reshape(-1, 2)
        uvn = np.c_[(uv[:, 0] - cx) / fx, (uv[:, 1] - cy) / fy].astype(np.float32)
        pose = np.r_[rot_quat(R_GtoI), p]
        out.append((pose, fid, uv, uvn))
    calib = np.r_[rot_quat(sim.R_ItoC), sim.p_IinC]
    return out, calib


@pytest.mark.parametrize("name,opts", [("defaults", api.PLANE_TRACK_DEFAULTS), ("euroc_mav", EUROC), ("rpng_plane", RPNG),
                                       ("no_old_feats", dict(api.PLANE_TRACK_DEFAULTS, check_old_feats=0, max_norm_count=1, min_norms=1)),
                                       ("tight", dict(api.PLANE_TRACK_DEFAULTS, filter_num_feat=2, filter_z_thresh=0.8, max_tri_side_px=120,
                                                      max_pairwise_px=60, max_cond_number=300.0, max_dist=6.0))])
def test_sequence_matches_restatement(name, opts):
    frames, calib = sequence(3, 110)
    ctx = make_ctx()
    ctx.plane_track_set_options(opts)
    R = ref.PlaneTrackRef(opts)
    ev = {}
    for k, (pose, fid, uv, uvn) in enumerate(frames):
        ctx.plane_track_frame(pose, calib, fid, uv, uvn)
        tri, nrm = ctx.plane_track_mesh()
        R.frame(pose, calib, fid, uv, uvn)
        assert np.array_equal(tri, R.tri), "frame %d: mesh differs from CDT's" % k
        for e, v in R.events.items():
            ev[e] = ev.get(e, 0) + v
        assert ctx.plane_track_feature2plane() == R.f2p, "frame %d" % k
        assert ctx.plane_track_plane2oldplane() == R.p2o, "frame %d" % k
        np.testing.assert_allclose(nrm, R.tri_norms, rtol=0, atol=1e-9, err_msg="frame %d" % k)
        vid, vuv = ctx.plane_track_vertices()  # what tri3 indexes: the triangulated features, in the frame's order
        assert [int(f) for f in vid] == R.survivors, "frame %d" % k
        assert np.array_equal(vuv, uv[[i for i, f in enumerate(fid) if int(f) in R.inG]])
        if len(tri):
            assert np.array_equal(vid[tri], np.array(R.survivors)[R.tri])
        hist = ctx.plane_track_history(fid)
        for f, h in zip(fid, hist):
            f = int(f)
            assert h["count"] == R.cnt[f] and h["has"] == (f in R.inG)
            np.testing.assert_allclose(h["A"], R.A[f], rtol=1e-12, atol=1e-12)
            if f in R.inG:
                np.testing.assert_allclose(h["p_FinG"], R.inG[f], rtol=1e-9, atol=1e-9)
            w = np.array(R.norms.get(f, [])).reshape(-1, 3)
            assert h["window"].shape == w.shape, "frame %d feature %d" % (k, f)
            np.testing.assert_allclose(h["window"], w, rtol=0, atol=1e-9)
    ctx.close()
    if name in ("defaults", "euroc_mav", "rpng_plane"):  # the sequence reaches every branch of the matching, filter and pruning
        for e in ("new_plane", "merge", "merge_nonneighbour", "z_removed", "pruned", "removed_feats"):
            assert ev[e] > 0, (name, e, ev)


# ---- refusals and bookkeeping ---------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_tracker_untouched():
    frames, calib = sequence(4, 12, n_feats=60)
    runs = []
    for refuse in (False, True):
        ctx = make_ctx()
        with pytest.raises(api.OvpError):
            ctx.plane_track_frame(*frames[0][:1], calib, *frames[0][1:])  # options not set
        ctx.plane_track_set_options(None)
        for k, (pose, fid, uv, uvn) in enumerate(frames):
            if refuse and k == 6:
                with pytest.raises(api.OvpError):  # duplicate featid
                    ctx.plane_track_frame(pose, calib, np.r_[fid, fid[:1]], np.r_[uv, uv[:1] + 1], np.r_[uvn, uvn[:1]])
                for bad in (np.nan, np.inf):
                    with pytest.raises(api.OvpError):  # a non-finite pixel
                        ctx.plane_track_frame(pose, calib, fid, np.r_[uv[:-1], [[bad, 3.0]]], uvn)
                with pytest.raises(api.OvpError):  # two features on one pixel
                    ctx.plane_track_frame(pose, calib, np.r_[fid, [10 ** 9]], np.r_[uv, uv[:1]], np.r_[uvn, uvn[:1]])
                big = api.PLANE_TRACK_MAX_POINTS + 1
                with pytest.raises(api.OvpError):
                    ctx.plane_track_frame(pose, calib, np.arange(big), np.c_[np.arange(big), np.arange(big)], np.zeros((big, 2)))
                with pytest.raises(api.OvpError):  # null pointer
                    ctx._ck(ctx.lib.ovp_plane_track_frame(ctx.h, None, None, 3, None, None, None))
                with pytest.raises(api.OvpError):  # options after the first frame
                    ctx.plane_track_set_options(None)
            ctx.plane_track_frame(pose, calib, fid, uv, uvn)
        runs.append((ctx.plane_track_feature2plane(), ctx.plane_track_plane2oldplane(), ctx.plane_track_mesh(), ctx.plane_track_history(fid)))
        ctx.close()
    a, b = runs
    assert a[0] == b[0] and a[1] == b[1]
    assert np.array_equal(a[2][0], b[2][0]) and np.array_equal(a[2][1], b[2][1])
    for x, y in zip(a[3], b[3]):
        assert np.array_equal(x["A"], y["A"]) and np.array_equal(x["window"], y["window"])


def test_bad_options_keep_the_held_ones():
    ctx = make_ctx()
    ctx.plane_track_set_options(dict(api.PLANE_TRACK_DEFAULTS, max_norm_count=7))
    for bad in (dict(filter_num_feat=1), dict(max_norm_count=0), dict(max_norm_count=api.PLANE_TRACK_MAX_NORM_COUNT + 1),
                dict(filter_num_feat=33), dict(check_old_feats=2), dict(max_norm_deg=float("nan"))):
        with pytest.raises(api.OvpError) as e:
            ctx.plane_track_set_options(dict(api.PLANE_TRACK_DEFAULTS, **bad))
        assert e.value.status == 1
    frames, calib = sequence(5, 8, n_feats=40)
    R = ref.PlaneTrackRef(dict(api.PLANE_TRACK_DEFAULTS, max_norm_count=7))
    for pose, fid, uv, uvn in frames:
        ctx.plane_track_frame(pose, calib, fid, uv, uvn)
        R.frame(pose, calib, fid, uv, uvn)
    for f, h in zip(frames[-1][1], ctx.plane_track_history(frames[-1][1])):
        assert len(h["window"]) == len(R.norms.get(int(f), []))
    ctx.close()


def test_frame_upload_is_one_counted_copy():
    frames, calib = sequence(6, 3, n_feats=50)
    ctx = make_ctx(debug=False)
    ctx.plane_track_set_options(None)
    h2d, d2h = C.c_int64(), C.c_int64()
    prev = None
    for pose, fid, uv, uvn in frames:
        ctx._ck(ctx.lib.ovp_transfer_bytes(ctx.h, C.byref(h2d), C.byref(d2h)))
        b0, d0 = h2d.value, d2h.value
        ctx.plane_track_frame(pose, calib, fid, uv, uvn)
        ctx._ck(ctx.lib.ovp_transfer_bytes(ctx.h, C.byref(h2d), C.byref(d2h)))
        n = len(fid)
        nstale = 0 if prev is None else len(set(prev) - set(int(f) for f in fid))
        top = 0
        for b in (14 * 8, 4 * n, 8 * n, 8 * n, 4 * n, 4 * nstale):
            top = (top + b + 15) & ~15
        assert h2d.value - b0 == top
        assert d2h.value == d0
        prev = [int(f) for f in fid]
    ctx.close()


def test_two_contexts_track_independently():
    fa, calib = sequence(7, 20, n_feats=80)
    fb, _ = sequence(8, 20, n_feats=80)
    both = [make_ctx(debug=False), make_ctx(debug=False)]
    solo = [make_ctx(debug=False), make_ctx(debug=False)]
    for c in both + solo:
        c.plane_track_set_options(EUROC)
    for k in range(20):
        for c, fr in zip(both, (fa, fb)):
            c.plane_track_frame(fr[k][0], calib, *fr[k][1:])
    for c, fr in zip(solo, (fa, fb)):
        for f in fr:
            c.plane_track_frame(f[0], calib, *f[1:])
    for x, y in zip(both, solo):
        assert x.plane_track_feature2plane() == y.plane_track_feature2plane()
        assert x.plane_track_plane2oldplane() == y.plane_track_plane2oldplane()
    for c in both + solo:
        c.close()


# ---- thresholds: each rule on both sides of one of its values, with margin --------------------------------------------------------------
FLOAT_RULES = ["min_dist", "max_dist", "max_cond_number", "max_norm_avg_var", "max_norm_avg_max", "max_norm_deg", "max_dist_between_z",
               "filter_z_thresh"]
INT_OPTION_RULES = ["max_tri_side_px", "max_pairwise_px"]  # integer options compared with float pixel distances
MARGIN = 1e-6  # relative; device and restatement agree to about 1e-12 in every compared value


def _run_both(opts, frames, calib):
    """device and restatement over frames, compared after every frame; returns (per-frame outcome, every traced value per rule, whether
    the run stopped at a decision made by rounding).  Two identical average normals (identical windows) make acos(n . n) NaN or 0 by the
    last bits of the normals, in the reference too: such a frame compares rounding, not the tracker (DESIGN.md 4.6), and ends the run."""
    ctx = make_ctx()
    ctx.plane_track_set_options(opts)
    R = ref.PlaneTrackRef(opts)
    sig, traces = [], {}
    for k, (pose, fid, uv, uvn) in enumerate(frames):
        ctx.plane_track_frame(pose, calib, fid, uv, uvn)
        R.frame(pose, calib, fid, uv, uvn)
        if R.trace.get("unit_dot"):
            ctx.close()
            return sig, traces, True
        tri, nrm = ctx.plane_track_mesh()
        assert np.array_equal(tri, R.tri), k
        np.testing.assert_allclose(nrm, R.tri_norms, rtol=0, atol=1e-9)
        assert ctx.plane_track_feature2plane() == R.f2p, k
        assert ctx.plane_track_plane2oldplane() == R.p2o, k
        hist = ctx.plane_track_history(fid)
        assert [h["has"] for h in hist] == [int(f) in R.inG for f in fid], k
        assert [len(h["window"]) for h in hist] == [len(R.norms.get(int(f), [])) for f in fid], k
        sig.append((sorted(R.inG), sorted(R.f2p.items()), sorted((f, len(w)) for f, w in R.norms.items()), tuple(np.abs(R.tri_norms).sum(1) > 0)))
        for r, v in R.trace.items():
            traces.setdefault(r, []).extend(v)
    ctx.close()
    return sig, traces, False


def _candidates(rule, frames, calib, opts):
    """thresholds either side of one value the rule compares in the first frame it compares anything, largest gaps first"""
    R = ref.PlaneTrackRef(opts)
    for pose, fid, uv, uvn in frames:
        R.frame(pose, calib, fid, uv, uvn)
        vals = sorted(set(v for v in R.trace.get(rule, []) if np.isfinite(v)))
        if rule == "max_dist":  # depths the other end of the range rejects anyway
            vals = [v for v in vals if v > opts["min_dist"]]
        if len(vals) >= 3:
            break
    out = []
    for i in range(1, len(vals) - 1):
        v, a, b = vals[i], vals[i - 1], vals[i + 1]
        if rule in INT_OPTION_RULES:
            lo, hi = math.floor(v), math.ceil(v)
            if lo > a and hi < b and v - lo > MARGIN and hi - v > MARGIN:
                out.append((min(v - lo, hi - v), lo, hi))
        else:
            out.append((min(v - a, b - v) / max(abs(v), 1e-12), 0.5 * (a + v), 0.5 * (v + b)))
    out.sort(reverse=True)
    return [(lo, hi) for _, lo, hi in out]


@pytest.mark.parametrize("rule", FLOAT_RULES + INT_OPTION_RULES)
def test_threshold_both_sides(rule):
    frames, calib = sequence(11, 14)
    base = dict(api.PLANE_TRACK_DEFAULTS, feat_init_min_obs=3, min_norms=2)
    if rule in ("min_dist", "max_dist"):  # the depth rules decide only where the condition number passes
        base["max_cond_number"] = 1e6
    for lo, hi in _candidates(rule, frames, calib, base)[:6]:
        runs = [_run_both(dict(base, **{rule: t}), frames, calib) for t in (lo, hi)]
        if runs[0][2] or runs[1][2]:
            continue
        near = [v for (_, tr, _), t in zip(runs, (lo, hi)) for v in tr.get(rule, []) if np.isfinite(v) and abs(v - t) <= MARGIN * max(1.0, abs(t))]
        if runs[0][0] != runs[1][0] and not near:
            return  # the rule decided differently on the two sides, and no compared value came within the margin
    pytest.fail("no threshold pair of %s changed the outcome with every value outside the margin" % rule)


@pytest.mark.parametrize("rule,lo,hi", [("feat_init_min_obs", 3, 4), ("min_norms", 2, 4), ("max_norm_count", 3, 6), ("check_old_feats", 0, 1),
                                        ("filter_num_feat", 3, 12)])
def test_integer_rule_both_sides(rule, lo, hi):
    frames, calib = sequence(12, 14)
    base = dict(api.PLANE_TRACK_DEFAULTS, feat_init_min_obs=3, min_norms=2)
    a, ta, amb_a = _run_both(dict(base, **{rule: lo}), frames, calib)
    b, tb, amb_b = _run_both(dict(base, **{rule: hi}), frames, calib)
    assert not amb_a and not amb_b
    assert a != b
    if rule == "filter_num_feat":  # planes of more than lo but at most hi features are filtered only on the lo side
        assert any(lo < s <= hi for s in ta["filter_num_feat"])


def test_prune_keeps_planes_of_more_than_three():
    frames, calib = sequence(13, 30)
    _, tr, amb = _run_both(dict(api.PLANE_TRACK_DEFAULTS, feat_init_min_obs=3, min_norms=2), frames, calib)
    assert not amb
    counts = set(tr["prune"])
    assert any(c <= 3 for c in counts) and any(c >= 4 for c in counts), counts
