"""tests/plane_track_reference.py pinned without a GPU: the reference's CDT on known point sets, avg_norm on both sides of its thresholds,
hand-built merge / relabel sequences, the k-NN mean against a brute-force float evaluation, and the TrackPlane adapter's syntax."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import plane_track_reference as ref  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPT = dict(max_tri_side_px=200, max_norm_count=5, max_norm_avg_max=25.0, max_norm_avg_var=25.0, max_norm_deg=25.0, max_dist_between_z=0.10,
           max_pairwise_px=100, min_norms=3, check_old_feats=1, filter_num_feat=4, filter_z_thresh=1.2, feat_init_min_obs=4, min_dist=0.10,
           max_dist=60.0, max_cond_number=8000.0)


def test_cdt_known_triangulations():
    # a square with its centre: four triangles around the centre, none without it
    sq = np.array([[0, 0], [10, 0], [10, 10], [0, 10], [5, 5]], dtype=np.float32)
    t = ref.cdt_triangulate(sq)
    assert len(t) == 4 and all(4 in tt for tt in t)
    # a triangle: itself, counter-clockwise
    t = ref.cdt_triangulate(np.array([[0, 0], [10, 0], [0, 10]], dtype=np.float32))
    assert len(t) == 1 and sorted(t[0]) == [0, 1, 2]
    a, b, c = np.array([[0, 0], [10, 0], [0, 10]], dtype=np.float64)[t[0]]
    assert (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0]) > 0
    # collinear points: no triangle
    assert len(ref.cdt_triangulate(np.array([[0, 0], [1, 1], [2, 2], [3, 3]], dtype=np.float32))) == 0


def _unit_deg(deg):
    r = math.radians(deg)
    return np.array([math.sin(r), 0.0, math.cos(r)])


@pytest.mark.parametrize("spread,ok", [(5.0, True), (40.0, False)])
def test_avg_norm_max_deviation(spread, ok):
    norms = [_unit_deg(0.0), _unit_deg(spread), _unit_deg(-spread / 4)]
    out = ref.avg_norm(norms, dict(OPT, max_norm_avg_var=1e9))
    assert (np.linalg.norm(out) > 0) == ok


@pytest.mark.parametrize("thr,ok", [(10.0, True), (3.0, False)])
def test_avg_norm_variance(thr, ok):
    norms = [_unit_deg(0.0), _unit_deg(8.0), _unit_deg(-8.0)]
    out = ref.avg_norm(norms, dict(OPT, max_norm_avg_var=thr, max_norm_avg_max=1e9))
    assert (np.linalg.norm(out) > 0) == ok  # sqrt of the sum of squared deviations / 2 is 8 deg


def test_avg_norm_needs_two_normals():
    assert np.linalg.norm(ref.avg_norm([_unit_deg(3.0)], OPT)) == 0
    assert np.linalg.norm(ref.avg_norm([], OPT)) == 0
    n = ref.avg_norm([_unit_deg(3.0), _unit_deg(3.0)], OPT)  # identical normals: acos(1 + eps) may be NaN, which passes
    assert np.linalg.norm(n) > 0


def test_merge_relabels_non_neighbours_and_keeps_history():
    R = ref.PlaneTrackRef(OPT)
    R.f2p = {1: 3, 2: 3, 3: 5, 4: 5, 9: 5, 7: 8}
    R.p2o = {5: {2}, 8: {6}}
    R.update_plane_ids(3, 5)
    assert R.f2p == {1: 3, 2: 3, 3: 3, 4: 3, 9: 3, 7: 8}
    assert R.p2o == {3: {2, 5}, 8: {6}}
    R.update_plane_ids(3, 8)
    assert set(R.f2p.values()) == {3} and R.p2o == {3: {2, 5, 6, 8}}
    R.update_plane_ids(3, 3)
    assert R.p2o == {3: {2, 5, 6, 8}}


def test_knn_mean_against_brute_force():
    rng = np.random.RandomState(0)
    P = rng.uniform(-3, 3, (30, 3)).astype(np.float32)
    for i in range(len(P)):
        d = []
        for j in range(len(P)):
            if j != i:
                e = (P[i] - P[j]).astype(np.float32)
                d.append(np.float32(np.float32(e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]))
        want = sum(float(v) for v in sorted(d)[:4]) / 4
        assert ref.knn_mean(list(P), i, 4) == want


def test_track_plane_adapter_syntax_check():
    cmd = ["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-Werror", "-I", os.path.join(ROOT, "adapter", "stubs"), "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "adapter", "TrackPlaneB200.cpp")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]


def _merge_setup(f2p, close, check_old_feats=1):
    """features 1..5 on the plane z = 1, each with three normals along z, 10 px apart: every mesh neighbour matches"""
    R = ref.PlaneTrackRef(dict(OPT, check_old_feats=check_old_feats))
    R.events = {"new_plane": 0, "merge": 0, "merge_nonneighbour": 0, "z_removed": 0, "pruned": 0, "removed_feats": 0}
    z = np.array([0.0, 0.0, 1.0])
    for f in range(1, 6):
        R.inG[f] = np.array([0.1 * f, 0.0, 1.0])
        R.norms[f] = [z, z, z]
    R.f2p = dict(f2p)
    pix = {f: np.array([10.0 * f, 0.0], dtype=np.float32) for f in range(1, 6)}
    avg = {f: ref.avg_norm(R.norms[f], R.o) for f in R.norms}
    R.merge_loop(close, pix, avg)
    return R


def test_merge_loop_new_plane_then_done_feature():
    # 1 and 2 unlabelled: 1 opens plane 1 with 2 (not marked done); 2 then matches 1 into plane 1 and is marked done
    R = _merge_setup({}, {1: {2}, 2: {1}})
    assert R.f2p == {1: 1, 2: 1} and R.currplaneid == 1 and R.events["new_plane"] == 1


def test_merge_loop_takes_the_smallest_plane_and_relabels_non_neighbours():
    # 1 (plane 7) matches 2 (plane 4): everything on 7 moves to 4, feature 3 too though it is no neighbour; 2 then skips 1 (done)
    R = _merge_setup({1: 7, 2: 4, 3: 7, 9: 4}, {1: {2}, 2: {1}})
    assert R.f2p == {1: 4, 2: 4, 3: 4, 9: 4} and R.p2o == {4: {7}} and R.currplaneid == 0
    assert R.events["merge_nonneighbour"] == 1


def test_merge_loop_merge_history_follows_the_merged_plane():
    R = ref.PlaneTrackRef(OPT)
    R.p2o = {6: {2, 3}}
    R.f2p = {1: 6, 2: 5}
    R.update_plane_ids(5, 6)
    assert R.p2o == {5: {2, 3, 6}} and R.f2p == {1: 5, 2: 5}


def test_merge_loop_check_old_feats_off_skips_labelled_features():
    # 1 is labelled and skipped as a seed; 2 still matches it and joins its plane
    R = _merge_setup({1: 5}, {1: {2}, 2: {1}}, check_old_feats=0)
    assert R.f2p == {1: 5, 2: 5}
    # without a neighbour that can match, nothing changes
    R = _merge_setup({1: 5}, {1: {2}}, check_old_feats=0)
    assert R.f2p == {1: 5}
