"""The update's kernel choices at their size boundaries, against the oracle.

The MSCKF update runs a batch on the warp-per-feature kernels when every track has at most 32 measurements and on the
one-block-per-feature kernel otherwise; a point system that fits the innovation workspace and one factorisation launch goes into the
EKF update directly, a larger one through the Gram compression.  The synthetic configs only reach one side of several of these choices,
so the tests here generate scenarios at the edges: tracks of 2, 3, 31, 32 (warp kernels) and 33, 37, 39 (block kernel) measurements,
each with the direct and the compressed form; the longest tracks each kernel holds and the refusal one measurement beyond; SLAM
updates of 1, 2 and 29 measurements per landmark; a process whose first feature update is a SLAM update; a point system just wider
than one factorisation launch holds.  Tolerances are those of test_gpu_parity: gates and Hx_order exact, state and covariance 1e-6,
per-feature chi2 1e-7 (1e-6 after plane updates), the well-defined part of the plane chi2 1e-5."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import make_pair
from ov_plane_b200 import api, synth
from test_gpu_parity import _check_msckf, oracle_msckf_update, relerr

pytestmark = pytest.mark.gpu

OVP_ERR_CAPACITY = 7
MAX_TRACK_POINTS, MAX_TRACK_PLANES, MAX_TRACK_SLAM = 39, 37, 29
# max_state of the sweep: Nmax = 896, so the innovation workspace (Rcap = Nmax + 64 = 960 rows) equals the widest system one
# factorisation launch holds on a 132-SM H100 (15 x 64 columns): point plans up to 960 rows go direct, larger ones are compressed
SWEEP_MAX_STATE = 896
DIRECT_ROWS = 960


def scenario(base, m, F, seed=0, **kw):
    """`base` with every track m measurements long; the clone window turns slowly enough that long tracks stay in view"""
    cfg = synth.CONFIGS[base]
    C = max(cfg["n_clones"], m + 3)
    return synth.make_scenario(base, seed=seed, n_clones=C, m_min=m, m_max=m, dtheta=min(cfg["dtheta"], 0.5 / C), F=F, **kw)


def keep_last(S, lengths):
    """S with feature f cut to its newest lengths[f] measurements (in place)"""
    offs, mc, uv = [0], [], []
    for f in range(S.F):
        a, b = S.meas_offset[f], S.meas_offset[f + 1]
        n = min(int(lengths[f]), b - a)
        mc.append(S.meas_clone_idx[b - n:b])
        uv.append(S.uv[b - n:b])
        offs.append(offs[-1] + n)
    S.meas_offset = np.array(offs, dtype=np.int32)
    S.meas_clone_idx = np.concatenate(mc).astype(np.int32)
    S.uv = np.ascontiguousarray(np.concatenate(uv), dtype=np.float32)
    return S


def tail_batch(b, m):
    """batch dict with every track cut to its newest m measurements"""
    offs, mc, uv = [0], [], []
    for f in range(int(b["F"])):
        a, e = b["meas_offset"][f], b["meas_offset"][f + 1]
        n = min(m, e - a)
        mc.append(b["meas_clone"][e - n:e])
        uv.append(b["uv"][e - n:e])
        offs.append(offs[-1] + n)
    out = dict(b)
    out.update(meas_offset=np.array(offs, dtype=np.int32), meas_clone=np.ascontiguousarray(np.concatenate(mc), dtype=np.int32),
               uv=np.ascontiguousarray(np.concatenate(uv), dtype=np.float32))
    return out


def plane_batches(S, chg, cho, planes):
    bg, bo = synth.feature_batch(S, chg), synth.feature_batch(S, cho)
    if planes is not None:  # planes that are not state variables: the batch carries their estimates
        for b in (bg, bo):
            b["plane_ids"] = np.array([p[0] for p in planes], dtype=np.int64)
            b["plane_cp"] = np.ascontiguousarray([p[1] for p in planes], dtype=np.float64)
    return bg, bo


def point_rows(S):
    return int(sum(2 * (S.meas_offset[f + 1] - S.meas_offset[f]) - 3 for f in range(S.F)))


def state_snapshot(ctx, handles):
    return ctx.cov().copy(), [ctx.var_get(int(h))[0].copy() for h in handles]


def assert_state_unchanged(ctx, handles, snap):
    P0, v0 = snap
    assert np.array_equal(ctx.cov(), P0), "the covariance changed"
    for h, v in zip(handles, v0):
        assert np.array_equal(ctx.var_get(int(h))[0], v), "a state value changed"


def all_handles(ctx, S, chg):
    return [ctx.handle_imu(), ctx.handle_calib(), ctx.handle_intrinsics()] + list(chg) + [ctx.plane_handle(p[0]) for p in S.planes]


# ---- 1. track-length sweep of ovp_msckf_update ---------------------------------------------------------------------------------------
KINDS = {"points": "tiny_points", "planes": "tiny_planes", "planes_out": "tiny_planes"}
SWEEP = [(k, m, form) for k in KINDS for m in (2, 3, 31, 32, 33, 37, 39) for form in ("direct", "compressed")
         if not (k != "points" and m > MAX_TRACK_PLANES)]


@pytest.mark.parametrize("kind,m,form", SWEEP)
def test_msckf_track_length_sweep(kind, m, form, chi2_table):
    per = 2 * m - 3
    # direct: as many features as fit 960 point rows (at most 300: every plane keeps more rows than columns, so its system has a clean
    # rank gap); compressed: a few more
    F = min(DIRECT_ROWS // per, 300) if form == "direct" else DIRECT_ROWS // per + 6
    S = scenario(KINDS[kind], m, F, seed=m)
    planes = synth.drop_planes_from_state(S) if kind == "planes_out" else None
    rows = point_rows(S)
    assert (rows <= DIRECT_ROWS) == (form == "direct")
    ctx, orc, chg, cho = make_pair(S, chi2_table, max_state=SWEEP_MAX_STATE)
    bg, bo = plane_batches(S, chg, cho, planes)
    g = ctx.msckf_update(bg, 1.0, 1.0)
    o = oracle_msckf_update(orc, bo, 1.0, 1.0)
    e = _check_msckf(S, ctx, orc, chg, cho, g, o, chi_tol=1e-7 if kind == "points" else 1e-6)
    print("%s m=%d %s: F=%d point rows %d, cov rel err %.2e, accepted %d, plane status %s" % (kind, m, form, S.F, rows, e,
          int((g["feat_status"] == 1).sum()), g["plane_status"]))
    ctx.close()


@pytest.mark.parametrize("kind", ["points", "planes"])
def test_msckf_mixed_batch_one_long_track(kind, chi2_table):
    """Many 10-measurement tracks and one of 33: the long track moves the whole batch to the one-block-per-feature kernel."""
    S = scenario(KINDS[kind], 33, 40, seed=5)
    lengths = np.full(S.F, 10)
    lengths[17] = 33
    keep_last(S, lengths)
    ctx, orc, chg, cho = make_pair(S, chi2_table, max_state=SWEEP_MAX_STATE)
    bg, bo = plane_batches(S, chg, cho, None)
    g = ctx.msckf_update(bg, 1.0, 1.0)
    o = oracle_msckf_update(orc, bo, 1.0, 1.0)
    e = _check_msckf(S, ctx, orc, chg, cho, g, o, chi_tol=1e-7 if kind == "points" else 1e-6)
    print("mixed %s: point rows %d, cov rel err %.2e" % (kind, point_rows(S), e))
    ctx.close()


@pytest.mark.parametrize("m", [2, MAX_TRACK_PLANES])
def test_plane_init_track_lengths(m, chi2_table):
    import oracle_backend
    S = scenario("tiny_planes", m, 24, seed=20 + m)
    planes = synth.drop_planes_from_state(S)
    ctx, orc, chg, cho = make_pair(S, chi2_table, max_state=SWEEP_MAX_STATE)
    bg, bo = plane_batches(S, chg, cho, planes)
    g = ctx.plane_init(bg, 1.0, 1.0)
    with oracle_backend.GaugeProbe(gate_without=True) as gp:
        o = orc.plane_init(bo, 1.0)
    print("plane_init m=%d: status %s / %s, round-off-row chi2 share %s" % (m, g["plane_status"], o["plane_status"], np.round(gp.junk(), 2)))
    assert np.array_equal(g["plane_status"], o["plane_status"])
    assert ctx.cov_rows() == orc.cov_rows()
    for hg, ho in zip(g["new_handles"], o["new_handles"]):
        assert (hg >= 0) == (ho >= 0)
        if hg >= 0:
            assert ctx.var_id(int(hg)) == orc.var_id(int(ho))
            assert np.allclose(ctx.var_get(int(hg))[0], orc.var_get(int(ho))[0], rtol=1e-6, atol=1e-7)
    e = relerr(ctx.cov(), orc.cov())
    print("cov rel err after plane init %.3e" % e)
    assert e < 1e-6
    ctx.close()


# ---- 2. SLAM update with few and many measurements per landmark ------------------------------------------------------------------------
def _slam_pair(m_track, nslam, chi2_table, seed):
    S = scenario("small_planes", m_track, 60, seed=seed)
    ctx, orc, chg, cho = make_pair(S, chi2_table, max_state=S.N + 3 * nslam + 64)
    sel = np.arange(nslam)
    return S, ctx, orc, chg, cho, synth.feature_batch(S, chg, sel), synth.feature_batch(S, cho, sel)


def _slam_init(ctx, orc, bg, bo):
    g = ctx.slam_delayed_init(bg, 1.0, 1.0)
    o = orc.slam_delayed_init(bo, 1.0, 1.0)
    assert np.array_equal(g["feat_status"], o["feat_status"])
    assert ctx.cov_rows() == orc.cov_rows() and (g["feat_status"] > 0).any()
    assert relerr(ctx.cov(), orc.cov()) < 1e-6
    return g, o


def _slam_update_and_compare(ctx, orc, ug, uo, g_init, o_init, keep):
    g2 = ctx.slam_update(ug, 1.0, 1.0)
    o2 = orc.slam_update(uo, 1.0, 1.0)
    assert np.array_equal(g2["feat_status"], o2["feat_status"])
    assert np.allclose(g2["feat_chi2"], o2["feat_chi2"], rtol=1e-6, atol=1e-8)
    for fid in ug["featid"]:
        assert ctx.slam_should_marg(fid) == orc.slam_should_marg(fid)
    e = relerr(ctx.cov(), orc.cov())
    assert e < 1e-6, e
    for hg, ho in zip(g_init["new_handles"][keep], o_init["new_handles"][keep]):
        vg, vo = ctx.var_get(int(hg))[0], orc.var_get(int(ho))[0]
        assert np.allclose(vg, vo, rtol=1e-6, atol=1e-7)
    assert np.allclose(ctx.var_get(ctx.handle_imu())[0], orc.var_get(orc.handle_imu())[0], rtol=1e-7, atol=1e-9)
    return g2, e


@pytest.mark.parametrize("m", [1, 2, MAX_TRACK_SLAM])
def test_slam_update_track_lengths(m, chi2_table):
    """delayed_init on tracks of max(m, 8), then an update with each landmark's newest m measurements (re-observed with pixel noise)"""
    S, ctx, orc, chg, cho, bg, bo = _slam_pair(max(m, 8), 20, chi2_table, seed=40 + m)
    g, o = _slam_init(ctx, orc, bg, bo)
    keep = np.nonzero(g["feat_status"] > 0)[0]
    ug = tail_batch(synth.feature_batch(S, chg, keep), m)
    uo = tail_batch(synth.feature_batch(S, cho, keep), m)
    noise = np.random.default_rng(m).normal(0.0, 0.5, ug["uv"].shape).astype(np.float32)
    ug["uv"] = ug["uv"] + noise
    uo["uv"] = uo["uv"] + noise
    g2, e = _slam_update_and_compare(ctx, orc, ug, uo, g, o, keep)
    print("slam m=%d: %d landmarks, status %s, cov rel err %.2e" % (m, len(keep), np.bincount(g2["feat_status"], minlength=4), e))
    ctx.close()


# ---- 3. refusals one measurement beyond each limit (and at 65), before anything is launched -----------------------------------------------
@pytest.mark.parametrize("kind,m", [("points", MAX_TRACK_POINTS + 1), ("points", 65), ("planes", MAX_TRACK_PLANES + 1), ("planes", 65)])
def test_msckf_refuses_tracks_beyond_the_limit(kind, m, chi2_table):
    limit = MAX_TRACK_POINTS if kind == "points" else MAX_TRACK_PLANES
    # the seed gives the follow-up's plane systems a clean rank gap (smallest kept singular value >= 4e-6 of the largest): the Gram
    # compression's chi2 error grows like eps / s^2 (test_gpu_parity._check_msckf), and some seeds of these short batches sit near 3e-7
    S = scenario(KINDS[kind], m, 19, seed=64 + m)
    ctx, orc, chg, cho = make_pair(S, chi2_table)
    handles = all_handles(ctx, S, chg)
    snap = state_snapshot(ctx, handles)
    bg = synth.feature_batch(S, chg)
    for call in (lambda: ctx.msckf_prepare(bg, 1.0, 1.0), lambda: ctx.msckf_update(bg, 1.0, 1.0)):
        with pytest.raises(api.OvpError) as err:
            call()
        print(kind, m, "->", err.value)
        assert err.value.status == OVP_ERR_CAPACITY
        assert "%d measurements" % m in str(err.value) and "longest supported track is %d" % limit in str(err.value)
        assert_state_unchanged(ctx, handles, snap)
    # the same context then runs a supported update: the same features cut to the limit
    keep_last(S, np.full(S.F, limit))
    g = ctx.msckf_update(synth.feature_batch(S, chg), 1.0, 1.0)
    o = oracle_msckf_update(orc, synth.feature_batch(S, cho), 1.0, 1.0)
    e = _check_msckf(S, ctx, orc, chg, cho, g, o, chi_tol=1e-7 if kind == "points" else 1e-6)
    print("follow-up update at m=%d: cov rel err %.2e" % (limit, e))
    ctx.close()


@pytest.mark.parametrize("m", [MAX_TRACK_SLAM + 1, 65])
def test_slam_refuses_tracks_beyond_the_limit(m, chi2_table):
    S, ctx, orc, chg, cho, bg, bo = _slam_pair(m, 12, chi2_table, seed=70 + m)
    g, o = _slam_init(ctx, orc, tail_batch(bg, 20), tail_batch(bo, 20))  # delayed_init takes up to 64; the landmarks start from 20
    keep = np.nonzero(g["feat_status"] > 0)[0]
    ug, uo = synth.feature_batch(S, chg, keep), synth.feature_batch(S, cho, keep)
    handles = all_handles(ctx, S, chg) + [int(h) for h in g["new_handles"][keep]]
    snap = state_snapshot(ctx, handles)
    with pytest.raises(api.OvpError) as err:
        ctx.slam_update(ug, 1.0, 1.0)
    print("slam", m, "->", err.value)
    assert err.value.status == OVP_ERR_CAPACITY
    assert "%d measurements" % m in str(err.value) and "longest supported track is %d" % MAX_TRACK_SLAM in str(err.value)
    assert_state_unchanged(ctx, handles, snap)
    _, e = _slam_update_and_compare(ctx, orc, tail_batch(ug, MAX_TRACK_SLAM), tail_batch(uo, MAX_TRACK_SLAM), g, o, keep)
    print("follow-up slam update at m=%d: cov rel err %.2e" % (MAX_TRACK_SLAM, e))
    ctx.close()


# ---- 4. call order: a process whose first feature update is a SLAM update --------------------------------------------------------------
CALL_ORDER_SCRIPT = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests")
from conftest import make_pair
from ov_plane_b200 import synth
from test_gpu_parity import _check_msckf, oracle_msckf_update, relerr
from test_gpu_boundaries import _slam_init, _slam_update_and_compare, point_rows

chi2 = synth.chi2_table()
S = synth.make_scenario("small_planes", seed=2, m_min=14, m_max=14)
ctx, orc, chg, cho = make_pair(S, chi2, max_state=S.N + 3 * 10 + 64)
slam = np.arange(10)
g, o = _slam_init(ctx, orc, synth.feature_batch(S, chg, slam), synth.feature_batch(S, cho, slam))
keep = slam[g["feat_status"] > 0]
_slam_update_and_compare(ctx, orc, synth.feature_batch(S, chg, keep), synth.feature_batch(S, cho, keep), g, o, keep)
print("delayed_init and slam_update match the oracle")
rest = np.arange(10, S.F)
bg, bo = synth.feature_batch(S, chg, rest), synth.feature_batch(S, cho, rest)
rows = int(sum(2 * (bg["meas_offset"][f + 1] - bg["meas_offset"][f]) - 3 for f in range(bg["F"])))
rcap = (S.N + 3 * 10 + 64 + 63) // 64 * 64 + 64
assert rows > rcap, (rows, rcap)  # more rows than the innovation workspace: compressed, on the warp-per-feature kernels
g2 = ctx.msckf_update(bg, 1.0, 1.0)
o2 = oracle_msckf_update(orc, bo, 1.0, 1.0)
e = _check_msckf(S, ctx, orc, chg, cho, g2, o2, chi_tol=1e-6)
print("msckf_update after slam_update matches the oracle: %d point rows, cov rel err %.2e" % (rows, e))
ctx.close()
"""


def test_slam_first_then_msckf_in_a_fresh_process():
    """The >48 KB shared-memory opt-in is process-wide per kernel: only a process whose first feature update is a SLAM update shows
    whether the warp-per-feature kernel is opted in by then."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", CALL_ORDER_SCRIPT, root], cwd=root, capture_output=True, text=True, timeout=900)
    print(r.stdout)
    print(r.stderr[-4000:])
    assert r.returncode == 0


# ---- 5. a point system just wider than one factorisation launch holds ------------------------------------------------------------------
@pytest.mark.parametrize("F", [25, 27, 29])  # 925 point rows (direct), 999 and 1073 (wider than 960: compressed)
def test_direct_form_respects_factorisation_width(F, chi2_table):
    S = synth.make_scenario("cfg3_n512_f600_p8", seed=1, F=F)
    rows = point_rows(S)
    assert rows == 37 * F
    ctx, orc, chg, cho = make_pair(S, chi2_table, max_state=1024, max_meas_rows=8192)  # Rcap = 1088 >= rows
    g = ctx.msckf_update(synth.feature_batch(S, chg), 1.0, 1.0)
    o = oracle_msckf_update(orc, synth.feature_batch(S, cho), 1.0, 1.0)
    e = _check_msckf(S, ctx, orc, chg, cho, g, o, chi_tol=1e-6)
    print("cfg3 max_state 1024, %d point rows: cov rel err %.2e, plane status %s" % (rows, e, g["plane_status"]))
    ctx.close()
