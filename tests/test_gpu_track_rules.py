"""Every entry point that takes feature tracks refuses malformed ones before it reads them, launches or copies anything: offsets that do not
start at 0 or decrease, null arrays, a handle that is not a clone, a clone observed twice where the mono rule holds, a track outside the
entry point's length bounds.  A refusal leaves the covariance, every value and the variable order bit-identical; ovp_slam_delayed_init
refuses a malformed last track before it initialises the landmarks of the tracks in front of it.  The accepted case at each bound runs
last."""
import ctypes as C

import numpy as np
import pytest

from conftest import make_pair
from ov_plane_b200 import api
from ov_plane_b200 import plane_init_chain as pic
from ov_plane_b200 import slam_init_chain as sic

pytestmark = pytest.mark.gpu

BAD, CAP = 1, 7
# status per case (None: the rule does not apply to the entry point; 0: accepted).  short / at_min: the last track one below / at the
# entry point's shortest track; long: one above its longest, where that bound is checked with the tracks (the MSCKF bound of 39 / 37
# comes after planning: tests/test_gpu_boundaries.py)
CASES = ("start1", "decreasing", "non_clone", "twice", "short", "long", "at_min")
EXPECT = {
    "msckf_update": dict(start1=BAD, decreasing=BAD, non_clone=BAD, twice=BAD, short=BAD, at_min=0),
    "msckf_shard_compress": dict(start1=BAD, decreasing=BAD, non_clone=BAD, twice=BAD, short=BAD, at_min=0),
    "plane_init": dict(start1=BAD, decreasing=BAD, non_clone=BAD, twice=BAD, short=BAD, at_min=0),
    "slam_update": dict(start1=BAD, decreasing=BAD, non_clone=BAD, twice=BAD, short=BAD, long=CAP),
    "slam_delayed_init": dict(start1=BAD, decreasing=BAD, non_clone=BAD, twice=BAD, short=BAD, long=BAD, at_min=0),
    "feature_jacobian_full": dict(non_clone=BAD, twice=BAD, short=BAD, long=BAD, at_min=0),
    "triangulate_features": dict(start1=BAD, decreasing=BAD, non_clone=BAD, twice=0),
    "optimize_plane": dict(start1=BAD, decreasing=BAD, non_clone=BAD, twice=0),
    "plane_init_tracks": dict(start1=BAD, decreasing=BAD, non_clone=BAD, twice=BAD, short=0, long=CAP, at_min=0),
    "slam_delayed_init_tracks": dict(start1=BAD, decreasing=BAD, non_clone=BAD, twice=BAD, short=0, long=CAP, at_min=0),
}
MIN_M = dict(msckf_update=2, msckf_shard_compress=2, plane_init=2, slam_update=1, slam_delayed_init=1, feature_jacobian_full=1, plane_init_tracks=2,
             slam_delayed_init_tracks=2)
MAX_M = dict(slam_update=29, slam_delayed_init=64, feature_jacobian_full=64, plane_init_tracks=37, slam_delayed_init_tracks=64)
PLANE = 99  # plane_init: a plane that is not in the state, carried by every feature of the batch


def _subset(t, keep):
    mo = t["meas_offset"]
    sel = np.concatenate([np.arange(mo[f], mo[f + 1]) for f in keep])
    return dict(meas_offset=np.concatenate([[0], np.cumsum(np.diff(mo)[keep])]).astype(np.int32), meas_clone=t["meas_clone"][sel].copy(),
                uv=t["uv"][sel].copy(), uv_norm=t["uv_norm"][sel].copy(), featid=t["featid"][keep].copy(), planeid=t["planeid"][keep].copy())


def _last_track_length(t, m):
    """t with its last track cut to (or, repeating its measurements, grown to) m measurements"""
    mo = t["meas_offset"]
    a, b = int(mo[-2]), int(mo[-1])
    idx = np.concatenate([np.arange(a), a + np.resize(np.arange(b - a), m)]).astype(int)
    return dict(t, meas_offset=np.concatenate([mo[:-1], [a + m]]).astype(np.int32), meas_clone=t["meas_clone"][idx].copy(),
                uv=t["uv"][idx].copy(), uv_norm=t["uv_norm"][idx].copy())


def _case(t, name, entry, ctx):
    t = {k: np.array(v, copy=True) for k, v in t.items()}
    mo, mc = t["meas_offset"], t["meas_clone"]
    a = int(mo[-2])
    if name == "start1":  # one more measurement in front of the first track, which nothing indexes
        t = dict(t, meas_offset=mo + 1, **{k: np.concatenate([t[k][:1], t[k]]) for k in ("meas_clone", "uv", "uv_norm")})
    elif name == "decreasing":
        mo[-1] = mo[-2] - 1
    elif name == "non_clone":
        mc[a] = ctx.handle_imu()
    elif name == "twice":
        mc[a + 1] = mc[a]
    elif name in ("short", "at_min"):
        t = _last_track_length(t, MIN_M[entry] - (name == "short"))
    elif name == "long":
        t = _last_track_length(t, MAX_M[entry] + 1)
    return t


def _batch(t, p, plane=False):
    F = len(t["meas_offset"]) - 1
    return dict(F=F, meas_offset=t["meas_offset"], meas_clone=t["meas_clone"], uv=t["uv"], p_FinG=p[:F], p_FinG_original=p[:F], featid=t["featid"],
                planeid=np.full(F, PLANE if plane else 0, dtype=np.int64), plane_ids=np.array([PLANE] if plane else [], dtype=np.int64),
                plane_cp=np.array([[0.0, 0.0, 1.0]] if plane else np.zeros((0, 3))))


def _call(entry, ctx, t, p, chg):
    F = len(t["meas_offset"]) - 1
    if entry == "msckf_update":
        return ctx.msckf_update(_batch(t, p))
    if entry == "msckf_shard_compress":
        import torch
        n = ctx.msckf_shard_columns(chg)
        d = torch.zeros((n + 1) ** 2, dtype=torch.float64, device="cuda")
        return ctx.msckf_shard_compress(_batch(t, p), chg, d.data_ptr())
    if entry == "plane_init":
        return ctx.plane_init(_batch(t, p, plane=True))
    if entry == "slam_update":
        return ctx.slam_update(dict(F=F, meas_offset=t["meas_offset"], meas_clone=t["meas_clone"], uv=t["uv"], featid=t["featid"], planeid=t["planeid"]))
    if entry == "slam_delayed_init":
        return ctx.slam_delayed_init(dict(F=F, meas_offset=t["meas_offset"], meas_clone=t["meas_clone"], uv=t["uv"], p_FinG=p[:F], p_FinG_original=p[:F],
                                          featid=t["featid"], planeid=t["planeid"]))
    if entry == "feature_jacobian_full":
        a = int(t["meas_offset"][-2])
        return ctx.feature_jacobian_full(t["meas_clone"][a:], t["uv"][a:], p[F - 1], p[F - 1], 0, None, None, 1.0, 1.0)
    if entry == "triangulate_features":
        return ctx.triangulate_features(t["meas_offset"], t["meas_clone"], t["uv_norm"])
    if entry == "optimize_plane":
        return ctx.optimize_plane(np.array([0, F], dtype=np.int32), t["meas_offset"], t["meas_clone"], t["uv_norm"], p[:F], [[0.0, 0.0, 1.0]], [1],
                                  1e-3, 0.01)
    if entry == "plane_init_tracks":
        return ctx.plane_init_tracks(t)
    return ctx.slam_delayed_init_tracks(t)


def _state(ctx):
    order = ctx.variable_order()
    return ctx.cov(), [ctx.var_get(h) for h in order], order


def _scene(entry, chi2_table):
    """the context and its tracks: the four-measurement-or-longer tracks of a scene whose planes are not in the state (plane_init_tracks) or
    are (every other entry point), and positions for them"""
    if entry == "plane_init_tracks":
        S, mk = pic.tracks_scene(seed=0)
    else:
        S, mk, _ = sic.tracks_scene(seed=0)
    ctx, _, chg, _ = make_pair(S, chi2_table)
    t = mk(chg)
    n = np.diff(t["meas_offset"])
    keep = [f for f in range(len(n)) if n[f] >= 4 and (entry != "plane_init_tracks" or t["planeid"][f] != 0)]
    t = _subset(t, keep)
    p, _ = ctx.triangulate_features(t["meas_offset"], t["meas_clone"], t["uv_norm"])
    return ctx, t, np.ascontiguousarray(p), chg


@pytest.mark.parametrize("entry", sorted(EXPECT))
def test_malformed_tracks_are_refused_before_anything_runs(entry, chi2_table):
    ctx, t, p, chg = _scene(entry, chi2_table)
    s0 = _state(ctx)
    for name in CASES:
        code = EXPECT[entry].get(name)
        if code is None or code == 0:
            continue
        tr = _case(t, name, entry, ctx)
        l0, b0 = ctx.launch_count(), ctx.transfer_bytes()  # reading the state back is a device->host copy itself
        with pytest.raises(api.OvpError) as e:
            _call(entry, ctx, tr, p, chg)
        assert e.value.status == code, (entry, name, str(e.value))
        assert ctx.launch_count() == l0 and ctx.transfer_bytes() == b0, (entry, name)
        P, v, o = _state(ctx)
        assert o == s0[2] and np.array_equal(P, s0[0]), (entry, name)
        assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(v, s0[1])), (entry, name)
        assert all(ctx.slam_handle(int(f)) == -1 for f in t["featid"]), (entry, name)  # no landmark of the tracks exists
    ctx.close()
    for name in CASES:  # the accepted case at each rule's bound, each on a fresh state
        if EXPECT[entry].get(name) == 0:
            ctx, t, p, chg = _scene(entry, chi2_table)
            out = _call(entry, ctx, _case(t, name, entry, ctx), p, chg)
            if name == "short" and entry.endswith("_tracks"):
                assert out["feat_status"][-1] == -1
            ctx.close()


def test_null_batch_arrays_are_refused(chi2_table):
    """the MSCKF batch's arrays, read on the host by the plan before this check existed"""
    ctx, t, p, chg = _scene("msckf_update", chi2_table)
    s0 = _state(ctx)
    l0, b0 = ctx.launch_count(), ctx.transfer_bytes()
    for plane in (False, True):
        for k in ("meas_offset", "meas_clone", "uv", "p_FinG", "planeid"):
            fb, keep = ctx._batch_struct(_batch(t, p, plane))
            setattr(fb, k, None)
            uo = api.UpdaterOptions(1.0, 1.0)
            F = fb.F
            fs, ps, nh = np.zeros(F, dtype=np.int32), np.zeros(1, dtype=np.int32), np.zeros(1, dtype=np.int32)
            if plane:
                st = ctx.lib.ovp_plane_init(ctx.h, C.byref(fb), C.byref(uo), fs.ctypes.data, nh.ctypes.data)
            else:
                st = ctx.lib.ovp_msckf_update(ctx.h, C.byref(fb), C.byref(uo), fs.ctypes.data, None, ps.ctypes.data, None, None, None)
            assert st == BAD, (plane, k, st)
    assert ctx.launch_count() == l0 and ctx.transfer_bytes() == b0
    P, v, o = _state(ctx)
    assert o == s0[2] and np.array_equal(P, s0[0])
    ctx.close()


def test_plane_fitting_refuses_malformed_feat_offset(chi2_table):
    """a decreasing feat_offset is a malformed argument, not a plane of negative size"""
    ctx, t, p, chg = _scene("triangulate_features", chi2_table)
    l0, b0 = ctx.launch_count(), ctx.transfer_bytes()
    F = len(p)
    for fo in ([1, F], [0, F, F - 1], [0, F - 2, F - 3, F]):
        with pytest.raises(api.OvpError) as e:
            ctx.plane_fitting(np.array(fo, dtype=np.int32), p, 3, 200.0)
        assert e.value.status == BAD and "feat_offset" in str(e.value), fo
    assert ctx.launch_count() == l0 and ctx.transfer_bytes() == b0
    ctx.plane_fitting(np.array([0, F // 2, F], dtype=np.int32), p, 3, 200.0)
    ctx.close()
