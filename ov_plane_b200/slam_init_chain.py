"""UpdaterSLAM::delayed_init (UpdaterSLAM.cpp:66-374) restated as a chain of the C ABI's stage calls, plus synthetic track scenes for it.

`chain(be, tracks, ...)` runs triangulate_features -> optimize_plane (one single-feature problem per refinement candidate, plane fixed) ->
slam_delayed_init on any object with the C ABI's method names: on an `api.Context` it is the hand-chained counterpart of
`Context.slam_delayed_init_tracks` (same kernels, the tracks uploaded by every stage, the in-state planes read back to seed the refinement); on
the test oracle it is the reference's orchestration over the oracle's own stages.

`tracks_scene(...)` builds raw tracks on a synthetic room (ov_plane_b200.plane_init_chain.tracks_scene) with planes 1-3 in the state and
plane 4 out of it, and the hazards the function has to handle.  Pure numpy.
"""
import numpy as np

from . import plane_init_chain as pic
from . import synth


def chain(be, tracks, sigma_constraint, sigma_pix=1.0, chi2_mult=1.0, use_plane_constraint=True, use_refine_plane_feat=True, tri=None, plane_of=None,
          set_plane_of=None):
    """delayed_init from the stage calls of `be` (sigma_constraint: StateOptions of the state in `be`).  tri = optional (p_FinG, status) of the
    tracks with >= 2 measurements, in input order, used instead of be.triangulate_features.  plane_of(featid): _features_SLAM_to_PLANE entry
    (-1 = none; default be.slam_plane_of).  set_plane_of(featid, planeid) (optional) writes the refinement's side effect on that map; without
    it a feature whose refinement failed is handed to slam_delayed_init without its plane, which initialises it the same way.  Returns the
    outputs of Context.slam_delayed_init_tracks."""
    plane_of = plane_of or be.slam_plane_of
    mo, mc = np.asarray(tracks["meas_offset"]), np.asarray(tracks["meas_clone"])
    uv, uvn = np.asarray(tracks["uv"], dtype=np.float32).reshape(-1, 2), np.asarray(tracks["uv_norm"], dtype=np.float32).reshape(-1, 2)
    fid, pid = np.asarray(tracks["featid"]), np.asarray(tracks["planeid"])
    F = len(mo) - 1
    count = np.diff(mo)
    fs, ps, pout, nh = np.where(count < 2, -1, 0).astype(np.int32), np.full(F, -1, dtype=np.int32), np.zeros((F, 3)), np.full(F, -1, dtype=np.int32)
    trk = [f for f in range(F) if count[f] >= 2]
    if not trk:
        return dict(feat_status=fs, plane_status=ps, p_FinG=pout, new_handles=nh)

    def sub(idx):
        offs = np.concatenate([[0], np.cumsum(count[idx])]).astype(np.int32)
        sel = np.concatenate([np.arange(mo[f], mo[f + 1]) for f in idx]).astype(np.int64)
        return offs, np.ascontiguousarray(mc[sel], dtype=np.int32), np.ascontiguousarray(uvn[sel]), np.ascontiguousarray(uv[sel])

    if tri is None:
        offs, cl, un, _ = sub(trk)
        p_tri, ok = be.triangulate_features(offs, cl, un)
    else:
        p_tri, ok = np.asarray(tri[0]).reshape(-1, 3), np.asarray(tri[1])
    for k, f in enumerate(trk):
        pout[f] = p_tri[k]
    # :147-186 the candidates, decided before the triangulation's verdict is looked at
    cand = [k for k, f in enumerate(trk) if use_plane_constraint and use_refine_plane_feat and pid[f] != 0 and be.plane_handle(int(pid[f])) >= 0
            and plane_of(int(fid[f])) != 0]
    ref_ok = {}
    if cand:
        fx = float(be.var_get(be.handle_intrinsics())[0][0])
        cp = np.array([be.var_get(be.plane_handle(int(pid[trk[k]])))[0][:3] for k in cand])
        omo, omc, oun, _ = sub([trk[k] for k in cand])
        o_st, o_p, _, _, _ = be.optimize_plane(np.arange(len(cand) + 1, dtype=np.int32), omo, omc, oun, p_tri[cand], cp, np.ones(len(cand), dtype=np.int32),
                                               sigma_pix / fx, sigma_constraint)
        for q, k in enumerate(cand):
            f = trk[k]
            ref_ok[f] = bool(o_st[q])
            ps[f] = int(o_st[q])
            pout[f] = o_p[q]
            if set_plane_of and o_st[q]:
                set_plane_of(int(fid[f]), int(pid[f]))
    # :188-201 triangulation failures leave; a failed refinement falls back to the triangulated position, without the plane
    init, plane = [], []
    for k, f in enumerate(trk):
        if not ok[k]:
            fs[f] = -2
            continue
        if not ref_ok.get(f, True):
            pout[f] = p_tri[k]
            if set_plane_of:
                set_plane_of(int(fid[f]), 0)
        init.append((k, f))
        plane.append(int(pid[f]) if use_plane_constraint and ref_ok.get(f, True) else 0)
    if init:
        idx = [f for _, f in init]
        bmo, bmc, _, buv = sub(idx)
        b = dict(F=len(idx), meas_offset=bmo, meas_clone=bmc, uv=buv, p_FinG=np.ascontiguousarray(pout[idx]),
                 p_FinG_original=np.ascontiguousarray(p_tri[[k for k, _ in init]]), featid=np.ascontiguousarray(fid[idx], dtype=np.int64),
                 planeid=np.array(plane, dtype=np.int64))
        r = be.slam_delayed_init(b, sigma_pix, chi2_mult)
        fs[idx] = r["feat_status"]
        nh[idx] = r["new_handles"]
    return dict(feat_status=fs, plane_status=ps, p_FinG=pout, new_handles=nh)


def tracks_scene(seed=0, px_noise=0.1, per_plane=(6, 4, 4, 5), n_free=6, **override):
    """Scenario + raw tracks for SLAM delayed initialisation on the small_planes room, planes 1, 2, 3 in the state, plane 4 not.  The tracks
    handed to the function: per_plane[p - 1] features of plane p and n_free features without a plane.  Hazards: plane 2's points lie 4.5 cm
    off it, plane 3's 2.5 cm (the refinement accepts some of either, depending on the triangulation's depth error; the cameras see the planes
    mostly along their normals, so the rays move onto the plane at little reprojection cost and the chi2 test with the plane passes what the
    refinement accepted; a test that needs a chi2 rejection with the plane tightens the gate, see tests/test_cpu_slam_init_tracks.py); plane 4 carries a one-measurement track and a feature placed 100 m out (a triangulation failure off a refinement candidate), and
    the first plane 1 feature is placed 100 m out too (a triangulation failure on a candidate).  Returns (S, make_tracks, hazards): hazards
    names the input indices of the far features ("far_cand", "far_free"), the single track ("single") and `outlier`, a feature without a plane
    whose last pixel make_tracks(..., outlier=True) moves by 40 px (a plain chi2 rejection)."""
    S0 = synth.make_scenario("small_planes", seed=seed, **override)
    first1 = int(np.nonzero(S0.planeid == 1)[0][0])
    S, mk = pic.tracks_scene(name="small_planes", seed=seed, px_noise=px_noise, keep_in_state=(1, 2, 3), off_plane=((2, 0.045), (3, 0.025)), n_single=1,
                             n_far=1, far_features=(first1,), **override)
    # the in-state planes where they are, and known to 1 mm: the off-plane offsets above are then what the refinement and the plane constraint
    # see, and a plane constraint the feature does not satisfy shows in the chi2 test instead of being absorbed by the plane's uncertainty
    S.planes = [(p, pic.true_plane_cp(p), pic.true_plane_cp(p) + (f - v)) for p, v, f in S.planes]
    assert max(S.ids["plane%d" % p] for p in (1, 2, 3)) < S.ids["plane4"]  # the rows tracks_scene removed come after these
    for p in (1, 2, 3):
        b = S.ids["plane%d" % p]
        S.P0[b:b + 3, :] = 0.0
        S.P0[:, b:b + 3] = 0.0
        S.P0[b:b + 3, b:b + 3] = 1e-6 * np.eye(3)
    pid = S.scene_planeid
    pick = []
    for p, n in enumerate(per_plane, 1):
        pick += list(np.nonzero(pid == p)[0][:n])
    free = list(np.nonzero(pid == 0)[0][:n_free])
    pick = sorted(pick + free)
    t0 = mk(np.zeros(64, dtype=np.int32))
    cnt = np.diff(t0["meas_offset"])
    on4 = [f for f in np.nonzero(pid == 4)[0]]
    hz = dict(far_cand=pick.index(first1), far_free=pick.index(on4[0]), single=pick.index(on4[1]), outlier=pick.index(free[-1]))
    assert cnt[on4[1]] == 1 and cnt[on4[0]] >= 2

    def make_tracks(clone_handles, outlier=True):
        t = mk(clone_handles)
        mo = t["meas_offset"]
        sel = np.concatenate([np.arange(mo[f], mo[f + 1]) for f in pick]).astype(np.int64)
        out = dict(meas_offset=np.concatenate([[0], np.cumsum(np.diff(mo)[pick])]).astype(np.int32),
                   meas_clone=np.ascontiguousarray(t["meas_clone"][sel]), uv=np.array(t["uv"][sel]), uv_norm=np.ascontiguousarray(t["uv_norm"][sel]),
                   featid=np.ascontiguousarray(t["featid"][pick]), planeid=np.ascontiguousarray(t["planeid"][pick]))
        if outlier:
            out["uv"][out["meas_offset"][hz["outlier"] + 1] - 1] += 40.0
        return out
    return S, make_tracks, hz
