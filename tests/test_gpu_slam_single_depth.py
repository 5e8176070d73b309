"""SLAM landmarks in ANCHORED_INVERSE_DEPTH_SINGLE (representation 5; ovp_set_landmark_representations), against the long-double restatement
of tests/single_depth_reference.py and against chains of the library's own tested primitives:
- the setter takes 0..5, refuses -1 and 6 and keeps what it held; {0, 0} through it gives the bits of no options in all three SLAM entry
  points; the old setter keeps refusing 5;
- ovp_slam_delayed_init_tracks in form 5 (an ArUco tag in feat_rep_aruco = 5): rho and the two bearings against set_from_xyz of the
  long-double triangulation's p_FinA; statuses and covariance against the twin chain ovp_triangulate_features ->
  ovp_feature_jacobian_full_rep(4) -> ovp_nullspace_project_inplace(2 columns) -> ovp_initialize(s = 1), each step of which is checked
  against update_reference.initialize of the long-double projection;
- ovp_slam_update of a batch mixing forms 0..5 (anchors inside and outside the track, a tag in form 5, do_fej 0 / 1) against long double:
  statuses, chi2 with 2m - 2 dof, the posterior of slam_update_reference; a form-5 tag just either side of its threshold;
- a form-5 landmark with one measurement: status -1, nothing launched or copied, the rest of a batch bit-identical to the batch without it;
- perform_anchor_change against long double (Phi, covariance, rho and the bearings), and a 12-frame lifecycle whose every update and anchor
  change is held to long double;
- refusals leave the state bit-identical with no launch and no copy; ovp_slam_get_xyz is get_xyz of the stored value for every form."""
import numpy as np
import pytest

import feature_jacobian_reference as fjr
import gate_reference as gr
import single_depth_reference as sd
import slam_reference as sr
import test_gpu_slam_reference as srt
import test_gpu_slam_representations as rt
import triangulation_reference as tr
import update_reference as ur
from conftest import make_pair
from test_cpu_slam_init_tracks import plane_gate
from test_gpu_slam_init_tracks import _state, _tri_of
from ov_plane_b200 import api, synth
from ov_plane_b200 import plane_init_chain as pic
from ov_plane_b200 import slam_init_chain as sic

pytestmark = pytest.mark.gpu

LD = np.longdouble
TAG = 7  # an ArUco tag id (below max_aruco_features)
ARUCO = (0.8, 1.3)


def _subset(t, idx):
    """the tracks idx of the track dict t"""
    mo = t["meas_offset"]
    sel = np.concatenate([np.arange(mo[f], mo[f + 1]) for f in idx]).astype(np.int64)
    return dict(meas_offset=np.concatenate([[0], np.cumsum(np.diff(mo)[idx])]).astype(np.int32), meas_clone=np.ascontiguousarray(t["meas_clone"][sel]),
                uv=np.ascontiguousarray(t["uv"][sel]), uv_norm=np.ascontiguousarray(t["uv_norm"][sel]),
                featid=np.ascontiguousarray(t["featid"][idx]), planeid=np.ascontiguousarray(t["planeid"][idx]))


CAL = {0: (0, 0), 6: (1, 0), 14: (1, 1)}  # calibration columns -> (extrinsics, intrinsics) estimated


def _scene(chi2_table, do_fej=0, tag=True, ncal=14, debug=False):
    """the delayed-init tracks scene (sic.tracks_scene) with ncal calibration columns on a fresh context (debug: on the library with the
    test hooks, for the update's Gram matrix); with tag, its first plane-free track is the ArUco tag TAG"""
    S, mk, _ = sic.tracks_scene(seed=1, calib_pose=CAL[ncal][0], calib_intr=CAL[ncal][1])
    S.options = dict(S.options, do_fej=do_fej)
    if debug:
        ctx = api.Context(S.options, device=0, max_state=max(128, S.N + 64), max_meas_rows=60000, debug=True)
        ctx.set_chi2_table(plane_gate(chi2_table))
        ch = synth.load_scenario_into(ctx, S)
    else:
        ctx, orc, ch, _ = make_pair(S, plane_gate(chi2_table))
        orc.close()
    t = mk(ch)
    t["featid"] = np.array(t["featid"], dtype=np.int64)
    if tag:
        t["featid"][int(np.nonzero(t["planeid"] == 0)[0][0])] = TAG
        ctx.set_aruco_options(*ARUCO)
    return S, t, ctx, ch


def _init_groups(ctx, t, reps, tag_rep=5):
    """delayed-init the tracks of t with at least two measurements, track k in representation reps[k % len(reps)] (the tag in tag_rep), no
    plane constraint; returns {featid: rep} of the landmarks created"""
    cnt = np.diff(t["meas_offset"])
    out = {}
    for i, rep in enumerate(reps):
        idx = [f for f in range(len(cnt)) if cnt[f] >= 2 and f % len(reps) == i]
        if not idx:
            continue
        ctx.set_landmark_representations(rep, tag_rep)
        r = ctx.slam_delayed_init_tracks(_subset(t, idx), 1.0, 1.0, use_plane_constraint=False)
        for k, f in enumerate(idx):
            if r["new_handles"][k] >= 0:
                fid = int(t["featid"][f])
                out[fid] = tag_rep if fid == TAG else rep
    return out


def _thr(table, mult, rows):
    return mult * table[rows if rows < len(table) else len(table) - 1]


def _opts(fid, sigma, mult):
    return ARUCO if int(fid) < 1024 else (sigma, mult)


def _ld_reference(ctx, b, sigma, mult, table, do_fej, calib_pose=True, aruco=ARUCO):
    """statuses, chi2 and the long-double posterior of ovp_slam_update on b: the bearing rows of ovp_feature_jacobian_full at p_FinG, chained
    in long double (representation_jacobians; form 5 as form 4, then its bearing columns projected out), gated and stacked in long double"""
    calib = ctx.var_get(ctx.handle_calib())
    P = ctx.cov()
    sizes = {}
    parts, st, chi = [], [], []
    for f in range(b["F"]):
        fid = int(b["featid"][f])
        track, uv = rt._track(b, f)
        rep, anc = ctx.slam_get_representation(fid)
        hl = ctx.slam_handle(fid)
        v, fe = ctx.var_get(hl)
        if rep >= 2:
            pF = fjr.ld(ctx.slam_get_xyz(fid)) if rep == 5 else fjr.get_xyz(rep, fjr.ld(v[:3]))
            terms = fjr.representation_jacobians(4 if rep == 5 else rep, do_fej, pF, pF, *ctx.var_get(anc), calib[0])
        else:
            pF, pFf = fjr.get_xyz(rep, fjr.ld(v[:3])), fjr.get_xyz(rep, fjr.ld(fe[:3]))
            terms = fjr.representation_jacobians(rep, do_fej, pF, pFf)
        pG = terms[0]
        pGd = np.asarray(pG, dtype=np.float64)
        pGfd = pGd if rep >= 2 else np.asarray(terms[1], dtype=np.float64)
        s, mu = aruco if fid < 1024 else (sigma, mult)
        Hf, Hx, r, xo = ctx.feature_jacobian_full(track, uv, pGd, pGfd, 0, None, None, s, 1.0)
        for h in list(xo) + ([anc] if anc >= 0 else []):
            sizes[h] = ctx.var_size(h)
        if rep >= 2:
            Jf, Hx, xo = sd.chain(Hf, Hx, xo, anc, sizes, terms, calib_pose)
        else:
            Jf, Hx, xo = fjr.ld(Hf) @ terms[2], fjr.ld(Hx), list(xo)
        r = fjr.ld(r)
        if rep == 5:
            Hr, Hx, r = sd.project(Jf, Hx, r)
            J = np.hstack([Hr[:, None], Hx])
        else:
            J = np.hstack([Jf, Hx])
        ids = gr.block_ids(ctx, [hl]) + gr.block_ids(ctx, xo)
        c2 = gr.slam_gate(J, r, fjr.ld(P)[np.ix_(ids, ids)])[0]
        ok = c2 <= _thr(table, mu, len(r))
        st.append(1 if ok else 0)
        chi.append(float(c2))
        if ok:
            parts.append((J, r, ids))
    cols = sorted({int(i) for _, _, ids in parts for i in ids})
    ref = sr.slam_update_reference(fjr.ld(P), cols, sr.stack(parts, cols)) if parts else None
    _ld_reference.parts = parts  # the accepted long-double blocks (J, r, covariance indices) of the last call
    return np.array(st), np.array(chi), ref


_refused = rt._refused


# ---- 1. the setter ---------------------------------------------------------------------------------------------------------------------
def test_setter_takes_0_to_5_and_keeps_what_it_held(chi2_table):
    S, t, ctx, _ = _scene(chi2_table)
    ctx.set_landmark_representations(5)
    for bad in ((-1, 0), (0, -1), (6, 0), (0, 6)):
        with pytest.raises(api.OvpError) as e:
            ctx.set_landmark_representations(*bad)
        assert e.value.status == 1
    with pytest.raises(api.OvpError) as e:
        ctx.set_landmark_options(5, 5)
    assert e.value.status == 1 and "ANCHORED_INVERSE_DEPTH_SINGLE" in str(e.value)
    r = ctx.slam_delayed_init_tracks(t, 1.0, 1.0, use_plane_constraint=False)  # {5, 5} still held
    made = [int(t["featid"][f]) for f in range(len(t["featid"])) if r["new_handles"][f] >= 0]
    assert len(made) >= 10 and all(ctx.slam_get_representation(fid)[0] == 5 for fid in made)
    assert all(ctx.var_size(ctx.slam_handle(fid)) == 1 for fid in made)
    ctx.close()


def test_zero_options_through_the_new_setter_give_equal_bits(chi2_table):
    out = []
    for opts in (None, (0, 0)):
        cs = rt._case(6, 1)
        ctx, chg, b, _ = srt.new_ctx(cs)
        if opts is not None:
            ctx.set_landmark_representations(*opts)
        r = ctx.slam_update(b, 1.0, 1.0, True)
        out.append((r["feat_status"].copy(), r["feat_chi2"].copy(), _state(ctx)))
        ctx.close()
        S = cs.S
        ctx = api.Context(S.options, device=0, max_state=S.N + 3 * S.F + 64, max_meas_rows=60000)
        ctx.set_chi2_table(plane_gate(chi2_table))
        ch = synth.load_scenario_into(ctx, S)
        if opts is not None:
            ctx.set_landmark_representations(*opts)
        r = ctx.slam_delayed_init(synth.feature_batch(S, ch), 1.0, 1.0)
        out.append((r["feat_status"].copy(), r["new_handles"].copy(), _state(ctx)))
        ctx.close()
        S2, mk, _ = sic.tracks_scene(seed=1)
        ctx, orc, ch, _ = make_pair(S2, plane_gate(chi2_table))
        orc.close()
        if opts is not None:
            ctx.set_landmark_representations(*opts)
        r = ctx.slam_delayed_init_tracks(mk(ch), 1.0, 1.0)
        out.append((np.concatenate([r["feat_status"], r["new_handles"]]), r["p_FinG"].copy(), _state(ctx)))
        ctx.close()
    for a, b in zip(out[:3], out[3:]):
        assert rt._bits_equal(a[0], b[0]) and rt._bits_equal(a[1], b[1]) and rt._same_state(a[2], b[2])


# ---- 2. delayed initialisation ---------------------------------------------------------------------------------------------------------
def test_delayed_init_tracks_in_the_single_depth_form(chi2_table):
    ur.require_long_double()
    S, t, ctx, _ = _scene(chi2_table)
    _, t2, twin, _ = _scene(chi2_table)
    ctx.set_landmark_representations(5, 5)
    poses = tr.camera_poses(twin, sorted({int(h) for h in t["meas_clone"]}))
    r = ctx.slam_delayed_init_tracks(t, 1.0, 1.0, use_plane_constraint=False)
    p_tri, tri_ok = _tri_of(twin, t)
    pFs = rt._anchor_positions(twin, t, p_tri, tri_ok, 5)
    table = plane_gate(chi2_table)
    k, n, worst_ld, worst_p = 0, 0, 0.0, 0.0
    for f in range(len(t["featid"])):
        fid = int(t["featid"][f])
        a, e = int(t["meas_offset"][f]), int(t["meas_offset"][f + 1])
        if e - a < 2:
            assert r["feat_status"][f] == -1
            continue
        ok, pF = tri_ok[k], pFs[k]
        k += 1
        if not ok:
            assert r["new_handles"][f] < 0
            continue
        track = [int(h) for h in t["meas_clone"][a:e]]
        s, mu = _opts(fid, 1.0, 1.0)
        # the twin: form-4 Jacobians, the two bearing columns projected out, ovp_initialize with s = 1
        Hf, Hx, res, xo = twin.feature_jacobian_full_rep(track, t["uv"][a:e], 4, track[-1], pF, pF, s)
        Hxp, rp = twin.nullspace_project_inplace(Hf[:, :2], np.hstack([Hf[:, 2:3], Hx]), res)
        P0 = twin.cov()
        ids = gr.block_ids(twin, xo)
        Hr, Hxl, rl = sd.project(fjr.ld(Hf), fjr.ld(Hx), fjr.ld(res))
        ref = ur.initialize(fjr.ld(P0), ids, Hxl, Hr[:, None], rl, LD(1))
        rho = np.array([1.0 / pF[2]])
        acc, nh = twin.initialize(api.OVP_KIND_LANDMARK, rho, rho, fid, xo, Hxp[:, 1:], Hxp[:, :1], rp, 1.0, mu)
        want = float(ref["chi2"]) <= _thr(table, mu, len(rl))
        assert bool(acc) == want, (f, float(ref["chi2"]))
        assert (r["new_handles"][f] >= 0) == bool(acc), f
        if not acc:
            continue
        n += 1
        Pref = ref["upd"]["P"] if ref["upd"] is not None else ref["P_init"]
        worst_ld = max(worst_ld, rt._rel(twin.cov(), np.asarray(Pref, dtype=np.float64)))
        # rho and the bearings against set_from_xyz of the long-double triangulation's p_FinA (anchor: the newest measurement)
        assert ctx.slam_get_representation(fid) == (5, track[-1])
        lref = tr.triangulate([poses[x][0] for x in track], [poses[x][1] for x in track], t["uv_norm"][a:e], tr.DEFAULTS)
        RA, pAc = poses[track[-1]]
        pF_ref = RA @ (lref["p_FinG"] - pAc)
        got_f = ctx.slam_get_xyz(fid, fej=True)  # uv_norm_zero_fej / rho_fej: the first estimate keeps the initial value
        rho_f = ctx.var_get(ctx.slam_handle(fid))[1][0]
        err = float(np.abs(np.asarray(fjr.ld(got_f) - pF_ref, dtype=np.float64)).max())
        bound = lref["p_bound"] + 64 * np.finfo(np.float64).eps * float(np.abs(np.asarray(pF_ref, dtype=np.float64)).max())
        assert err <= bound, (f, err, bound)
        worst_p = max(worst_p, err / bound)
        want_v = sd.set_from_xyz(fjr.ld(got_f))
        assert abs(rho_f - float(want_v[0])) <= 4e-16 * abs(rho_f) and abs(rho_f * got_f[2] - 1.0) < 1e-15
        # the update moved rho, not the bearing: value and first estimate share it
        rho_v = ctx.var_get(ctx.slam_handle(fid))[0][0]
        assert np.allclose(rho_v * ctx.slam_get_xyz(fid), rho_f * got_f, rtol=1e-14, atol=1e-15)
        assert ctx.var_size(ctx.slam_handle(fid)) == 1
    eP, ev = rt._state_rel(_state(ctx), _state(twin))
    print("form 5: %d landmarks; twin vs long double %.2e; fused vs twin P %.2e values %.2e; p_FinA error / bound %.2e" % (n, worst_ld, eP, ev, worst_p))
    assert n >= 10 and worst_ld < 1e-9 and eP < 1e-9 and ev < 1e-9
    assert ctx.slam_get_representation(TAG)[0] == 5
    ctx.close()
    twin.close()


# ---- 3. the update of a mixed batch ----------------------------------------------------------------------------------------------------
def _mixed(chi2_table, do_fej, ncal=14, debug=False):
    S, t, ctx, ch = _scene(chi2_table, do_fej, ncal=ncal, debug=debug)
    reps = _init_groups(ctx, t, (0, 1, 2, 3, 4, 5))
    # anchors: half the anchored landmarks move to the newest clone their track does not see (outside the track), the rest keep the clone of
    # their newest measurement (inside)
    k = 0
    for f in range(len(t["featid"])):
        fid = int(t["featid"][f])
        if reps.get(fid, 0) < 2:
            continue
        track = [int(h) for h in t["meas_clone"][t["meas_offset"][f]:t["meas_offset"][f + 1]]]
        outside = [h for h in ch if h not in track]
        if k % 2 == 0 and outside:
            ctx.slam_perform_anchor_change(fid, int(outside[-1]))
        k += 1
    return S, t, ctx, reps


def _check_get_xyz(ctx, reps, bearings=None):
    """ovp_slam_get_xyz of every landmark against get_xyz of its stored value; for form 5, whose value is [rho] alone, the bearing rho p_FinA
    against the one the landmark was given (bearings: featid -> (value's, first estimate's)).  Returns the bearings it read."""
    out = {}
    for fid, rep in reps.items():
        v, fe = ctx.var_get(ctx.slam_handle(fid))
        got = [ctx.slam_get_xyz(fid, fej) for fej in (False, True)]
        if rep == 5:
            assert len(v) == 1 and len(fe) == 1
            b = (v[0] * got[0], fe[0] * got[1])
            for x in b:
                assert abs(x[2] - 1.0) < 1e-15
            if bearings is not None:
                for x, want in zip(b, bearings[fid]):
                    assert np.abs(x - want).max() <= 1e-15, (fid, x, want)
            out[fid] = b
        else:
            for g, val in zip(got, (v, fe)):
                assert np.allclose(g, np.asarray(fjr.get_xyz(rep, fjr.ld(val[:3])), dtype=np.float64), rtol=1e-15, atol=0)
    return out


@pytest.mark.parametrize("do_fej", [0, 1])
@pytest.mark.parametrize("ncal", [0, 6, 14])
def test_mixed_batch_against_long_double(ncal, do_fej, chi2_table):
    ur.require_long_double()
    S, t, ctx, reps = _mixed(chi2_table, do_fej, ncal, debug=True)
    assert sorted(set(reps.values())) == [0, 1, 2, 3, 4, 5] and reps[TAG] == 5
    # each form-5 bearing as set_from_xyz left it: the same in the value and the first estimate until an anchor change re-anchors them apart
    bearings = _check_get_xyz(ctx, reps)
    for fid, (bv, bf) in bearings.items():
        if ctx.slam_get_representation(fid)[1] in [int(h) for h in rt._track(rt._batch_of(ctx, t, {fid}), 0)[0]]:
            assert np.abs(bv - bf).max() <= 1e-15
    b = rt._batch_of(ctx, t, set(reps))
    table = plane_gate(chi2_table)
    st_ref, chi_ref, ref = _ld_reference(ctx, b, 1.0, 1.0, table, do_fej, bool(S.options["do_calib_camera_pose"]))
    assert ref is not None and st_ref.sum() > 5
    # the a-priori bound of the update's Gram / Cholesky path (slam_reference.slam_bounds, from the library's own Gram matrix of this batch),
    # which the SLAM update tests hold every update to: the landmarks' conditioning (GLOBAL_FULL_INVERSE_DEPTH's above all) sets it
    g = srt.debug_gram(ctx, b, False)
    cols = [int(c) for c in g["cols"]]
    P0 = fjr.ld(ctx.cov())
    X = sr.stack(_ld_reference.parts, cols)
    ref_g = sr.slam_update_reference(P0, cols, X)
    _, dPb, _ = sr.slam_bounds(P0, cols, X, g["G"], ref_g)
    res = ctx.slam_update(b, 1.0, 1.0, False)
    assert np.array_equal(res["feat_status"], st_ref), (res["feat_status"], st_ref)
    assert rt._rel(res["feat_chi2"], chi_ref) < 1e-9
    sd = np.sqrt(np.diag(np.asarray(P0, dtype=np.float64)))
    q = float((np.abs(ctx.cov() - np.asarray(ref_g["P"], dtype=np.float64)) / np.outer(sd, sd) / np.where(dPb > 0, dPb, 1.0)).max())
    eP = rt._rel(ctx.cov(), np.asarray(ref_g["P"], dtype=np.float64))
    print("ncal %d do_fej %d: %d of %d accepted, P+ rel err %.2e, error / a-priori bound %.2e" % (ncal, do_fej, int(st_ref.sum()), b["F"], eP, q))
    assert q <= 1.0
    _check_get_xyz(ctx, reps, bearings)  # the update moves rho only
    ctx.close()


@pytest.mark.parametrize("side", [-1, 1])
@pytest.mark.parametrize("ncal", [0, 6, 14])
def test_single_depth_tag_on_either_side_of_its_threshold(ncal, side, chi2_table):
    S, t, ctx, reps = _mixed(chi2_table, 0, ncal)
    b = rt._batch_of(ctx, t, {TAG})
    table = plane_gate(chi2_table)
    _, chi, _ = _ld_reference(ctx, b, 1.0, 1.0, table, 0, bool(S.options["do_calib_camera_pose"]), aruco=(ARUCO[0], 1.0))
    m = int(b["meas_offset"][1])
    ctx.set_aruco_options(ARUCO[0], chi[0] / _thr(table, 1.0, 2 * m - 2) * (1.0 + side * 1e-9))
    res = ctx.slam_update(b, 1.0, 1.0, False)
    assert abs(res["feat_chi2"][0] - chi[0]) <= 1e-11 * chi[0]
    assert res["feat_status"][0] == (1 if side > 0 else 0)
    assert ctx.slam_should_marg(TAG) == 0
    ctx.close()


# ---- 4. one measurement ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ncal", [0, 6, 14])
def test_one_measurement_landmark_is_not_updated(ncal, chi2_table):
    runs = []
    for with_single in (False, True):
        S, t, ctx, reps = _mixed(chi2_table, 0, ncal)
        b = rt._batch_of(ctx, t, set(reps))
        f5 = next(f for f in range(b["F"]) if reps[int(b["featid"][f])] == 5 and int(b["featid"][f]) != TAG)
        one = _cut(b, [f5], [1])
        if with_single:
            fid5 = int(b["featid"][f5])
            snap, n0, t0 = _state(ctx), ctx.launch_count(), ctx.transfer_bytes()
            r1 = ctx.slam_update(one, 1.0, 1.0, False)
            assert r1["feat_status"][0] == -1 and np.isnan(r1["feat_chi2"][0])
            assert ctx.launch_count() == n0 and ctx.transfer_bytes() == t0 and rt._same_state(snap, _state(ctx))
            assert ctx.slam_should_marg(fid5) == 0 and ctx.slam_plane_of(fid5) == -1
            # the batch with the one-measurement landmark in the middle
            rest = [f for f in range(b["F"]) if f != f5]
            half = len(rest) // 2
            bb = _concat([_cut(b, rest[:half]), one, _cut(b, rest[half:])])
            r = ctx.slam_update(bb, 1.0, 1.0, False)
            assert r["feat_status"][half] == -1 and np.isnan(r["feat_chi2"][half])
            st = np.delete(r["feat_status"], half)
            chi = np.delete(r["feat_chi2"], half)
        else:
            r = ctx.slam_update(_cut(b, [f for f in range(b["F"]) if f != f5]), 1.0, 1.0, False)
            st, chi = r["feat_status"], r["feat_chi2"]
        runs.append((st.copy(), chi.copy(), _state(ctx), [ctx.slam_should_marg(int(x)) for x in b["featid"]]))
        ctx.close()
    (a_st, a_chi, a_s, a_m), (b_st, b_chi, b_s, b_m) = runs
    assert rt._bits_equal(a_st, b_st) and rt._bits_equal(a_chi, b_chi) and rt._same_state(a_s, b_s) and a_m == b_m


def _cut(b, sel, lengths=None):
    """the features sel of the batch b, each with its newest lengths[i] measurements (all: None)"""
    parts = []
    for i, f in enumerate(sel):
        a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
        n = e - a if lengths is None else lengths[i]
        parts.append(dict(F=1, meas_offset=np.array([0, n], dtype=np.int32), meas_clone=np.asarray(b["meas_clone"][e - n:e]),
                          uv=np.asarray(b["uv"][e - n:e]), featid=np.asarray(b["featid"][f:f + 1]), planeid=np.asarray(b["planeid"][f:f + 1])))
    return _concat(parts)


def _concat(bs):
    offs, mc, uv, fid, pid = [0], [], [], [], []
    for b in bs:
        mo = np.asarray(b["meas_offset"])
        offs += list(offs[-1] + mo[1:])
        mc += list(b["meas_clone"])
        uv.append(np.asarray(b["uv"]).reshape(-1, 2))
        fid += list(b["featid"])
        pid += list(b.get("planeid", np.zeros(b["F"], dtype=np.int64)))
    return dict(F=len(fid), meas_offset=np.array(offs, dtype=np.int32), meas_clone=np.array(mc, dtype=np.int32),
                uv=np.ascontiguousarray(np.concatenate(uv), dtype=np.float32), featid=np.array(fid, dtype=np.int64), planeid=np.array(pid, dtype=np.int64))


# ---- 5. anchor change and lifecycle ----------------------------------------------------------------------------------------------------
def _ld_anchor_change(ctx, fid, new, do_fej):
    hl = ctx.slam_handle(fid)
    _, old = ctx.slam_get_representation(fid)
    rho, rho_f = ctx.var_get(hl)[0][0], ctx.var_get(hl)[1][0]
    v = np.concatenate([[rho], rho * ctx.slam_get_xyz(fid)])
    vf = np.concatenate([[rho_f], rho_f * ctx.slam_get_xyz(fid, True)])
    calib_pose = ctx.var_id(ctx.handle_calib()) >= 0
    ref = sd.anchor_change(v, vf, *ctx.var_get(old), *ctx.var_get(new), ctx.var_get(ctx.handle_calib())[0], do_fej, calib_pose)
    order = [old] + ([ctx.handle_calib()] if calib_pose else []) + ([] if new == old else [new]) + [hl]
    P = sd.propagate(ctx.cov(), gr.block_ids(ctx, order), ctx.var_id(hl), ref["Phi"])
    return ref, P


@pytest.mark.parametrize("do_fej", [0, 1])
def test_perform_anchor_change_against_long_double(do_fej, chi2_table):
    ur.require_long_double()
    S, t, ctx, ch = _scene(chi2_table, do_fej)
    reps = _init_groups(ctx, t, (5,))
    n = 0
    for fid in sorted(reps):
        _, old = ctx.slam_get_representation(fid)
        new = int(ch[0]) if old != int(ch[0]) else int(ch[1])
        ref, Pref = _ld_anchor_change(ctx, fid, new, do_fej)
        ctx.slam_perform_anchor_change(fid, new)
        assert ctx.slam_get_representation(fid) == (5, new)
        eP = rt._rel(ctx.cov(), np.asarray(Pref, dtype=np.float64))
        hl = ctx.slam_handle(fid)
        got_v = np.concatenate([[ctx.var_get(hl)[0][0]], ctx.var_get(hl)[0][0] * ctx.slam_get_xyz(fid)])
        got_f = np.concatenate([[ctx.var_get(hl)[1][0]], ctx.var_get(hl)[1][0] * ctx.slam_get_xyz(fid, True)])
        ev = max(rt._rel(got_v, np.asarray(ref["value"], dtype=np.float64)), rt._rel(got_f, np.asarray(ref["fej"], dtype=np.float64)))
        assert eP < 1e-12 and ev < 1e-13, (fid, eP, ev)
        n += 1
    assert n >= 10
    ctx.close()


def test_lifecycle(chi2_table):
    """delayed init from tracks -> update, then FRAMES frames of propagate_and_clone -> change_anchors -> marginalize_old_clone -> update ->
    marginalize_slam, every landmark in form 5: each update against the long-double update of its projected blocks on the context's own
    prior; marginalize_slam removes one covariance column per landmark"""
    S, mk, _ = sic.tracks_scene(seed=1)
    S.options = dict(S.options, max_clone_size=S.cfg["n_clones"] - 1)
    ctx, orc, ch, _ = make_pair(S, plane_gate(chi2_table))
    orc.close()
    t = mk(ch)
    ctx.set_landmark_representations(5, 5)
    t0 = ctx.get_timestamp()
    rt._feed_imu((ctx,), t0, t0 + 0.1 * rt.FRAMES)
    r = ctx.slam_delayed_init_tracks(t, 1.0, 1.0, use_plane_constraint=False)
    fids = {int(t["featid"][f]) for f in range(len(t["featid"])) if r["new_handles"][f] >= 0}
    table = plane_gate(chi2_table)
    worst, moved, log = 0.0, 0, []

    def update(name):
        nonlocal worst
        b = rt._batch_of(ctx, t, fids)
        st, chi, ref = _ld_reference(ctx, b, 1.0, 1.0, table, int(S.options["do_fej"]), bool(S.options["do_calib_camera_pose"]))
        res = ctx.slam_update(b, 1.0, 1.0, False)
        live = res["feat_status"] >= 0
        assert np.array_equal(res["feat_status"][live], st[live])
        if ref is not None:
            e = rt._rel(ctx.cov(), np.asarray(ref["P"], dtype=np.float64))
            worst = max(worst, e)
            log.append("%s %.1e" % (name, e))

    update("update")
    for k in range(rt.FRAMES):
        ctx.propagate_and_clone(t0 + 0.1 * (k + 1))
        moved += ctx.slam_change_anchors()
        ctx.marginalize_old_clone()
        update("f%d" % k)
        n0 = ctx.cov_rows()
        gone = [fid for fid in fids if ctx.slam_should_marg(fid) == 1]
        ctx.marginalize_slam()
        assert ctx.cov_rows() == n0 - len(gone)  # each form-5 landmark is one column
        fids = {f for f in fids if ctx.slam_handle(f) >= 0}
    print("lifecycle form 5: %d landmarks left, %d anchor changes, worst update vs long double %.2e\n  %s" % (len(fids), moved, worst, "; ".join(log)))
    assert moved > 0 and worst < 1e-9
    ctx.close()


# ---- 6. refusals ------------------------------------------------------------------------------------------------------------------------
def test_refusals(chi2_table):
    S, t, ctx, ch = _scene(chi2_table, tag=False)
    reps = _init_groups(ctx, t, (5,), tag_rep=5)
    on_plane = [f for f in range(len(t["featid"])) if int(t["featid"][f]) in reps and 1 <= int(t["planeid"][f]) <= 3]
    assert on_plane
    b = rt._batch_of(ctx, t, {int(t["featid"][on_plane[0]])})
    b["planeid"] = np.array([int(t["planeid"][on_plane[0]])], dtype=np.int64)
    assert "plane" in _refused(ctx, lambda: ctx.slam_update(b, 1.0, 1.0, True), 1)
    fid = int(b["featid"][0])
    _refused(ctx, lambda: ctx.slam_set_representation(fid, 5, int(ch[-1])), 1)
    # a single-depth landmark (size 1) cannot be relabelled into a 3-vector form
    assert "size 1" in _refused(ctx, lambda: ctx.slam_set_representation(fid, 4, int(ch[-1])), 1)
    assert "size 1" in _refused(ctx, lambda: ctx.slam_set_representation(fid, 0, -1), 1)
    # a form-5 landmark joining an MSCKF plane update of a plane that is not in the state (plane 4)
    sel = [i for i in np.nonzero(S.planeid == 4)[0] if int(S.featid[i]) not in reps]
    cnt = np.diff(synth.feature_batch(S, ch, sel)["meas_offset"])
    fb = synth.feature_batch(S, ch, [i for i, n in zip(sel, cnt) if 2 <= n <= 37])
    fb["plane_ids"] = np.array([4], dtype=np.int64)
    fb["plane_cp"] = np.ascontiguousarray([pic.true_plane_cp(4)], dtype=np.float64)
    assert "GLOBAL_3D" in _refused(ctx, lambda: ctx.msckf_update_landmarks(fb, [fid], [4]), 1)
    # a landmark whose size does not match its representation: a size-1 variable that ovp_initialize registered as a (GLOBAL_3D) landmark
    free = next(f for f in range(len(t["featid"])) if int(t["featid"][f]) not in reps and np.diff(t["meas_offset"])[f] >= 2)
    one = _subset(t, [free])
    one["F"] = 1
    track = [int(h) for h in one["meas_clone"]]
    H_R = np.zeros((2 * len(track), ctx.var_size(track[0]) * len(track)))
    H_R[::2, 0] = 1.0
    acc, nh = ctx.initialize(api.OVP_KIND_LANDMARK, np.array([0.5]), np.array([0.5]), int(one["featid"][0]), track, H_R,
                             np.ones((2 * len(track), 1)), np.zeros(2 * len(track)), 1.0, 1e9)
    assert acc and ctx.var_size(nh) == 1 and ctx.slam_get_representation(int(one["featid"][0]))[0] == 0
    assert "size 1" in _refused(ctx, lambda: ctx.slam_update(one, 1.0, 1.0, False), 1)
    ctx.close()
    cs = rt._case(0, 0)
    c2 = api.Context(cs.S.options, device=0, max_state=cs.S.N + 3 * cs.S.F + 64, max_meas_rows=60000)
    c2.set_chi2_table(synth.chi2_table())
    ch2 = synth.load_scenario_into(c2, cs.S)
    c2.set_landmark_representations(0, 5)
    assert "ovp_slam_delayed_init_tracks" in _refused(c2, lambda: c2.slam_delayed_init(synth.feature_batch(cs.S, ch2), 1.0, 1.0), 1)
    c2.close()
