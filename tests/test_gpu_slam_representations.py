"""SLAM landmarks in UpdaterSLAM's other representations (ovp_set_landmark_options): StateOptions::feat_rep_slam / feat_rep_aruco, numbered
0 GLOBAL_3D, 1 GLOBAL_FULL_INVERSE_DEPTH, 2 ANCHORED_3D, 3 ANCHORED_FULL_INVERSE_DEPTH, 4 ANCHORED_MSCKF_INVERSE_DEPTH.
- options {0, 0} give the bits of a context without them in ovp_slam_update, ovp_slam_delayed_init and ovp_slam_delayed_init_tracks;
- the setter refuses 5, 6 and -1 and keeps what it held; clearing the options brings the GLOBAL_3D-only refusals back;
- ovp_slam_update on a batch that mixes the five representations (anchors inside and outside the track, an ArUco tag in its own
  representation, do_fej 0 / 1, 0 / 6 / 14 calibration columns, a correlated covariance) against a long-double reference: the bearing rows
  of ovp_feature_jacobian_full at p_FinG, chained in long double with feature_jacobian_reference.representation_jacobians, gated in long
  double and updated with slam_reference.slam_update_reference; an anchored tag whose chi2 sits just on either side of its threshold;
- the same update against a twin context that chains the library's tested primitives: ovp_feature_jacobian_full_rep per landmark, the gate
  from ovp_get_marginal_covariance, ovp_ekf_update of the accepted stack;
- parametrisation invariance: one landmark as GLOBAL_3D and in each other representation, its covariance mapped through the chain terms,
  gives the same long-double posterior on every other block and the same global position; each computed posterior lies within the
  a-priori bound of the SLAM update path;
- ovp_slam_delayed_init_tracks in each representation: the first estimate against set_from_xyz of the long-double triangulation's p_FinA
  (tests/triangulation_reference.py) within that reference's bound, the covariance against the twin chain ovp_triangulate_features ->
  ovp_feature_jacobian_full_rep -> ovp_initialize;
- the lifecycle over 12 frames: delayed init -> update, then propagate_and_clone -> change_anchors -> marginalize_old_clone -> update ->
  marginalize_slam, against the twin chain, with GLOBAL_3D as the baseline;
- the refusals (plane constraint, ovp_slam_delayed_init, track limits) leave the state bit-identical with no launch and no copy."""
import numpy as np
import pytest

import feature_jacobian_reference as fjr
import gate_reference as gr
import slam_reference as sr
import test_gpu_slam_reference as srt
import triangulation_reference as tr
from conftest import make_pair
from test_cpu_slam_init_tracks import plane_gate
from test_gpu_slam_init_tracks import _state, _tri_of
from ov_plane_b200 import api, synth
from ov_plane_b200 import slam_init_chain as sic

pytestmark = pytest.mark.gpu

LD = np.longdouble
TAG = srt.ARUCO_FEATID  # the scenario's ArUco tag (featid 7 < max_aruco_features)


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _same_state(a, b):
    return a[2] == b[2] and _bits_equal(a[0], b[0]) and all(_bits_equal(x[0], y[0]) and _bits_equal(x[1], y[1]) for x, y in zip(a[1], b[1]))


def _case(ncal, do_fej, use_plane=False, seed=0):
    cs = srt.make_case(ncal, "correlated", ("batch", use_plane), seed)
    cs.S.options = dict(cs.S.options, do_fej=do_fej)
    return cs


def _track(b, f):
    a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
    return [int(h) for h in b["meas_clone"][a:e]], b["uv"][a:e]


def _mixed_plan(b, chg, tag_rep=3):
    """featid -> (rep, anchor): representation f % 5 for landmark f of the batch, anchors alternately inside the track (its middle clone)
    and outside it (the newest clone it does not see); the tag in tag_rep anchored outside its track"""
    plan, k = {}, 0
    for f in range(b["F"]):
        fid = int(b["featid"][f])
        track, _ = _track(b, f)
        rep = tag_rep if fid == TAG else f % 5
        outside = [h for h in chg if h not in track]
        if rep >= 2:
            inside = (k % 2 == 0) and fid != TAG
            anc = track[len(track) // 2] if inside or not outside else outside[-1]
            k += 1
        else:
            anc = -1
        plan[fid] = (rep, anc)
    return plan


def _convert(ctx, plan):
    """re-express every landmark of plan in its representation: value and first estimate through the anchor's value and first estimate"""
    calib = ctx.var_get(ctx.handle_calib())[0]
    for fid, (rep, anc) in plan.items():
        hl = ctx.slam_handle(fid)
        v, fe = ctx.var_get(hl)
        pG, pGf = v[:3].copy(), fe[:3].copy()
        if rep >= 2:
            av, af = ctx.var_get(anc)
            lam, lamf = fjr.to_lambda(rep, fjr.global_to_anchor(av, calib, pG)), fjr.to_lambda(rep, fjr.global_to_anchor(af, calib, pGf))
        else:
            lam, lamf = fjr.to_lambda(rep, pG), fjr.to_lambda(rep, pGf)
        ctx.var_set(hl, np.asarray(lam, dtype=np.float64), np.asarray(lamf, dtype=np.float64))
        ctx.slam_set_representation(fid, rep, anc)


def _positions(ctx, fid, rep):
    """p_F, p_F_fej as ovp_feature_jacobian_full_rep takes them for the landmark of fid"""
    v, fe = ctx.var_get(ctx.slam_handle(fid))
    if rep == 0:
        return v[:3].copy(), fe[:3].copy()
    if rep == 1:
        return fjr.get_xyz(1, v[:3]), fjr.get_xyz(1, fe[:3])
    p = fjr.get_xyz(rep, v[:3])
    return p, p


def _opts(fid, sigma, mult, aruco):
    return aruco if (aruco is not None and int(fid) < 1024) else (sigma, mult)


def _thr(table, mult, rows):
    return mult * table[rows if rows < len(table) else len(table) - 1]


def _fused(cs, plan_of, sigma=1.0, mult=1.0, aruco=None):
    ctx, chg, b, _ = srt.new_ctx(cs)
    plan = plan_of(ctx, chg, b)
    _convert(ctx, plan)
    ctx.set_landmark_options(0, 0)
    if aruco is not None:
        ctx.set_aruco_options(*aruco)
    res = ctx.slam_update(b, sigma, mult, cs.use_plane)
    return ctx, chg, b, plan, res


def _twin_blocks(ctx, b, sigma, mult, aruco, table):
    """per landmark of b, the primitive chain's gate: ovp_feature_jacobian_full_rep, then the chi2 against ovp_get_marginal_covariance.
    Returns (statuses, chi2, the accepted blocks (H, r, handles))"""
    parts, st, chi = [], [], []
    for f in range(b["F"]):
        fid = int(b["featid"][f])
        track, uv = _track(b, f)
        rep, anc = ctx.slam_get_representation(fid)
        pF, pFf = _positions(ctx, fid, rep)
        s, mu = _opts(fid, sigma, mult, aruco)
        Hf, Hx, r, xo = ctx.feature_jacobian_full_rep(track, uv, rep, anc, pF, pFf, s)
        hs = [ctx.slam_handle(fid)] + list(xo)
        H = np.hstack([Hf, Hx])
        Pm = ctx.get_marginal_covariance(hs)
        S = H @ Pm @ H.T + np.eye(len(r))
        c2 = float(r @ np.linalg.solve(S, r))
        ok = c2 <= _thr(table, mu, len(r))
        st.append(1 if ok else 0)
        chi.append(c2)
        if ok:
            parts.append((H, r, hs))
    return np.array(st), np.array(chi), parts


def _ld_posterior(ctx, parts):
    """the long-double EKF update (slam_reference.slam_update_reference, R = I) of the blocks parts on ctx's current covariance"""
    stacked = [(fjr.ld(H), fjr.ld(r), gr.block_ids(ctx, hs)) for H, r, hs in parts]
    cols = sorted({int(i) for _, _, ids in stacked for i in ids})
    return sr.slam_update_reference(fjr.ld(ctx.cov()), cols, sr.stack(stacked, cols))


def _twin_update(ctx, b, sigma, mult, aruco, table):
    """the update chained from the library's primitives; returns (statuses, chi2)"""
    st, chi, parts = _twin_blocks(ctx, b, sigma, mult, aruco, table)
    if parts:
        order = []
        for _, _, hs in parts:
            order += [h for h in hs if h not in order]
        off = np.concatenate([[0], np.cumsum([ctx.var_size(h) for h in order])])
        at = {h: int(off[i]) for i, h in enumerate(order)}
        rows = sum(p[0].shape[0] for p in parts)
        Hb, rb, i = np.zeros((rows, int(off[-1]))), np.zeros(rows), 0
        for H, r, hs in parts:
            c = 0
            for h in hs:
                n = ctx.var_size(h)
                Hb[i:i + len(r), at[h]:at[h] + n] = H[:, c:c + n]
                c += n
            rb[i:i + len(r)] = r
            i += len(r)
        # [H r] = Q R: the update with R's leading rows equals the one with the stack (UpdaterHelper::measurement_compress_inplace)
        k = Hb.shape[1]
        R = np.linalg.qr(np.hstack([Hb, rb[:, None]]), mode="r")[:min(rows, k)]
        ctx.ekf_update(order, R[:, :k], R[:, k])
    return st, chi


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(1e-300, np.abs(np.asarray(b)).max()))


def _state_rel(sa, sb):
    """(max rel error of P, max abs error of the values scaled by their size) between two _state snapshots over the same variables"""
    assert sa[2] == sb[2]
    ev = max(float(np.abs(x[0] - y[0]).max() / max(1.0, np.abs(y[0]).max())) for x, y in zip(sa[1], sb[1]))
    return _rel(sa[0], sb[0]), ev


# ---- 1. options {0, 0} change nothing ---------------------------------------------------------------------------------------------------
def test_noop_options_give_equal_bits(chi2_table):
    out = []
    for opts in (None, (0, 0)):
        cs = _case(6, 1)
        ctx, chg, b, _ = srt.new_ctx(cs)
        if opts is not None:
            ctx.set_landmark_options(*opts)
        r = ctx.slam_update(b, 1.0, 1.0, True)
        out.append((r["feat_status"].copy(), r["feat_chi2"].copy(), _state(ctx), [ctx.slam_should_marg(int(f)) for f in b["featid"]]))
        ctx.close()
        S = cs.S
        ctx = api.Context(S.options, device=0, max_state=S.N + 3 * S.F + 64, max_meas_rows=60000)
        ctx.set_chi2_table(plane_gate(chi2_table))
        ch = synth.load_scenario_into(ctx, S)
        if opts is not None:
            ctx.set_landmark_options(*opts)
        r = ctx.slam_delayed_init(synth.feature_batch(S, ch), 1.0, 1.0)
        out.append((r["feat_status"].copy(), r["new_handles"].copy(), _state(ctx), []))
        ctx.close()
        S2, mk, _ = sic.tracks_scene(seed=1)
        ctx, orc, ch, _ = make_pair(S2, plane_gate(chi2_table))
        orc.close()
        if opts is not None:
            ctx.set_landmark_options(*opts)
        r = ctx.slam_delayed_init_tracks(mk(ch), 1.0, 1.0)
        out.append((np.concatenate([r["feat_status"], r["new_handles"]]), r["p_FinG"].copy(), _state(ctx), []))
        ctx.close()
    for a, b in zip(out[:3], out[3:]):
        assert _bits_equal(a[0], b[0]) and _bits_equal(a[1], b[1]) and _same_state(a[2], b[2]) and a[3] == b[3]


# ---- 2. the setter ---------------------------------------------------------------------------------------------------------------------
def test_setter_refuses_bad_values_and_clearing_restores_the_refusals():
    cs = _case(0, 0)
    ctx, chg, b, _ = srt.new_ctx(cs)
    fid = int(b["featid"][3])
    track, _ = _track(b, 3)
    ctx.set_landmark_options(4, 2)
    for bad in ((5, 0), (0, 5), (6, 0), (-1, 0), (0, -1)):
        with pytest.raises(api.OvpError) as e:
            ctx.set_landmark_options(*bad)
        assert e.value.status == 1
        if 5 in bad:
            assert "ANCHORED_INVERSE_DEPTH_SINGLE" in str(e.value)
    # the options held before are kept: an anchored landmark still updates
    _convert(ctx, {fid: (4, track[-1])})
    one = srt._cut(b, [3])
    ctx.slam_update(one, 1.0, 1.0, False)
    ctx.set_landmark_options(None)
    assert "GLOBAL_3D" in _refused(ctx, lambda: ctx.slam_update(one, 1.0, 1.0, False), 1)
    ctx.close()


# ---- 3. the update against long double --------------------------------------------------------------------------------------------------
def _ld_reference(ctx, b, sigma, mult, aruco, table, do_fej, calib_pose):
    """statuses, chi2 and the long-double posterior of the update, from the bearing rows of ovp_feature_jacobian_full at p_FinG chained in
    long double (representation_jacobians), gated and stacked in long double"""
    calib = ctx.var_get(ctx.handle_calib())
    P = ctx.cov()
    parts, st, chi = [], [], []
    for f in range(b["F"]):
        fid = int(b["featid"][f])
        track, uv = _track(b, f)
        rep, anc = ctx.slam_get_representation(fid)
        v, fe = ctx.var_get(ctx.slam_handle(fid))
        if rep >= 2:
            pF, pFf = fjr.get_xyz(rep, fjr.ld(v[:3])), None
            pG, _, L, Ha, Hc = fjr.representation_jacobians(rep, do_fej, pF, pF, *ctx.var_get(anc), calib[0])
        else:
            pF, pFf = fjr.get_xyz(rep, fjr.ld(v[:3])), fjr.get_xyz(rep, fjr.ld(fe[:3]))
            pG, _, L, Ha, Hc = fjr.representation_jacobians(rep, do_fej, pF, pFf)
        pGd = np.asarray(pG, dtype=np.float64)
        pGfd = pGd if rep >= 2 else np.asarray(pFf, dtype=np.float64)
        s, mu = _opts(fid, sigma, mult, aruco)
        Hf, Hx, r, xo = ctx.feature_jacobian_full(track, uv, pGd, pGfd, 0, None, None, s, 1.0)
        Hf, Hx, r = fjr.ld(Hf), fjr.ld(Hx).copy(), fjr.ld(r)
        xo = list(xo)
        if rep >= 2:
            if anc not in xo:
                xo.append(anc)
                Hx = np.hstack([Hx, np.zeros((Hx.shape[0], 6), dtype=LD)])
            c = sum(ctx.var_size(h) for h in xo[:xo.index(anc)])
            Hx[:, c:c + 6] += Hf @ Ha
            if calib_pose:
                Hx[:, 0:6] += Hf @ Hc
        J = np.hstack([Hf @ L, Hx])
        ids = gr.block_ids(ctx, [ctx.slam_handle(fid)]) + gr.block_ids(ctx, xo)
        Pm = fjr.ld(P)[np.ix_(ids, ids)]
        c2 = gr.slam_gate(J, r, Pm)[0]
        ok = c2 <= _thr(table, mu, len(r))
        st.append(1 if ok else 0)
        chi.append(float(c2))
        if ok:
            parts.append((J, r, ids))
    cols = sorted({int(i) for _, _, ids in parts for i in ids})
    ref = sr.slam_update_reference(fjr.ld(P), cols, sr.stack(parts, cols)) if parts else None
    return np.array(st), np.array(chi), ref, cols



@pytest.mark.parametrize("do_fej", [0, 1])
@pytest.mark.parametrize("ncal", [0, 6, 14])
def test_mixed_batch_against_long_double(ncal, do_fej):
    gr.require_long_double()
    cs = _case(ncal, do_fej)
    table = synth.chi2_table()
    aruco = (0.8, 1.3)
    ctx, chg, b, _ = srt.new_ctx(cs)
    plan = _mixed_plan(b, chg)
    _convert(ctx, plan)
    ctx.set_landmark_options(0, 3)
    ctx.set_aruco_options(*aruco)
    st_ref, chi_ref, ref, cols = _ld_reference(ctx, b, 1.0, 1.0, aruco, table, do_fej, ncal in (6, 14))
    P0 = ctx.cov()
    lm0 = {fid: ctx.var_get(ctx.slam_handle(fid))[0][:3].copy() for fid in plan}
    res = ctx.slam_update(b, 1.0, 1.0, False)
    assert np.array_equal(res["feat_status"], st_ref), (res["feat_status"], st_ref)
    assert _rel(res["feat_chi2"], chi_ref) < 1e-9
    assert ref is not None and st_ref.sum() > 5
    eP = _rel(ctx.cov(), np.asarray(ref["P"], dtype=np.float64))
    dx = np.asarray(ref["dx"], dtype=np.float64)  # over the whole state
    ev = 0.0
    for fid in plan:
        i0 = ctx.var_id(ctx.slam_handle(fid))
        want = lm0[fid] + dx[i0:i0 + 3]
        ev = max(ev, float(np.abs(ctx.var_get(ctx.slam_handle(fid))[0][:3] - want).max() / max(1.0, np.abs(want).max())))
    reps = sorted({r for r, _ in plan.values()})
    print("ncal %d do_fej %d reps %s: %d of %d accepted, P+ rel err %.2e (P- scale %.2e), landmark values %.2e" % (
        ncal, do_fej, reps, int(st_ref.sum()), b["F"], eP, np.abs(P0).max(), ev))
    assert reps == [0, 1, 2, 3, 4]
    assert eP < 1e-9 and ev < 1e-9
    for f in range(b["F"]):
        fid = int(b["featid"][f])
        assert ctx.slam_should_marg(fid) == (1 if res["feat_status"][f] == 0 and fid >= 1024 else 0)
    ctx.close()


@pytest.mark.parametrize("side", [-1, 1])
def test_anchored_tag_on_either_side_of_its_threshold(side):
    """the tag in ANCHORED_MSCKF_INVERSE_DEPTH alone; its ArUco chi2 multiplier puts the threshold 1e-9 above or below its chi2"""
    cs = _case(6, 0)
    ctx, chg, b, _ = srt.new_ctx(cs)
    f = [int(x) for x in b["featid"]].index(TAG)
    one = srt._cut(b, [f])
    track, _ = _track(one, 0)
    _convert(ctx, {TAG: (4, [h for h in chg if h not in track][-1])})
    ctx.set_landmark_options(0, 4)
    ctx.set_aruco_options(1.0, 1.0)
    table = synth.chi2_table()
    chi = _twin_chi2(ctx, one)
    ctx.set_aruco_options(1.0, chi / _thr(table, 1.0, 2 * len(track)) * (1.0 + side * 1e-9))
    res = ctx.slam_update(one, 1.0, 1.0, False)
    assert abs(res["feat_chi2"][0] - chi) <= 1e-12 * chi
    assert res["feat_status"][0] == (1 if side > 0 else 0)
    assert ctx.slam_should_marg(TAG) == 0  # a rejected tag is not flagged
    ctx.close()


def _twin_chi2(ctx, one):
    fid = int(one["featid"][0])
    track, uv = _track(one, 0)
    rep, anc = ctx.slam_get_representation(fid)
    pF, pFf = _positions(ctx, fid, rep)
    Hf, Hx, r, xo = ctx.feature_jacobian_full_rep(track, uv, rep, anc, pF, pFf, 1.0)
    H = np.hstack([Hf, Hx])
    Pm = ctx.get_marginal_covariance([ctx.slam_handle(fid)] + list(xo))
    return float(r @ np.linalg.solve(H @ Pm @ H.T + np.eye(len(r)), r))


# ---- 4. against the library's own primitives --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("do_fej", [0, 1])
@pytest.mark.parametrize("ncal", [0, 6, 14])
def test_mixed_batch_against_the_primitive_chain(ncal, do_fej):
    cs = _case(ncal, do_fej)
    aruco = (0.8, 1.3)
    ctx, chg, b, plan, res = _fused(cs, lambda c, ch, bb: _mixed_plan(bb, ch), aruco=aruco)
    twin, chg2, b2, _ = srt.new_ctx(cs)
    _convert(twin, plan)
    st, chi = _twin_update(twin, b2, 1.0, 1.0, aruco, synth.chi2_table())
    assert np.array_equal(res["feat_status"], st), (res["feat_status"], st)
    eP, ev = _state_rel(_state(ctx), _state(twin))
    ec = _rel(res["feat_chi2"], chi)
    print("ncal %d do_fej %d: %d accepted; fused vs primitive chain: P %.2e values %.2e chi2 %.2e" % (ncal, do_fej, int(st.sum()), eP, ev, ec))
    assert st.sum() > 5 and eP < 1e-9 and ev < 1e-9 and ec < 1e-9
    ctx.close()
    twin.close()


# ---- 5. parametrisation invariance ------------------------------------------------------------------------------------------------------
def _inv3(L):
    """the inverse of a 3 x 3 matrix in long double (adjugate over determinant)"""
    c = np.array([[L[(i + 1) % 3, (j + 1) % 3] * L[(i + 2) % 3, (j + 2) % 3] - L[(i + 1) % 3, (j + 2) % 3] * L[(i + 2) % 3, (j + 1) % 3]
                   for i in range(3)] for j in range(3)], dtype=LD)
    return c / (L[0] @ c[:, 0])


@pytest.mark.parametrize("rep", [1, 2, 3, 4])
def test_parametrisation_invariance(rep):
    """one landmark, its pixels set to its predicted ones (float rounding aside): the correction is ~1e-6 of the state's, so the global
    position agrees to second order in it.  In exact arithmetic the covariance blocks of every other variable agree: the two long-double
    posteriors (of each run's own float64 prior and primitive-chain Jacobian) agree to 1e-12.  Each run's P+ lies within the a-priori
    bound of the Gram / Cholesky path that tests/test_gpu_slam_reference.py holds every SLAM update to (slam_reference.slam_bounds, from
    the run's own Gram matrix); the two computed posteriors then differ by at most the sum of their distances to those long-double
    posteriors.  That sum depends on the parametrisation's conditioning: 5.6e-9 for GLOBAL_FULL_INVERSE_DEPTH, below 1e-10 for the others."""
    cs = _case(6, 0)
    runs = []
    for r in (0, rep):
        ctx, chg, b, _ = srt.new_ctx(cs)
        f = max(range(b["F"]), key=lambda i: (int(b["meas_offset"][i + 1] - b["meas_offset"][i]), -i))
        fid = int(b["featid"][f])
        one = srt._cut(b, [f], [min(12, int(b["meas_offset"][f + 1] - b["meas_offset"][f]))])
        track, uv = _track(one, 0)
        v = ctx.var_get(ctx.slam_handle(fid))[0][:3].copy()
        _, _, res0, _ = ctx.feature_jacobian_full(track, uv, v, v, 0, None, None, 1.0, 1.0)
        one["uv"] = np.ascontiguousarray((uv.astype(np.float64) - res0.reshape(-1, 2)).astype(np.float32))
        anc = [h for h in chg if h not in track][-1]
        hl = ctx.slam_handle(fid)
        i0 = ctx.var_id(hl)
        if r:
            calib = ctx.var_get(ctx.handle_calib())[0]
            av = ctx.var_get(anc)
            pF = fjr.global_to_anchor(fjr.ld(av[0]), fjr.ld(calib), fjr.ld(v)) if r >= 2 else fjr.ld(v)
            if r >= 2:
                pG, _, L, Ha, Hc = fjr.representation_jacobians(r, 0, pF, pF, av[0], av[1], calib)
            else:  # d p / d (theta, phi, rho) in closed form
                th, ph, rho = fjr.to_lambda(1, pF)
                L = np.array([[-np.sin(th) * np.sin(ph), np.cos(th) * np.cos(ph), -np.cos(th) * np.sin(ph) / rho],
                              [np.cos(th) * np.sin(ph), np.sin(th) * np.cos(ph), -np.sin(th) * np.sin(ph) / rho],
                              [0 * th, -np.sin(ph), -np.cos(ph) / rho]], dtype=LD) / rho
            T = np.eye(ctx.cov_rows(), dtype=LD)
            Li = _inv3(fjr.ld(L))
            kappa = float(np.linalg.cond(np.asarray(L, dtype=np.float64)))
            T[i0:i0 + 3, i0:i0 + 3] = Li
            if r >= 2:
                ia, ic = ctx.var_id(anc), ctx.var_id(ctx.handle_calib())
                T[i0:i0 + 3, ia:ia + 6] = -Li @ Ha
                T[i0:i0 + 3, ic:ic + 6] = -Li @ Hc
            P = fjr.ld(ctx.cov())
            ctx.cov_upload(np.asarray(T @ P @ T.T, dtype=np.float64))
            _convert(ctx, {fid: (r, anc if r >= 2 else -1)})
        ctx.set_landmark_options(0, 0)
        _, _, parts = _twin_blocks(ctx, one, 1.0, 1.0, None, synth.chi2_table())
        ref = _ld_posterior(ctx, parts)
        g = srt.debug_gram(ctx, one, False)
        cols = [int(c) for c in g["cols"]]
        P0 = fjr.ld(ctx.cov())
        X = sr.stack([(fjr.ld(H), fjr.ld(rr), gr.block_ids(ctx, hs)) for H, rr, hs in parts], cols)
        ref_g = sr.slam_update_reference(P0, cols, X)
        _, dPb, _ = sr.slam_bounds(P0, cols, X, g["G"], ref_g)
        out = ctx.slam_update(one, 1.0, 1.0, False)
        assert out["feat_status"][0] == 1
        sd = np.sqrt(np.diag(np.asarray(P0, dtype=np.float64)))
        q = float((np.abs(ctx.cov() - np.asarray(ref_g["P"], dtype=np.float64)) / np.outer(sd, sd) / np.where(dPb > 0, dPb, 1.0)).max())
        assert q <= 1.0, "rep %d: P+ error / a-priori bound %.3e" % (r, q)
        lam = ctx.var_get(hl)[0][:3]
        if r >= 2:
            pos = fjr.anchor_to_global(ctx.var_get(anc)[0], ctx.var_get(ctx.handle_calib())[0], fjr.get_xyz(r, lam))
        else:
            pos = fjr.get_xyz(r, lam)
        keep = [i for i in range(ctx.cov_rows()) if not i0 <= i < i0 + 3]
        Pref = np.asarray(ref["P"], dtype=np.float64)
        runs.append((ctx.cov()[np.ix_(keep, keep)], np.asarray(pos, dtype=np.float64), v, _rel(ctx.cov(), Pref), Pref[np.ix_(keep, keep)], q))
        ctx.close()
    (Pa, pa, v0, ea, Ra, qa), (Pb, pb, _, eb, Rb, qb) = runs
    eP, ep, eR = _rel(Pb, Pa), float(np.abs(pb - pa).max() / np.abs(pa).max()), _rel(Rb, Ra)
    print("rep %d vs GLOBAL_3D: other blocks of P+ rel %.2e, global position rel %.2e (moved %.2e); kappa(dpfg_dlambda) %.2e; each update vs "
          "its long-double posterior %.2e / %.2e (error / a-priori bound %.2f / %.2f); the two long-double posteriors' other blocks %.2e" % (
              rep, eP, ep, np.abs(pa - v0).max() / np.abs(v0).max(), kappa, ea, eb, qa, qb, eR))
    assert eR < 1e-12 and ep < 1e-10
    assert eP <= ea + eb + eR + 1e-12  # each P+ within its bound (above): what separates them is each one's own rounding
    if rep != 1:
        assert eP < 1e-10


# ---- 6. delayed initialisation from tracks ----------------------------------------------------------------------------------------------
def _init_scene(chi2_table, rep):
    S, mk, _ = sic.tracks_scene(seed=1)
    ctx, orc, ch, _ = make_pair(S, plane_gate(chi2_table))
    orc.close()
    twin, orc, ch2, _ = make_pair(S, plane_gate(chi2_table))
    orc.close()
    assert list(ch) == list(ch2)
    ctx.set_landmark_options(rep, rep)
    return S, mk(ch), ctx, twin


def _anchor_positions(be, t, p_tri, tri_ok, rep):
    """per triangulated track, the position ovp_feature_jacobian_full_rep takes: p_FinA in the camera of its newest measurement at the poses
    of the triangulation (UpdaterSLAM.cpp:238-243: every initialisation's update rows move the clones afterwards), p_FinG for rep 0 / 1"""
    calib = be.var_get(be.handle_calib())[0]
    out, k = [], 0
    for f in range(len(t["featid"])):
        a, e = int(t["meas_offset"][f]), int(t["meas_offset"][f + 1])
        if e - a < 2:
            continue
        pG = p_tri[k]
        out.append(fjr.global_to_anchor(be.var_get(int(t["meas_clone"][e - 1]))[0], calib, pG) if rep >= 2 and tri_ok[k] else pG)
        k += 1
    return out


def _twin_init(twin, t, p_tri, tri_ok, rep, sigma=1.0, mult=1.0):
    """ovp_triangulate_features -> ovp_feature_jacobian_full_rep -> ovp_initialize, feature by feature in input order"""
    pFs = _anchor_positions(twin, t, p_tri, tri_ok, rep)
    handles, k = [], 0
    for f in range(len(t["featid"])):
        a, e = int(t["meas_offset"][f]), int(t["meas_offset"][f + 1])
        if e - a < 2:
            handles.append(-1)
            continue
        ok, pF = tri_ok[k], pFs[k]
        k += 1
        if not ok:
            handles.append(-1)
            continue
        track = [int(h) for h in t["meas_clone"][a:e]]
        anc = track[-1]
        Hf, Hx, r, xo = twin.feature_jacobian_full_rep(track, t["uv"][a:e], rep, anc, pF, pF, sigma)
        lam = np.asarray(fjr.to_lambda(rep, fjr.ld(pF)), dtype=np.float64)
        acc, nh = twin.initialize(api.OVP_KIND_LANDMARK, lam, lam, int(t["featid"][f]), xo, Hx, Hf, r, 1.0, mult)
        handles.append(nh if acc else -1)
        if acc:
            twin.slam_set_representation(int(t["featid"][f]), rep, anc if rep >= 2 else -1)
    return handles



@pytest.mark.parametrize("rep", [1, 2, 3, 4])
def test_delayed_init_tracks_in_a_representation(rep, chi2_table):
    S, t, ctx, twin = _init_scene(chi2_table, rep)
    poses = tr.camera_poses(twin, sorted({int(h) for h in t["meas_clone"]}))  # before any initialisation moves the clones
    r = ctx.slam_delayed_init_tracks(t, 1.0, 1.0, use_plane_constraint=False)
    p_tri, tri_ok = _tri_of(twin, t)
    handles = _twin_init(twin, t, p_tri, tri_ok, rep)
    n, ev = 0, 0.0
    for f in range(len(t["featid"])):
        fid, h = int(t["featid"][f]), int(r["new_handles"][f])
        assert (h >= 0) == (handles[f] >= 0), (f, h, handles[f])
        if h < 0:
            continue
        n += 1
        a, e = int(t["meas_offset"][f]), int(t["meas_offset"][f + 1])
        got_rep, anc = ctx.slam_get_representation(fid)
        assert got_rep == rep and anc == (int(t["meas_clone"][e - 1]) if rep >= 2 else -1)
        assert twin.slam_get_representation(fid) == (got_rep, anc)
        # the long-double triangulation of the track (anchor: its newest measurement); p_FinA = R_GtoA (p_FinG - p_AinG)
        cl = [int(x) for x in t["meas_clone"][a:e]]
        ref = tr.triangulate([poses[x][0] for x in cl], [poses[x][1] for x in cl], t["uv_norm"][a:e], tr.DEFAULTS)
        assert ref["status"] == 1
        RA, pA = poses[cl[-1]]
        pF_ref = RA @ (ref["p_FinG"] - pA) if rep >= 2 else ref["p_FinG"]
        # the first estimate keeps the initial value (the value moves with the initialisation's update rows): get_xyz of it is the
        # library's p_FinA (p_FinG for rep 1), within the reference's bound plus the rounding of set_from_xyz / get_xyz
        fe = fjr.ld(ctx.var_get(h)[1][:3])
        got = fjr.get_xyz(rep, fe)
        err = float(np.abs(np.asarray(got - pF_ref, dtype=np.float64)).max())
        bound = ref["p_bound"] + 64 * np.finfo(np.float64).eps * float(np.abs(np.asarray(pF_ref, dtype=np.float64)).max())
        assert err <= bound, (f, err, bound)
        ev = max(ev, err / bound)
    eP, evt = _state_rel(_state(ctx), _state(twin))
    print("rep %d: %d landmarks; first estimate vs the long-double p_FinA: worst error / bound %.2e; against the primitive chain P %.2e values %.2e"
          % (rep, n, ev, eP, evt))
    assert n >= 10 and eP < 1e-9 and evt < 1e-9
    ctx.close()
    twin.close()


# ---- 7. lifecycle ---------------------------------------------------------------------------------------------------------------------
def _batch_of(ctx, t, fids):
    """the tracks of the landmarks fids that still have a measurement from a clone in the state, without the measurements of clones that
    have left it"""
    offs, mc, uv, ids = [0], [], [], []
    for f in range(len(t["featid"])):
        if int(t["featid"][f]) not in fids:
            continue
        keep = [k for k in range(int(t["meas_offset"][f]), int(t["meas_offset"][f + 1])) if ctx.var_id(int(t["meas_clone"][k])) >= 0]
        if not keep:
            continue
        mc += [int(t["meas_clone"][k]) for k in keep]
        uv += [t["uv"][k] for k in keep]
        offs.append(len(mc))
        ids.append(int(t["featid"][f]))
    return dict(F=len(ids), meas_offset=np.array(offs, dtype=np.int32), meas_clone=np.array(mc, dtype=np.int32),
                uv=np.ascontiguousarray(np.array(uv).reshape(-1, 2), dtype=np.float32), featid=np.array(ids, dtype=np.int64),
                planeid=np.zeros(len(ids), dtype=np.int64))


def _feed_imu(bes, t0, t1):
    rng = np.random.RandomState(3)
    for be in bes:
        be.propagator_set_noise(1.6968e-04, 1.9393e-05, 2.0e-3, 3.0e-3, 9.81)
    t = t0 - 0.0123
    while t < t1 + 0.01:
        wm = np.array([0.1, -0.05, 0.2]) + 0.01 * rng.randn(3)
        am = np.array([0.2, 9.7, 0.4]) + 0.05 * rng.randn(3)
        for be in bes:
            be.feed_imu(t, wm, am)
        t += 0.0025


FRAMES = 12  # the window is full (max_clone_size = clones - 1): from frame 9 on the oldest clone anchors landmarks and change_anchors moves them


@pytest.mark.parametrize("rep", [0, 4])
def test_lifecycle(rep, chi2_table):
    """delayed init from tracks -> update, then FRAMES frames of propagate_and_clone -> change_anchors -> marginalize_old_clone -> update ->
    marginalize_slam, on the fused entry points and on the twin primitive chain (ovp_feature_jacobian_full_rep + gate + ovp_ekf_update for
    the updates; propagation, anchor change and marginalisation are the same calls on both).  After each step the two states are compared,
    and each update is compared with the long-double EKF update of the primitive chain's blocks on that context's own prior covariance.
    rep 0 (GLOBAL_3D) runs the same sequence as the baseline of what the two update paths' rounding does over the frames."""
    S, mk, _ = sic.tracks_scene(seed=1)
    S.options = dict(S.options, max_clone_size=S.cfg["n_clones"] - 1)
    bes = []
    for _ in range(2):
        c, orc, ch, _ = make_pair(S, plane_gate(chi2_table))
        orc.close()
        bes.append((c, ch))
    (ctx, ch), (twin, _) = bes
    t = mk(ch)
    for be in (ctx, twin):
        be.set_landmark_options(rep, rep)
    t0 = ctx.get_timestamp()
    _feed_imu((ctx, twin), t0, t0 + 0.1 * FRAMES)
    r = ctx.slam_delayed_init_tracks(t, 1.0, 1.0, use_plane_constraint=False)
    p_tri, tri_ok = _tri_of(twin, t)
    _twin_init(twin, t, p_tri, tri_ok, rep)
    fids = {int(t["featid"][f]) for f in range(len(t["featid"])) if r["new_handles"][f] >= 0}
    table = plane_gate(chi2_table)
    log, worst, worst_ld, moved = [], 0.0, 0.0, 0

    def step(name):
        nonlocal worst
        e = max(_state_rel(_state(ctx), _state(twin)))
        worst = max(worst, e)
        log.append("%s %.1e" % (name, e))

    def update(name):
        nonlocal worst_ld
        b = _batch_of(ctx, t, fids)
        refs = []
        for be in (ctx, twin):
            st_be, _, parts = _twin_blocks(be, b, 1.0, 1.0, None, table)
            refs.append((st_be, _ld_posterior(be, parts) if parts else None))
        res = ctx.slam_update(b, 1.0, 1.0, False)
        st, _ = _twin_update(twin, b, 1.0, 1.0, None, table)
        assert np.array_equal(res["feat_status"], st) and np.array_equal(refs[0][0], st)
        for be, (_, ref) in zip((ctx, twin), refs):
            if ref is not None:
                e = _rel(be.cov(), np.asarray(ref["P"], dtype=np.float64))
                worst_ld = max(worst_ld, e)
                log.append("%s %s vs long double %.1e" % (name, "fused" if be is ctx else "twin", e))
        step(name)

    step("init")
    update("update")
    for k in range(FRAMES):
        for be in (ctx, twin):
            be.propagate_and_clone(t0 + 0.1 * (k + 1))
        step("f%d clone" % k)
        n1, n2 = ctx.slam_change_anchors(), twin.slam_change_anchors()
        assert n1 == n2
        moved += n1
        step("f%d anchors(%d)" % (k, n1))
        for be in (ctx, twin):
            be.marginalize_old_clone()
        step("f%d marg" % k)
        update("f%d update" % k)
        for be in (ctx, twin):
            be.marginalize_slam()
        fids = {f for f in fids if ctx.slam_handle(f) >= 0}
        assert fids == {f for f in fids if twin.slam_handle(f) >= 0}
        step("f%d marg_slam" % k)
    print("lifecycle rep %d: %d landmarks left, %d anchor changes; worst fused vs twin %.2e, worst update vs long double %.2e\n  %s" % (
        rep, len(fids), moved, worst, worst_ld, "; ".join(log)))
    assert rep == 0 or moved > 0
    # the two chains are each within worst_ld of the exact update at every step; 4x covers their sum and its carry over the frames
    assert worst < max(1e-9, 4 * worst_ld)
    if rep:
        assert worst < 1e-9
    ctx.close()
    twin.close()


# ---- 8. refusals ------------------------------------------------------------------------------------------------------------------------
def _refused(ctx, call, status):
    snap = _state(ctx)
    n0, t0 = ctx.launch_count(), ctx.transfer_bytes()
    with pytest.raises(api.OvpError) as e:
        call()
    assert e.value.status == status, str(e.value)
    assert ctx.launch_count() == n0 and ctx.transfer_bytes() == t0 and _same_state(snap, _state(ctx))
    return str(e.value)


def test_update_refuses_a_relative_landmark_on_its_plane():
    cs = _case(0, 0, use_plane=True)
    ctx, chg, b, attached = srt.new_ctx(cs)
    f = next(i for i in range(b["F"]) if int(b["featid"][i]) in attached and srt.on_plane(ctx, b, i, True))
    track, _ = _track(b, f)
    _convert(ctx, {int(b["featid"][f]): (2, track[0])})
    ctx.set_landmark_options(0, 0)
    msg = _refused(ctx, lambda: ctx.slam_update(b, 1.0, 1.0, True), 1)
    assert "plane" in msg
    ctx.slam_update(b, 1.0, 1.0, False)  # the same batch without the plane constraint runs
    ctx.close()


def test_delayed_init_refusals(chi2_table):
    S, t, ctx, twin = _init_scene(chi2_table, 2)
    twin.close()
    msg = _refused(ctx, lambda: ctx.slam_delayed_init_tracks(t, 1.0, 1.0, use_plane_constraint=True), 1)
    assert "plane" in msg
    cs = _case(0, 0)
    c2 = api.Context(cs.S.options, device=0, max_state=cs.S.N + 3 * cs.S.F + 64, max_meas_rows=60000)
    c2.set_chi2_table(synth.chi2_table())
    ch = synth.load_scenario_into(c2, cs.S)
    c2.set_landmark_options(0, 3)  # the tag alone takes a relative representation: the whole batch is refused
    msg = _refused(c2, lambda: c2.slam_delayed_init(synth.feature_batch(cs.S, ch), 1.0, 1.0), 1)
    assert "ovp_slam_delayed_init_tracks" in msg
    c2.close()
    ctx.close()


def test_update_track_limit_with_an_anchor_outside_the_track():
    cs = _case(14, 1)
    ctx, chg, b, _ = srt.new_ctx(cs)
    full = synth.feature_batch(cs.S, chg, [i for i in range(cs.S.F) if ctx.slam_handle(int(cs.S.featid[i])) >= 0])
    lens = np.diff(full["meas_offset"])
    f = int(np.argmax(lens))
    assert lens[f] >= 30
    fid = int(full["featid"][f])
    longest = srt._cut(full, [f], [30])
    track, _ = _track(longest, 0)
    _convert(ctx, {fid: (4, track[0])})  # outside the newest 29 measurements, inside the 30
    ctx.set_landmark_options(0, 0)
    _refused(ctx, lambda: ctx.slam_update(longest, 1.0, 1.0, False), 7)
    res = ctx.slam_update(srt._cut(full, [f], [29]), 1.0, 1.0, False)
    assert res["feat_status"][0] in (0, 1)
    ctx.close()
