"""ArUco tags in UpdaterSLAM (ovp_set_aruco_options): a feature with featid < max_aruco_features is whitened and gated with the updater's
options_aruco instead of the call's options (UpdaterSLAM.cpp:164, 257, 302-304, 500, 545-547).
- ArUco options equal to the call's give the bits of a context without them, in ovp_slam_update, ovp_slam_delayed_init and
  ovp_slam_delayed_init_tracks (the last against the same tracks with the tags renumbered, since without options it refuses tags);
- ovp_slam_update with distinct ArUco sigma_pix and chi2_multipler on a correlated covariance against the long-double references of
  tests/test_gpu_slam_reference.py, over blocks whitened per feature with its own sigma; one tag on its plane and one on a wrong plane have a
  chi2 between the SLAM and the ArUco thresholds (plane try, retry), a tag rejected by its own multiplier is not flagged;
- ovp_slam_delayed_init and ovp_slam_delayed_init_tracks against the oracle's stages with each feature's own options, in the reference's
  order (every refinement first, then the initialisations one feature at a time); a tag's refinement equals ovp_optimize_plane at
  sigma_aruco / fx;
- the setter's refusals, and a cleared context that behaves as one that never set the options."""
import numpy as np
import pytest

import gate_reference as gr
import oracle_slam_init as osi
import slam_reference as sr
import test_gpu_slam_reference as srt
import update_reference as ur
from conftest import make_pair
from test_cpu_slam_init_tracks import plane_gate
from test_gpu_slam_init_tracks import _state, _tri_of
from ov_plane_b200 import api, synth
from ov_plane_b200 import slam_init_chain as sic

pytestmark = pytest.mark.gpu

TAG0 = 100  # tag ids: TAG0, TAG0 + 1, ... (below max_aruco_features = 1024; 7 is test_gpu_slam_reference's own tag)


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _same_state(a, b):
    return a[2] == b[2] and _bits_equal(a[0], b[0]) and all(_bits_equal(x[0], y[0]) and _bits_equal(x[1], y[1]) for x, y in zip(a[1], b[1]))


def _tag_update_case(seed=0, ncal=0):
    """test_gpu_slam_reference's 24-landmark batch with tags: the first six landmarks on a plane (the first three of those are the batch's
    wrong-plane landmarks) and two without one, besides its own featid 7"""
    cs = srt.make_case(ncal, "correlated", ("batch", True), seed)
    on = [int(i) for i in np.nonzero(cs.S.planeid != 0)[0] if i != 1]
    off = [int(i) for i in np.nonzero(cs.S.planeid == 0)[0] if i != 1]
    for k, i in enumerate(on[:6] + off[:2]):
        cs.S.featid[i] = TAG0 + k
    return cs


def _is_tag(fid):
    return int(fid) < 1024


# ---- equal options, equal bits ---------------------------------------------------------------------------------------------------------
def _update_run(cs, aruco, sigma, mult):
    ctx, chg, b, _ = srt.new_ctx(cs)
    assert any(_is_tag(f) for f in b["featid"])
    if aruco is not None:
        ctx.set_aruco_options(*aruco)
    res = ctx.slam_update(b, sigma, mult, True)
    out = (res["feat_status"].copy(), res["feat_chi2"].copy(), _state(ctx), [(ctx.slam_should_marg(int(f)), ctx.slam_plane_of(int(f))) for f in b["featid"]])
    ctx.close()
    return out


def _init_run(cs, aruco, sigma, mult, table):
    S = cs.S
    ctx = api.Context(S.options, device=0, max_state=S.N + 3 * S.F + 64, max_meas_rows=60000)
    ctx.set_chi2_table(table)
    chg = synth.load_scenario_into(ctx, S)
    if aruco is not None:
        ctx.set_aruco_options(*aruco)
    r = ctx.slam_delayed_init(synth.feature_batch(S, chg), sigma, mult)
    out = (r["feat_status"].copy(), r["new_handles"].copy(), _state(ctx), [ctx.slam_plane_of(int(f)) for f in S.featid])
    ctx.close()
    return out


@pytest.mark.parametrize("sigma,mult", [(1.0, 1.0), (1.7, 0.6)])
def test_equal_options_give_equal_bits_update_and_delayed_init(sigma, mult, chi2_table):
    cs = _tag_update_case()
    a, b = _update_run(cs, None, sigma, mult), _update_run(cs, (sigma, mult), sigma, mult)
    assert _bits_equal(a[0], b[0]) and _bits_equal(a[1], b[1]), (a[0], b[0])
    assert _same_state(a[2], b[2]) and a[3] == b[3]
    assert np.count_nonzero(a[0]) > 0
    a, b = _init_run(cs, None, sigma, mult, plane_gate(chi2_table)), _init_run(cs, (sigma, mult), sigma, mult, plane_gate(chi2_table))
    assert _bits_equal(a[0], b[0]) and _bits_equal(a[1], b[1]), (a[0], b[0])
    assert _same_state(a[2], b[2]) and a[3] == b[3]
    print("sigma %g mult %g: delayed_init statuses %s" % (sigma, mult, np.bincount(b[0], minlength=4).tolist()))


def _tag_tracks(t, every=2):
    """t with every `every`-th feature renumbered to a tag id"""
    v = {k: np.array(x, copy=True) for k, x in t.items()}
    idx = np.arange(0, len(v["featid"]), every)
    v["featid"][idx] = TAG0 + np.arange(len(idx))
    return v


@pytest.mark.parametrize("sigma,mult", [(1.0, 1.0), (1.7, 0.6)])
def test_equal_options_give_equal_bits_delayed_init_tracks(sigma, mult, chi2_table):
    S, mk, hz = sic.tracks_scene(seed=1)
    out = []
    for tagged in (False, True):
        ctx, orc, ch, _ = make_pair(S, plane_gate(chi2_table))
        orc.close()
        t = mk(ch)
        if tagged:
            t = _tag_tracks(t)
            ctx.set_aruco_options(sigma, mult)
        r = ctx.slam_delayed_init_tracks(t, sigma, mult)
        out.append((r, _state(ctx), [ctx.slam_plane_of(int(f)) for f in t["featid"]]))
        ctx.close()
    (ra, sa, pa), (rb, sb, pb) = out
    for k in ("feat_status", "plane_status", "p_FinG", "new_handles"):
        assert _bits_equal(ra[k], rb[k]), (k, ra[k], rb[k])
    assert _same_state(sa, sb) and pa == pb
    assert (ra["plane_status"] == 1).any() and (ra["feat_status"] >= 1).sum() > 10


# ---- the update against long double ---------------------------------------------------------------------------------------------------
SIGMA_A = 0.25  # a power of two: the whitened rows are the raw rows times 4, exactly


def _thr(table, dof):
    return table[dof if dof < len(table) else len(table) - 1]


def _blocks(ctx, cs, b, raw):
    """per landmark: (ids, H = [H_f | H_x] with sigma_pix 1, r, on its plane, m)"""
    cal = gr.calib_ids(ctx, cs.S.options)
    out = []
    for f in range(b["F"]):
        a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
        hp = srt.on_plane(ctx, b, f, True)
        Hf, Hx, r = gr.raw_block(raw, a, e, len(cal), hp)
        ids = gr.block_ids(ctx, [ctx.slam_handle(int(b["featid"][f]))]) + cal + gr.block_ids(ctx, b["meas_clone"][a:e], 6)
        if hp:
            ids += gr.block_ids(ctx, [ctx.plane_handle(int(b["planeid"][f]))])
        out.append((ids, np.hstack([Hf, Hx]), r, hp, e - a))
    return out


def _whiten(J, r, m, sigma):
    J, r = J.copy(), r.copy()
    w = gr.LD(1) / gr.LD(sigma)
    J[:2 * m] *= w
    r[:2 * m] *= w
    return J, r


def _gates(P, blocks, sig):
    """per landmark (chi2, bound, dof) of the try with its plane (or its only try) and of the retry without it (None off a plane)"""
    out = []
    for f, (ids, J, r, hp, m) in enumerate(blocks):
        Jw, rw = _whiten(J, r, m, sig[f])
        first = gr.slam_gate(Jw, rw, P[np.ix_(ids, ids)])
        retry = gr.slam_gate(Jw[:2 * m, :len(ids) - 3], rw[:2 * m], P[np.ix_(ids[:-3], ids[:-3])]) if hp else None
        out.append((first, retry))
    return out


def _statuses(gates, blocks, mults, table):
    st = []
    for (first, retry), (ids, J, r, hp, m), mu in zip(gates, blocks, mults):
        if first[0] <= mu * _thr(table, first[2]):
            st.append(1)
        elif hp and retry[0] <= mu * _thr(table, retry[2]):
            st.append(3)
        else:
            st.append(0)
    return np.array(st, dtype=np.int32)


def _pick_multipliers(gates, blocks, tags, moved, table):
    """(SLAM multiplier, ArUco multiplier, tag A, tag B): tag A is on its plane and its first chi2 lies between the two thresholds; tag B is on
    a wrong plane, rejected on it under both multipliers, and its retry's chi2 lies between them.  The band is a factor 1.5 from either chi2."""
    ratio = lambda g: float(g[0]) / _thr(table, g[2])  # noqa: E731
    A = [f for f in tags if blocks[f][3] and f not in moved]
    B = [f for f in tags if blocks[f][3] and f in moved]
    best = None
    for a in A:
        for b in B:
            ra, rb, rbp = ratio(gates[a][0]), ratio(gates[b][1]), ratio(gates[b][0])
            lo, hi = min(ra, rb) / 1.5, max(ra, rb) * 1.5
            if rbp > 1.5 * hi and (best is None or hi / lo < best[0]):
                best = (hi / lo, lo, hi, a, b)
    if best is None:
        print("no tag pair with a chi2 band: A %s, B %s" % ([ratio(gates[f][0]) for f in A], [(ratio(gates[f][1]), ratio(gates[f][0])) for f in B]))
        return None
    _, lo, hi, a, b = best
    # ArUco the lenient side, so that the two tags are accepted (1 and 3) where the SLAM multiplier would reject them
    return lo, hi, a, b


def test_slam_update_with_aruco_options_against_long_double():
    ur.require_long_double()
    table = synth.chi2_table()
    for seed in range(srt.SEEDS):
        cs = _tag_update_case(seed)
        ctx0, chg, b, attached = srt.new_ctx(cs)
        P = ctx0.cov().copy()
        g0 = srt.debug_gram(ctx0, b, True)  # the raw rows at sigma_pix 1
        blocks = _blocks(ctx0, cs, b, g0["raw"])
        kinds = srt.kinds_of(ctx0, cs, chg, b)
        ids = {h: ctx0.var_id(h) for h in kinds}
        ctx0.close()
        tags = [f for f in range(b["F"]) if _is_tag(b["featid"][f])]
        moved = [f for f in range(b["F"]) if int(b["planeid"][f]) != 0 and int(b["planeid"][f]) != int(cs.S.planeid[list(cs.S.featid).index(b["featid"][f])])]
        sig = [SIGMA_A if f in tags else 1.0 for f in range(b["F"])]
        gates = _gates(P, blocks, sig)
        pick = _pick_multipliers(gates, blocks, tags, moved, table)
        if pick is None:
            continue
        m_slam, m_aruco, ta, tb = pick
        mults = [m_aruco if f in tags else m_slam for f in range(b["F"])]
        st = _statuses(gates, blocks, mults, table)
        assert st[ta] == 1 and st[tb] == 3, (st[ta], st[tb])
        slam_only = _statuses(gates, blocks, [m_slam] * b["F"], table)
        assert slam_only[ta] != 1 and slam_only[tb] == 0
        # the stack the reference forms, each landmark's rows whitened with its own sigma
        parts = []
        for f, (fid, J, r, hp, m) in enumerate(blocks):
            Jw, rw = _whiten(J, r, m, sig[f])
            out = sr.landmark_rows(Jw[:, :3], Jw[:, 3:], rw, int(st[f]), hp, m)
            if out is not None:
                parts.append((out[0], out[1], fid[:out[0].shape[1]]))
        # the library's Gram matrix and gates with the options
        ctx1, _, b1, _ = srt.new_ctx(cs)
        ctx1.set_aruco_options(SIGMA_A, m_aruco)
        g1 = srt.debug_gram(ctx1, b1, True, 1.0, m_slam)
        ctx1.close()
        tag = "seed %d: SLAM multiplier %.4g, ArUco %.4g (sigma %g), tags A %d B %d, statuses %s" % (seed, m_slam, m_aruco, SIGMA_A, ta, tb,
                                                                                                  np.bincount(st, minlength=4).tolist())
        assert np.array_equal(g1["status"], st), "%s: device %s" % (tag, g1["status"])
        for f, ((first, retry), blk) in enumerate(zip(gates, blocks)):
            g = retry if (blk[3] and st[f] != 1) else first
            assert abs(float(g1["chi2"][f]) - float(g[0])) <= g[1], (tag, f, g1["chi2"][f], g[0], g[1])
        cols = [int(s) for s in g1["cols"]]
        X = sr.stack(parts, cols)
        G = g1["G"]
        low = np.tril(np.ones_like(G, dtype=bool))
        eG = np.abs(np.asarray(G - sr.gram_ld(X), dtype=np.float64))[low]
        assert np.all(eG <= sr.gram_bound(X)[low]), "%s: G error above the Gram bound" % tag
        tol = srt.pick_tolerance(G, len(cols))
        if tol is None:
            print("%s: no tolerance leaves every pivot 100x clear; next scenario" % tag)
            continue
        ref = sr.slam_update_reference(P, cols, X)
        assert ref is not None
        ctx2, chg2, b2, _ = srt.new_ctx(cs)
        ctx2.set_aruco_options(SIGMA_A, m_aruco)
        ctx2.set_rank_tolerance(tol)
        s0 = srt.snapshot(ctx2, kinds, list(cs.S.featid))
        res = ctx2.slam_update(b2, 1.0, m_slam, True)
        assert np.array_equal(res["feat_status"], st), (tag, res["feat_status"])
        got = srt.snapshot(ctx2, kinds, list(cs.S.featid))
        dxb, dPb, _ = sr.slam_bounds(P, cols, X, G, ref, tol)
        qP, qv = ur.check_update(got[0], got[1], got[2], P, kinds, ids, s0[1], s0[2], ref["dx"], dxb, dPb, ref["P"])
        for f in range(b2["F"]):
            fid = int(b2["featid"][f])
            assert ctx2.slam_should_marg(fid) == (1 if st[f] == 0 and not _is_tag(fid) else 0), (tag, f, fid)
        print("%s: tol %g, worst error / bound P+ %.3e values %.3e" % (tag, tol, qP, qv))
        ctx2.close()
        return
    pytest.fail("no scenario with a rank decision clear of rounding")


def test_tag_rejected_by_its_own_multiplier_is_not_flagged():
    """an ArUco multiplier of 1e-12 rejects every tag (UpdaterSLAM.cpp:600-605, 613-618: warned about, not flagged); the other landmarks get
    the statuses of a context without ArUco options"""
    cs = _tag_update_case()
    plain = _update_run(cs, None, 1.0, 1.0)
    ctx, chg, b, _ = srt.new_ctx(cs)
    ctx.set_aruco_options(1.0, 1e-12)
    res = ctx.slam_update(b, 1.0, 1.0, True)
    tags = np.array([_is_tag(f) for f in b["featid"]])
    assert np.all(res["feat_status"][tags] == 0) and np.array_equal(res["feat_status"][~tags], plain[0][~tags])
    assert (plain[0][tags] != 0).any()  # some of them pass the SLAM multiplier
    for f, fid in enumerate(b["featid"]):
        assert ctx.slam_should_marg(int(fid)) == (0 if tags[f] else int(res["feat_status"][f] == 0)), (f, fid)
    ctx.close()


# ---- delayed initialisation against the oracle ----------------------------------------------------------------------------------------
def _opts(fid, slam, aruco):
    return aruco if _is_tag(fid) else slam


def test_slam_delayed_init_with_aruco_options_against_the_oracle(chi2_table):
    """ovp_slam_delayed_init on a mixed batch against the oracle's slam_delayed_init called feature by feature in input order, each with its
    own options (the reference initialises one feature at a time)"""
    slam, aruco = (1.0, 1.0), (0.5, 4.0)
    cs = _tag_update_case()
    S = cs.S
    ctx, orc, chg, cho = make_pair(S, plane_gate(chi2_table), max_state=S.N + 3 * S.F + 64)
    ctx.set_aruco_options(*aruco)
    bg, bo = synth.feature_batch(S, chg), synth.feature_batch(S, cho)
    g = ctx.slam_delayed_init(bg, *slam)
    fs, nh = np.zeros(S.F, dtype=np.int32), np.zeros(S.F, dtype=np.int32)
    for f in range(S.F):
        a, e = int(bo["meas_offset"][f]), int(bo["meas_offset"][f + 1])
        one = dict(F=1, meas_offset=np.array([0, e - a], dtype=np.int32), meas_clone=np.ascontiguousarray(bo["meas_clone"][a:e]),
                   uv=np.ascontiguousarray(bo["uv"][a:e]), p_FinG=np.ascontiguousarray(bo["p_FinG"][f:f + 1]),
                   p_FinG_original=np.ascontiguousarray(bo["p_FinG_original"][f:f + 1]), featid=bo["featid"][f:f + 1].copy(),
                   planeid=bo["planeid"][f:f + 1].copy())
        r = orc.slam_delayed_init(one, *_opts(bo["featid"][f], slam, aruco))
        fs[f], nh[f] = r["feat_status"][0], r["new_handles"][0]
    tags = np.array([_is_tag(f) for f in S.featid])
    print("statuses: tags %s, others %s" % (g["feat_status"][tags].tolist(), g["feat_status"][~tags].tolist()))
    assert np.array_equal(g["feat_status"], fs) and np.array_equal(g["new_handles"], nh), (g["feat_status"], fs)
    assert (g["feat_status"][tags] >= 1).any()
    _compare_states(ctx, orc, S.featid, g["new_handles"])
    ctx.close()
    orc.close()


def _compare_states(ctx, orc, featids, new_handles):
    assert ctx.cov_rows() == orc.cov_rows()
    Pg, Po = ctx.cov(), orc.cov()
    assert np.linalg.norm(Pg - Po) / np.linalg.norm(Po) < 1e-6
    for h in new_handles[new_handles >= 0]:
        vg, vo = ctx.var_get(int(h)), orc.var_get(int(h))
        assert np.abs(vg[0] - vo[0]).max() < 1e-6 and np.abs(vg[1] - vo[1]).max() < 1e-6, h
    for f in featids:
        assert ctx.slam_plane_of(int(f)) == osi.slam_plane_of(orc, int(f)), f


def _oracle_tracks(orc, t, tri, sigma_constraint, slam, aruco):
    """UpdaterSLAM::delayed_init on the oracle's stages in the reference's order with each feature's own options: every refinement candidate
    refined onto its plane (:147-186, sigma_pix / fx of its option set), then the initialisations one feature at a time in input order"""
    mo, mc = np.asarray(t["meas_offset"]), np.asarray(t["meas_clone"])
    fid, pid = np.asarray(t["featid"]), np.asarray(t["planeid"])
    F = len(mo) - 1
    count = np.diff(mo)
    fs, ps, pout, nh = np.where(count < 2, -1, 0).astype(np.int32), np.full(F, -1, dtype=np.int32), np.zeros((F, 3)), np.full(F, -1, dtype=np.int32)
    trk = [f for f in range(F) if count[f] >= 2]
    p_tri, ok = np.asarray(tri[0]).reshape(-1, 3), np.asarray(tri[1])
    fx = float(orc.var_get(orc.handle_intrinsics())[0][0])
    one = lambda f: (np.array([0, count[f]], dtype=np.int32), np.ascontiguousarray(mc[mo[f]:mo[f + 1]], dtype=np.int32))  # noqa: E731
    ref_ok = {}
    for k, f in enumerate(trk):
        pout[f] = p_tri[k]
        if pid[f] == 0 or orc.plane_handle(int(pid[f])) < 0 or osi.slam_plane_of(orc, int(fid[f])) == 0:
            continue
        cp = orc.var_get(orc.plane_handle(int(pid[f])))[0][:3]
        omo, omc = one(f)
        st, p, _, _, _ = orc.optimize_plane(np.array([0, 1], dtype=np.int32), omo, omc, np.ascontiguousarray(t["uv_norm"][mo[f]:mo[f + 1]]),
                                            p_tri[k:k + 1], cp[None], np.ones(1, dtype=np.int32), _opts(fid[f], slam, aruco)[0] / fx,
                                            sigma_constraint)
        ref_ok[f], ps[f], pout[f] = bool(st[0]), int(st[0]), p[0]
        if st[0]:
            osi.set_slam_plane_of(orc, int(fid[f]), int(pid[f]))
    for k, f in enumerate(trk):
        if not ok[k]:
            fs[f] = -2
            continue
        if not ref_ok.get(f, True):
            pout[f] = p_tri[k]
            osi.set_slam_plane_of(orc, int(fid[f]), 0)
        omo, omc = one(f)
        b = dict(F=1, meas_offset=omo, meas_clone=omc, uv=np.ascontiguousarray(t["uv"][mo[f]:mo[f + 1]], dtype=np.float32),
                 p_FinG=np.ascontiguousarray(pout[f:f + 1]), p_FinG_original=np.ascontiguousarray(p_tri[k:k + 1]),
                 featid=np.array([fid[f]], dtype=np.int64), planeid=np.array([pid[f] if ref_ok.get(f, True) else 0], dtype=np.int64))
        r = orc.slam_delayed_init(b, *_opts(fid[f], slam, aruco))
        fs[f], nh[f] = r["feat_status"][0], r["new_handles"][0]
    return dict(feat_status=fs, plane_status=ps, p_FinG=pout, new_handles=nh)


@pytest.mark.parametrize("seed", [0, 1])
def test_slam_delayed_init_tracks_with_aruco_options_against_the_oracle(seed, chi2_table):
    slam, aruco = (1.0, 1.0), (0.5, 4.0)
    S, mk, hz = sic.tracks_scene(seed=seed)
    ctx, orc, chg, cho = make_pair(S, plane_gate(chi2_table))
    tg, to = _tag_tracks(mk(chg)), _tag_tracks(mk(cho))
    tri = _tri_of(ctx, tg)
    # every refinement candidate refined alone by ovp_optimize_plane at its own sigma / fx, before the call (same state, same inputs)
    mo, count = tg["meas_offset"], np.diff(tg["meas_offset"])
    trk = [f for f in range(len(count)) if count[f] >= 2]
    fx = float(ctx.var_get(ctx.handle_intrinsics())[0][0])
    alone = {}
    for k, f in enumerate(trk):
        if tg["planeid"][f] == 0 or ctx.plane_handle(int(tg["planeid"][f])) < 0:
            continue
        cp = ctx.var_get(ctx.plane_handle(int(tg["planeid"][f])))[0][:3]
        st, p, _, _, _ = ctx.optimize_plane(np.array([0, 1], dtype=np.int32), np.array([0, count[f]], dtype=np.int32),
                                            np.ascontiguousarray(tg["meas_clone"][mo[f]:mo[f + 1]]), np.ascontiguousarray(tg["uv_norm"][mo[f]:mo[f + 1]]),
                                            tri[0][k:k + 1], cp[None], np.ones(1, dtype=np.int32), _opts(tg["featid"][f], slam, aruco)[0] / fx,
                                            S.options["sigma_constraint"])
        alone[f] = (int(st[0]), p[0].copy())
    ctx.set_aruco_options(*aruco)
    g = ctx.slam_delayed_init_tracks(tg, *slam)
    o = _oracle_tracks(orc, to, tri, S.options["sigma_constraint"], slam, aruco)
    tags = np.array([_is_tag(f) for f in tg["featid"]])
    print("seed %d: feat_status %s plane_status %s tags %s" % (seed, g["feat_status"].tolist(), g["plane_status"].tolist(), np.nonzero(tags)[0].tolist()))
    for k in ("feat_status", "plane_status", "new_handles"):
        assert np.array_equal(g[k], o[k]), (k, g[k], o[k])
    assert np.abs(g["p_FinG"] - o["p_FinG"]).max() < 1e-7
    refined_tags = [f for f in alone if tags[f] and g["plane_status"][f] == 1]
    assert refined_tags and (g["feat_status"][tags] >= 1).any()
    for f, (st, p) in alone.items():
        assert st == g["plane_status"][f], f
        if st == 1:
            assert _bits_equal(g["p_FinG"][f], p), (f, g["p_FinG"][f], p)
    _compare_states(ctx, orc, tg["featid"], g["new_handles"])
    ctx.close()
    orc.close()


# ---- the setter ------------------------------------------------------------------------------------------------------------------------
def test_setter_refuses_bad_options_and_clearing_restores_the_default(chi2_table):
    S, mk, hz = sic.tracks_scene(seed=0)
    ctx, orc, ch, _ = make_pair(S, chi2_table)
    orc.close()
    l0, b0 = ctx.launch_count(), ctx.transfer_bytes()
    for bad in ((0.0, 1.0), (-1.0, 1.0), (float("nan"), 1.0), (1.0, 0.0), (1.0, -2.0), (1.0, float("nan"))):
        with pytest.raises(api.OvpError) as e:
            ctx.set_aruco_options(*bad)
        assert e.value.status == 1, bad
    ctx.set_aruco_options(0.5, 4.0)
    ctx.set_aruco_options(None)
    assert ctx.launch_count() == l0 and ctx.transfer_bytes() == b0  # host-only
    t = _tag_tracks(mk(ch))
    with pytest.raises(api.OvpError) as e:
        ctx.slam_delayed_init_tracks(t)
    assert e.value.status == 1 and "ArUco" in str(e.value)
    ctx.close()
    # a cleared context gives the bits of one that never set the options: ovp_slam_delayed_init, then ovp_slam_update, with tags
    cs = _tag_update_case()
    outs = []
    for clear in (False, True):
        ctx, chg, b, _ = srt.new_ctx(cs)
        if clear:
            ctx.set_aruco_options(0.5, 4.0)
            ctx.set_aruco_options(None)
        r = ctx.slam_update(b, 1.0, 1.0, True)
        outs.append((r["feat_status"].copy(), r["feat_chi2"].copy(), _state(ctx), [ctx.slam_should_marg(int(f)) for f in b["featid"]]))
        ctx.close()
    assert _bits_equal(outs[0][0], outs[1][0]) and _bits_equal(outs[0][1], outs[1][1])
    assert _same_state(outs[0][2], outs[1][2]) and outs[0][3] == outs[1][3]
    a = _init_run(cs, None, 1.0, 1.0, plane_gate(chi2_table))
    S2 = cs.S
    ctx = api.Context(S2.options, device=0, max_state=S2.N + 3 * S2.F + 64, max_meas_rows=60000)
    ctx.set_chi2_table(plane_gate(chi2_table))
    chg = synth.load_scenario_into(ctx, S2)
    ctx.set_aruco_options(0.5, 4.0)
    ctx.set_aruco_options(None)
    r = ctx.slam_delayed_init(synth.feature_batch(S2, chg), 1.0, 1.0)
    assert _bits_equal(a[0], r["feat_status"]) and _bits_equal(a[1], r["new_handles"]) and _same_state(a[2], _state(ctx))
    ctx.close()
