"""The references of tests/slam_reference.py pinned on the CPU: the SLAM update reference (the accepted landmarks' rows stacked, EKFUpdate
with R = I in long double) against the oracle's UpdaterSLAM::update on a correlated covariance, the Gram route (a long-double factor of
X^T X with the zero-pivot rule) against the uncompressed update on rank-deficient stacks, marginalize_slam against the oracle, and the
planted mistakes the GPU tests rely on the references to catch."""
import numpy as np
import pytest

import gate_reference as gr
import oracle_backend
import slam_reference as sr
import update_reference as ur
from ov_plane_b200 import synth

ARUCO_FEATID = 7  # below max_aruco_features (1024): an ArUco tag, never flagged for marginalisation


def _setup(ncal, cond, seed=0):
    """oracle with gr.slam_scenario's landmarks initialised, the first one under an ArUco id, a correlated covariance and the update
    batch (an outlier of 30 px on every measurement of the ArUco landmark and of one more landmark, so that both are rejected)"""
    S = gr.slam_scenario(ncal, seed=seed)
    S.featid[0] = ARUCO_FEATID
    orc = oracle_backend.OracleContext(S.options)
    orc.set_chi2_table(synth.chi2_table())
    ch = synth.load_scenario_into(orc, S)
    g = orc.slam_delayed_init(synth.feature_batch(S, ch), 1.0, 1.0)
    keep = np.nonzero(g["feat_status"] > 0)[0]
    assert 0 in keep
    attached = {int(S.featid[f]) for f in keep if g["feat_status"][f] == 1 and S.planeid[f] != 0}
    orc.cov_upload(gr.correlated_cov(S, orc.cov_rows(), seed=7 + ncal, cond=cond))
    b = gr.slam_update_batch(S, ch, keep, seed=ncal, wrong_plane=3)
    for f in (0, 5):
        a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
        b["uv"][a:e] += np.float32(30.0)
    return S, orc, ch, b, attached


def _kinds(orc, S, ch, b):
    kinds = {orc.handle_imu(): ur.IMU}
    if S.options["do_calib_camera_pose"]:
        kinds[orc.handle_calib()] = ur.POSE
    if S.options["do_calib_camera_intrinsics"]:
        kinds[orc.handle_intrinsics()] = ur.VEC
    for h in ch:
        kinds[int(h)] = ur.POSE
    for pid in S.plane_ids:
        kinds[orc.plane_handle(int(pid))] = ur.VEC
    for fid in b["featid"]:
        kinds[orc.slam_handle(int(fid))] = ur.LANDMARK
    return kinds


def _parts(orc, S, b, statuses, attached, **mistakes):
    """(J, r, ids) of every landmark that stacks rows, from the oracle's get_feature_jacobian_full at the current state (with the plane
    when the landmark is on it)"""
    parts = []
    for f in range(b["F"]):
        a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
        lm = orc.slam_handle(int(b["featid"][f]))
        val, fej = orc.var_get(lm)
        has_plane = int(b["featid"][f]) in attached
        pid = int(b["planeid"][f]) if has_plane else 0
        cp = cpf = None
        if has_plane:
            cp, cpf = orc.var_get(orc.plane_handle(pid))
        Hf, Hx, r, xo = orc.feature_jacobian_full(b["meas_clone"][a:e], b["uv"][a:e], val, fej, pid, cp, cpf, 1.0, S.options["sigma_constraint"])
        out = sr.landmark_rows(Hf, Hx, r, int(statuses[f]), has_plane, e - a, **mistakes)
        if out is None:
            continue
        ids = gr.block_ids(orc, [lm]) + gr.block_ids(orc, xo)
        parts.append((out[0], out[1], ids[:out[0].shape[1]]))
    return parts


def _scaled_err(Pa, Pb, P0):
    sd = np.sqrt(np.diag(np.asarray(P0, dtype=np.float64)))
    return np.abs(np.asarray(Pa - Pb, dtype=np.float64)) / np.outer(sd, sd)


@pytest.mark.parametrize("ncal,cond", [(0, None), (14, None), (8, 1e10)])
def test_update_reference_equals_the_oracle(ncal, cond):
    ur.require_long_double()
    S, orc, ch, b, attached = _setup(ncal, cond)
    kinds = _kinds(orc, S, ch, b)
    P = orc.cov()
    vals = {h: orc.var_get(h)[0] for h in kinds}
    ids = {h: orc.var_id(h) for h in kinds}
    # the raw layout landmark_rows relies on: with the plane, the 2m bearing rows come first and equal the rows built without it
    f = next(f for f in range(b["F"]) if int(b["featid"][f]) in attached)
    a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
    lm = orc.slam_handle(int(b["featid"][f]))
    val, fej = orc.var_get(lm)
    cp, cpf = orc.var_get(orc.plane_handle(int(b["planeid"][f])))
    with_p = orc.feature_jacobian_full(b["meas_clone"][a:e], b["uv"][a:e], val, fej, int(b["planeid"][f]), cp, cpf, 1.0, S.options["sigma_constraint"])
    without = orc.feature_jacobian_full(b["meas_clone"][a:e], b["uv"][a:e], val, fej, 0, None, None, 1.0, S.options["sigma_constraint"])
    m = e - a
    assert np.array_equal(with_p[0][:2 * m], without[0]) and np.array_equal(with_p[1][:2 * m, :-3], without[1])
    assert np.array_equal(with_p[2][:2 * m], without[2])
    o = orc.slam_update(b, 1.0, 1.0)
    st = o["feat_status"]
    assert st[0] == 0 and st[5] == 0 and np.count_nonzero(st == 1) >= 8 and np.count_nonzero(st == 3) >= 1, st
    # the update is linearised at the prior state: restore it on a second oracle to build the rows there
    S2, orc2, ch2, b2, _ = _setup(ncal, cond)
    parts = _parts(orc2, S2, b2, st, attached)
    cols = sorted({int(s) for p in parts for s in p[2]})
    X = sr.stack(parts, cols)
    ref = sr.slam_update_reference(P, cols, X)
    e = _scaled_err(orc.cov(), ref["P"], P)
    assert e.max() < 1e-10, "oracle P+ against the reference: %.3e" % e.max()
    new = ur.apply_dx(kinds, vals, ids, ref["dx"])
    worst_v = max(float(np.abs(np.asarray(orc.var_get(h)[0] - new[h], dtype=np.float64)).max()) for h in kinds)
    assert worst_v < 1e-10, worst_v
    # the bookkeeping: the ArUco landmark is not flagged, every other rejected one is
    for f in range(b["F"]):
        fid = int(b["featid"][f])
        assert orc.slam_should_marg(fid) == (1 if st[f] == 0 and fid >= 1024 else 0), (f, fid, st[f])
    # the bounds of the GPU tests, on a Gram matrix formed in float64 as the library forms it
    X64 = np.asarray(X, dtype=np.float64)
    G = X64.T @ X64
    dxb, dPb, fac = sr.slam_bounds(P, cols, X, G, ref)
    print("ncal %d cond %s: %d rows over %d columns, %d zero pivots; oracle P+ scaled error %.3e, values %.3e" % (
        ncal, cond, X.shape[0], len(cols), len(fac["zero"]), e.max(), worst_v))
    # planted mistakes: each moves P+ by more than twice its bound
    for name, mistakes in (("a rejected landmark's rows stacked", dict(stack_rejected=True)),
                           ("the retry keeping its plane row", dict(retry_keeps_plane=True))):
        bad_parts = _parts(orc2, S2, b2, st, attached, **mistakes)
        bcols = sorted(set(cols) | {int(s) for p in bad_parts for s in p[2]})
        bad = sr.slam_update_reference(P, bcols, sr.stack(bad_parts, bcols))
        q = float((_scaled_err(bad["P"], ref["P"], P) / dPb).max())
        assert q > 2.0, "%s: P+ moves by only %.3g bounds" % (name, q)
    orc.close()
    orc2.close()


@pytest.mark.parametrize("rows,nc,seed", [(2, 9, 0), (3, 12, 1), (4, 23, 2), (58, 183, 3), (40, 30, 4)])
def test_gram_route_equals_the_uncompressed_update(rows, nc, seed):
    """Rank-deficient stacks (rows < nc: a landmark with m measurements has 2m or 3m rows over 3 + 6m (+ 3) + ncal columns): the update with
    H = L^T, r = the last row of the long-double factor of X^T X (zero-pivot rule at the default tolerance) is the update with X itself."""
    ur.require_long_double()
    rng = np.random.default_rng(seed)
    N = nc + 20
    d = np.exp(rng.uniform(-4.0, 0.0, N))
    P = ur.correlated(d, seed)
    cols = sorted(rng.choice(N, size=nc, replace=False).tolist())
    H = rng.standard_normal((rows, nc)) / d[cols][None, :] / np.sqrt(nc)
    X = np.hstack([H, rng.standard_normal((rows, 1))]).astype(ur.LD)
    ref = sr.slam_update_reference(P, cols, X)
    L, zero, _ = sr.ld_factor(sr.gram_ld(X), nc)
    assert len(zero) == max(0, nc - rows)
    Hk, rk = sr.kept_system(L)
    got = ur.kalman(P, cols, Hk, rk, None)
    e = float(_scaled_err(got["P"], ref["P"], P).max())
    edx = float(np.abs(np.asarray((got["dx"] - ref["dx"]) / d, dtype=np.float64)).max())
    assert e < 1e-12 and edx < 1e-12, (e, edx)


def test_marginalize_slam_reference_equals_the_oracle():
    S, orc, ch, b, attached = _setup(14, None)
    o = orc.slam_update(b, 1.0, 1.0)
    P = np.asarray(orc.cov())
    lms = {int(fid): (orc.var_id(orc.slam_handle(int(fid))), orc.slam_should_marg(int(fid)) == 1) for fid in S.featid
           if orc.slam_handle(int(fid)) >= 0}
    assert sum(v[1] for v in lms.values()) >= 1 and o["feat_status"][0] == 0
    want, removed = sr.marginalize_slam(P, lms, S.options["max_aruco_features"])
    orc.marginalize_slam()
    got = orc.cov()
    assert got.shape == want.shape and np.array_equal(got.view(np.uint64), want.view(np.uint64))
    for fid in lms:
        assert (orc.slam_handle(fid) < 0) == (fid in removed)
    # the planted mistake: >= at featid 4 max_aruco_features
    lim = 4 * S.options["max_aruco_features"]
    two = {lim: (3, True), lim + 1: (9, True), lim + 2: (15, False)}
    Q = ur.correlated(np.ones(21), 3)
    good, gr_ = sr.marginalize_slam(Q, two, S.options["max_aruco_features"])
    bad, br_ = sr.marginalize_slam(Q, two, S.options["max_aruco_features"], rule=">=")
    assert gr_ == [lim + 1] and br_ == [lim, lim + 1] and good.shape != bad.shape
    orc.close()


def test_gate_dof_against_the_oracle():
    """The table entries the oracle's gates read, against gate_dof: a table non-zero at one entry accepts a landmark on its plane with
    status 1 at 3m and with status 3 (the retry) at 2m, and one without a plane at 2m; the planted dof 2m for a plane landmark
    mispredicts."""
    S, orc, ch, b, attached = _setup(0, None)
    P = orc.cov()
    m = np.diff(b["meas_offset"])
    on = [int(fid) in attached for fid in b["featid"]]
    wrong = 0
    for idx in sorted({int(3 * x) for x in m} | {int(2 * x) for x in m}):
        table = np.zeros(3 * int(m.max()) + 1)
        table[idx] = 1e300
        S2, o2, ch2, b2, _ = _setup(0, None)
        o2.cov_upload(P)
        o2.set_chi2_table(table)
        st = o2.slam_update(b2, 1.0, 1.0)["feat_status"]
        o2.close()
        want = [sr.status_one_hot(int(m[f]), on[f], idx) for f in range(b["F"])]
        assert list(st) == want, "table non-zero at %d: statuses %s, expected %s" % (idx, list(st), want)
        bad = [sr.status_one_hot(int(m[f]), on[f], idx, dof=lambda mm, p: sr.gate_dof(mm, p, plane_rows=2)) for f in range(b["F"])]
        wrong += int(bad != want)
    assert wrong >= 2, "the planted dof 2m for a plane landmark changes no prediction"
    orc.close()
