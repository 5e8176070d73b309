"""The reference of tests/msckf_point_reference.py pinned on the CPU: the direct-form reference (the accepted features' rows projected
in long double, stacked, EKFUpdate with R = I) against the oracle's msckf_update on a correlated covariance, the Gram route (a long-double
factor of X^T X with the zero-pivot rule) against the direct form within its bound on systems with gauge directions, and the planted
mistakes the GPU test relies on the bounds to catch, each at least 10 times over its bound."""
import numpy as np
import pytest

import gate_reference as gr
import msckf_point_reference as mr
import oracle_backend
import slam_reference as sr
import update_reference as ur
from ov_plane_b200 import synth

# the GPU test's direct-form and compressed shapes, small enough for the oracle: (ncal, clones, features, m_min, m_max)
SHAPES = {0: (0, 12, 24, 3, 10), 14: (14, 12, 24, 3, 10)}


def _setup(ncal, cond=None, seed=0):
    """the oracle with a point scenario loaded and gate_reference.correlated_cov uploaded; one feature moved by 30 px (rejected)"""
    _, C, F, m0, m1 = SHAPES[ncal]
    S = mr.point_scenario(ncal, C, F, m0, m1, seed=seed)
    k = (S.meas_offset[5] + S.meas_offset[6]) // 2
    S.uv[k] += np.float32(30.0)
    orc = oracle_backend.OracleContext(S.options)
    orc.set_chi2_table(synth.chi2_table())
    ch = synth.load_scenario_into(orc, S)
    orc.cov_upload(gr.correlated_cov(S, orc.cov_rows(), seed=31 + ncal + seed, cond=cond))
    return S, orc, ch, synth.feature_batch(S, ch)


def _feats(orc, S, b, status):
    """(H_f, H_x, r, ids) of every accepted feature from the oracle's get_feature_jacobian_full at the current state"""
    out = []
    for f in range(b["F"]):
        if int(status[f]) != 1:
            continue
        a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
        pf = b["p_FinG_original"][f]
        Hf, Hx, r, xo = orc.feature_jacobian_full(b["meas_clone"][a:e], b["uv"][a:e], pf, pf, 0, None, None, 1.0, S.options["sigma_constraint"])
        out.append((Hf, Hx, r, gr.block_ids(orc, xo)))
    return out


def _kinds(orc, S, ch):
    kinds = {orc.handle_imu(): ur.IMU}
    if S.options["do_calib_camera_pose"]:
        kinds[orc.handle_calib()] = ur.POSE
    if S.options["do_calib_camera_intrinsics"]:
        kinds[orc.handle_intrinsics()] = ur.VEC
    for h in ch:
        kinds[int(h)] = ur.POSE
    return kinds


def _scaled(Pa, Pb, P0):
    sd = np.sqrt(np.diag(np.asarray(P0, dtype=np.float64)))
    return np.abs(np.asarray(Pa - Pb, dtype=np.float64)) / np.outer(sd, sd)


def _case(ncal, cond=None):
    """(P, cols, feats, statuses, oracle after its update, kinds, prior values, ids)"""
    S, orc, ch, b = _setup(ncal, cond)
    P = orc.cov()
    kinds = _kinds(orc, S, ch)
    vals = {h: orc.var_get(h)[0] for h in kinds}
    ids = {h: orc.var_id(h) for h in kinds}
    o = orc.msckf_update(b, 1.0, 1.0)
    st = o["feat_status"]
    assert st[5] == 0 and np.count_nonzero(st == 1) >= 15, st
    # the rows are linearised at the prior state: a second oracle with the prior builds them
    S2, orc2, ch2, b2 = _setup(ncal, cond)
    feats = _feats(orc2, S2, b2, st)
    orc2.close()
    cols = sorted({i for fe in feats for i in fe[3]})
    assert cols == sorted(gr.block_ids(orc, o["hx_order"])), "Hx_order does not span the accepted features' columns"
    return P, cols, feats, st, orc, kinds, vals, ids


@pytest.mark.parametrize("ncal", [0, 14])
def test_direct_reference_equals_the_oracle(ncal):
    ur.require_long_double()
    P, cols, feats, st, orc, kinds, vals, ids = _case(ncal)
    X, Xb = mr.stacked_rows(feats, cols)
    assert X.shape[0] == sum(2 * (fe[0].shape[0] // 2) - 3 for fe in feats)
    d = mr.direct_reference(P, cols, X, Xb)
    e = _scaled(orc.cov(), d["ref"]["P"], P).max()
    assert e < 1e-10, "oracle P+ against the reference: %.3e" % e
    new = ur.apply_dx(kinds, vals, ids, d["ref"]["dx"])
    ev = max(float(np.abs(np.asarray(orc.var_get(h)[0] - new[h], dtype=np.float64)).max()) for h in kinds)
    assert ev < 1e-10, ev
    print("ncal %d: %d rows over %d columns; oracle P+ scaled error %.3e, values %.3e" % (ncal, X.shape[0], len(cols), e, ev))
    orc.close()


@pytest.mark.parametrize("ncal,cond", [(0, None), (14, None), (14, 1e10)])
def test_gram_route_equals_the_direct_form(ncal, cond):
    """The point system over clones alone has gauge directions (a global translation and yaw): the Gram route on the long-double X^T X
    zeroes them and lands within its bound of the stacked reference."""
    ur.require_long_double()
    P, cols, feats, st, orc, kinds, vals, ids = _case(ncal, cond)
    orc.close()
    X, Xb = mr.stacked_rows(feats, cols)
    d = mr.direct_reference(P, cols, X, Xb)
    g = mr.gram_reference(P, cols, sr.gram_ld(X))
    assert len(g["zero"]) >= 1, "no zero pivot"
    qP = float((_scaled(g["ref"]["P"], d["ref"]["P"], P) / g["dPb"]).max())
    qx = float((np.abs(np.asarray(g["ref"]["dx"] - d["ref"]["dx"], dtype=np.float64)) / g["dxb"]).max())
    print("ncal %d cond %s: %d zero pivots; Gram route against the stacked rows: P+ %.3e, dx %.3e of the bound" % (ncal, cond, len(g["zero"]), qP, qx))
    assert qP <= 1.0 and qx <= 1.0, (qP, qx)


def _clone_blocks(cols, ncal):
    return [cols[ncal + 6 * k:ncal + 6 * k + 6] for k in range((len(cols) - ncal) // 6)]


def _misread(P, Pread, cols, H, r):
    """the update with M = P[:, cols] H^T read from Pread (S and the prior from P): a product item that reads P wrongly"""
    P, Pread, H, r = (np.asarray(a, dtype=ur.LD) for a in (P, Pread, H, r))
    M = Pread[:, cols] @ H.T
    L = ur.ld_cholesky(H @ P[np.ix_(cols, cols)] @ H.T + np.eye(H.shape[0], dtype=ur.LD))
    Y = ur.ld_solve_lower(L, M.T).T
    return dict(P=P - Y @ Y.T, dx=Y @ ur.ld_solve_lower(L, r))


def _over(bad, good):
    """the planted mistake's change of the update against the bound: max over P+ (Jacobi-scaled by the prior) and dx"""
    qP = float((_scaled(bad["P"], good["ref"]["P"], good["P0"]) / good["dPb"]).max())
    qx = float((np.abs(np.asarray(bad["dx"] - good["ref"]["dx"], dtype=np.float64)) / good["dxb"]).max())
    return max(qP, qx)


@pytest.mark.parametrize("form", ["direct", "gram"])
@pytest.mark.parametrize("cond", [None, 1e10])
def test_planted_mistakes_exceed_ten_times_the_bound(form, cond):
    ur.require_long_double()
    ncal = 14
    P, cols, feats, st, orc, kinds, vals, ids = _case(ncal, cond)
    orc.close()
    X, Xb = mr.stacked_rows(feats, cols)
    G = np.asarray(X, dtype=np.float64).T @ np.asarray(X, dtype=np.float64)  # in float64, as the library forms it
    tol = mr.GRAM_TOL

    def run(cols_, X_, Xb_, tol_=tol):
        if form == "direct":
            return mr.direct_reference(P, cols_, X_, Xb_)
        return mr.gram_reference(P, cols_, np.asarray(X_, dtype=np.float64).T @ np.asarray(X_, dtype=np.float64), tol_)

    good = run(cols, X, Xb)
    good["P0"] = P
    nc = len(cols)
    if form == "gram":
        assert len(good["zero"]) >= 1
        H, r = sr.kept_system(good["L"])
    else:
        H, r = X[:, :nc], X[:, nc]
    blocks = _clone_blocks(cols, ncal)
    cal = cols[:ncal]
    out = {}
    # one clone x clone block of P read transposed (and its mirror)
    a, c = blocks[1], blocks[4]
    Pt = P.copy()
    Pt[np.ix_(a, c)] = P[np.ix_(a, c)].T
    Pt[np.ix_(c, a)] = P[np.ix_(c, a)].T
    out["a clone block of P read transposed"] = _over(_misread(P, Pt, cols, H, r), good)
    # the calibration x clone covariance dropped
    Pd = P.copy()
    clo = [i for bl in blocks for i in bl]
    Pd[np.ix_(cal, clo)] = 0.0
    Pd[np.ix_(clo, cal)] = 0.0
    out["calibration x clone covariance dropped"] = _over(_misread(P, Pd, cols, H, r), good)
    # two clone blocks of cols swapped
    cs = list(cols)
    cs[ncal + 6:ncal + 12], cs[ncal + 24:ncal + 30] = cols[ncal + 24:ncal + 30], cols[ncal + 6:ncal + 12]
    out["two clone blocks of cols swapped"] = _over(run(cs, X, Xb)["ref"], good)
    # one accepted feature's rows left out
    X1, Xb1 = mr.stacked_rows(feats[1:], cols)
    out["an accepted feature's rows left out"] = _over(run(cols, X1, Xb1)["ref"], good)
    # the zero-pivot rule (the Gram route), printed, not asserted: keeping the zero pivots (tol = 0) moves the posterior by ~1e-8 of the
    # bound (their information is rounding's), and zeroing the weakest real pivot by less than the bound (it carries little next to the
    # prior); the bound holds the rule's first-order effect by construction (tol G_jj on every dropped pivot)
    if form == "gram":
        kept = np.array([j for j in range(nc) if j not in good["zero"]])
        weakest = float((good["ratio"][kept] * tol).min())  # its pivot over its column's original diagonal
        print("gram cond %s: zero pivots kept (tol = 0) %.3e, the weakest real pivot zeroed %.3e of the bound" % (
            cond, _over(run(cols, X, Xb, tol_=0.0)["ref"], good), _over(run(cols, X, Xb, tol_=2.0 * weakest)["ref"], good)))
    # R = 2 I: the rows whitened by sqrt(2) too little
    out["R = 2 I"] = _over(ur.kalman(P, cols, H, r, np.full(H.shape[0], 2.0)), good)
    # the quaternion error applied on the wrong side: the values against their bound
    dx = good["ref"]["dx"]
    right = ur.apply_dx(kinds, vals, ids, dx, quat=lambda q, d: ur.quat_update(q, d, order="right"))
    ref = ur.apply_dx(kinds, vals, ids, dx)
    vb = ur.value_bounds(kinds, vals, ids, good["dxb"])
    out["quaternion error on the wrong side"] = max(float((np.abs(np.asarray(right[h] - ref[h], dtype=np.float64)) / vb[h]).max()) for h in kinds)
    for k, v in out.items():
        print("%s cond %s: %-40s %.3e of the bound" % (form, cond, k, v))
    low = {k: v for k, v in out.items() if not v >= 10.0}
    assert not low, "planted mistakes within 10x of the bound: %s" % low
