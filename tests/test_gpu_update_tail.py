"""The tail of the EKF update (dx = Y w in OVP_DX_SPLIT fixed chunks, the manifold update of every variable kind, the downdate with its
negative-diagonal check) through ovp_ekf_update, and StateHelper::initialize through ovp_initialize, against the long-double references
of tests/update_reference.py on a state that holds every variable kind, has holes in its handle table and a recycled handle, and a
covariance that correlates everything with everything.  Bounds are the first-order bounds of update_reference.kalman_bounds; the planted
mistakes of tests/test_cpu_update_references.py show that they are tight enough to catch a wrong dx, quaternion or variable offset."""
import numpy as np
import pytest

import update_reference as ur
from ov_plane_b200 import api
from test_gpu_boundaries import assert_state_unchanged, state_snapshot

pytestmark = pytest.mark.gpu

OVP_ERR_NEGATIVE_DIAGONAL = 2
EXTRA = {1: 2, 63: 44}  # N % 64 -> extra landmarks of build_state (N = 129 and 255)
ROWS = (1, 7, 8, 9, 63, 64, 65, 500)


def new_ctx(chi2_table):
    ctx = api.Context(ur.STATE_OPTIONS, device=0, max_state=640, max_meas_rows=4096)
    ctx.set_chi2_table(chi2_table)
    return ctx


def read_state(ctx, kinds):
    vals, fejs = {}, {}
    for h in kinds:
        vals[h], fejs[h] = ctx.var_get(h)
    return ctx.cov(), vals, fejs


CASES = [(m, rows, rd) for m in (1, 63) for rows in ROWS for rd in (None, "nonunit")]
CASES += [(m, rows, "kappa") for m in (1, 63) for rows in (63, 64, 65, 500)]


@pytest.mark.parametrize("nmod,rows,rdiag", CASES)
def test_ekf_update_tail_against_long_double(nmod, rows, rdiag, chi2_table):
    ur.require_long_double()
    ctx = new_ctx(chi2_table)
    c = ur.update_case(ctx, EXTRA[nmod], rows, rdiag, seed=rows + nmod)
    assert ctx.cov_rows() % 64 == nmod
    assert len(set(c["kinds"])) == len(c["kinds"])
    ctx.ekf_update(c["handles"], c["H"], c["r"], c["Rdiag"])
    P_got, vals_got, fejs_got = read_state(ctx, c["kinds"])
    ref = ur.kalman(c["P"], c["cols"], c["H"], c["r"], c["Rdiag"])
    dxb, dPb, kS = ur.kalman_bounds(c["P"], c["cols"], c["H"], ref)
    if rdiag == "kappa":
        assert 1e7 <= kS <= 1e9, kS
    qP, qv = ur.check_update(P_got, vals_got, fejs_got, c["P"], c["kinds"], c["ids"], c["vals"], c["fejs"], ref["dx"], dxb, dPb, ref["P"])
    flips = ur.flipped(c["kinds"], c["vals"], c["ids"], ref["dx"])
    print("N %d rows %d R %s: kappa(S) %.2e, worst error / bound: P+ %.3e values %.3e; %d quaternion sign flips" % (
        ctx.cov_rows(), rows, rdiag, kS, qP, qv, len(flips)))
    ctx.close()


def test_ekf_update_negative_diagonal_is_reported_and_cleared(chi2_table):
    """P_dt,dt = 1e-12 with cov(dt, f_x) = 1e-3 and var(f_x) = 1: an update of f_x with R = 1e-6 drives P_dt,dt to about -1e-6, which
    the update reports as OVP_ERR_NEGATIVE_DIAGONAL (the reference exits there).  The next update on a valid P succeeds, so the
    device-side flag was cleared."""
    ctx = new_ctx(chi2_table)
    kinds, sig, hs = ur.build_state(ctx, EXTRA[1], 3)
    ids, vals, fejs, d = ur.state_arrays(ctx, kinds, sig)
    P = np.diag(d * d)
    idt, ix = ctx.var_id(ctx.handle_dt()), ctx.var_id(ctx.handle_intrinsics())
    P[idt, idt], P[ix, ix] = 1e-12, 1.0
    P[idt, ix] = P[ix, idt] = 1e-3
    ctx.cov_upload(P)
    H = np.zeros((1, 8))
    H[0, 0] = 1.0
    with pytest.raises(api.OvpError) as e:
        ctx.ekf_update([ctx.handle_intrinsics()], H, [0.0], [1e-6])
    assert e.value.status == OVP_ERR_NEGATIVE_DIAGONAL
    ctx.cov_upload(np.diag(d * d))
    ctx.ekf_update([ctx.handle_intrinsics()], H, [0.0], [1e-6])
    assert np.all(np.diag(ctx.cov()) > 0)
    ctx.close()


# ---- ovp_initialize --------------------------------------------------------------------------------------------------------------
INIT_CASES = [(s, rows, wide) for s in (1, 3) for rows in sorted({s, s + 1, 33, 65, 300}) for wide in (False, True)]


def init_case(ctx, s, rows, wide, seed, scale=1.0):
    kinds, sig, hs = ur.build_state(ctx, EXTRA[63] if wide else EXTRA[1], seed)
    ids, vals, fejs, d = ur.state_arrays(ctx, kinds, sig)
    P = ur.correlated(d, seed)
    ctx.cov_upload(P)
    # wide: every variable, so that [H_L | H_R | r] has s + N + 1 > 256 columns
    handles = sorted(kinds, key=lambda h: -ids[h]) if wide else ur.update_handles(ctx, hs)
    cols = ur.columns(ctx, handles)
    rng = np.random.default_rng(seed)
    sigma2 = 0.5
    H_R, r = ur.measurement(rng, P, cols, rows, d, np.full(rows, sigma2))
    H_L = rng.standard_normal((rows, s))
    r = scale * (r + H_L @ (0.1 * rng.standard_normal(s)))
    value = 3.0 + rng.standard_normal(s)
    return kinds, ids, vals, fejs, P, handles, cols, H_R, H_L, r, sigma2, value


@pytest.mark.parametrize("s,rows,wide", INIT_CASES)
def test_initialize_against_long_double(s, rows, wide, chi2_table):
    ur.require_long_double()
    ctx = new_ctx(chi2_table)
    kinds, ids, vals, fejs, P, handles, cols, H_R, H_L, r, sigma2, value = init_case(ctx, s, rows, wide, seed=rows + 7 * s)
    N = P.shape[0]
    kind = ur.LANDMARK if s == 3 else ur.VEC
    acc, nh = ctx.initialize(kind, value, value, 7000000 + rows, handles, H_R, H_L, r, sigma2, 1.0)
    ref = ur.initialize(P, cols, H_R, H_L, r, sigma2)
    thr = chi2_table[rows]
    assert acc == (ref["chi2"] <= thr), "chi2 %.6g against %.6g" % (float(ref["chi2"]), thr)
    assert acc, "the case is built to pass the gate: chi2 %.6g against %.6g" % (float(ref["chi2"]), thr)
    assert ctx.var_id(nh) == N and ctx.cov_rows() == N + s
    P_got, vals_got, fejs_got = read_state(ctx, kinds)
    vals_got[nh], fejs_got[nh] = ctx.var_get(nh)
    # the new variable enters the update at value + R_1^-1 Q_1^T r; its dx bound carries the initialisation's error below
    kinds2, ids2 = {**kinds, nh: kind}, {**ids, nh: N}
    vals2 = {**vals, nh: np.asarray(value, dtype=ur.LD) + ref["dxn"]}
    fejs2 = {**fejs, nh: np.asarray(value)}
    # the initialisation's own error (R_1^-1 and the s x s products) on the new rows, first order in kappa(R_1)
    sv = np.linalg.svd(H_L, compute_uv=False)
    kR = sv[0] / sv[-1]
    e_init = ur.BOUND_C * (rows + len(cols) + 2) * ur.EPS * kR * kR
    e_dxn = ur.BOUND_C * (rows + 2) * ur.EPS * kR * float(np.linalg.norm(r)) / sv[-1]
    if ref["upd"] is None:
        P_ref, dx = ref["P_init"], np.zeros(N + s, dtype=ur.LD)
        dxb, dPb = np.zeros(N + s), np.zeros((N + s, N + s))
    else:
        P_ref, dx = ref["upd"]["P"], ref["upd"]["dx"]
        dxb, dPb, _ = ur.kalman_bounds(ref["P_init"], cols, ref["H2"], ref["upd"])
    dPb[N:, :] += e_init
    dPb[:, N:] += e_init
    dxb[N:] += e_dxn
    # P stays exactly symmetric also without update rows: P_LL (formed on the host, symmetric to rounding) enters P from its lower triangle
    qP, qv = ur.check_update(P_got, vals_got, fejs_got, ref["P_init"], kinds2, ids2, vals2, fejs2, dx, dxb, dPb, P_ref)
    print("s %d rows %d columns %d: chi2 %.4g, worst error / bound: P+ %.3e values %.3e" % (s, rows, s + len(cols) + 1, float(ref["chi2"]),
                                                                                          qP, qv))
    ctx.close()


@pytest.mark.parametrize("s", [1, 3])
def test_initialize_rejected_leaves_state_bit_identical(s, chi2_table):
    ur.require_long_double()
    ctx = new_ctx(chi2_table)
    kinds, ids, vals, fejs, P, handles, cols, H_R, H_L, r, sigma2, value = init_case(ctx, s, 65, False, seed=11 + s, scale=30.0)
    ref = ur.initialize(P, cols, H_R, H_L, r, sigma2)
    assert ref["chi2"] > 2 * chi2_table[65]
    order = ctx.variable_order()
    snap = state_snapshot(ctx, list(kinds))
    fej0 = [ctx.var_get(h)[1].copy() for h in kinds]
    acc, nh = ctx.initialize(ur.LANDMARK if s == 3 else ur.VEC, value, value, 7100000 + s, handles, H_R, H_L, r, sigma2, 1.0)
    assert not acc and nh == -1
    assert_state_unchanged(ctx, list(kinds), snap)
    assert all(np.array_equal(ctx.var_get(h)[1], f) for h, f in zip(kinds, fej0)), "a FEJ changed"
    assert ctx.variable_order() == order and ctx.cov_rows() == P.shape[0]
    ctx.close()
