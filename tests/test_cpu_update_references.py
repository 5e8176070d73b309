"""The long-double references of tests/update_reference.py (the projection, the EKF update's tail, StateHelper::initialize) against numpy
and the oracle on the same inputs the GPU tests use, and the bounds of tests/test_gpu_update_tail.py against planted mistakes: each
mistake applied to the reference moves some value by more than twice its bound, so a kernel that made it could not pass."""
import functools

import numpy as np
import pytest

import oracle_backend
import update_reference as ur
from test_gpu_update_tail import CASES, EXTRA, init_case


def _oracle(chi2_table):
    orc = oracle_backend.OracleContext(ur.STATE_OPTIONS)
    orc.set_chi2_table(chi2_table)
    return orc


def _state(be, kinds):
    vals, fejs = {}, {}
    for h in kinds:
        vals[h], fejs[h] = be.var_get(h)
    return be.cov(), vals, fejs


@pytest.mark.parametrize("hf,rows,plane", [(1, 5, False), (3, 33, True), (3, 65, False), (2, 300, True)])
def test_householder_reference_against_numpy_qr(hf, rows, plane):
    """R and Q_1^T X of the reference equal numpy's QR up to the sign of each row; the remaining rows have the Gram matrix of the
    projection onto the left null space of numpy's Q_1."""
    ur.require_long_double()
    rng = np.random.default_rng(rows)
    Hf = rng.standard_normal((rows, hf))
    X = rng.standard_normal((rows, 12 + (3 if plane else 0)))
    A = np.asarray(ur.householder_project(np.column_stack([Hf, X]), hf), dtype=np.float64)
    Q, R = np.linalg.qr(Hf, mode="complete")
    sgn = np.sign(np.diag(R[:hf]))[:, None] * np.sign(np.diag(A[:hf, :hf]))[:, None]
    assert np.allclose(A[:hf, :hf], sgn * R[:hf], rtol=0, atol=1e-13 * np.abs(R).max())
    assert np.allclose(A[:hf, hf:], sgn * (Q[:, :hf].T @ X), rtol=0, atol=1e-12)
    assert np.allclose(A[hf:, :hf], 0.0, atol=0)
    O, N = A[hf:, hf:], Q[:, hf:]
    assert np.allclose(O.T @ O, (N.T @ X).T @ (N.T @ X), rtol=0, atol=1e-10)


def test_householder_reference_skips_a_zero_column():
    Hf = np.random.default_rng(1).standard_normal((9, 3))
    Hf[:, 1] = 0.0
    A = ur.householder_project(Hf, 3)
    assert A[1, 1] != 0 or np.all(A[1:, 1] == 0)
    assert np.all(A[2:, 1] == 0)


@pytest.mark.parametrize("nmod,rows,rdiag", [(1, 9, None), (63, 65, "nonunit"), (1, 500, "kappa")])
def test_kalman_reference_against_oracle(nmod, rows, rdiag, chi2_table):
    """The oracle (StateHelper::EKFUpdate in double) stays within the same bounds the GPU update is held to."""
    ur.require_long_double()
    orc = _oracle(chi2_table)
    c = ur.update_case(orc, EXTRA[nmod], rows, rdiag, seed=rows + nmod)
    orc.ekf_update(c["handles"], c["H"], c["r"], c["Rdiag"])
    P_got, vals_got, fejs_got = _state(orc, c["kinds"])
    ref = ur.kalman(c["P"], c["cols"], c["H"], c["r"], c["Rdiag"])
    dxb, dPb, kS = ur.kalman_bounds(c["P"], c["cols"], c["H"], ref)
    P_got = 0.5 * (P_got + P_got.T)  # the oracle symmetrises P at its own pace; the kernel's exact symmetry is a GPU test
    qP, qv = ur.check_update(P_got, vals_got, fejs_got, c["P"], c["kinds"], c["ids"], c["vals"], c["fejs"], ref["dx"], dxb, dPb, ref["P"])
    print("oracle N %d rows %d R %s: kappa(S) %.2e, worst error / bound: P+ %.3e values %.3e" % (P_got.shape[0], rows, rdiag, kS, qP, qv))


@pytest.mark.parametrize("s,rows,wide", [(1, 1, False), (3, 33, False), (3, 65, True), (1, 300, False)])
def test_initialize_reference_against_oracle(s, rows, wide, chi2_table):
    """The oracle's StateHelper::initialize (Givens rotations) against the reference built on Householder reflectors: the gate's chi2,
    the new variable's value and the grown, updated covariance do not depend on the rotation."""
    ur.require_long_double()
    orc = _oracle(chi2_table)
    kinds, ids, vals, fejs, P, handles, cols, H_R, H_L, r, sigma2, value = init_case(orc, s, rows, wide, seed=rows + 7 * s)
    N = P.shape[0]
    acc, nh = orc.initialize(ur.LANDMARK if s == 3 else ur.VEC, value, value, 7000000 + rows, handles, H_R, H_L, r, sigma2, 1.0)
    ref = ur.initialize(P, cols, H_R, H_L, r, sigma2)
    assert acc and ref["chi2"] <= chi2_table[rows]
    P_ref = ref["P_init"] if ref["upd"] is None else ref["upd"]["P"]
    dx = np.zeros(N + s, dtype=ur.LD) if ref["upd"] is None else ref["upd"]["dx"]
    P_got = orc.cov()
    sd = np.sqrt(np.diag(np.asarray(ref["P_init"], dtype=np.float64)))
    assert np.abs(np.asarray(P_got - P_ref, dtype=np.float64) / np.outer(sd, sd)).max() < 1e-9
    new = np.asarray(value, dtype=ur.LD) + ref["dxn"] + dx[N:]
    assert np.abs(np.asarray(orc.var_get(nh)[0] - new, dtype=np.float64)).max() < 1e-9 * (1 + np.abs(value).max())
    got = _state(orc, kinds)[1]
    exp = ur.apply_dx(kinds, vals, ids, dx)
    for h in kinds:
        assert np.abs(np.asarray(got[h] - exp[h], dtype=np.float64)).max() < 1e-10 * (1 + np.abs(vals[h]).max())


# ---- planted mistakes ------------------------------------------------------------------------------------------------------------
def _values_exceed(c, dx, dxb, bad):
    """How far `bad` (a dict like apply_dx's) fails check_update's value checks, in units of their bounds: the distance of every value
    from the reference's, and of every quaternion's norm from 1 (8 eps)."""
    good = ur.apply_dx(c["kinds"], c["vals"], c["ids"], dx)
    vb = ur.value_bounds(c["kinds"], c["vals"], c["ids"], dxb)
    q = max(float((np.abs(np.asarray(bad[h] - good[h], dtype=np.float64)) / vb[h]).max()) for h in c["kinds"])
    for h in c["kinds"]:
        if c["kinds"][h] in (ur.POSE, ur.IMU):
            q = max(q, float(abs(np.sqrt((bad[h][:4] ** 2).sum()) - 1)) / (8 * ur.EPS))
    return q


def _chunks(ref, drop):
    """dx = Y w summed over the OVP_DX_SPLIT chunks of w except `drop`."""
    rr = len(ref["w"])
    chunk = -(-rr // ur.DX_SPLIT)
    w = ref["w"].copy()
    w[drop * chunk:(drop + 1) * chunk] = 0
    return ref["Y"] @ w


@pytest.mark.parametrize("nmod,rows,rdiag", [k for k in CASES if k[1] in (1, 9, 65, 500)])
def test_planted_mistakes_exceed_the_bounds(nmod, rows, rdiag, chi2_table):
    ur.require_long_double()
    orc = _oracle(chi2_table)
    c = ur.update_case(orc, EXTRA[nmod], rows, rdiag, seed=rows + nmod)
    ref = ur.kalman(c["P"], c["cols"], c["H"], c["r"], c["Rdiag"])
    dxb, dPb, _ = ur.kalman_bounds(c["P"], c["cols"], c["H"], ref)
    dx, N = ref["dx"], len(ref["dx"])
    k, v, ids = c["kinds"], c["vals"], c["ids"]
    ratios = {}
    # 7 of the 8 chunks of w: the first chunk holds rows whatever rr is
    ratios["dx from 7 of 8 chunks"] = _values_exceed(c, dx, dxb, ur.apply_dx(k, v, ids, _chunks(ref, 0)))
    # the last 64-row block of state rows (N % 64 of them) left without dx
    bad = dx.copy()
    bad[64 * (N // 64):] = 0
    ratios["last partial 64-row block dropped"] = _values_exceed(c, dx, dxb, ur.apply_dx(k, v, ids, bad))
    ratios["q (x) dq"] = _values_exceed(c, dx, dxb, ur.apply_dx(k, v, ids, dx, functools.partial(ur.quat_update, order="right")))
    ratios["dq not normalised"] = _values_exceed(c, dx, dxb, ur.apply_dx(k, v, ids, dx, functools.partial(ur.quat_update, normalise=False)))
    if ur.flipped(k, v, ids, dx):
        ratios["no sign flip"] = _values_exceed(c, dx, dxb, ur.apply_dx(k, v, ids, dx, functools.partial(ur.quat_update, flip=False)))
    # dx of a landmark applied at its neighbour's state id (the next landmark, same size)
    lm = sorted(c["hs"]["lms"], key=lambda h: ids[h])
    shifted = {**ids, lm[0]: ids[lm[1]]}
    ratios["dx at the neighbour's id"] = _values_exceed(c, dx, dxb, ur.apply_dx(k, v, shifted, dx))
    print("N %d rows %d R %s: %s" % (N, rows, rdiag, ", ".join("%s %.1e" % kv for kv in ratios.items())))
    for name, q in ratios.items():
        assert q > 2.0, "%s moves no value beyond twice its bound (%.3e)" % (name, q)


def test_some_update_case_runs_the_sign_flip_branch(chi2_table):
    """The clones near a half turn give dq (x) q a negative scalar part in the GPU test's cases (same inputs, built here on the oracle)."""
    ur.require_long_double()
    n = 0
    for nmod, rows, rdiag in [k for k in CASES if k[1] in (64, 500)]:
        orc = _oracle(chi2_table)
        c = ur.update_case(orc, EXTRA[nmod], rows, rdiag, seed=rows + nmod)
        ref = ur.kalman(c["P"], c["cols"], c["H"], c["r"], c["Rdiag"])
        n += len(ur.flipped(c["kinds"], c["vals"], c["ids"], ref["dx"]))
    assert n >= 1


def test_initialize_cases_cross_256_columns(chi2_table):
    orc = _oracle(chi2_table)
    out = init_case(orc, 1, 33, True, seed=0)
    assert 1 + len(out[6]) + 1 > 256
