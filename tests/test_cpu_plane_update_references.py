"""Pins tests/plane_update_reference.py on the CPU: the long-double kept system against a Givens restatement of
UpdaterPlane::measurement_compress_inplace, its chi2 and posterior against numpy, and planted mistakes (the wrong dof, the dropped Schur
rows kept, the plane's columns in the wrong order) moving a checked quantity by more than twice its bound."""
import numpy as np
import pytest

import plane_update_reference as pr
import update_reference as ur


def givens_compress(X, ncx):
    """measurement_compress_inplace on [H_x | H_cp | r] in long double with Givens rotations (UpdaterPlane.cpp:522-551): zero every
    column of H_x below its diagonal from the bottom up, keep the top min(rows, ncx) rows."""
    A = np.array(X, dtype=ur.LD)
    rows = A.shape[0]
    for j in range(ncx):
        for i in range(rows - 1, j, -1):
            a, b = A[i - 1, j], A[i, j]
            if b == 0:
                continue
            rr = np.sqrt(a * a + b * b)
            c, s = a / rr, b / rr
            top, bot = A[i - 1].copy(), A[i].copy()
            A[i - 1], A[i] = c * top + s * bot, -s * top + c * bot
    return A[:min(rows, ncx)]


def case(rows, ncx, seed, N=None):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((rows, ncx + 4))
    N = N or ncx + 12
    d = np.exp(rng.uniform(-3.0, 0.0, N))
    P = ur.correlated(d, seed)
    ids = sorted(rng.choice(N, size=ncx + 3, replace=False).tolist())
    return X, P, ids[:ncx], ids[ncx:]


@pytest.mark.parametrize("rows,ncx", [(40, 24), (61, 30), (90, 60)])
def test_kept_system_against_givens(rows, ncx):
    """G's long-double factor over the x columns spans the same kept system as the Givens compression (rows > ncx: the kept rows' Gram
    matrices agree; it does not depend on the rotations)."""
    ur.require_long_double()
    X, _, _, _ = case(rows, ncx, rows)
    G = X.T @ X
    L, zero, _ = pr.ld_factor(G, ncx)
    assert zero == []
    K = np.asarray(L, dtype=ur.LD) @ np.asarray(L, dtype=ur.LD).T
    R = givens_compress(X, ncx)
    Kg = R.T @ R
    err = float(np.abs(np.asarray(K - Kg, dtype=np.float64)).max() / np.abs(G).max())
    assert err < 1e-15, err


@pytest.mark.parametrize("in_state", [True, False])
@pytest.mark.parametrize("rows,ncx", [(20, 24), (40, 24)])
def test_chi2_and_posterior_against_numpy(in_state, rows, ncx):
    """well-conditioned systems: the reference's chi2 and P+ against numpy's float64 Kalman update of the same kept system"""
    ur.require_long_double()
    X, P, x_ids, pl = case(rows, ncx, 7 * rows + in_state)
    X[:, -1] *= 0.1
    G = X.T @ X
    form, npiv, dof, _ = pr.form_of(in_state, rows, ncx)
    if form == "direct":
        rf = pr.plane_reference(P, x_ids, pl, ncx, form, X=X.astype(ur.LD), Xb=np.zeros_like(X))
    else:
        rf = pr.plane_reference(P, x_ids, pl if in_state else None, ncx, form, G=G, npiv=npiv)
    H, r = np.asarray(rf["H"], dtype=np.float64), np.asarray(rf["r"], dtype=np.float64)
    ids = x_ids + (pl if in_state else [])
    S = H @ P[np.ix_(ids, ids)] @ H.T + np.eye(H.shape[0])
    chi2 = r @ np.linalg.solve(S, r)
    Pp = P - P[:, ids] @ H.T @ np.linalg.solve(S, H @ P[ids, :])
    assert abs(chi2 - float(rf["chi2"])) <= 1e-10 * chi2
    assert np.abs(Pp - np.asarray(rf["ref"]["P"], dtype=np.float64)).max() <= 1e-12 * np.abs(P).max()
    # the chi2 does not depend on the rotation that compresses the system: the reference's own definition from the raw rows
    own, _ = pr.reference_chi2(X.astype(ur.LD), ncx, P, x_ids, pl if in_state else None)
    assert abs(float(own) - float(rf["chi2"])) <= 1e-12 * float(own) + rf["chi2b"]


def test_form_and_dof():
    assert pr.form_of(True, 57, 60)[0::2] == ("direct", 57)
    assert pr.form_of(True, 60, 60)[0::2] == ("direct", 60)
    assert pr.form_of(True, 61, 60)[:3] == ("compressed", 60, 60)
    assert pr.form_of(False, 60, 60)[:3] == ("out", 63, 57)
    assert pr.form_of(False, 61, 60)[:4] == ("out", 60, 57, 60)
    assert pr.form_of(False, 3, 60)[2] == 1


def test_planted_mistakes_exceed_twice_their_bound(chi2_table):
    """the wrong dof (min(rows, ncx) for max(1, min(rows, ncx) - 3), a plane not in the state) turns the reference's gate decision, its
    chi2 more than twice its bound from both thresholds; keeping the rows the compression drops moves chi2; reversing the plane's three
    columns moves P+ (Jacobi-scaled) by more than twice its bound"""
    ur.require_long_double()
    rows, ncx = 40, 24
    X, P, x_ids, pl = case(rows, ncx, 3)
    X[:, -1] *= 0.3
    X[ncx:, ncx:ncx + 3] *= 4.0  # H_cp content on the rows the compression drops
    form, npiv, dof, rows_ref = pr.form_of(False, rows, ncx)
    assert dof == rows_ref - 3
    lo, hi = chi2_table[dof], chi2_table[rows_ref]
    out = pr.plane_reference(P, x_ids, None, ncx, form, G=X.T @ X, npiv=npiv)
    X[:, -1] *= np.sqrt(0.5 * (lo + hi) / float(out["chi2"]))  # chi2 scales with |r|^2: halfway between the two thresholds
    out = pr.plane_reference(P, x_ids, None, ncx, form, G=X.T @ X, npiv=npiv)
    c, b = float(out["chi2"]), out["chi2b"]
    assert lo + 2 * b < c < hi - 2 * b
    assert (c <= lo) != (c <= hi), "the planted dof does not change the decision"
    G = X.T @ X
    rf = pr.plane_reference(P, x_ids, pl, ncx, "compressed", G=G, npiv=ncx)
    full = ur.kalman(P, x_ids + pl, X[:, :ncx + 3], X[:, ncx + 3], None)
    assert abs(float(pr.chi2_of(full)) - float(rf["chi2"])) > 2 * rf["chi2b"]
    bad = ur.kalman(P, x_ids + pl[::-1], rf["H"], rf["r"], None)
    sd = np.sqrt(np.diag(P))
    e = np.abs(np.asarray(bad["P"] - rf["ref"]["P"], dtype=np.float64)) / np.outer(sd, sd)
    assert (e / np.maximum(rf["dPb"], 1e-300)).max() > 2.0


@pytest.mark.parametrize("rows,ncx", [(20, 24), (40, 24)])
def test_well_defined_chi2_and_dropped_share(rows, ncx):
    """The raw rows' QR with the zero-pivot rule gives the factor's system (rotation-independent chi2); with rows <= ncx and a plane not
    in the state, the reference's chi2 is that part plus the residual on the rows without Jacobian (three planted ones here)."""
    ur.require_long_double()
    X, P, x_ids, _ = case(rows, ncx, 11 * rows)
    X[:, -1] *= 0.2
    if rows <= ncx:
        X[-3:, :-1] = 0.0  # three rows without Jacobian
    form, npiv, _, _ = pr.form_of(False, rows, ncx)
    rf = pr.plane_reference(P, x_ids, None, ncx, form, G=X.T @ X, npiv=npiv)
    wd, dropped, zero, _, rest = pr.reference_chi2_well_defined(X.astype(ur.LD), ncx, npiv, P, x_ids, None)
    assert zero == rf["zero"]
    assert abs(float(wd) - float(rf["chi2"])) <= 1e-12 * float(wd) + rf["chi2b"]
    if rows <= ncx:
        assert len(zero) == ncx + 3 - (rows - 3) and float(dropped) > 0  # rank: the rows with Jacobian
        own, _ = pr.reference_chi2(X.astype(ur.LD), ncx, P, x_ids, None)
        assert abs(float(own) - float(wd) - float(dropped)) <= 1e-12 * float(own)
        assert abs(float(dropped) - float((X[-3:, -1] ** 2).sum())) <= 1e-12 * float(dropped)
