"""Long-double references of UpdaterSLAM::update's EKF update and of StateHelper::marginalize_slam, with a-priori bounds of the library's
route to the same update.  Used by tests/test_gpu_slam_reference.py and pinned against the oracle, planted mistakes included, by
tests/test_cpu_slam_references.py.

The reference (UpdaterSLAM.cpp:536-673) stacks the rows of every accepted landmark and hands them to EKFUpdate with R = I: the 3m rows
with the plane for status 1 on a plane (2m bearing rows without one), the 2m bearing rows without the plane columns for status 3 (the
retry without the plane), nothing for status 0; with no row stacked it returns before the update.  The library (slam_host.inc) forms
G = [H r]^T [H r] of the same stack with the split-k Gram kernel (a rejected landmark's rows are zero), factors it with the zero-pivot rule
and updates with H = L^T, r = the factor's last row.  Its error is collected as an element-wise bound dK of the information over [x | r],
carried to the posterior by plane_update_reference.info_effects:
- the Gram sum's rounding: 2 (rows + 2) eps |X|^T |X| (X = the stacked rows);
- the factorisation's backward error: 2 (n + 1) eps |L| |L^T| (n = nc + 1);
- tol G_jj on every dropped pivot, and sqrt(tol G_jj G_kk) on the rest of its column;
then kalman_bounds of the arithmetic of the update itself, on the stacked system and on the kept one (the larger of the two).
Nothing here is measured."""
import numpy as np

from plane_update_reference import GRAM_TOL, factor_dK, info_effects, ld_factor
from update_reference import EPS, LD, kalman, kalman_bounds
from state_reference import marginalize


# ---- the stacked system --------------------------------------------------------------------------------------------------------------
def landmark_rows(Hf, Hx, r, status, has_plane, m, retry_keeps_plane=False, stack_rejected=False):
    """The rows of one landmark the reference stacks, as (J, r) with J = [H_f | H_x] over the landmark's columns then x_ids (H_x's
    columns: calibration, clones, then the plane's 3 when the rows were built with it).  Returns None for a landmark that stacks nothing.
    retry_keeps_plane, stack_rejected: planted mistakes."""
    J = np.hstack([np.asarray(Hf, dtype=LD), np.asarray(Hx, dtype=LD)])
    r = np.asarray(r, dtype=LD)
    if status == 0 and not stack_rejected:
        return None
    if status == 1 or (status == 3 and retry_keeps_plane) or not has_plane:
        return J, r
    return J[:2 * m, :J.shape[1] - 3], r[:2 * m]  # the retry: bearing rows, no plane columns


def gate_dof(m, with_plane, plane_rows=3):
    """The chi2 table entry a landmark's gate reads (UpdaterSLAM.cpp:587-596, res.rows()): 3m with the plane row, 2m on the bearing rows
    (without a plane, or on the retry).  plane_rows=2: the planted mistake."""
    return (plane_rows if with_plane else 2) * m


def status_one_hot(m, on_plane, idx, dof=gate_dof):
    """The status a landmark gets from a table that is zero except at entry idx (every positive chi2 fails a zero threshold and passes
    an unbounded one): 1 when its first gate reads idx, 3 when it is on a plane and its retry reads idx, else 0."""
    if idx == dof(m, on_plane):
        return 1
    if on_plane and idx == dof(m, False):
        return 3
    return 0


def stack(parts, cols):
    """X = [H | r] (rows x (nc + 1), long double) of the landmarks' stacked rows over the compact columns `cols` (state indices).  parts:
    a list of (J, r, ids) with ids the state indices of J's columns (a landmark without rows is left out)."""
    col_of = {int(s): c for c, s in enumerate(cols)}
    nc = len(cols)
    rows = sum(p[0].shape[0] for p in parts)
    X = np.zeros((rows, nc + 1), dtype=LD)
    at = 0
    for J, r, ids in parts:
        k = J.shape[0]
        idx = [col_of[int(s)] for s in ids]
        X[at:at + k, idx] = J
        X[at:at + k, nc] = r
        at += k
    return X


def slam_update_reference(P, cols, X):
    """EKFUpdate with R = I of the stacked rows X over the state columns cols, in long double (update_reference.kalman), or None when
    nothing was stacked (the reference returns before the update)."""
    if X.shape[0] == 0:
        return None
    nc = len(cols)
    return kalman(P, list(cols), X[:, :nc], X[:, nc], None)


# ---- the library's route: the Gram factor --------------------------------------------------------------------------------------------
def gram_ld(X):
    """X^T X in long double: the Gram matrix the library forms."""
    X = np.asarray(X, dtype=LD)
    return X.T @ X


def gram_bound(X):
    """Element-wise bound of the Gram kernel's rounding of X^T X: 2 (rows + 2) eps |X|^T |X|."""
    aX = np.abs(np.asarray(X, dtype=np.float64))
    return 2.0 * (X.shape[0] + 2) * EPS * (aX.T @ aX)


def kept_system(L):
    """(H, r) of the update the library runs from the factor L (nc1 x nc) of G: H = L^T over the x columns, r the factor's last row."""
    nc = L.shape[1]
    return L[:nc, :].T.copy(), L[nc, :].copy()


def slam_bounds(P, cols, X, G, ref, tol=GRAM_TOL):
    """(dx bound, P+ bound Jacobi-scaled by P, factor info) of the library's update against slam_update_reference(P, cols, X): G the
    library's Gram matrix (nc1 x nc1, lower triangle read), ref the reference.  The factor info: dict(L, zero, ratio)."""
    nc = len(cols)
    L, zero, ratio = ld_factor(G, nc, tol)
    aL = np.abs(np.asarray(L, dtype=np.float64))
    dG = gram_bound(X) + 2.0 * (nc + 2) * EPS * (aL @ aL.T)
    dK = factor_dK(L, zero, G, tol, dG=dG)
    # a dropped pivot discards its whole column of the Schur complement, not only its diagonal: |S_kj| <= sqrt(S_jj S_kk) <=
    # sqrt(tol G_jj G_kk) off the diagonal
    g = np.sqrt(np.abs(np.diag(np.asarray(G, dtype=np.float64))))
    for j in zero:
        off = np.sqrt(tol) * g[j] * g
        off[j] = 0.0
        dK[j, :] += off
        dK[:, j] += off
    Pp, dx = np.asarray(ref["P"], dtype=np.float64), np.asarray(ref["dx"], dtype=np.float64)
    dPi, ddx, _ = info_effects(Pp[:, list(cols)], dx[list(cols)], dK)
    dxb, dPb, _ = kalman_bounds(P, list(cols), X[:, :nc], ref)
    Hk, rk = kept_system(L)
    kref = kalman(P, list(cols), Hk, rk, None)
    dxk, dPk, _ = kalman_bounds(P, list(cols), Hk, kref)
    sd = np.sqrt(np.diag(np.asarray(P, dtype=np.float64)))
    return np.maximum(dxb, dxk) + ddx, np.maximum(dPb, dPk) + dPi / np.outer(sd, sd), dict(L=L, zero=zero, ratio=ratio)


# ---- StateHelper::marginalize_slam ---------------------------------------------------------------------------------------------------
def marginalize_slam(P, landmarks, max_aruco_features, rule=">"):
    """StateHelper::marginalize_slam (StateHelper.cpp:638-652): every landmark with should_marg and featid > 4 max_aruco_features is
    marginalised (state_reference.marginalize), in ascending featid (the order of State::_features_SLAM), the ids behind it shifting
    by 3.  landmarks: {featid: (state id, should_marg)}.  rule ">=": the planted mistake.  Returns (P, removed featids)."""
    P = np.asarray(P)
    ids = {f: i for f, (i, _) in landmarks.items()}
    removed = []
    for f in sorted(landmarks):
        flag = landmarks[f][1]
        lim = 4 * max_aruco_features
        if not (flag and (f > lim if rule == ">" else f >= lim)):
            continue
        mid = ids[f]
        P = marginalize(P, mid, 3)
        for g in ids:
            if ids[g] > mid:
                ids[g] -= 3
        removed.append(f)
    return P, removed
