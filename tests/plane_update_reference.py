"""Long-double references of the per-plane stacked system of the MSCKF update: what msckf_launch_body does with a plane's rows after the
feature kernel, in each of its forms, and what ovp_plane_init hands to StateHelper::initialize.  Used by
tests/test_gpu_plane_update_reference.py and pinned, planted mistakes included, by tests/test_cpu_plane_update_references.py.

The forms (features_host.inc, msckf_prepare and msckf_launch_body), with ncx the plan's x columns and rows = sum(3 m - 3):
- in-state direct (rows <= ncx): the stacked projected rows [H_x | H_cp | r] go into the EKF update as they are, chi2 dof = rows;
- in-state compressed (rows > ncx): the Gram matrix G of [H_x | H_cp | r] is factored over the ncx x columns; the update uses
  H = L^T over [x | cp], r = the factor's last row; dof = ncx;
- not in the state: G is factored over ncx columns (rows > ncx) or ncx + 3 (rows <= ncx); W = [R_xc | R | z] (plane_W_kernel), three
  reflectors on its cp columns, the remaining rowsW - 3 rows update the state; dof = max(1, min(rows, ncx) - 3);
- ovp_plane_init: the same W to StateHelper::initialize, dof = min(rows, ncx).

Error bounds are first-order and a priori.  Every perturbation of the library's system is collected as an element-wise bound dK of the
kept information K = [H r]^T [H r] over [x | cp | r]; its effect on the posterior is that of a perturbed information matrix on the
joint (state, cp) problem (cp with a flat prior when the plane is not in the state):
    |dP+| <= |A| dK |A|^T,   |d dx| <= |A| (dK[:, r] + dK |x^|),   |d chi2| <= v^T dK v,  v = [|x^|; 1],
with A the posterior cross-covariance of the state with the system's unknowns and x^ their posterior mean (chi2 = min over the unknowns
of the whitened residual plus the prior term, whose derivative in K is [-x^; 1] [-x^; 1]^T).  dK collects:
- the Gram factorisation's backward error: the computed L is the exact factor of G + dG, |dG| <= 2 (n + 1) eps |L| |L^T| (the bound
  tests/test_gpu_compression.py checks); on the rows the factor does not pivot, K = G_tp G_pp^-1 G_pt, so with E = G_pp^-1 G_pt
  dK_tt <= |dG_tp| |E| + |E^T| |dG_pt| + |E^T| |dG_pp| |E|;
- the zero-pivot rule: tol G_jj on every dropped direction;
- the Householder projections of the feature rows (direct form) and of W's cp columns: projection_bound per column.
Nothing here is measured."""
import numpy as np

from gate_reference import gate_bound, householder_q3, raw_block
from update_reference import BOUND_C, EPS, LD, householder_project, kalman, kalman_bounds, projection_bound

GRAM_TOL = 1e-11  # Ctx::gram_tol, the zero-pivot rule of the Gram factorisation
PIVOT_MARGIN = 100.0  # every pivot must lie this far from the threshold, on either side


# ---- the plan's forms -------------------------------------------------------------------------------------------------------------
def form_of(in_state, rows, ncx):
    """(form, npiv, dof, rows_ref) of a plane plan, restating msckf_prepare / msckf_launch_body."""
    rows_ref = min(rows, ncx)
    if in_state:
        return ("direct", None, rows, rows_ref) if rows <= ncx else ("compressed", ncx, ncx, rows_ref)
    return ("out", ncx if rows > ncx else ncx + 3, max(1, rows_ref - 3), rows_ref)


# ---- the direct form: raw rows, projected and stacked ------------------------------------------------------------------------------
def stacked_rows(raw, batch, sel, ncal, ncx, col_of, var_id):
    """The plan's stacked system [H_x | H_cp | r] (rows x (ncx + 4), long double) from the raw whitened rows of its features: each
    feature's rows projected onto the left null space of its H_f (householder_q3), in the plan's column order (col_of: state index ->
    compact column).  Also returns the element-wise bound of the projection's error (projection_bound per column, on every row of the
    feature) and the list of (H_f, X) blocks."""
    blocks, bnds, parts = [], [], []
    for f in sel:
        a, b = int(batch["meas_offset"][f]), int(batch["meas_offset"][f + 1])
        Hf, Hx, r = raw_block(raw, a, b, ncal, True)
        X = np.hstack([Hx, r[:, None]])
        _, N = householder_q3(Hf, null_basis=True)
        Z = N.T @ X
        idx = list(range(ncal))
        for k in range(a, b):
            c0 = col_of[var_id(int(batch["meas_clone"][k]))]
            idx += list(range(c0, c0 + 6))
        idx += [ncx, ncx + 1, ncx + 2, ncx + 3]
        out = np.zeros((Z.shape[0], ncx + 4), dtype=LD)
        out[:, idx] = Z
        bd = np.zeros((Z.shape[0], ncx + 4))
        bd[:, idx] = projection_bound(Hf, X)[None, :]
        blocks.append(out)
        bnds.append(bd)
        parts.append((Hf, X))
    return np.vstack(blocks), np.vstack(bnds), parts


def dK_of_rows(X, bound):
    """|dX|^T |X| + |X|^T |dX| + |dX|^T |dX|: the information's bound for rows X known to |dX| <= bound element-wise."""
    aX = np.abs(np.asarray(X, dtype=np.float64))
    return bound.T @ aX + aX.T @ bound + bound.T @ bound


# ---- the compressed forms: the Gram factor ------------------------------------------------------------------------------------------
def ld_factor(G, npiv, tol=GRAM_TOL):
    """Right-looking long-double Cholesky of the lower triangle of G over its first npiv columns with the zero-pivot rule (pivot <= tol
    times the column's original diagonal: the column is zero).  Returns (L (n x npiv), zeroed columns, pivot / threshold per column)."""
    n = G.shape[0]
    A = np.tril(np.asarray(G)).astype(LD)
    A = A + np.tril(A, -1).T
    d0 = np.diag(np.asarray(G)).astype(LD).copy()
    L = np.zeros((n, npiv), dtype=LD)
    zero, ratio = [], []
    for j in range(npiv):
        d = A[j, j]
        ratio.append(float(d / (tol * d0[j])) if d0[j] > 0 else 0.0)
        if not d > tol * d0[j]:
            zero.append(j)
            continue
        l = A[j:, j] / np.sqrt(d)
        L[j:, j] = l
        A[j:, j:] -= np.outer(l, l)
    return L, zero, np.array(ratio)


def kept_system(L, ncx, in_state):
    """The system the library updates with, from the factor L ((ncx + 4) x npiv) of G: in the state, H = L^T over [x | cp] and r the
    factor's last row; not in the state, W = [R_xc | R | z] (plane_W_kernel's layout), projected by three reflectors on its cp columns
    (householder_cols_kernel's), and the rowsW - 3 rows below them over the x columns.  Returns dict(H, r, W, Wp)."""
    npiv = L.shape[1]
    R = L.T  # npiv x (ncx + 4): [x | cp | r]
    if in_state:
        return dict(H=R[:, :ncx + 3].copy(), r=R[:, ncx + 3].copy(), W=None, Wp=None)
    W = np.hstack([R[:, ncx:ncx + 3], R[:, :ncx], R[:, ncx + 3:ncx + 4]])
    Wp = householder_project(W, 3)
    return dict(H=Wp[3:, 3:3 + ncx].copy(), r=Wp[3:, 3 + ncx].copy(), W=W, Wp=Wp)


def factor_dK(L, zero, G, tol=GRAM_TOL, dG=None):
    """Element-wise bound of the kept information's error over [x | cp | r] from the factorisation (module docstring).  dG: another
    element-wise bound of G's error to carry through instead of the factorisation's backward error."""
    n, npiv = L.shape
    aL = np.abs(np.asarray(L, dtype=np.float64))
    if dG is None:
        dG = 2.0 * (n + 1) * EPS * (aL @ aL.T)
    p, t = np.arange(npiv), np.arange(npiv, n)
    keep = np.array([j for j in p if j not in zero], dtype=int)
    E = np.zeros((npiv, len(t)))
    if len(t) and len(keep):
        Lp = np.asarray(L[np.ix_(keep, keep)], dtype=np.float64)
        Lt = np.asarray(L[np.ix_(t, keep)], dtype=np.float64)
        E[keep] = np.linalg.solve(Lp.T, Lt.T)  # G_pp^-1 G_pt over the kept pivots
    aE = np.abs(E)
    dK = dG.copy()
    if len(t):
        dK[np.ix_(t, t)] = dG[np.ix_(t, p)] @ aE + aE.T @ dG[np.ix_(p, t)] + aE.T @ dG[np.ix_(p, p)] @ aE
    for j in zero:
        dK[j, j] += tol * abs(float(G[j, j]))
    return dK


# ---- sensitivity of the update to its information -----------------------------------------------------------------------------------
def joint_unknowns(ref, K, x_ids, plane_ids, ncx):
    """(A, xhat): the posterior cross-covariance of the whole state with the system's unknowns [x columns | cp] and their posterior
    mean.  ref: kalman() of the kept system; K: its information over [x | cp | r] (float64).  A plane in the state: its columns are
    state columns.  Not in the state: cp has a flat prior, cp^ = K_cc^-1 (k_c - K_cx dx_x) and Cov(state, cp) = -P+[:, x] K_xc K_cc^-1."""
    Pp = np.asarray(ref["P"], dtype=np.float64)
    dx = np.asarray(ref["dx"], dtype=np.float64)
    if plane_ids is not None:
        ids = list(x_ids) + list(plane_ids)
        return Pp[:, ids], dx[ids]
    x, c = np.arange(ncx), np.arange(ncx, ncx + 3)
    Kcc_inv = np.linalg.inv(K[np.ix_(c, c)])
    T = K[np.ix_(x, c)] @ Kcc_inv
    A = np.hstack([Pp[:, x_ids], -Pp[:, x_ids] @ T])
    cph = Kcc_inv @ (K[c, ncx + 3] - K[np.ix_(c, x)] @ dx[x_ids])
    return A, np.concatenate([dx[x_ids], cph])


def info_effects(A, xhat, dK):
    """(dP (N x N), ddx (N), dchi2) of an information error dK over [unknowns | r] (module docstring), times BOUND_C."""
    u = len(xhat)
    aA = np.abs(A)
    dKu = dK[:u, :u]
    dP = aA @ dKu @ aA.T
    ddx = aA @ (dK[:u, u] + dKu @ np.abs(xhat))
    v = np.concatenate([np.abs(xhat), [1.0]])
    return BOUND_C * dP, BOUND_C * ddx, BOUND_C * float(v @ dK[:u + 1, :u + 1] @ v)


def plane_reference(P, x_ids, plane_ids, ncx, form, X=None, Xb=None, G=None, npiv=None, tol=GRAM_TOL):
    """The long-double update of one plane plan with its bounds.  form "direct": X, Xb = stacked_rows(); "compressed" / "out": G (the
    library's Gram matrix) and npiv.  plane_ids: the plane's state columns, None when it is not in the state.  Returns dict(ref (kalman of
    the kept system), H, r, dx, dxb, dPb (Jacobi-scaled by P), chi2, chi2b, zero, ratio, sys, K, dK)."""
    Pl = np.asarray(P, dtype=np.float64)
    zero, ratio, sysd = [], None, None
    if form == "direct":
        H, r = X[:, :ncx + 3], X[:, ncx + 3]
        K = np.asarray(X, dtype=np.float64).T @ np.asarray(X, dtype=np.float64)
        dK = dK_of_rows(X, Xb)
    else:
        L, zero, ratio = ld_factor(G, npiv, tol)
        sysd = kept_system(L, ncx, plane_ids is not None)
        H, r = sysd["H"], sysd["r"]
        L64 = np.asarray(L, dtype=np.float64)
        K = L64 @ L64.T
        dK = factor_dK(L, zero, G, tol)
        if plane_ids is None:  # the three reflectors on W's cp columns, on the rows below them over [x | r]
            W = sysd["W"]
            pb = projection_bound(W[:, :3], W[:, 3:])
            idx = list(range(ncx)) + [ncx + 3]
            dK[np.ix_(idx, idx)] += dK_of_rows(sysd["Wp"][3:, 3:], np.broadcast_to(pb, (W.shape[0] - 3, ncx + 1)))
    ids = list(x_ids) + (list(plane_ids) if plane_ids is not None else [])
    ref = kalman(P, ids, H, r, None)
    dxb, dPb, _ = kalman_bounds(P, ids, H, ref)
    A, xhat = joint_unknowns(ref, K, x_ids, plane_ids, ncx)
    dPi, ddx, dchi = info_effects(A, xhat, dK)
    sd = np.sqrt(np.diag(Pl))
    return dict(ref=ref, H=H, r=r, dx=ref["dx"], dxb=dxb + ddx, dPb=dPb + dPi / np.outer(sd, sd), chi2=chi2_of(ref),
                chi2b=kept_gate_bound(ref, H, r, P, ids) + dchi, zero=zero, ratio=ratio, sys=sysd, K=K, dK=dK, A=A, xhat=xhat,
                L=None if form == "direct" else L)


def raw_chi2_bound(rf, G, X, Xb, tol=GRAM_TOL):
    """Bound of the chi2 difference between the reference built on the library's G (rf) and the same reference built on the raw rows X
    the feature kernel produced (long-double projection, error bound Xb): G differs from X^T X by the kernel's projection and by the
    rounding of the sum, |dG| <= dK_of_rows(X, Xb) + 2 (rows + 2) eps |X|^T |X|, carried through the factor as factor_dK does."""
    aX = np.abs(np.asarray(X, dtype=np.float64))
    dG = dK_of_rows(X, Xb) + 2.0 * (X.shape[0] + 2) * EPS * (aX.T @ aX)
    dK = factor_dK(rf["L"], rf["zero"], G, tol, dG=dG)
    return info_effects(rf["A"], rf["xhat"], dK)[2]


def chi2_of(ref):
    return (ref["w"] * ref["w"]).sum()


def kept_gate_bound(ref, H, r, P, ids):
    """gate_reference.gate_bound of the kept system (no projection: kappa_f = 1)."""
    P = np.asarray(P)
    return gate_bound(chi2_of(ref), ref["S"], H, r, P[np.ix_(ids, ids)], 1.0, H.shape[0] + H.shape[1])


# ---- the reference's own chi2 definition --------------------------------------------------------------------------------------------
def reference_chi2(X, ncx, P, x_ids, plane_ids):
    """UpdaterPlane's chi2 from the stacked raw system X = [H_x | H_cp | r] (long double): no compression when rows <= ncx, else the top
    ncx rows of a Householder QR over the x columns (measurement_compress_inplace keeps them); then, without the plane in the state, its
    3 columns projected away (3 reflectors).  Returns (chi2, rows of the system it is taken on)."""
    X = np.asarray(X, dtype=LD)
    if X.shape[0] > ncx:
        X = householder_project(X, ncx)[:ncx]
    if plane_ids is None:
        W = np.hstack([X[:, ncx:ncx + 3], X[:, :ncx], X[:, ncx + 3:]])
        W = householder_project(W, 3)[3:]
        H, r, ids = W[:, 3:3 + ncx], W[:, 3 + ncx], list(x_ids)
    else:
        H, r, ids = X[:, :ncx + 3], X[:, ncx + 3], list(x_ids) + list(plane_ids)
    ref = kalman(P, ids, H, r, None)
    return chi2_of(ref), H.shape[0]


def skip_qr(X, npiv, tol=GRAM_TOL):
    """Householder QR of X (long double) over its first npiv columns with the zero-pivot rule restated on the rows: column j is skipped
    (no reflector, no row consumed) when what is left of it below the consumed rows has |x|^2 <= tol times its original |x|^2, the
    Schur pivot the Gram factor compares.  Returns (R: the k consumed rows, rest: the rows below, whose pivoted columns are zero,
    skipped columns, pivot / threshold per column)."""
    A = np.array(X, dtype=LD)
    d0 = (A * A).sum(axis=0)
    k, zero, ratio = 0, [], []
    for j in range(npiv):
        x = A[k:, j]
        nrm2 = (x * x).sum()
        ratio.append(float(nrm2 / (tol * d0[j])) if d0[j] > 0 else 0.0)
        if not nrm2 > tol * d0[j]:
            zero.append(j)
            continue
        nrm = np.sqrt(nrm2)
        alpha = -nrm if x[0] > 0 else nrm
        v = x.copy()
        v[0] -= alpha
        A[k:, j:] -= (2 / (v * v).sum()) * np.outer(v, v @ A[k:, j:])
        A[k + 1:, j] = 0
        k += 1
    return A[:k], A[k:], zero, np.array(ratio)


def reference_chi2_well_defined(X, ncx, npiv, P, x_ids, plane_ids, tol=GRAM_TOL):
    """The reference's own chi2 from the raw rows on its well-defined part: the rows of a QR of X over the pivot columns whose Jacobian
    lies outside the numerical null space of [H_x (H_cp)] (skip_qr, rank decided by the same relative tolerance); then, without the plane
    in the state, its 3 columns projected away.  Returns (chi2, dropped, zero, ratio): dropped = |r|^2 on the rows left below, the
    residual's own Schur pivot."""
    R, rest, zero, ratio = skip_qr(X, npiv, tol)
    if plane_ids is None:
        W = np.hstack([R[:, ncx:ncx + 3], R[:, :ncx], R[:, ncx + 3:]])
        W = householder_project(W, 3)[3:]
        H, r, ids = W[:, 3:3 + ncx], W[:, 3 + ncx], list(x_ids)
    else:
        H, r, ids = R[:, :ncx + 3], R[:, ncx + 3], list(x_ids) + list(plane_ids)
    ref = kalman(P, ids, H, r, None)
    return chi2_of(ref), (rest[:, -1] * rest[:, -1]).sum(), zero, ratio, rest


def rest_dK(rest):
    """The information the rows below a skip_qr carry besides their residual's square (their Jacobian is at most the pivot rule's
    size): |J|^T |X| + |X|^T |J| with J = those rows without their residual column."""
    aX = np.abs(np.asarray(rest, dtype=np.float64))
    aJ = aX.copy()
    aJ[:, -1] = 0.0
    return aJ.T @ aX + aX.T @ aJ
