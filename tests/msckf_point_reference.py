"""Long-double reference of the MSCKF point update (the last plan of every ovp_msckf_update call), with a-priori bounds of the library's
two routes to it.  Used by tests/test_gpu_msckf_point_reference.py and pinned against the oracle, planted mistakes included, by
tests/test_cpu_msckf_point_reference.py.

The reference (UpdaterMSCKF.cpp) takes every feature its gate accepts, projects the whitened rows [H_x | r] onto the left null space of
H_f (2m - 3 rows), stacks them over the plan's columns (calibration, then the clones of every track) and hands them to EKFUpdate with
R = I.  The library updates in one of two forms (features_host.inc, msckf_prepare):
- direct: a plan whose stacked rows fit the innovation workspace and one factorisation launch goes into ekf_update_core as it is.  The
  reference is kalman() of the stacked rows; the bound is kalman_bounds plus the projection's rounding (update_reference.projection_bound
  per column, on every row of the feature), carried to the posterior as an information error by plane_update_reference.info_effects;
- compressed: G = [H r]^T [H r] is factored with the zero-pivot rule and the update runs with H = L^T, r = the factor's last row.  The
  reference is built on the library's own G (its accuracy against the stacked rows is tests/test_gpu_compression.py's): the long-double
  factor, its kept system, kalman().  The bound is slam_reference.gram_route_bounds: the factorisation's backward error and the dropped
  pivots through info_effects, plus kalman_bounds of the kept system.
Nothing here is measured."""
import numpy as np

from gate_reference import householder_q3, raw_block
from plane_update_reference import GRAM_TOL, dK_of_rows, info_effects, ld_factor
from slam_reference import gram_bound, gram_route_bounds, kept_system, stack
from update_reference import LD, kalman, kalman_bounds, projection_bound


# ---- the stacked rows (direct form) -------------------------------------------------------------------------------------------------
def project_feature(Hf, Hx, r):
    """(N^T H_x, N^T r, per-column bound of [H_x | r]'s projection) of one feature, N the long-double basis of the left null space of H_f
    (2m - 3 rows)."""
    _, N = householder_q3(np.asarray(Hf, dtype=LD), null_basis=True)
    X = np.hstack([np.asarray(Hx, dtype=LD), np.asarray(r, dtype=LD)[:, None]])
    Z = N.T @ X
    return Z[:, :-1], Z[:, -1], projection_bound(np.asarray(Hf, dtype=np.float64), X)


def stacked_rows(feats, cols):
    """(X, Xb): the projected rows of the accepted features stacked over the plan's columns `cols` (state indices), X = [H | r]
    (long double), and the element-wise bound of their projection's error.  feats: (H_f, H_x, r, ids) per accepted feature, ids the
    state indices of H_x's columns (calibration, then 6 per measurement's clone)."""
    parts, bparts = [], []
    for Hf, Hx, r, ids in feats:
        H, z, pb = project_feature(Hf, Hx, r)
        k = H.shape[0]
        parts.append((H, z, ids))
        bparts.append((np.broadcast_to(pb[:-1], (k, len(pb) - 1)), np.full(k, pb[-1]), ids))
    return stack(parts, cols), np.asarray(stack(bparts, cols), dtype=np.float64)


def raw_features(raw, batch, status, ncal, calib, var_id):
    """(H_f, H_x, r, ids) of every feature with status 1, from the raw whitened rows of ovp_debug_msckf_gram (gate_reference.raw_block):
    ids = the calibration's state indices, then the 6 of each measurement's clone."""
    out = []
    for f in range(int(batch["F"])):
        if int(status[f]) != 1:
            continue
        a, b = int(batch["meas_offset"][f]), int(batch["meas_offset"][f + 1])
        Hf, Hx, r = raw_block(raw, a, b, ncal, False)
        ids = list(calib)
        for k in range(a, b):
            i0 = var_id(int(batch["meas_clone"][k]))
            ids += list(range(i0, i0 + 6))
        out.append((Hf, Hx, r, ids))
    return out


def direct_reference(P, cols, X, Xb):
    """The point update of the stacked rows X (stacked_rows) with its bounds: dict(ref, dxb, dPb (Jacobi-scaled by P))."""
    nc = len(cols)
    cols = list(cols)
    ref = kalman(P, cols, X[:, :nc], X[:, nc], None)
    dxb, dPb, _ = kalman_bounds(P, cols, X[:, :nc], ref)
    Pp, dx = np.asarray(ref["P"], dtype=np.float64), np.asarray(ref["dx"], dtype=np.float64)
    dPi, ddx, _ = info_effects(Pp[:, cols], dx[cols], dK_of_rows(X, Xb))
    sd = np.sqrt(np.diag(np.asarray(P, dtype=np.float64)))
    return dict(ref=ref, dxb=dxb + ddx, dPb=dPb + dPi / np.outer(sd, sd))


# ---- the Gram route (compressed form) -----------------------------------------------------------------------------------------------
def gram_reference(P, cols, G, tol=GRAM_TOL, X=None):
    """The point update on the library's Gram matrix G (nc1 x nc1, lower triangle read) with its bounds: dict(ref, dxb, dPb (Jacobi-
    scaled by P), L, zero, ratio).  X: the stacked rows G was formed from, when G is not the one the update factors (another launch of
    the same rows): their Gram rounding, gram_bound(X) twice, enters the bound."""
    cols = list(cols)
    L, _, _ = ld_factor(G, len(cols), tol)
    Hk, rk = kept_system(L)
    ref = kalman(P, cols, Hk, rk, None)
    dG = None if X is None else 2.0 * gram_bound(X)
    ddx, dPi, dxk, dPk, fac = gram_route_bounds(P, cols, G, ref, tol, dG=dG, kref=ref)
    return dict(ref=ref, dxb=dxk + ddx, dPb=dPk + dPi, **fac)


# ---- point-only scenarios -----------------------------------------------------------------------------------------------------------
CALIB = {0: (0, 0), 6: (1, 0), 8: (0, 1), 14: (1, 1)}  # calibration columns -> (calib_pose, calib_intr)


def point_scenario(ncal, n_clones, F, m_min, m_max, seed=0, dtheta=0.02):
    """synth's point tracks without the time offset (its column is in no MSCKF row) and with ncal calibration columns."""
    from ov_plane_b200 import synth
    cal = CALIB[ncal]
    return synth.make_scenario("tiny_points", seed=seed, n_clones=n_clones, F=F, m_min=m_min, m_max=m_max, dtheta=dtheta, calib_dt=0,
                               calib_pose=cal[0], calib_intr=cal[1])


def cut_to_rows(batch, rows):
    """The batch's features in order, each cut to its newest measurements, until the point plan's rows sum(2m - 3) reach `rows`
    exactly (the last feature taken is cut to what is left).  Returns the cut batch."""
    offs, mc, uv, sel = [0], [], [], []
    left = rows
    for f in range(int(batch["F"])):
        if left == 0:
            break
        a, e = int(batch["meas_offset"][f]), int(batch["meas_offset"][f + 1])
        m = min(e - a, (left + 3) // 2)
        if m < 2:
            continue
        mc.append(batch["meas_clone"][e - m:e])
        uv.append(batch["uv"][e - m:e])
        offs.append(offs[-1] + m)
        sel.append(f)
        left -= 2 * m - 3
    assert left == 0, "the batch has too few measurements for %d rows" % rows
    out = dict(batch)
    for k in ("p_FinG", "p_FinG_original", "featid", "planeid"):
        out[k] = np.ascontiguousarray(batch[k][sel])
    out.update(F=len(sel), meas_offset=np.array(offs, dtype=np.int32), meas_clone=np.ascontiguousarray(np.concatenate(mc), dtype=np.int32),
               uv=np.ascontiguousarray(np.concatenate(uv), dtype=np.float32))
    return out
