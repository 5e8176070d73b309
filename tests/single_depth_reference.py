"""Long-double restatement of UpdaterSLAM's single-depth landmarks, ANCHORED_INVERSE_DEPTH_SINGLE (representation 5), built on the helpers of
feature_jacobian_reference (the representation Jacobians), update_reference (the Householder projection, StateHelper::initialize) and
slam_reference (the EKF update of a stack).

ov_type::Landmark of representation 5 (ov_core, not in the tree): a Landmark of size 1 whose value is the inverse depth rho = 1/z of the point
in its anchor camera; it carries the bearing it was set from, uv_norm_zero = rho p_FinA = [x/z, y/z, 1], and a first-estimate copy
uv_norm_zero_fej; get_xyz = uv_norm_zero / rho.  The library keeps [rho, uv_norm_zero] in one value row (ovp_slam_get_xyz reads it back).

- jacobian_block: the rows UpdaterSLAM::update / delayed_init stack for such a landmark (UpdaterSLAM.cpp:260-283, 503-516): the Jacobians of
  ANCHORED_MSCKF_INVERSE_DEPTH at p_FinA, H_f's last column moved to the state side, the two bearing columns projected out.
- anchor_change: UpdaterSLAM::perform_anchor_change (:706-850) for the form: Phi (1 x cols) with H_f_new's pseudo-inverse, the re-anchored
  point, rho and the bearing of value and first estimate."""
import numpy as np

import feature_jacobian_reference as fjr
import update_reference as ur

LD = np.longdouble


def set_from_xyz(p):
    """Landmark::set_from_xyz for representation 5: [rho, uv_norm_zero] of the anchored point p (generic dtype)"""
    rho = 1 / p[2]
    return np.array([rho, rho * p[0], rho * p[1], rho * p[2]], dtype=np.asarray(p).dtype)


def get_xyz(v):
    """Landmark::get_xyz for representation 5: uv_norm_zero / rho of the 4-vector [rho, uv_norm_zero]"""
    return np.asarray(v[1:4]) / v[0]


def chain(Hf_bearing, Hx, xo, anc, sizes, rep_terms, calib_pose):
    """the bearing rows (w dz/dp_FinG of ovp_feature_jacobian_full at p_FinG, long double) chained onto ANCHORED_MSCKF_INVERSE_DEPTH with
    rep_terms = fjr.representation_jacobians(4, ...): (J_f (rows x 3), H_x with the anchor's columns (appended when no measurement was taken
    from it), x order)"""
    _, _, L, Ha, Hc = rep_terms
    Hx, xo = fjr.ld(Hx).copy(), list(xo)
    if anc not in xo:
        xo.append(anc)
        Hx = np.hstack([Hx, np.zeros((Hx.shape[0], 6), dtype=LD)])
    c = sum(sizes[h] for h in xo[:xo.index(anc)])
    Hf = fjr.ld(Hf_bearing)
    Hx[:, c:c + 6] += Hf @ Ha
    if calib_pose:
        Hx[:, 0:6] += Hf @ Hc
    return Hf @ L, Hx, xo


def project(Jf, Hx, r):
    """[H_rho | H_x | r] after the two bearing columns of J_f are projected out (update_reference.householder_project: the kernel's
    reflectors): (H_rho (rows - 2), H_x (rows - 2 x n), r (rows - 2))"""
    X = ur.householder_project(np.hstack([Jf, Hx, np.asarray(r, dtype=LD)[:, None]]), 2)[2:, 2:]
    return X[:, 0], X[:, 1:-1], X[:, -1]


def anchor_change(v, vf, old_val, old_fej, new_val, new_fej, calib, do_fej, calib_pose):
    """perform_anchor_change of a single-depth landmark [rho, uv_norm_zero] (value v, first estimate vf) from the old to the new anchor
    clone (7-vectors: JPL quaternion, position; value and first estimate) with extrinsics calib.  Returns dict(Phi (1 x cols, long double)
    over [old anchor 6][extrinsics 6 when calibrated][new anchor 6 when another clone][landmark 1], value, fej (the new 4-vectors),
    pA, pAf (the re-anchored points))."""
    v, vf = fjr.ld(v), fjr.ld(vf)
    ov, of, nv, nf, cal = (fjr.ld(a) for a in (old_val, old_fej, new_val, new_fej, calib))
    pA, pAf = get_xyz(v), get_xyz(vf)
    # the point seen from the new anchor camera, best and first estimates (:739-777; the extrinsics have no first estimate)
    pA_new = fjr.global_to_anchor(nv, cal, fjr.anchor_to_global(ov, cal, pA))
    pAf_new = fjr.global_to_anchor(nf, cal, fjr.anchor_to_global(of, cal, pAf))
    _, _, Lo, Hao, Hco = fjr.representation_jacobians(5, do_fej, pA, pA, ov, of, cal)
    _, _, Ln, Han, Hcn = fjr.representation_jacobians(5, do_fej, pA_new, pA_new, nv, nf, cal)
    Hinv = Ln.T / (Ln * Ln).sum()  # 1 x 3 (:807-808)
    same = np.array_equal(np.asarray(old_val), np.asarray(new_val)) and np.array_equal(np.asarray(old_fej), np.asarray(new_fej))
    cols = 6 + (6 if calib_pose else 0) + (0 if same else 6) + 1
    Phi = np.zeros((1, cols), dtype=LD)
    c_cal = 6 if calib_pose else -1
    c_new = 0 if same else 6 + (6 if calib_pose else 0)
    Phi[:, 0:6] += Hinv @ Hao
    if calib_pose:
        Phi[:, c_cal:c_cal + 6] += Hinv @ Hco - Hinv @ Hcn
    Phi[:, cols - 1:] = Hinv @ Lo
    Phi[:, c_new:c_new + 6] -= Hinv @ Han
    return dict(Phi=Phi, value=set_from_xyz(pA_new), fej=set_from_xyz(pAf_new), pA=pA_new, pAf=pAf_new)


def propagate(P, ids_old, id_lm, Phi):
    """StateHelper::EKFPropagation with Q = 0 of the landmark at covariance index id_lm (size 1) through Phi over the covariance indices
    ids_old (long double): the new row / column Phi P[ids_old, :] and the new variance Phi P[ids_old, ids_old] Phi^T"""
    P = np.array(P, dtype=LD)
    row = (Phi @ P[ids_old, :])[0]
    var = (Phi @ P[np.ix_(ids_old, ids_old)] @ Phi.T)[0, 0]
    out = P.copy()
    out[id_lm, :] = row
    out[:, id_lm] = row
    out[id_lm, id_lm] = var
    return out
