"""Long-double references of PlaneFitting (PlaneFitting.cpp:43-514): the plane fit, the RANSAC loop with the margin of every decision, the
refinement's robust cost with its gradient and Gauss-Newton matrix, and the refinement's inlier / status rule (tests/test_gpu_planefit_reference.py,
tests/test_cpu_planefit_reference.py).  numpy's linalg does not take long double, so the 3 x 3 eigen solve and the 3-column least squares are
written out.

Bounds (eps = 2^-53, c = BOUND_C; each an a-priori bound on the double-precision kernels of csrc/planefit.cu):
- plane fit, A n = -1 with K rows: the least-squares perturbation bound |dn| / |n| <= c K eps (kappa + kappa^2 |r| / (|A| |n|)), kappa = s1 / s3
  from the long-double singular values; abcd = (n, 1) / |n| moves by at most 2 |dn| / |n| in every entry (times max(1, |abcd_3|) for the offset).
- condition number: the kernel forms A^T A (error <= c eps |A|_F^2 <= 3 c eps s1^2) and takes its extreme eigenvalues in closed form through
  acos(r); the smallest eigenvalue moves by at most c eps lambda1 (1 + amp), amp = min(1 / sqrt(1 - r^2), 1 / sqrt(c eps)) the acos amplification.
  The decision cond > thr is lambda3 < lambda1 / thr^2; its margin lambda3 - lambda1 / thr^2 is compared with that bound.
- |cp| > 0.02: |cp| = 1 / |n|, relative error the least-squares bound.
- point separation |p_i - p_j| < 0.05: c eps (|p_i|_1 + |p_j|_1); none when the two points differ in one coordinate by an exact double
  (sqrt(fl(x^2)) = |x|), so a separation of exactly fl(0.05) is decided.
- point-to-plane distance |p . abcd_123 + abcd_4|: |p|_1 |d abcd_123| + |d abcd_4| + c eps (|p|_1 + |abcd_4|).
- mean inlier error: the mean of the distance bounds plus c K eps avg (summation in any order).
- refinement cost: each residual is formed with relative rounding of its inputs; for a reprojection block on the camera point (X, Y, Z)
  |d(X / Z)| <= c eps (|p|_1 + |p_C|_1) (1 + |X / Z|) / |Z| + c eps |X / Z|, the residual adds eps (|u| + |u_meas|) and is scaled by 1 / sigma_px;
  a point-on-plane residual w (n . p - d) moves by w c eps (|p|_1 + d).  A block's s = |r|^2 moves by ds <= 2 |r| |dr| + |dr|^2 + c eps s and
  1/2 log(1 + s) by 1/2 (ds / (1 + s) + c eps (1 + log(1 + s))); the sum of the block costs adds depth eps cost with depth the longest
  chain of additions (measurements per lane, butterfly, features per warp, warps).
"""
import numpy as np

from gate_reference import LD, EPS, require_long_double  # noqa: F401

BOUND_C = 8.0
SEP, INL_DIST, CP_MIN = 0.05, 0.05, 0.02   # PlaneFitting.cpp:90-91, 78
REF_DIST, MIN_DEPTH = 0.03, 0.1              # :205, :472
N_HYP, N_SET = 200, 5                        # :87-88


def _ld(x):
    return np.asarray(x, dtype=np.float64).astype(LD)


def jacobi_eig3(M):
    """eigenvalues (descending) of a symmetric 3 x 3 by cyclic Jacobi sweeps in long double"""
    A = np.array(M, dtype=LD)
    for _ in range(50):
        off = A[0, 1] ** 2 + A[0, 2] ** 2 + A[1, 2] ** 2
        if off <= (LD(1e-40) * (A * A).sum()):
            break
        for p, q in ((0, 1), (0, 2), (1, 2)):
            if A[p, q] == 0:
                continue
            theta = (A[q, q] - A[p, p]) / (2 * A[p, q])
            t = (LD(1) if theta >= 0 else LD(-1)) / (abs(theta) + np.sqrt(theta * theta + 1))
            c = 1 / np.sqrt(t * t + 1)
            s = t * c
            J = np.eye(3, dtype=LD)
            J[p, p] = J[q, q] = c
            J[p, q], J[q, p] = s, -s
            A = J.T @ A @ J
    return np.sort(np.diag(A))[::-1]


def lstsq3_ld(A, b):
    """least squares min |A x - b| (K x 3) by a long-double Householder QR; returns x and the residual norm"""
    R = np.hstack([np.array(A, dtype=LD), np.array(b, dtype=LD).reshape(-1, 1)])
    for j in range(3):
        x = R[j:, j].copy()
        nrm = np.sqrt((x * x).sum())
        alpha = -nrm if x[0] > 0 else nrm
        v = x
        v[0] -= alpha
        vtv = (v * v).sum()
        if vtv > 0:
            R[j:, j:] -= (2 / vtv) * np.outer(v, v @ R[j:, j:])
    y = np.zeros(3, dtype=LD)
    for j in (2, 1, 0):
        y[j] = (R[j, 3] - (R[j, j + 1:3] * y[j + 1:]).sum()) / R[j, j]
    return y, np.sqrt((R[3:, 3] ** 2).sum())


def fit_plane_ld(P, cond_thresh, cond_check=True):
    """PlaneFitting::fit_plane (:43-81).  Returns a dict: ok, abcd, the margins (positive = the check passes) and bounds of the condition
    and |cp| decisions, the bound of the kernel's abcd, cond."""
    A = _ld(P).reshape(-1, 3)
    K = len(A)
    out = dict(ok=False, abcd=None, cond=np.inf, cond_margin=np.inf, cond_bound=0.0, cp=0.0, cp_margin=-np.inf, cp_bound=0.0, abcd_bound=np.inf)
    if K < 3:
        return out
    G = A.T @ A
    lam = np.maximum(jacobi_eig3(G), LD(0))
    out["cond"] = float(np.sqrt(lam[0] / lam[2])) if lam[2] > 0 else np.inf
    if cond_check:
        # the kernel's closed-form solve: r = det((G - q I) / p) / 2, phi = acos(r) / 3
        q = np.trace(G) / 3
        p = np.sqrt((((G - q * np.eye(3, dtype=LD)) ** 2).sum()) / 6)
        r = np.linalg.det(np.asarray((G - q * np.eye(3, dtype=LD)) / p, dtype=np.float64)) / 2 if p > 0 else 1.0
        amp = min(1.0 / np.sqrt(max(1.0 - r * r, 1e-300)), 1.0 / np.sqrt(BOUND_C * EPS))
        out["cond_margin"] = float(lam[2] - lam[0] / LD(cond_thresh) ** 2)
        out["cond_bound"] = BOUND_C * EPS * float(lam[0]) * (1.0 + amp) * (1.0 + 1.0 / cond_thresh ** 2)
        if not (lam[2] > 0 and np.sqrt(lam[0] / lam[2]) <= LD(cond_thresh)):
            return out
    n, res = lstsq3_ld(A, -np.ones(K, dtype=LD))
    nn = np.sqrt((n * n).sum())
    abcd = np.append(n, LD(1)) / nn
    s1 = np.sqrt(lam[0])
    kappa = float(np.sqrt(lam[0] / lam[2])) if lam[2] > 0 else np.inf
    rel = BOUND_C * K * EPS * (kappa + kappa ** 2 * float(res / (s1 * nn)))
    cp = 1 / nn
    out.update(abcd=abcd, cp=float(cp), cp_margin=float(cp - LD(CP_MIN)), cp_bound=float(cp) * rel + BOUND_C * EPS * float(cp),
               abcd_bound=2.0 * rel * max(1.0, float(cp)) + 4 * EPS, ok=bool(cp > LD(CP_MIN)))
    return out


def _dist_bounds(P1, f, abcd_bound):
    return abcd_bound * (P1 + 1.0) + BOUND_C * EPS * (P1 + abs(float(f["abcd"][3])))


def ransac_ld(P, min_inlier_num, max_cond, perms, mistake=None):
    """PlaneFitting::plane_fitting (:83-195) on the 200 draws perms (200 x F).  Returns a dict:
    status, inlier (bool per point), abcd (long double refit on the reference's inlier set) with abcd_bound, draws (per draw: sel, fit, count,
    avg, avg_bound), undecided (every decision whose margin is inside its bound, other than single inlier flags), decided (the status follows
    from decided decisions), inlier_decided (per point: the flag follows from decided decisions), winners (the draws that may win within the mean-error bounds), gap (runner-up mean error - winner's)
    with gap_bound.  mistake plants a bug in the reference (tests of the tests): "sep<=", "count>=", "tiebreak", "avg_all"."""
    P = np.asarray(P, dtype=np.float64).reshape(-1, 3)
    F = len(P)
    A = _ld(P)
    P1 = np.abs(P).sum(axis=1)
    out = dict(status=0, inlier=np.zeros(F, bool), inlier_decided=np.ones(F, bool), abcd=None, abcd_bound=np.inf, draws=[], undecided=[],
               winners=[], gap=np.inf, gap_bound=0.0, short=False, decided=True, refit=None)
    if F < min_inlier_num or F == 0:
        return out
    thr = max(min_inlier_num, int(F * 0.80))
    for h in range(N_HYP):
        sel = []
        for c in perms[h]:
            if len(sel) == N_SET:
                break
            good = True
            for qq in sel:
                dd = P[qq] - P[c]
                if np.count_nonzero(dd) <= 1 and (A[qq] - A[c] == dd.astype(LD)).all():
                    d, bnd = LD(np.abs(dd).sum()), 0.0  # one exact nonzero difference: sqrt(fl(x^2)) = |x| in binary64, no rounding at all
                else:
                    d = np.sqrt(((A[qq] - A[c]) ** 2).sum())
                    bnd = BOUND_C * EPS * (P1[qq] + P1[c])
                if bnd > 0 and abs(float(d) - SEP) <= bnd:
                    out["undecided"].append(("separation", h, int(qq), int(c), float(d) - SEP, bnd))
                if (d <= SEP) if mistake == "sep<=" else (d < SEP):
                    good = False
                    break
            if good:
                sel.append(int(c))
        if len(sel) != N_SET:  # :137-140: the reference returns false at the first short draw; the kernel after looking at all draws
            out["short"] = True
            out["draws"].append(dict(sel=sel, fit=None, valid=False))
            out["decided"] = not out["undecided"]
            return out
        f = fit_plane_ld(P[sel], max_cond)
        D = dict(sel=sel, fit=f, valid=False)
        out["draws"].append(D)
        if abs(f["cond_margin"]) <= f["cond_bound"]:
            out["undecided"].append(("condition", h, f["cond_margin"], f["cond_bound"]))
        if f["abcd"] is None:
            continue
        if abs(f["cp_margin"]) <= f["cp_bound"]:
            out["undecided"].append(("cp", h, f["cp_margin"], f["cp_bound"]))
        if not f["ok"]:
            continue
        e = np.abs(A @ f["abcd"][:3] + f["abcd"][3])
        eb = _dist_bounds(P1, f, f["abcd_bound"])
        close = np.abs(e.astype(np.float64) - INL_DIST) <= eb
        inl = e < LD(INL_DIST)
        cnt = int(inl.sum())
        avg = (e.sum() / F) if mistake == "avg_all" else (e[inl].sum() / cnt if cnt else LD(np.nan))
        D.update(inl=inl, close=close, count=cnt, avg=avg, avg_bound=float(eb[inl].mean()) + BOUND_C * max(cnt, 1) * EPS * float(avg) if cnt else 0.0)
        D["count_open"] = bool(close.any())  # the count is only decided when every point's distance is
        valid = (cnt >= thr) if mistake == "count>=" else (cnt > thr)
        D["valid"] = bool(valid and avg < LD(INL_DIST))
        if close.any() and any(abs(cnt + k - thr) <= int(close.sum()) for k in (0, 1)):
            out["undecided"].append(("count", h, cnt, thr, int(close.sum())))
    valid = [h for h, D in enumerate(out["draws"]) if D["valid"]]
    if not valid:
        out["decided"] = not out["undecided"]
        return out
    best_cnt = max(out["draws"][h]["count"] for h in valid)
    top = [h for h in valid if out["draws"][h]["count"] == best_cnt]
    key = (lambda h: -out["draws"][h]["avg"]) if mistake == "tiebreak" else (lambda h: out["draws"][h]["avg"])
    win = min(top, key=lambda h: (key(h), h))
    Dw = out["draws"][win]
    winners = [h for h in top if abs(float(out["draws"][h]["avg"] - Dw["avg"])) <= out["draws"][h]["avg_bound"] + Dw["avg_bound"]]
    others = sorted(float(out["draws"][h]["avg"] - Dw["avg"]) for h in top if h != win)
    out["winners"], out["gap"] = winners, (others[0] if others else np.inf)
    out["gap_bound"] = 2 * Dw["avg_bound"]
    inl = Dw["inl"]
    dec = ~Dw["close"]
    for h in winners:  # a flag is decided when every draw that may win puts the point on the same side, away from the threshold
        dec &= ~out["draws"][h]["close"] & (out["draws"][h]["inl"] == inl)
    f = fit_plane_ld(P[inl], max_cond, cond_check=False)
    out["refit"] = f
    if abs(f["cp_margin"]) <= f["cp_bound"]:
        out["undecided"].append(("refit cp", win, f["cp_margin"], f["cp_bound"]))
    out["decided"] = not out["undecided"]
    out["inlier_decided"] = dec if out["decided"] else np.zeros(F, bool)
    if f["ok"]:
        out.update(status=1, inlier=inl.copy(), abcd=f["abcd"], abcd_bound=f["abcd_bound"])
    return out


# ---- refinement (PlaneFitting.cpp:197-514) ------------------------------------------------------------------------------------------------
def quat_2_rot_ld(q):
    """JPL quaternion (x, y, z, w) to the rotation matrix, in long double (ov_core quat_2_Rot)"""
    q = _ld(q)
    v, w = q[:3], q[3]
    sk = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]], dtype=LD)
    return (2 * w * w - 1) * np.eye(3, dtype=LD) - 2 * w * sk + 2 * np.outer(v, v)


def camera_pose_ld(imu_value, calib_value):
    """R_GtoC = R_ItoC R_GtoI, p_CinG = p_IinG - R_GtoC^T p_IinC from a pose value (q_GtoI, p_IinG) and the extrinsics (q_ItoC, p_IinC)"""
    R = quat_2_rot_ld(calib_value[:4]) @ quat_2_rot_ld(imu_value[:4])
    return R, _ld(imu_value[4:7]) - R.T @ _ld(calib_value[4:7])


class RefineProblem(object):
    """one plane's optimize_plane inputs in long double: meas_offset (local, F + 1), the camera pose of every measurement, uv_norm (float32
    widened exactly), fix_plane, sigma_px_norm, sigma_c"""

    def __init__(self, meas_offset, Rm, pm, uv_norm, fix_plane, sigma_px_norm, sigma_c):
        self.mo = np.asarray(meas_offset, dtype=np.int64)
        self.F = len(self.mo) - 1
        self.m = np.diff(self.mo)
        self.fidx = np.repeat(np.arange(self.F), self.m)
        self.R, self.pc = np.asarray(Rm, dtype=LD).reshape(-1, 3, 3), np.asarray(pm, dtype=LD).reshape(-1, 3)
        self.uv = np.asarray(uv_norm, dtype=np.float32).reshape(-1, 2).astype(np.float64).astype(LD)
        self.fix = bool(fix_plane)
        self.w, self.sc = LD(1) / LD(sigma_px_norm), LD(sigma_c)

    def evaluate(self, p, cp, derivatives=False, mistake=None):
        """cost 1/2 sum rho(|r|^2) (Cauchy, a = 1) at (p, cp), its a-priori rounding bound, and with derivatives the gradient and Gauss-Newton
        blocks with Ceres' corrector (residual and Jacobian scaled by sqrt(rho')): g_f (F x 3), U_f (F x 3 x 3), W_f (F x 3 x 3), g_c, V.
        mistake: "jc_without_dn" (the point-on-plane Jacobian without its -d n term), "one_copy_short" (m - 1 copies of a measured feature's
        point-on-plane block)."""
        P, cp = _ld(p).reshape(-1, 3), _ld(cp)
        F, fi = self.F, self.fidx
        free = self.m > 0
        # reprojection blocks (one per measurement)
        dlt = P[fi] - self.pc
        c = np.einsum("kij,kj->ki", self.R, dlt)
        Z = c[:, 2]
        u = c[:, :2] / Z[:, None]
        r = self.w * (u - self.uv)
        s = (r * r).sum(axis=1)
        blk = np.log1p(s) / 2
        cost = blk.sum()
        # rounding bound of the reprojection blocks
        a = np.abs(np.asarray(P[fi], dtype=np.float64)).sum(axis=1) + np.abs(np.asarray(self.pc, dtype=np.float64)).sum(axis=1)
        uf, Zf, rf, sf = (np.asarray(x, dtype=np.float64) for x in (u, Z, r, s))
        du = BOUND_C * EPS * a[:, None] * (1 + np.abs(uf)) / np.abs(Zf)[:, None] + BOUND_C * EPS * np.abs(uf)
        dr = float(self.w) * (du + EPS * (np.abs(uf) + np.abs(np.asarray(self.uv, dtype=np.float64))))
        ds = (2 * np.abs(rf) * dr + dr * dr).sum(axis=1) + BOUND_C * EPS * sf
        bound = (0.5 * (ds / (1 + sf) + BOUND_C * EPS * (1 + np.log1p(sf)))).sum()
        # point-on-plane blocks: m copies for a measured feature, one at 2 sigma_c for a constant one, none when nothing is free
        d = np.sqrt((cp * cp).sum())
        nrm = cp / d
        ndp = P @ nrm
        wc = np.where(free, 1 / self.sc, 1 / (2 * self.sc))
        mult = np.where(free, self.m, 1).astype(LD)
        if mistake == "one_copy_short":
            mult = np.where(free, np.maximum(self.m - 1, 0), 1).astype(LD)
        active = free | (not self.fix)
        rp = wc * (ndp - d)
        sp = rp * rp
        cost += (np.where(active, mult, 0) * np.log1p(sp) / 2).sum()
        spf, rpf = np.asarray(sp, dtype=np.float64), np.asarray(rp, dtype=np.float64)
        drp = np.asarray(wc, dtype=np.float64) * BOUND_C * EPS * (np.abs(np.asarray(P, dtype=np.float64)).sum(axis=1) + float(d))
        dsp = 2 * np.abs(rpf) * drp + drp * drp + BOUND_C * EPS * spf
        bound += (np.where(active, np.asarray(mult, dtype=np.float64), 0) * 0.5 * (dsp / (1 + spf) + BOUND_C * EPS * (1 + np.log1p(spf)))).sum()
        depth = int(np.ceil(self.m.max() / 32.0)) + 5 + int(np.ceil(F / 8.0)) + 8 + 2 if F else 1
        bound += depth * EPS * float(cost)
        out = dict(cost=cost, bound=float(bound))
        if not derivatives:
            return out
        # Jacobians: reprojection w.r.t. p, Cauchy corrector sqrt(rho') = 1 / sqrt(1 + s)
        rho1 = 1 / (1 + s)
        iz = 1 / Z
        J = np.empty((len(s), 2, 3), dtype=LD)
        J[:, 0, :] = self.w * (iz[:, None] * self.R[:, 0, :] - (c[:, 0] * iz * iz)[:, None] * self.R[:, 2, :])
        J[:, 1, :] = self.w * (iz[:, None] * self.R[:, 1, :] - (c[:, 1] * iz * iz)[:, None] * self.R[:, 2, :])
        gf = np.zeros((F, 3), dtype=LD)
        Uf = np.zeros((F, 3, 3), dtype=LD)
        np.add.at(gf, fi, rho1[:, None] * np.einsum("kij,ki->kj", J, r))
        np.add.at(Uf, fi, rho1[:, None, None] * np.einsum("kij,kil->kjl", J, J))
        rho1p = 1 / (1 + sp)
        Jp = wc[:, None] * nrm[None, :]
        tail = P - ndp[:, None] * nrm[None, :] - (0 if mistake == "jc_without_dn" else d * nrm[None, :])
        Jc = wc[:, None] * tail / d
        k = np.where(active, mult, 0) * rho1p
        ff = free.astype(LD)
        gf += (ff * k * rp)[:, None] * Jp
        Uf += (ff * k)[:, None, None] * np.einsum("fi,fj->fij", Jp, Jp)
        cpf = LD(0 if self.fix else 1)
        Wf = (ff * k * cpf)[:, None, None] * np.einsum("fi,fj->fij", Jp, Jc)
        gc = cpf * ((k * rp)[:, None] * Jc).sum(axis=0)
        V = cpf * (k[:, None, None] * np.einsum("fi,fj->fij", Jc, Jc)).sum(axis=0)
        out.update(gf=gf * ff[:, None], Uf=Uf, Wf=Wf, gc=gc, V=V, free=free)
        return out

    def gradient(self, p, cp, mistake=None):
        """the gradient over the free parameters [free features, cp if free] as one vector"""
        e = self.evaluate(p, cp, True, mistake)
        g = [e["gf"][self.m > 0].ravel()]
        if not self.fix:
            g.append(e["gc"])
        return np.concatenate(g)

    def newton_decrement(self, p, cp):
        """1/2 g^T H^-1 g with H the Gauss-Newton matrix (Ceres' corrector), through the Schur complement on the plane; returns (value, cost)"""
        e = self.evaluate(p, cp, True)
        free = e["free"]
        gf, Uf, Wf = e["gf"][free], e["Uf"][free], e["Wf"][free]
        Ui = np.array([_inv3(U) for U in Uf], dtype=LD).reshape(-1, 3, 3)
        Uig = np.einsum("fij,fj->fi", Ui, gf)
        val = (gf * Uig).sum()
        if not self.fix:
            S = e["V"] - np.einsum("fki,fkl,flj->ij", Wf, Ui, Wf)
            rc = e["gc"] - np.einsum("fki,fk->i", Wf, Uig)
            val += rc @ (_inv3(S) @ rc)
        return val / 2, e["cost"]


def problem_from_context(backend, meas_offset, meas_clone, uv_norm, fix_plane, sigma_px_norm, sigma_c):
    """RefineProblem of one plane whose measurements observe clone handles of a context (api.Context or the oracle mirror): the camera poses
    from the clone values and the extrinsics the context holds"""
    calib = backend.var_get(backend.handle_calib())[0]
    poses = {}
    for h in set(int(x) for x in meas_clone):
        poses[h] = camera_pose_ld(backend.var_get(h)[0], calib)
    Rm = [poses[int(h)][0] for h in meas_clone]
    pm = [poses[int(h)][1] for h in meas_clone]
    return RefineProblem(meas_offset, np.array(Rm, dtype=LD).reshape(-1, 3, 3), np.array(pm, dtype=LD).reshape(-1, 3), uv_norm, fix_plane,
                         sigma_px_norm, sigma_c)


def current_camera_ld(backend):
    """the current camera pose (R_GtoC, p_CinG) of the in-front-of-camera test, from the IMU state and the extrinsics (:439-448)"""
    return camera_pose_ld(backend.var_get(backend.handle_imu())[0], backend.var_get(backend.handle_calib())[0])


def _inv3(M):
    M = np.asarray(M, dtype=LD)
    a, b, c, d, e, f, g, h, i = M.ravel()
    adj = np.array([[e * i - f * h, c * h - b * i, b * f - c * e], [f * g - d * i, a * i - c * g, c * d - a * f], [d * h - e * g, b * g - a * h,
                                                                                                                   a * e - b * d]], dtype=LD)
    return adj / (a * adj[0, 0] + b * adj[1, 0] + c * adj[2, 0])


def refine_status_ld(p0, p_after, cp, R_cur, p_cur, fix_plane, mistake=None):
    """the inlier pass and status rule (:441-514) on the refined plane cp and positions p_after (long double), with each threshold's margin and
    bound.  Returns inlier (bool), status, decided (the status follows from decided flags), flag_decided (per feature).
    mistake: "refined_distance" (the 0.03 test made on the refined position)."""
    p0, pa = _ld(p0).reshape(-1, 3), _ld(p_after).reshape(-1, 3)
    F = len(p0)
    cp = _ld(cp)
    cn = np.sqrt((cp * cp).sum())
    nrm = cp / cn
    q = pa if mistake == "refined_distance" else p0
    err = q @ nrm - cn
    db = BOUND_C * EPS * (np.abs(np.asarray(q, dtype=np.float64)).sum(axis=1) + float(cn))
    Rc, pc = _ld(R_cur).reshape(3, 3), _ld(p_cur)
    z = (pa - pc) @ Rc[2]
    zb = BOUND_C * EPS * (np.abs(np.asarray(pa, dtype=np.float64)).sum(axis=1) + np.abs(np.asarray(pc, dtype=np.float64)).sum())
    inl = (np.abs(err) < LD(REF_DIST)) & (z >= LD(MIN_DEPTH))
    near = np.abs(np.abs(np.asarray(err, dtype=np.float64)) - REF_DIST) <= db
    near |= (np.abs(np.asarray(err, dtype=np.float64)) < REF_DIST + db) & (np.abs(np.asarray(z, dtype=np.float64) - MIN_DEPTH) <= zb)
    thr = max(4, int(F * 0.80))
    n = int(inl.sum())
    fail = (F != 1 and n < thr) or (bool(fix_plane) and F == 1 and n == 0)
    n_open = int(near.sum())
    decided = not ((F != 1 and n - n_open < thr <= n + n_open) or (F == 1 and n_open > 0))
    return dict(inlier=inl, status=0 if fail else 1, decided=decided, flag_decided=~near, dist_margin=REF_DIST - np.abs(np.asarray(err, np.float64)),
                depth_margin=np.asarray(z, np.float64) - MIN_DEPTH)
