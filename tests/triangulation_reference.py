"""Long-double reference of FeatureInitializer::single_triangulation + single_gaussnewton (csrc/triangulate_core.h, the device's
triangulate_kernel) with the margin of every decision it takes, and a generator of tracks that sit on those decisions
(tests/test_gpu_triangulation_reference.py, tests/test_cpu_triangulation_reference.py).

Numerics.  Every double quantity of the kernel is carried in long double; the float32 steps are reproduced exactly:
- z = h / h3 is rounded to float32 once from the long-double quotient.  The kernel rounds its double quotient, so the two agree
  whenever z's error bound (below) does not straddle a float32 rounding boundary; such a z is "decided".
- r = uvn - z and |r|^2 in float32.  The sm_90a build of triangulate_kernel contracts the norm: its SASS is FMUL t = r1 * r1 then
  FFMA(r0, r0, t), so |r|^2 = fmaf(r0, r0, fl(r1 * r1)), emulated exactly (long-double sum, an exact fraction on a float32 tie).  The
  square root is the IEEE-rounded sqrtf (MUFU.RSQ with its correction step).  The evaluation inside the Hessian pass discards the
  cost, and the compiler drops that norm.
- lambda is kept in double: its updates (lam * lam_mult, lam / lam_mult) are single correctly rounded operations that the kernel
  makes bit for bit, so `lam < max_lamda` is exact.
- The 3 x 3 solves are long-double Gaussian elimination with partial pivoting, which like ov_core's colPivHouseholderQr carries on
  where the kernel's Cholesky meets a non-positive pivot.  The smallest long-double Cholesky pivot is recorded ("lin_chol",
  "lm_chol"), so a case where the kernel's Cholesky would stop and ov_core would not shows as a decided mismatch.
- cond(A) comes from long-double eigenvalues of the symmetric 3 x 3 (cyclic Jacobi).

Bounds (first order, eps = 2^-53, c = BOUND_C; m measurements).  Each is an a-priori bound on the double-precision kernel, pose table
included (cam_pose_kernel's R_GtoC and p_CinG carry a relative error of a few eps):
- A and b: every entry of A_i is at most 1 in magnitude, so |dA| <= c eps m; b adds |p_CiinA| c eps per measurement.
- cond: the closed-form smallest eigenvalue moves by c eps lambda_max (m + amp), amp = min(1 / sqrt(1 - r^2), 1 / sqrt(c eps)) the
  acos amplification of the trigonometric form (near cond 1e4, about eps lambda_max / lambda_min ~ 1e-12 relative).
- linear solution: |dp| <= (3 |dA| |p| + |db|) / lambda_min(A); alpha, beta, rho inherit it through the divisions by z.
- LM state: ds (per component) starts from the linear bound and grows by the step's error at every accepted step.  With every z
  decided the residuals are the kernel's floats bit for bit, so the step map s -> dx(s) has fixed residuals; its error is its rounding
  at s, |Hl^-1| c eps (m + 2) (sum |H_k| |r_k| + (1 + lam) sum |H_k|^2 |dx|), plus its change across ds, taken as the long-double
  central difference of dx over +-ds_j in every component (first order in ds, the actual sensitivity rather than a norm bound).
  Hl's error, for the Cholesky pivots: c eps (m + 2) (1 + lam) sum |H_k|^2 plus the same central differences.
- z_k: |dz_k| <= c eps sum|terms of h_k| (1 + |z_k|) / |h3_k| + |H_k| ds.
- cost: with every z decided the kernel sums the same float squares in double: |dcost| <= c eps m cost.  An undecided z adds a
  one-float-ulp flip of that residual, 4 (|r_k| + u_k) u_k with u_k the float32 ulp of z_k.  When the float residual vectors of the
  new and the old point are bitwise equal (every z decided) both costs are the same double and the tie is exact in both.
- |dx| against min_dx: the step bound above; depth against min_dist / max_dist: |p_FinA| ds / rho plus c eps; baseline ratio
  |p_FinA| / max_k b_k: b_k^2 = |p_CiinA|^2 - along_k^2 moves by 2 |along_k| |p_CiinA| |dn| + c eps |p_CiinA|^2.
- position: |dp_FinG| <= |dp_FinA| + c eps (|p_FinA| + |p_AinG|).
A comparison is decided when its margin (value - threshold) clears its bound.  A status is decided when a rejecting comparison is
decided, or every comparison on the path is decided and passes.
"""
from fractions import Fraction

import numpy as np

from gate_reference import LD, EPS, require_long_double  # noqa: F401
from planefit_reference import jacobi_eig3
from update_reference import rot

BOUND_C = 4.0
F32 = np.float32
FIELDS = ("max_runs", "init_lamda", "max_lamda", "min_dx", "min_dcost", "lam_mult", "min_dist", "max_dist", "max_baseline", "max_cond_number")
DEFAULTS = dict(max_runs=5, init_lamda=1e-3, max_lamda=1e10, min_dx=1e-6, min_dcost=1e-6, lam_mult=10.0, min_dist=0.10, max_dist=60.0,
                max_baseline=40.0, max_cond_number=10000.0)
# every field differs from the defaults and from every other field
NON_DEFAULT = dict(max_runs=3, init_lamda=1e-2, max_lamda=1e6, min_dx=3e-7, min_dcost=2e-5, lam_mult=4.0, min_dist=0.3, max_dist=25.0,
                   max_baseline=15.0, max_cond_number=3000.0)
OPTION_SETS = {"defaults": DEFAULTS, "non_default": NON_DEFAULT}
# option sets that steer the LM loop to one exit: a lambda ceiling one rejection away, a single run, a coarse step threshold
LM_OPTION_SETS = {"max_lamda": dict(DEFAULTS, max_lamda=5e-3), "max_runs_1": dict(DEFAULTS, max_runs=1), "big_min_dx": dict(DEFAULTS, min_dx=1e-3)}
MISTAKES = ("swap_dx_dcost", "anchor_first", "baseline_full", "cond_sqrt", "depth_norm", "dcost_counts_run", "lam_add")


def _f(x):
    return float(np.float64(x))


def camera_poses(backend, handles):
    """(R_GtoC, p_CinG) in long double of every clone handle: R_GtoCi = R_ItoC R_GtoIi, p_CiinG = p_IiinG - R_GtoCi^T p_IinC"""
    calib = np.asarray(backend.var_get(backend.handle_calib())[0], dtype=np.float64).astype(LD)
    RC = rot(calib[:4])
    out = {}
    for h in handles:
        v = np.asarray(backend.var_get(int(h))[0], dtype=np.float64).astype(LD)
        R = RC @ rot(v[:4])
        out[int(h)] = (R, v[4:7] - R.T @ calib[4:7])
    return out


def _solve3(A, b):
    """long-double Gaussian elimination with partial pivoting; an exactly zero pivot leaves its unknown at 0 (a rank-deficient QR's basic
    solution)"""
    M = np.hstack([np.array(A, dtype=LD), np.array(b, dtype=LD).reshape(3, 1)])
    for j in range(3):
        k = j + int(np.argmax(np.abs(M[j:, j])))
        M[[j, k]] = M[[k, j]]
        if M[j, j] == 0:
            continue
        for i in range(j + 1, 3):
            M[i] -= M[i, j] / M[j, j] * M[j]
    x = np.zeros(3, dtype=LD)
    for j in (2, 1, 0):
        if M[j, j] == 0:
            continue
        x[j] = (M[j, 3] - M[j, j + 1:3] @ x[j + 1:]) / M[j, j]
    return x


def _chol_min_pivot(A):
    """smallest pivot (before the square root) of the kernel's 3 x 3 Cholesky, in long double; -inf once one is not positive"""
    l00 = A[0, 0]
    if not l00 > 0:
        return LD(l00) if l00 == l00 else LD(-np.inf)
    l00 = np.sqrt(l00)
    l10, l20 = A[1, 0] / l00, A[2, 0] / l00
    p1 = A[1, 1] - l10 * l10
    if not p1 > 0:
        return LD(p1) if p1 == p1 else LD(-np.inf)
    l21 = (A[2, 1] - l20 * l10) / np.sqrt(p1)
    p2 = A[2, 2] - l20 * l20 - l21 * l21
    if not p2 == p2:
        return LD(-np.inf)
    return min(A[0, 0], p1, p2)


def _closed_form_r(A):
    """r = det(B) / 2 of tri_eig_minmax: the cosine whose acos the kernel takes"""
    q = np.trace(A) / 3
    p1 = A[0, 1] ** 2 + A[0, 2] ** 2 + A[1, 2] ** 2
    p = np.sqrt(((A[0, 0] - q) ** 2 + (A[1, 1] - q) ** 2 + (A[2, 2] - q) ** 2 + 2 * p1) / 6)
    if not p > 0:
        return LD(1)
    B = (A - q * np.eye(3, dtype=LD)) / p
    r = (B[0, 0] * (B[1, 1] * B[2, 2] - B[1, 2] * B[2, 1]) - B[0, 1] * (B[1, 0] * B[2, 2] - B[1, 2] * B[2, 0])
         + B[0, 2] * (B[1, 0] * B[2, 1] - B[1, 1] * B[2, 0])) / 2
    return min(max(r, LD(-1)), LD(1))


def _fmaf_sq(r0, r1):
    """fmaf(r0, r0, fl(r1 * r1)) exactly: the product is exact in long double, the sum is rounded once to float32 (an exact fraction
    settles a long-double result that lands on a float32 tie)"""
    t = (r1 * r1).astype(F32)
    s = r0.astype(LD) * r0.astype(LD) + t.astype(LD)
    out = s.astype(F32)
    lo, hi = np.nextafter(out, F32(-np.inf)), np.nextafter(out, F32(np.inf))
    tie = (s == (out.astype(LD) + lo.astype(LD)) / 2) | (s == (out.astype(LD) + hi.astype(LD)) / 2)
    for k in np.nonzero(tie)[0]:
        exact = Fraction(float(r0[k])) ** 2 + Fraction(float(t[k]))
        cands = [F32(c) for c in (lo[k], out[k], hi[k])]
        best = min(cands, key=lambda c: (abs(Fraction(float(c)) - exact), int(np.frombuffer(c.tobytes(), np.uint32)[0]) & 1))
        out[k] = best
    return out


class _Geometry(object):
    """one track's constant geometry in the anchor frame: R_AtoCi, p_CiinA, p_AinCi"""

    def __init__(self, Rs, ps, anchor):
        self.RA, self.pA = Rs[anchor], ps[anchor]
        self.RAt = np.einsum("kij,lj->kil", Rs, self.RA)  # R_GtoCi R_GtoA^T
        self.pCA = np.einsum("ij,kj->ki", self.RA, ps - self.pA)
        self.pAC = -np.einsum("kij,kj->ki", self.RAt, self.pCA)


def _jacobian(g, s):
    """h (m x 3) and dz/d(alpha, beta, rho) (m x 2 x 3) at s, long double, as the kernel forms them"""
    a = np.array([s[0], s[1], LD(1)], dtype=LD)
    h = np.einsum("kij,j->ki", g.RAt, a) + s[2] * g.pAC
    H = np.empty((len(h), 2, 3), dtype=LD)
    h32 = h[:, 2] * h[:, 2]
    for row in range(2):
        H[:, row, 0] = (g.RAt[:, row, 0] * h[:, 2] - h[:, row] * g.RAt[:, 2, 0]) / h32
        H[:, row, 1] = (g.RAt[:, row, 1] * h[:, 2] - h[:, row] * g.RAt[:, 2, 1]) / h32
        H[:, row, 2] = (g.pAC[:, row] * h[:, 2] - h[:, row] * g.pAC[:, 2]) / h32
    return h, H


def _gn_step(g, s, r, lam):
    """the damped Gauss-Newton step at s for fixed float residuals r: dx and Hl"""
    _, H = _jacobian(g, s)
    rl = r.astype(LD)
    Hl = np.einsum("kij,kil->jl", H, H)
    for i in range(3):
        Hl[i, i] *= (LD(1) + LD(lam))
    return _solve3(Hl, np.einsum("kij,ki->j", H, rl)), Hl


def _evaluate(g, uvn, s, ds, jac=False):
    """cost at s = (alpha, beta, rho) with the kernel's float32 residuals; ds the state's error bound.  Returns a dict with the cost, its
    bound, the float residuals, whether every z is decided and (jac) H, grad, Hess and the relative Jacobian error e_H."""
    a = np.array([s[0], s[1], LD(1)], dtype=LD)
    h, H = _jacobian(g, s)
    z = h[:, :2] / h[:, 2:3]
    terms = np.einsum("kij,j->ki", np.abs(g.RAt), np.abs(a)) + abs(s[2]) * np.abs(g.pAC)
    h3 = np.abs(h[:, 2])
    Hf, zf = np.asarray(H, dtype=np.float64), np.asarray(z, dtype=np.float64)
    dsf = np.asarray(ds, dtype=np.float64)
    dz = BOUND_C * EPS * np.asarray(terms[:, :2] + terms[:, 2:3] * np.abs(z), dtype=np.float64) / np.asarray(h3, dtype=np.float64)[:, None] \
        + np.einsum("kij,j->ki", np.abs(Hf), dsf) + EPS * np.abs(zf)
    zlo, zhi = (zf - dz).astype(F32), (zf + dz).astype(F32)
    z32 = z.astype(F32)
    zdec = (zlo == zhi) & (zlo == z32)
    r = (uvn - z32).astype(F32)
    rn = np.sqrt(_fmaf_sq(r[:, 0], r[:, 1]))
    cost = (rn.astype(LD) ** 2).sum()
    ulp = np.spacing(np.abs(z32)).astype(np.float64)
    flip = (4 * (np.abs(r.astype(np.float64)) + ulp) * ulp).sum(axis=1)
    bound = BOUND_C * EPS * len(h) * _f(cost) + float(flip[~zdec.all(axis=1)].sum())
    out = dict(cost=cost, bound=bound, r=r, zdec=bool(zdec.all()))
    if jac:
        rl = r.astype(LD)
        out["grad"] = np.einsum("kij,ki->j", H, rl)
        out["Hess"] = np.einsum("kij,kil->jl", H, H)
        out["sum_Hr"] = float(np.einsum("kij,ki->", np.abs(Hf), np.abs(r.astype(np.float64))))
        out["sum_HH"] = float((Hf * Hf).sum())
    return out


def _cmp(name, value, thr, passes, bound_abs, scale):
    """one comparison: value against thr, margin = (value - thr) / scale, bound relative to the same scale"""
    margin = _f(value - thr) / scale if scale else 0.0
    bound = bound_abs / scale if scale else np.inf
    return dict(name=name, value=_f(value), thr=float(thr), passes=bool(passes), margin=margin, bound=float(bound),
                decided=bool(abs(margin) > bound))


def triangulate(Rs, ps, uvn, opt, mistake=None):
    """the reference on one track: Rs (m x 3 x 3, R_GtoCi) and ps (m x 3, p_CiinG) in long double, uvn (m x 2) float32, opt a dict of
    FIELDS.  Returns status, p_FinG (long double), p_bound, decided, reason (the first rejecting comparison or 'ok'), cmps (every
    comparison, in order), trace (one dict per LM iteration) and stop (the LM exit).  mistake: one of MISTAKES (planted variants)."""
    o = dict(opt)
    if mistake == "swap_dx_dcost":
        o["min_dx"], o["min_dcost"] = opt["min_dcost"], opt["min_dx"]
    m = len(uvn)
    # finding: a decided non-positive Cholesky pivot where ov_core's QR carries on (the kernel would return 0 there)
    res = dict(status=0, p_FinG=np.zeros(3, dtype=LD), p_bound=0.0, decided=True, reason="m<2", cmps=[], trace=[], stop=None, runs=0,
               finding=False)
    if m < 2:
        return res
    uvn = np.asarray(uvn, dtype=F32).reshape(m, 2)
    Rs, ps = np.asarray(Rs, dtype=LD).reshape(m, 3, 3), np.asarray(ps, dtype=LD).reshape(m, 3)
    g = _Geometry(Rs, ps, 0 if mistake == "anchor_first" else m - 1)
    cmps = res["cmps"]

    def finish(stage_cmps):
        """status decision over a group of rejecting comparisons (the kernel ORs them)"""
        fired = [c for c in stage_cmps if not c["passes"]]
        if any(c["decided"] for c in fired):
            res["reason"] = [c for c in fired if c["decided"]][0]["name"]
            return False, True
        if fired:
            res["reason"] = fired[0]["name"]
            return False, False
        return True, all(c["decided"] for c in stage_cmps)

    # ---- single_triangulation ----
    with np.errstate(all="ignore"):
        bvec = np.einsum("kji,kj->ki", g.RAt, np.c_[uvn.astype(LD), np.ones(m, dtype=LD)])  # R_AtoCi^T [u v 1]
        bvec = bvec / np.sqrt((bvec * bvec).sum(axis=1))[:, None]
        Ai = np.eye(3, dtype=LD)[None] - np.einsum("ki,kj->kij", bvec, bvec)
        A = Ai.sum(axis=0)
        b = np.einsum("kij,kj->i", Ai, g.pCA)
        pf = _solve3(A, b) if np.isfinite(np.asarray(A, np.float64)).all() else np.full(3, np.nan, dtype=LD)
    if not np.isfinite(np.asarray(pf, np.float64)).all():
        cmps.append(dict(name="lin_nan", value=np.nan, thr=0.0, passes=False, margin=np.inf, bound=0.0, decided=True))
        res["reason"] = "lin_nan"
        return res
    ev = jacobi_eig3(A)
    emax, emin = ev[0], ev[2]
    r = _closed_form_r(A)
    amp = min(1.0 / np.sqrt(max(1.0 - _f(r) ** 2, 1e-300)), 1.0 / np.sqrt(BOUND_C * EPS))
    de = BOUND_C * EPS * _f(emax) * (m + amp)
    Af = float(np.abs(np.asarray(A, np.float64)).max())
    lin = [_cmp("lin_chol", _chol_min_pivot(A), 0.0, _chol_min_pivot(A) > 0, BOUND_C * EPS * m * Af, Af)]
    # |cond| <= max_cond decided on the smallest eigenvalue: |lambda_min| >= lambda_max / max_cond (lambda_max / max_cond^2 for the
    # planted square root), so a singular A (lambda_min ~ 0 either sign) is decided as well
    cthr = o["max_cond_number"]
    e_thr = emax / cthr / (cthr if mistake == "cond_sqrt" else 1)
    cc = _cmp("cond", abs(emin), e_thr, abs(emin) >= e_thr, de + BOUND_C * EPS * _f(e_thr), _f(e_thr))
    cc["value"] = _f(emax / abs(emin)) if emin != 0 else np.inf
    lin.append(cc)
    npf = np.sqrt((pf * pf).sum())
    dpf = (3 * BOUND_C * EPS * m * _f(npf) + BOUND_C * EPS * float(np.abs(np.asarray(g.pCA, np.float64)).sum())) / max(abs(_f(emin)), 1e-300)
    depth_lin = npf if mistake == "depth_norm" else pf[2]
    lin.append(_cmp("lin_min", depth_lin, o["min_dist"], not depth_lin < o["min_dist"], dpf, o["min_dist"]))
    lin.append(_cmp("lin_max", depth_lin, o["max_dist"], not depth_lin > o["max_dist"], dpf, o["max_dist"]))
    cmps.extend(lin)
    # lin_chol: the kernel's Cholesky stops where ov_core's QR carries on: a decided failure there with an accepted cond is a finding
    ok, dec = finish(lin[1:])
    res["finding"] = bool(ok and not lin[0]["passes"] and lin[0]["decided"])
    if not lin[0]["decided"] and ok:
        dec = False
    if not ok:
        res["decided"] = dec
        return res
    # ---- single_gaussnewton ----
    z = pf[2]
    s = np.array([pf[0] / z, pf[1] / z, 1 / z], dtype=LD)
    rel = dpf / abs(_f(z))
    ds = np.array([(dpf + abs(_f(s[0])) * dpf) / abs(_f(z)), (dpf + abs(_f(s[1])) * dpf) / abs(_f(z)), abs(_f(s[2])) * rel], dtype=np.float64) \
        + BOUND_C * EPS * np.abs(np.asarray(s, np.float64))
    lam, eps_ = float(o["init_lamda"]), LD(10000)
    runs, recompute = 0, True
    path_decided = dec
    cur = _evaluate(g, uvn, s, ds)
    J = None
    stop = None
    while True:
        # the loop condition, in the kernel's order
        if not runs < o["max_runs"]:
            stop = "max_runs"
            break
        if not lam < o["max_lamda"]:
            stop = "max_lamda"
            break
        dx_cmp = None
        if res["trace"] and res["trace"][-1].get("dx_cmp") is not None and res["trace"][-1]["accepted"]:
            dx_cmp = res["trace"][-1]["dx_cmp"]
            if not dx_cmp["passes"]:
                stop = "min_dx"
                break
        if recompute:
            J = _evaluate(g, uvn, s, ds, jac=True)
        Hl = J["Hess"].copy()
        for i in range(3):
            Hl[i, i] *= (LD(1) + LD(lam))
        ev_h = jacobi_eig3(Hl)
        inv_norm = 1.0 / max(_f(ev_h[2]), 1e-300)
        dx = _solve3(Hl, J["grad"])
        ndx = np.sqrt((dx * dx).sum())
        # the step's error: its rounding at s, plus the change of the step map (residuals fixed) across the state's bound ds
        e_r = BOUND_C * EPS * (m + 2)
        dHl = e_r * (1 + lam) * J["sum_HH"]
        ddx = inv_norm * e_r * (J["sum_Hr"] + (1 + lam) * J["sum_HH"] * _f(ndx)) + BOUND_C * EPS * 3 * _f(ndx) + np.zeros(3)
        for j in range(3):
            if ds[j] > 0:
                sp, sm = s.copy(), s.copy()
                sp[j] += LD(ds[j])
                sm[j] -= LD(ds[j])
                (xp, Hp), (xm, Hm) = _gn_step(g, sp, J["r"], lam), _gn_step(g, sm, J["r"], lam)
                ddx = ddx + np.abs(np.asarray(xp - xm, np.float64)) / 2
                dHl += _f(np.abs(Hp - Hm).max()) / 2
        lm_chol = _cmp("lm_chol", _chol_min_pivot(Hl), 0.0, _chol_min_pivot(Hl) > 0, BOUND_C * EPS * 3 * _f(np.abs(Hl).max()) + dHl,
                       max(_f(np.abs(Hl).max()), 1e-300))
        new = _evaluate(g, uvn, s + dx, ds + ddx)
        it = dict(lam=lam, runs=runs, cost_old=_f(cur["cost"]), cost=_f(new["cost"]), lm_chol=lm_chol, accepted=False, event=None, dx=_f(ndx))
        if not lm_chol["passes"] and lm_chol["decided"]:
            res["finding"] = True
        path_decided = path_decided and lm_chol["decided"]
        tie = cur["zdec"] and new["zdec"] and np.array_equal(cur["r"], new["r"])
        co = cur["cost"]
        c1 = _cmp("cost_le", co - new["cost"], 0.0, new["cost"] <= co, cur["bound"] + new["bound"], _f(co) if co > 0 else 1.0)
        if tie:
            c1.update(passes=True, decided=True, margin=0.0)
        it["c1"] = c1
        path_decided = path_decided and c1["decided"]
        c2 = None
        if c1["passes"]:
            reldec = (co - new["cost"]) / co if co > 0 else LD(0)
            c2 = _cmp("dcost", reldec, o["min_dcost"], reldec < o["min_dcost"], (cur["bound"] + new["bound"]) / max(_f(co), 1e-300), o["min_dcost"])
            if tie:
                c2.update(passes=True, decided=True)
            it["c2"] = c2
            path_decided = path_decided and c2["decided"]
        if c1["passes"] and c2["passes"]:
            s = s + dx
            ds = ds + ddx + BOUND_C * EPS * np.abs(np.asarray(s, np.float64))
            eps_ = LD(0)
            if mistake == "dcost_counts_run":
                runs += 1
            it.update(accepted=True, event="min_dcost")
            res["trace"].append(it)
            stop = "min_dcost"
            break
        if c1["passes"]:
            recompute = True
            cur = new
            s = s + dx
            ds = ds + ddx + BOUND_C * EPS * np.abs(np.asarray(s, np.float64))
            runs += 1
            lam = lam / o["lam_mult"]
            eps_ = ndx
            it["dx_cmp"] = _cmp("min_dx", eps_, o["min_dx"], eps_ > o["min_dx"], float(np.sqrt((ddx * ddx).sum())) + BOUND_C * EPS * _f(ndx), o["min_dx"])
            path_decided = path_decided and it["dx_cmp"]["decided"]
            it.update(accepted=True, event="accept")
        else:
            recompute = False
            lam = lam + o["lam_mult"] if mistake == "lam_add" else lam * o["lam_mult"]
            it.update(event="reject")
        res["trace"].append(it)
    res["stop"], res["runs"] = stop, runs
    # ---- the final checks ----
    pfa = np.array([s[0] / s[2], s[1] / s[2], 1 / s[2]], dtype=LD)
    nf = np.sqrt((pfa * pfa).sum())
    dpfa = (float(ds[0]) + float(ds[1])) / abs(_f(s[2])) + _f(nf) * float(ds[2]) / abs(_f(s[2])) + BOUND_C * EPS * _f(nf)
    n = pfa / nf
    dn = 2 * dpfa / _f(nf)
    along = g.pCA @ n
    l2 = (g.pCA * g.pCA).sum(axis=1)
    bl2 = l2 if mistake == "baseline_full" else l2 - along * along
    bl = np.sqrt(np.maximum(bl2, 0))
    k = int(np.argmax(np.asarray(bl, np.float64)))
    bmax = bl[k]
    db2 = 2 * np.abs(np.asarray(along, np.float64)) * np.sqrt(np.asarray(l2, np.float64)) * dn + BOUND_C * EPS * np.asarray(l2, np.float64)
    bmaxf = _f(bmax)
    db = float(db2[k]) / (2 * bmaxf) if bmaxf > 0 else np.inf
    ratio = nf / bmax if bmax > 0 else LD(np.inf)
    dratio = _f(ratio) * (dpfa / _f(nf) + db / bmaxf + BOUND_C * EPS) if bmaxf > 0 else 0.0
    depth = nf if mistake == "depth_norm" else pfa[2]
    dz = dpfa
    fin = [_cmp("fin_min", depth, o["min_dist"], not depth < o["min_dist"], dz, o["min_dist"]),
           _cmp("fin_max", depth, o["max_dist"], not depth > o["max_dist"], dz, o["max_dist"]),
           _cmp("baseline", ratio, o["max_baseline"], not ratio > o["max_baseline"], dratio if np.isfinite(dratio) else 0.0, o["max_baseline"])]
    if not np.isfinite(np.asarray(pfa, np.float64)).all():
        fin.append(dict(name="fin_nan", value=np.nan, thr=0.0, passes=False, margin=np.inf, bound=0.0, decided=True))
    cmps.extend(fin)
    ok, dec = finish(fin)
    res["decided"] = bool(dec and path_decided)
    res["p_FinG"] = g.RA.T @ pfa + g.pA
    res["p_bound"] = dpfa + BOUND_C * EPS * (_f(nf) + float(np.abs(np.asarray(g.pA, np.float64)).sum()))
    if ok:
        res["status"], res["reason"] = 1, "ok"
    return res


def cmp_of(res, name):
    """the last comparison called name (None when the reference never made it)"""
    c = [x for x in res["cmps"] if x["name"] == name]
    return c[-1] if c else None


def path_of(res):
    """what the LM loop did: exit, whether a step was rejected, number of iterations"""
    return dict(stop=res["stop"], rejected=any(it["event"] == "reject" for it in res["trace"]), iters=len(res["trace"]), runs=res["runs"])


# ---- case generator ---------------------------------------------------------------------------------------------------------------------
class Context(object):
    """the clone poses of a context (api.Context or the oracle mirror), in long double, in clone order"""

    def __init__(self, backend, clone_handles, fx):
        self.handles = [int(h) for h in clone_handles]
        self.poses = camera_poses(backend, self.handles)
        self.fx = float(fx)

    def pose_arrays(self, track):
        return (np.array([self.poses[h][0] for h in track], dtype=LD).reshape(-1, 3, 3),
                np.array([self.poses[h][1] for h in track], dtype=LD).reshape(-1, 3))

    def project(self, track, p, noise_px=None):
        """normalised coordinates of p_FinG in every camera of the track, long double rounded to float32; noise_px (m x 2) pixels"""
        R, pc = self.pose_arrays(track)
        c = np.einsum("kij,kj->ki", R, np.asarray(p, dtype=LD)[None] - pc)
        uv = c[:, :2] / c[:, 2:3]
        if noise_px is not None:
            uv = uv + np.asarray(noise_px, dtype=np.float64).astype(LD) / LD(self.fx)
        return uv.astype(F32)

    def point(self, anchor, direction, depth):
        """p_FinG at depth along a direction given in the anchor camera frame (depth = the anchor camera z)"""
        R, p = self.poses[anchor]
        d = np.asarray(direction, dtype=np.float64).astype(LD)
        return R.T @ (d / d[2] * LD(depth)) + p

    def bisector(self, track, frac=1.0):
        """the mean optical axis of the track's cameras (frac = 1) or a direction frac of the way to it from the anchor's axis, in the
        anchor (last) camera's frame.  The mean axis sees the track's whole baseline, the anchor's axis the most depth per distance."""
        d = sum(self.poses[h][0][2] for h in track)
        d = np.asarray(self.poses[track[-1]][0] @ (d / np.sqrt((d * d).sum())), dtype=np.float64)
        d = frac * d + (1 - frac) * np.array([0.0, 0.0, 1.0])
        return d / np.linalg.norm(d)

    def run(self, case, opt, mistake=None):
        R, pc = self.pose_arrays(case["track"])
        return triangulate(R, pc, case["uvn"], opt, mistake)


def _case(ctx, name, track, p, noise=None, **kw):
    c = dict(name=name, track=[int(h) for h in track], uvn=ctx.project(track, p, noise) if len(track) else np.zeros((0, 2), F32))
    c.update(kw)
    return c


def _bisect(fun, t_lo, t_hi, iters=80):
    """t where the sign of fun changes between t_lo and t_hi (geometric bisection of a positive parameter)"""
    f_lo = fun(t_lo)
    for _ in range(iters):
        t = np.sqrt(t_lo * t_hi)
        if (fun(t) > 0) == (f_lo > 0):
            t_lo = t
        else:
            t_hi = t
        if t_hi / t_lo - 1 < 1e-12:
            break
    return np.sqrt(t_lo * t_hi)


REL_MIN, REL_MAX = 1e-6, 1e-3   # the relative margin every planted threshold case keeps


def _pair(ctx, opt, rule, family, t_lo, t_hi):
    """the two sides of rule: family(t) -> case; bisects the signed margin of rule's comparison, then steps off the crossing until the
    margin is between REL_MIN and REL_MAX on each side.  Returns None when the family does not isolate the rule (another comparison
    rejects the inside case, or one side does not reject by this rule alone)."""
    def margin(t):
        c = cmp_of(ctx.run(family(t), opt), rule)
        return np.nan if c is None else c["margin"]

    grid = np.geomspace(t_lo, t_hi, 48)
    ms = [margin(t) for t in grid]
    br = [i for i in range(47) if np.isfinite(ms[i]) and np.isfinite(ms[i + 1]) and (ms[i] > 0) != (ms[i + 1] > 0)]
    if not br:
        return None
    t0 = _bisect(margin, grid[br[0]], grid[br[0] + 1])
    out = {}
    for side in ("in", "out"):
        for step in (1e-4, 3e-5, 3e-4, 1e-5, 1e-3, 3e-6):
            for sgn in (1, -1):
                t = t0 * (1 + sgn * step)
                case = family(t)
                res = ctx.run(case, opt)
                c = cmp_of(res, rule)
                if c is None or c["passes"] != (side == "in") or not (REL_MIN <= abs(c["margin"]) <= REL_MAX) or not c["decided"]:
                    continue
                if side == "in" and not (res["status"] == 1 and res["decided"]):
                    continue
                if side == "out" and not (res["status"] == 0 and res["decided"] and res["reason"] == rule):
                    continue
                case.update(rule=rule, side=side, margin=c["margin"], bound=c["bound"], t=t)
                out[side] = case
                break
            if side in out:
                break
        if side not in out:
            return None
    return out["in"], out["out"]


def threshold_pairs(ctx, opt):
    """one inside / outside pair for each rejection rule of triangulate_feature under opt: cond(A), the linear depth at min_dist and
    max_dist, the final depth at max_dist, the baseline ratio.  Every track carries 1 px of noise (3 px for the final depth), so that the
    Gauss-Newton costs sit far above the float32 rounding of the residuals.  Raises when a rule finds no isolating geometry."""
    H = ctx.handles
    n = len(H)
    ax = (0.08, -0.05, 1.0)

    def family(rule, track, direction, lo, hi, px, seeds=range(4)):
        out = []
        for seed in seeds:
            nz = np.random.RandomState(1000 * len(track) + seed).randn(len(track), 2) * px
            d = ctx.bisector(track, 0.5) if direction is None else direction
            out.append(((lambda t, tr=track, nz=nz, d=d: _case(ctx, rule, tr, ctx.point(tr[-1], d, t), nz)), lo, hi))
        return out

    fam = {r: [] for r in ("cond", "lin_min", "lin_max", "fin_max", "baseline")}
    # cond(A): a far point over a short baseline; the tracks concentrated at the anchor keep the baseline ratio below max_baseline at
    # cond = max_cond (cond ~ m ratio^2 for m - 1 measurements at the anchor and one away from it)
    for a in (n - 1, n - 20):
        for track in ([H[a - 12 + k] for k in range(13)], [H[a - 10], H[a - 2], H[a - 1], H[a]], [H[a - 12]] + [H[a]] * 11,
                      [H[a - 20]] + [H[a]] * 29, [H[a - 30]] + [H[a]] * 39):
            fam["cond"] += family("cond", track, ax, 0.5, 200.0, 1.0)
    fam["lin_min"] += family("lin_min", [H[n - 4], H[n - 3], H[n - 1]], ax, 0.02, 2.0, 1.0)
    # the depth limits far out: the widest baselines, seen halfway between the anchor's axis and the track's mean axis
    for track in ([H[0], H[n - 1]], [H[0], H[n // 2], H[n - 1]], [H[0], H[n // 4], H[n // 2], H[3 * n // 4], H[n - 1]]):
        fam["lin_max"] += family("lin_max", track, None, 5.0, 400.0, 1.0)
        fam["fin_max"] += family("fin_max", track, None, 5.0, 400.0, 3.0, seeds=range(40))
    # the baseline ratio: two clusters at the ends of a short baseline (cond stays near 4 ratio^2)
    for span in (8, 12, 20, 30):
        fam["baseline"] += family("baseline", [H[n - 1 - span], H[n - 1]], ax, 0.5, 400.0, 1.0)
        fam["baseline"] += family("baseline", [H[n - 1 - span], H[n - span], H[n - 2], H[n - 1]], ax, 0.5, 400.0, 1.0)
    pairs = {}
    for rule, fams in fam.items():
        for f, lo, hi in fams:
            p = _pair(ctx, opt, rule, f, lo, hi)
            if p is None:
                continue
            if rule == "fin_max":  # the linear depth stays decided and inside on both sides
                lc = [cmp_of(ctx.run(c, opt), "lin_max") for c in p]
                if not all(c["passes"] and c["decided"] for c in lc):
                    continue
            pairs[rule] = p
            break
        if rule not in pairs:
            raise AssertionError("no geometry isolates rule %s under %s" % (rule, opt))
    return [c for p in pairs.values() for c in p]


def degenerate_cases(ctx):
    """tracks every option set rejects: a point behind the cameras, identical bearings, one clone only, pure forward motion, a NaN, m = 0, 1"""
    H = ctx.handles
    n = len(H)
    ax = (0.08, -0.05, 1.0)
    out = []
    tr = [H[n - 5], H[n - 3], H[n - 1]]
    out.append(_case(ctx, "behind", tr, ctx.point(tr[-1], ax, -4.0), expect="lin_min"))
    # identical bearings: every camera sees the direction of the anchor's ray, as if the point were at infinity
    RA = ctx.poses[tr[-1]][0]
    d = RA.T @ np.array(ax, dtype=LD)
    uv = []
    for h in tr:
        c = ctx.poses[h][0] @ d
        uv.append(c[:2] / c[2])
    out.append(dict(name="identical_bearings", track=list(tr), uvn=np.array(uv, dtype=LD).astype(F32), expect="cond"))
    out.append(_case(ctx, "one_clone", [H[n - 1]] * 4, ctx.point(H[n - 1], ax, 3.0), expect="cond"))
    # pure forward motion: the point on the line through the two camera centres
    pa, pb = ctx.poses[H[n - 9]][1], ctx.poses[H[n - 1]][1]
    out.append(_case(ctx, "forward", [H[n - 9], H[n - 1]], pb + 12 * (pb - pa), expect="cond"))
    c = _case(ctx, "nan", tr, ctx.point(tr[-1], ax, 3.0), expect="lin_nan")
    c["uvn"][1, 0] = np.nan
    out.append(c)
    out.append(_case(ctx, "m0", [], None, expect="m<2"))
    out.append(_case(ctx, "m1", [H[n - 1]], ctx.point(H[n - 1], ax, 3.0), expect="m<2"))
    return out


def random_cases(ctx, count, seed, lengths=(2, 3, 4, 6, 8, 12, 16, 20, 32, 33, 64, 100), noise_px=(1.0, 3.0)):
    """count noisy features: a track of consecutive clones (lengths drawn from `lengths`, capped by the window) ending at a random anchor,
    a point 1.5 .. 25 m out along the mean viewing direction of the track, 1 .. 3 px of noise"""
    H = ctx.handles
    n = len(H)
    rng = np.random.RandomState(seed)
    out = []
    for i in range(count):
        L = int(min(rng.choice(lengths), n))
        a = rng.randint(L - 1, n)
        tr = H[a - L + 1:a + 1]
        axes = np.array([np.asarray(ctx.poses[h][0][2], np.float64) for h in tr])
        d = axes.mean(axis=0)
        d /= np.linalg.norm(d)
        d = d + 0.15 * rng.randn(3) * np.array([1, 1, 0.2])
        d /= np.linalg.norm(d)
        centre = np.mean([np.asarray(ctx.poses[h][1], np.float64) for h in tr], axis=0)
        p = centre + d * rng.uniform(1.5, 25.0)
        nz = rng.randn(L, 2) * rng.uniform(*noise_px)
        out.append(_case(ctx, "random", tr, p.astype(LD), nz, length=L))
    return out


def lm_cases(ctx, opt_name, opt, pool):
    """from a pool of noisy features, one case per LM path the option set can take: a rejected step, and every exit the loop has.
    Returns {path: case}; each case carries the path it was chosen for."""
    want = {"reject": lambda p: p["rejected"], "max_runs": lambda p: p["stop"] == "max_runs", "min_dcost": lambda p: p["stop"] == "min_dcost",
            "min_dx": lambda p: p["stop"] == "min_dx", "max_lamda": lambda p: p["stop"] == "max_lamda"}
    out = {}
    for c in pool:
        res = ctx.run(c, opt)
        if res["status"] != 1 or not res["decided"]:
            continue
        p = path_of(res)
        for k, f in want.items():
            if k not in out and f(p):
                cc = dict(c, name="lm_" + k, path=k, opt_name=opt_name)
                out[k] = cc
    return out


def flatten(cases):
    """meas_offset, flat track (clone handles) and uvn of a list of cases, as ovp_triangulate_features takes them"""
    mo = np.zeros(len(cases) + 1, dtype=np.int32)
    for i, c in enumerate(cases):
        mo[i + 1] = mo[i] + len(c["track"])
    mc = np.array([h for c in cases for h in c["track"]], dtype=np.int32)
    uvn = np.concatenate([c["uvn"].reshape(-1, 2) for c in cases]).astype(F32) if mo[-1] else np.zeros((0, 2), F32)
    return mo, mc, np.ascontiguousarray(uvn)


def scenario():
    """the scenario every triangulation case is built on: 110 clones 3 cm apart on an arc of 2.2 rad (tracks of up to 100
    measurements, baselines up to 2.7 m), no planes in the state"""
    from ov_plane_b200 import synth
    return synth.make_scenario("cfg2_n256_f200", seed=5, n_clones=110, F=40)


def case_sets(ctx, n_random=2000, seed=11):
    """every generated case, per option set: {name: dict(opt, pairs, degenerate, lm, random)} for the defaults and the non-default set,
    and {name: dict(opt, lm)} for the LM option sets (their lm cases are drawn from the same noisy pool)"""
    pool = random_cases(ctx, n_random, seed)
    out = {}
    for name, opt in OPTION_SETS.items():
        out[name] = dict(opt=opt, pairs=threshold_pairs(ctx, opt), degenerate=degenerate_cases(ctx), lm=lm_cases(ctx, name, opt, pool),
                         random=pool)
    for name, opt in LM_OPTION_SETS.items():
        out[name] = dict(opt=opt, lm=lm_cases(ctx, name, opt, pool[:400]))
    return out


def trace_signature(res):
    """what a planted mistake may change: status, reason, exit, runs and the (event, lambda) sequence"""
    return (res["status"], res["reason"], res["stop"], res["runs"], tuple((it["event"], it["lam"]) for it in res["trace"]))
