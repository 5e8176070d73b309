"""Long-double reference of FeatureInitializer::single_triangulation_1d and of the unrefined exits of both linear stages
(csrc/triangulate_core.h, triangulate_kernel<OneD, Refine>), in the four modes of ovp_set_triangulation_mode, with the margin and an
a-priori bound of every decision, like triangulation_reference.py (tests/test_gpu_triangulation_modes.py,
tests/test_cpu_triangulation_1d_reference.py).

- 3-D, refined: triangulation_reference.triangulate.
- 3-D, unrefined: that reference with max_runs = 0, whose Gauss-Newton loop then exits before its first step; the status is decided on
  the linear stage's comparisons alone (lin_chol, cond, lin_min, lin_max, lin_nan), not on the final checks (fin_*, baseline), and the
  position is the linear one.
- 1-D (linear_1d): every double quantity of the kernel in long double.  Bounds (first order, eps = 2^-53, c = BOUND_C; per measurement
  k, a_k = b_k x b_A, w_k = b_k x p_CkinA, q_k = |p_CkinA| + |p_CkinG| + |p_AinG| the scale of p_CkinA's rounding):
    |dA| <= c eps sum (12 |a_k| + (m + 3) |a_k|^2),   |db| <= c eps sum (6 |w_k| + 6 |a_k| q_k + (m + 3) |a_k| |w_k|),
    |d depth| <= (|db| + |depth| |dA|) / A + c eps |depth|, and the same bound on every component of p_FinA (b_A is a unit vector).
  A track whose measurements all come from the anchor's clone has p_CkinA = 0 exactly on the device as well, so b = 0 and the depth is
  0 (or NaN when A rounds to 0): rejected either way while min_dist > 0, a decided "lin1_zero".
- 1-D, refined: the linear result starts refine(), the Gauss-Newton loop and final checks of triangulation_reference.triangulate
  restated from an arbitrary start (test_cpu_triangulation_1d_reference.py checks that from the 3-D start it reproduces that reference
  exactly).

MISTAKES are planted variants that the generated cases must catch."""
import numpy as np

import triangulation_reference as tr
from triangulation_reference import BOUND_C, EPS, F32, LD, cmp_of  # noqa: F401

MODES = {"3d_refine": (0, 1), "3d_linear": (0, 0), "1d_refine": (1, 1), "1d_linear": (1, 0)}
MISTAKES = ("anchor_first", "skip_anchor_clone", "depth_range", "baseline_unrefined", "cond_in_1d")
LIN3 = ("lin_chol", "cond", "lin_min", "lin_max", "lin_nan")
# the rejection rules of each mode (lin1_*: the 1-D stage's depth range; fin_* / baseline: single_gaussnewton's final checks)
RULES = {"3d_linear": ("cond", "lin_min", "lin_max"), "1d_linear": ("lin1_min", "lin1_max"),
         "1d_refine": ("lin1_min", "lin1_max", "fin_max", "baseline"), "3d_refine": ("cond", "lin_min", "lin_max", "fin_max", "baseline")}
_f = tr._f


def _empty():
    return dict(status=0, p_FinG=np.zeros(3, dtype=LD), p_FinA=np.zeros(3, dtype=LD), p_bound=0.0, decided=True, reason="m<2", cmps=[],
                trace=[], stop=None, runs=0, finding=False)


def _finish(res, cmps):
    """status decision over a group of rejecting comparisons (the kernel ORs them); returns ok"""
    fired = [c for c in cmps if not c["passes"]]
    if fired:
        dec = [c for c in fired if c["decided"]]
        res["reason"] = (dec or fired)[0]["name"]
        res["decided"] = res["decided"] and bool(dec)
        return False
    res["decided"] = res["decided"] and all(c["decided"] for c in cmps)
    return True


def linear_3d(Rs, ps, uvn, opt, mistake=None):
    """single_triangulation as the unrefined output: status, p_FinG, p_FinA, p_bound, decided, reason, cmps"""
    r = tr.triangulate(Rs, ps, uvn, dict(opt, max_runs=0))
    if mistake == "baseline_unrefined":  # the final checks of single_gaussnewton at the linear point
        out = dict(r)
    else:
        out = _empty()
        out["cmps"] = [c for c in r["cmps"] if c["name"] in LIN3]
        out["finding"] = r["finding"]
        if len(uvn) < 2:
            return out
        names = [c["name"] for c in out["cmps"]]
        if "lin_nan" in names:
            out["reason"] = "lin_nan"
            return out
        # lin_chol: the kernel's Cholesky stopping where ov_core's QR carries on is a finding, not a status (as in the refined reference)
        ok = _finish(out, out["cmps"][1:])
        chol = out["cmps"][0]
        if ok and not chol["decided"]:
            out["decided"] = False
        if not ok:
            return out
        out.update(status=1, reason="ok", p_FinG=r["p_FinG"], p_bound=r["p_bound"])
    if out["status"] == 1:
        g = tr._Geometry(np.asarray(Rs, dtype=LD).reshape(-1, 3, 3), np.asarray(ps, dtype=LD).reshape(-1, 3), len(uvn) - 1)
        out["p_FinA"] = g.RA @ (np.asarray(out["p_FinG"], dtype=LD) - g.pA)
    else:
        out["p_FinG"], out["p_FinA"] = np.zeros(3, dtype=LD), np.zeros(3, dtype=LD)
    return out


def linear_1d(Rs, ps, uvn, opt, mistake=None):
    """single_triangulation_1d: status, p_FinG, p_FinA, p_bound, decided, reason, cmps, and its internals (A, b, depth, rows)"""
    res = _empty()
    m = len(uvn)
    if m < 2:
        return res
    uvn = np.asarray(uvn, dtype=F32).reshape(m, 2)
    Rs, ps = np.asarray(Rs, dtype=LD).reshape(m, 3, 3), np.asarray(ps, dtype=LD).reshape(m, 3)
    anchor = 0 if mistake == "anchor_first" else m - 1
    g = tr._Geometry(Rs, ps, anchor)
    uvl = uvn.astype(LD)
    with np.errstate(all="ignore"):
        bA = np.array([uvl[anchor, 0], uvl[anchor, 1], LD(1)], dtype=LD)
        bA = bA / np.sqrt((bA * bA).sum())
        bk = np.einsum("kji,kj->ki", g.RAt, np.c_[uvl, np.ones(m, dtype=LD)])  # R_AtoCk^T [u v 1]
        bk = bk / np.sqrt((bk * bk).sum(axis=1))[:, None]
        a = np.cross(bk, bA[None])
        w = np.cross(bk, g.pCA)
        keep = np.arange(m) != anchor
        if mistake == "skip_anchor_clone":  # every observation from the anchor's clone skipped, not just the anchor measurement
            keep &= ~((ps == ps[anchor]).all(axis=1) & (Rs == Rs[anchor]).all(axis=(1, 2)))
        a, w = a[keep], w[keep]
        A = (a * a).sum()
        b = (a * w).sum()
        depth = b / A
        pfa = depth * bA
    res.update(A=A, b=b, depth=depth, a=a, w=w, pCA=g.pCA[keep], bA=bA)
    cmps = res["cmps"]
    if not (g.pCA[keep] != 0).any() and np.isfinite(np.asarray(A, np.float64)):
        # b = 0 exactly on the device too: depth 0, or NaN when A = 0; rejected by min_dist > 0 or by the NaN rule
        cmps.append(dict(name="lin1_zero", value=0.0, thr=float(opt["min_dist"]), passes=False, margin=-np.inf, bound=0.0,
                         decided=bool(opt["min_dist"] > 0)))
        res["reason"], res["decided"] = "lin1_zero", bool(opt["min_dist"] > 0)
        return res
    if not np.isfinite(np.asarray(pfa, np.float64)).all():
        cmps.append(dict(name="lin1_nan", value=np.nan, thr=0.0, passes=False, margin=np.inf, bound=0.0, decided=True))
        res["reason"] = "lin1_nan"
        return res
    na = np.sqrt(np.asarray((a * a).sum(axis=1), np.float64))
    nw = np.sqrt(np.asarray((w * w).sum(axis=1), np.float64))
    q = np.sqrt(np.asarray((g.pCA[keep] ** 2).sum(axis=1), np.float64)) + np.sqrt(np.asarray((ps[keep] ** 2).sum(axis=1), np.float64)) \
        + float(np.sqrt(np.asarray((g.pA ** 2).sum(), np.float64)))
    dA = BOUND_C * EPS * float((12 * na + (m + 3) * na * na).sum())
    db = BOUND_C * EPS * float((6 * nw + 6 * na * q + (m + 3) * na * nw).sum())
    Af, df = _f(A), abs(_f(depth))
    dd = (db + df * dA) / Af + BOUND_C * EPS * df if Af > dA else np.inf
    dval = np.sqrt((pfa * pfa).sum()) if mistake == "depth_range" else pfa[2]
    lin = [tr._cmp("lin1_min", dval, opt["min_dist"], not dval < opt["min_dist"], dd, opt["min_dist"]),
           tr._cmp("lin1_max", dval, opt["max_dist"], not dval > opt["max_dist"], dd, opt["max_dist"])]
    if mistake == "cond_in_1d":  # the 3-D stage's condition-number rule applied to the 1-D stage
        lin.append(cmp_of(tr.triangulate(Rs, ps, uvn, dict(opt, max_runs=0)), "cond"))
    cmps.extend(c for c in lin if c is not None)
    if not _finish(res, cmps):
        return res
    res.update(status=1, reason="ok", p_FinA=pfa, p_FinG=g.RA.T @ pfa + g.pA, dp=dd,
               p_bound=dd + BOUND_C * EPS * (_f(np.sqrt((pfa * pfa).sum())) + float(np.abs(np.asarray(g.pA, np.float64)).sum())))
    return res


def refine(Rs, ps, uvn, opt, lin):
    """single_gaussnewton started from the linear result lin (status 1, p_FinA, dp: its bound): triangulation_reference.triangulate's
    loop and final checks, the same comparisons and bounds"""
    res = _empty()
    res.update(cmps=list(lin["cmps"]), decided=lin["decided"])
    o = dict(opt)
    m = len(uvn)
    uvn = np.asarray(uvn, dtype=F32).reshape(m, 2)
    g = tr._Geometry(np.asarray(Rs, dtype=LD).reshape(m, 3, 3), np.asarray(ps, dtype=LD).reshape(m, 3), m - 1)
    pf, dpf = lin["p_FinA"], lin["dp"]
    z = pf[2]
    s = np.array([pf[0] / z, pf[1] / z, 1 / z], dtype=LD)
    rel = dpf / abs(_f(z))
    ds = np.array([(dpf + abs(_f(s[0])) * dpf) / abs(_f(z)), (dpf + abs(_f(s[1])) * dpf) / abs(_f(z)), abs(_f(s[2])) * rel], dtype=np.float64) \
        + BOUND_C * EPS * np.abs(np.asarray(s, np.float64))
    lam = float(o["init_lamda"])
    runs, recompute = 0, True
    path_decided = res["decided"]
    cur = tr._evaluate(g, uvn, s, ds)
    J, stop = None, None
    while True:
        if not runs < o["max_runs"]:
            stop = "max_runs"
            break
        if not lam < o["max_lamda"]:
            stop = "max_lamda"
            break
        if res["trace"] and res["trace"][-1].get("dx_cmp") is not None and res["trace"][-1]["accepted"]:
            if not res["trace"][-1]["dx_cmp"]["passes"]:
                stop = "min_dx"
                break
        if recompute:
            J = tr._evaluate(g, uvn, s, ds, jac=True)
        Hl = J["Hess"].copy()
        for i in range(3):
            Hl[i, i] *= (LD(1) + LD(lam))
        inv_norm = 1.0 / max(_f(tr.jacobi_eig3(Hl)[2]), 1e-300)
        dx = tr._solve3(Hl, J["grad"])
        ndx = np.sqrt((dx * dx).sum())
        e_r = BOUND_C * EPS * (m + 2)
        dHl = e_r * (1 + lam) * J["sum_HH"]
        ddx = inv_norm * e_r * (J["sum_Hr"] + (1 + lam) * J["sum_HH"] * _f(ndx)) + BOUND_C * EPS * 3 * _f(ndx) + np.zeros(3)
        for j in range(3):
            if ds[j] > 0:
                sp, sm = s.copy(), s.copy()
                sp[j] += LD(ds[j])
                sm[j] -= LD(ds[j])
                (xp, Hp), (xm, Hm) = tr._gn_step(g, sp, J["r"], lam), tr._gn_step(g, sm, J["r"], lam)
                ddx = ddx + np.abs(np.asarray(xp - xm, np.float64)) / 2
                dHl += _f(np.abs(Hp - Hm).max()) / 2
        lm_chol = tr._cmp("lm_chol", tr._chol_min_pivot(Hl), 0.0, tr._chol_min_pivot(Hl) > 0,
                          BOUND_C * EPS * 3 * _f(np.abs(Hl).max()) + dHl, max(_f(np.abs(Hl).max()), 1e-300))
        new = tr._evaluate(g, uvn, s + dx, ds + ddx)
        it = dict(lam=lam, runs=runs, cost_old=_f(cur["cost"]), cost=_f(new["cost"]), lm_chol=lm_chol, accepted=False, event=None, dx=_f(ndx))
        res["finding"] = res["finding"] or bool(not lm_chol["passes"] and lm_chol["decided"])
        path_decided = path_decided and lm_chol["decided"]
        tie = cur["zdec"] and new["zdec"] and np.array_equal(cur["r"], new["r"])
        co = cur["cost"]
        c1 = tr._cmp("cost_le", co - new["cost"], 0.0, new["cost"] <= co, cur["bound"] + new["bound"], _f(co) if co > 0 else 1.0)
        if tie:
            c1.update(passes=True, decided=True, margin=0.0)
        path_decided = path_decided and c1["decided"]
        c2 = None
        if c1["passes"]:
            reldec = (co - new["cost"]) / co if co > 0 else LD(0)
            c2 = tr._cmp("dcost", reldec, o["min_dcost"], reldec < o["min_dcost"], (cur["bound"] + new["bound"]) / max(_f(co), 1e-300), o["min_dcost"])
            if tie:
                c2.update(passes=True, decided=True)
            path_decided = path_decided and c2["decided"]
        if c1["passes"] and c2["passes"]:
            s = s + dx
            ds = ds + ddx + BOUND_C * EPS * np.abs(np.asarray(s, np.float64))
            it.update(accepted=True, event="min_dcost")
            res["trace"].append(it)
            stop = "min_dcost"
            break
        if c1["passes"]:
            recompute, cur = True, new
            s = s + dx
            ds = ds + ddx + BOUND_C * EPS * np.abs(np.asarray(s, np.float64))
            runs += 1
            lam = lam / o["lam_mult"]
            it["dx_cmp"] = tr._cmp("min_dx", ndx, o["min_dx"], ndx > o["min_dx"], float(np.sqrt((ddx * ddx).sum())) + BOUND_C * EPS * _f(ndx),
                                   o["min_dx"])
            path_decided = path_decided and it["dx_cmp"]["decided"]
            it.update(accepted=True, event="accept")
        else:
            recompute = False
            lam = lam * o["lam_mult"]
            it.update(event="reject")
        res["trace"].append(it)
    res["stop"], res["runs"] = stop, runs
    pfa = np.array([s[0] / s[2], s[1] / s[2], 1 / s[2]], dtype=LD)
    nf = np.sqrt((pfa * pfa).sum())
    dpfa = (float(ds[0]) + float(ds[1])) / abs(_f(s[2])) + _f(nf) * float(ds[2]) / abs(_f(s[2])) + BOUND_C * EPS * _f(nf)
    dn = 2 * dpfa / _f(nf)
    along = g.pCA @ (pfa / nf)
    l2 = (g.pCA * g.pCA).sum(axis=1)
    bl = np.sqrt(np.maximum(l2 - along * along, 0))
    k = int(np.argmax(np.asarray(bl, np.float64)))
    bmax, bmaxf = bl[k], _f(bl[k])
    db2 = 2 * np.abs(np.asarray(along, np.float64)) * np.sqrt(np.asarray(l2, np.float64)) * dn + BOUND_C * EPS * np.asarray(l2, np.float64)
    db = float(db2[k]) / (2 * bmaxf) if bmaxf > 0 else np.inf
    ratio = nf / bmax if bmax > 0 else LD(np.inf)
    dratio = _f(ratio) * (dpfa / _f(nf) + db / bmaxf + BOUND_C * EPS) if bmaxf > 0 else 0.0
    fin = [tr._cmp("fin_min", pfa[2], o["min_dist"], not pfa[2] < o["min_dist"], dpfa, o["min_dist"]),
           tr._cmp("fin_max", pfa[2], o["max_dist"], not pfa[2] > o["max_dist"], dpfa, o["max_dist"]),
           tr._cmp("baseline", ratio, o["max_baseline"], not ratio > o["max_baseline"], dratio if np.isfinite(dratio) else 0.0, o["max_baseline"])]
    if not np.isfinite(np.asarray(pfa, np.float64)).all():
        fin.append(dict(name="fin_nan", value=np.nan, thr=0.0, passes=False, margin=np.inf, bound=0.0, decided=True))
    res["cmps"].extend(fin)
    res["decided"] = path_decided
    ok = _finish(res, fin)
    if ok:
        res.update(status=1, reason="ok", p_FinA=pfa, p_FinG=g.RA.T @ pfa + g.pA,
                   p_bound=dpfa + BOUND_C * EPS * (_f(nf) + float(np.abs(np.asarray(g.pA, np.float64)).sum())))
    return res


def triangulate(Rs, ps, uvn, opt, mode, mistake=None):
    """the reference in one of MODES: status, p_FinG, p_FinA, p_bound, decided, reason, cmps"""
    one_d, ref = MODES[mode]
    if not one_d:
        if not ref:
            return linear_3d(Rs, ps, uvn, opt, mistake)
        res = tr.triangulate(Rs, ps, uvn, opt, mistake if mistake in tr.MISTAKES else None)
        if res["status"] == 1:
            g = tr._Geometry(np.asarray(Rs, dtype=LD).reshape(-1, 3, 3), np.asarray(ps, dtype=LD).reshape(-1, 3), len(uvn) - 1)
            res["p_FinA"] = g.RA @ (res["p_FinG"] - g.pA)
        return res
    lin = linear_1d(Rs, ps, uvn, opt, mistake)
    if not ref and mistake == "baseline_unrefined" and lin["status"] == 1:
        return refine(Rs, ps, uvn, dict(opt, max_runs=0), lin)
    if not ref or lin["status"] != 1:
        return lin
    return refine(Rs, ps, uvn, opt, lin)


class ModeContext(tr.Context):
    """triangulation_reference.Context whose run() is the reference in one mode (so that its case generators drive every mode)"""

    def __init__(self, base, mode):
        self.handles, self.poses, self.fx, self.mode = base.handles, base.poses, base.fx, mode

    def run(self, case, opt, mistake=None):
        R, pc = self.pose_arrays(case["track"])
        return triangulate(R, pc, case["uvn"], opt, self.mode, mistake)


def threshold_pairs(ctx, opt):
    """one inside / outside pair for each rejection rule of ctx.mode (RULES) under opt, on triangulation_reference's families: 1 px of
    noise (3 px for the final depth).  Raises when a rule finds no isolating geometry."""
    H = ctx.handles
    n = len(H)
    ax = (0.08, -0.05, 1.0)

    def family(rule, track, direction, lo, hi, px, seeds=range(4)):
        out = []
        for seed in seeds:
            nz = np.random.RandomState(1000 * len(track) + seed).randn(len(track), 2) * px
            d = ctx.bisector(track, 0.5) if direction is None else direction
            out.append(((lambda t, tr_=track, nz=nz, d=d: tr._case(ctx, rule, tr_, ctx.point(tr_[-1], d, t), nz)), lo, hi))
        return out

    fam = {}
    for a in (n - 1, n - 20):
        for track in ([H[a - 12 + k] for k in range(13)], [H[a - 10], H[a - 2], H[a - 1], H[a]], [H[a - 12]] + [H[a]] * 11,
                      [H[a - 20]] + [H[a]] * 29):
            fam.setdefault("cond", []).extend(family("cond", track, ax, 0.5, 200.0, 1.0))
    for rule in ("lin_min", "lin1_min"):
        fam[rule] = family(rule, [H[n - 4], H[n - 3], H[n - 1]], ax, 0.02, 2.0, 1.0) + family(rule, [H[n - 12], H[n - 1]], ax, 0.02, 2.0, 1.0)
    for track in ([H[0], H[n - 1]], [H[0], H[n // 2], H[n - 1]], [H[0], H[n // 4], H[n // 2], H[3 * n // 4], H[n - 1]]):
        for rule in ("lin_max", "lin1_max"):
            fam.setdefault(rule, []).extend(family(rule, track, None, 5.0, 400.0, 1.0))
        fam.setdefault("fin_max", []).extend(family("fin_max", track, None, 5.0, 400.0, 3.0, seeds=range(40)))
    for span in (8, 12, 20, 30):
        fam.setdefault("baseline", []).extend(family("baseline", [H[n - 1 - span], H[n - 1]], ax, 0.5, 400.0, 1.0))
        fam["baseline"] += family("baseline", [H[n - 1 - span], H[n - span], H[n - 2], H[n - 1]], ax, 0.5, 400.0, 1.0)
    lin_max = "lin1_max" if MODES[ctx.mode][0] else "lin_max"
    pairs = []
    for rule in RULES[ctx.mode]:
        for f, lo, hi in fam[rule]:
            p = tr._pair(ctx, opt, rule, f, lo, hi)
            if p is None:
                continue
            if rule == "fin_max":  # the linear depth stays decided and inside on both sides
                if not all(c["passes"] and c["decided"] for c in (cmp_of(ctx.run(x, opt), lin_max) for x in p)):
                    continue
            pairs += list(p)
            break
        else:
            raise AssertionError("no geometry isolates rule %s in mode %s under %s" % (rule, ctx.mode, opt))
    return pairs


def collinear_cases(ctx):
    """tracks whose rays are (nearly) collinear, so that the 1-D stage's A is 0 or tiny: the point at infinity seen along the anchor's
    ray (every bearing the anchor's), a point on the line through two camera centres, and one clone observed twice with the anchor's
    normalised coordinates (b = 0 exactly)"""
    H = ctx.handles
    n = len(H)
    ax = np.array((0.08, -0.05, 1.0))
    tr_ = [H[n - 5], H[n - 3], H[n - 1]]
    d = ctx.poses[tr_[-1]][0].T @ ax.astype(LD)
    uv = []
    for h in tr_:
        c = ctx.poses[h][0] @ d
        uv.append(c[:2] / c[2])
    out = [dict(name="identical_bearings", track=list(tr_), uvn=np.array(uv, dtype=LD).astype(F32))]
    pa, pb = ctx.poses[H[n - 9]][1], ctx.poses[H[n - 1]][1]
    out.append(tr._case(ctx, "forward", [H[n - 9], H[n - 1]], pb + 12 * (pb - pa)))
    c = tr._case(ctx, "anchor_twice", [H[n - 1], H[n - 1]], ctx.point(H[n - 1], ax, 3.0))
    c["uvn"][0] = c["uvn"][1]
    out.append(c)
    return out


def clone_twice_cases(ctx, seed=3):
    """tracks that observe a clone twice: the anchor's clone (which the 1-D stage sums, p_CkinA = 0) and a middle one, 1 px of noise"""
    H = ctx.handles
    n = len(H)
    rng = np.random.RandomState(seed)
    out = []
    for tr_ in ([H[n - 30], H[n - 20], H[n - 1], H[n - 1]], [H[n - 40], H[n - 25], H[n - 25], H[n - 10], H[n - 10]],
                [H[n - 60], H[n - 2], H[n - 2]], [H[n - 1], H[n - 50], H[n - 1]]):
        p = ctx.point(tr_[-1], ctx.bisector(tr_, 0.5), 4.0)
        out.append(tr._case(ctx, "clone_twice", tr_, p, rng.randn(len(tr_), 2)))
    return out
