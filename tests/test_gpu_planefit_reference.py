"""ovp_plane_fitting and ovp_optimize_plane (csrc/planefit.cu) against the long-double references of tests/planefit_reference.py: RANSAC at
its size limits (up to PF_MAX_POINTS = 1900 points, 1901 refused), in mixed batches, with every decision planted at 1e-6 relative of its
threshold on exactly planar data, on degenerate inputs and on a mean-error tie-break; the refinement on clean consistent problems (4 to 600
features, tracks of 1 to 64 measurements, constant features, fixed and free planes, 12 and 100 iterations) and at the thresholds of its
inlier / status rule.  Everything runs through the C ABI on api.Context."""
import ctypes as C

import numpy as np
import pytest

import planefit_reference as pr
from ov_plane_b200 import api, synth

pytestmark = pytest.mark.gpu

LD = pr.LD
EPS = pr.EPS
WORST = {}  # class -> worst error / bound over the module, printed at the end


def _note(cls, ratio):
    WORST[cls] = max(WORST.get(cls, 0.0), float(ratio))


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    pr.require_long_double()
    yield
    for cls, v in sorted(WORST.items()):
        print("planefit reference: %-34s worst error / bound %.3e" % (cls, v))


@pytest.fixture(scope="module")
def env():
    S = synth.make_scenario("small_planes", seed=2)
    ctx = api.Context(S.options, device=0, max_state=S.N + 64, max_meas_rows=60000)
    ch = synth.load_scenario_into(ctx, S)
    yield S, ctx, ch
    ctx.close()


_PERMS = {}


def perms_of(F, kind):
    if (F, kind) not in _PERMS:
        out = np.zeros((pr.N_HYP, max(F, 1)), dtype=np.int32)
        assert api.load_library().ovp_plane_shuffle(F, pr.N_HYP, kind, out.ctypes.data_as(C.c_void_p)) == 0
        _PERMS[(F, kind)] = out[:, :F]
    return _PERMS[(F, kind)]


# ---- RANSAC -------------------------------------------------------------------------------------------------------------------------------
def noisy_plane(F, seed, outlier_frac=0.15, noise=0.004):
    """F points on a tilted plane 2 m from the origin over 4 x 4 m, noise, and a share of outliers 0.08-0.4 m off the plane"""
    rng = np.random.RandomState(1000 + seed)
    n = np.array([0.3, -0.2, 1.0]) + 0.1 * rng.randn(3)
    n /= np.linalg.norm(n)
    B = np.linalg.svd(n[None, :])[2][1:]
    P = rng.uniform(-2, 2, size=(F, 2)) @ B + 2.0 * n + noise * rng.randn(F, 3)
    k = int(outlier_frac * F)
    if k:
        P[:k] += rng.uniform(0.08, 0.4, size=(k, 1)) * rng.choice([-1.0, 1.0], size=(k, 1)) * n
    return P[rng.permutation(F)]


def grid(nx, ny, h=0.25, z=2.0):
    return np.array([[i * h, j * h, z] for i in range(nx) for j in range(ny)])


def check_ransac(tag, sets, st, ab, inl, min_inlier_num, max_cond, kind, expect=None):
    """status exact, inlier flags exact where decided, abcd within the least-squares bound of the long-double refit, unit normal to 4 eps"""
    off = 0
    for p, P in enumerate(sets):
        F = len(P)
        ref = pr.ransac_ld(P, min_inlier_num, max_cond, perms_of(F, kind))
        flags = inl[off:off + F]
        off += F
        if expect is not None and expect[p] is not None:  # the case is built so: the reference decides it, as intended
            assert ref["decided"] and ref["status"] == expect[p], (tag, p, ref["undecided"], ref["status"])
        if ref["decided"]:
            assert st[p] == ref["status"], (tag, p, st[p], ref["status"])
        d = ref["inlier_decided"]
        assert np.array_equal(flags[d] == 1, ref["inlier"][d]), (tag, p)
        if st[p] == 1:
            # the refit is that of the returned inlier set: the reference's, unless an undecided flag went the other way
            f = ref if np.array_equal(flags == 1, ref["inlier"]) else pr.fit_plane_ld(P[flags == 1], max_cond, cond_check=False)
            assert f["abcd"] is not None
            err = np.abs(ab[p] - np.asarray(f["abcd"], np.float64)).max()
            assert err <= f["abcd_bound"], (tag, p, err, f["abcd_bound"])
            _note("ransac abcd", err / f["abcd_bound"])
            assert abs(np.sqrt((ab[p, :3].astype(LD) ** 2).sum()) - 1) <= 4 * EPS
        else:
            assert (flags == 0).all() and (ab[p] == 0).all()
        if len(ref["winners"]):
            print("%s plane %d (F %d): status %d, %d inliers, %d draws may win, mean-error gap to the runner-up %.3e (bound %.1e)" % (
                tag, p, F, st[p], int(flags.sum()), len(ref["winners"]), ref["gap"], ref["gap_bound"]))


def run_ransac(ctx, sets, min_inlier_num=5, max_cond=200.0, kind=0):
    fo = np.concatenate([[0], np.cumsum([len(P) for P in sets])]).astype(np.int32)
    pts = np.vstack([P for P in sets if len(P)]) if fo[-1] else np.zeros((0, 3))
    out = ctx.plane_fitting(fo, pts, min_inlier_num, max_cond, shuffle_kind=kind)
    again = ctx.plane_fitting(fo, pts, min_inlier_num, max_cond, shuffle_kind=kind)
    for a, b in zip(out, again):  # bit-identical from run to run
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    return out


@pytest.mark.parametrize("F", [4, 5, 6, 31, 32, 33, 64, 65, 255, 256, 257, 1000, 1899, 1900])
def test_ransac_sizes(env, F):
    S, ctx, ch = env
    sets = [noisy_plane(F, F)]
    st, ab, inl = run_ransac(ctx, sets)
    check_ransac("size %d" % F, sets, st, ab, inl, 5, 200.0, 0, expect=[0 if F < 6 else 1])


def test_ransac_capacity_refusal_keeps_the_outputs(env):
    S, ctx, ch = env
    P = noisy_plane(1901, 3)
    fo = np.array([0, 1901], dtype=np.int32)
    st, ab, inl = np.full(1, -7, np.int32), np.full((1, 4), -7.0), np.full(1901, -7, np.int32)
    opt = api.PlaneFitOptions(5, 200.0, 0)
    r = ctx.lib.ovp_plane_fitting(ctx.h, 1, fo.ctypes.data_as(C.c_void_p), np.ascontiguousarray(P).ctypes.data_as(C.c_void_p), C.byref(opt),
                                  st.ctypes.data_as(C.c_void_p), ab.ctypes.data_as(C.c_void_p), inl.ctypes.data_as(C.c_void_p))
    assert r == 7  # OVP_ERR_CAPACITY
    assert (st == -7).all() and (ab == -7.0).all() and (inl == -7).all()
    sets = [P[:1900]]
    st, ab, inl = run_ransac(ctx, sets)
    check_ransac("after the refusal", sets, st, ab, inl, 5, 200.0, 0, expect=[1])


@pytest.mark.parametrize("kind", [0, 1])
def test_ransac_mixed_batch(env, kind):
    S, ctx, ch = env
    rng = np.random.RandomState(40 + kind)
    sizes = [int(x) for x in rng.choice([6, 12, 20, 33, 64, 100, 257], size=36)] + [1900, 0, 3, 20]
    rng.shuffle(sizes)
    sets = [noisy_plane(F, 100 + i) for i, F in enumerate(sizes)]
    st, ab, inl = run_ransac(ctx, sets, kind=kind)
    check_ransac("batch kind %d" % kind, sets, st, ab, inl, 5, 200.0, kind, expect=[None if F >= 6 else 0 for F in sizes])
    assert st.sum() >= len(sizes) - 8


def _planted_sets():
    """exactly planar data (z = 2, coordinates on a binary grid): every on-plane hypothesis is that plane to rounding; each case plants one
    decision at 1e-6 relative of its threshold.  Returns (name, sets, min_inlier_num, max_cond, expected status per set)."""
    up, dn = 1 + 1e-6, 1 - 1e-6
    cases = []
    sq = np.array([[0.0, 0.0, 2.0], [1.0, 0.0, 2.0], [0.0, 1.0, 2.0], [1.0, 1.0, 2.0]])
    cases.append(("separation", [np.vstack([sq, [0.05 * up, 0.0, 2.0]]), np.vstack([sq, [0.05 * dn, 0.0, 2.0]])], 3, 200.0, [1, 0]))
    # exactly fl(0.05) apart along one axis: the double distance is exactly 0.05 (sqrt(fl(x^2)) = x), which "<" keeps apart and "<=" does not
    cases.append(("separation exactly 0.05", [np.vstack([sq, [0.05, 0.0, 2.0]])], 3, 200.0, [1]))
    g = grid(6, 4)
    dist = np.vstack([g, [[0.1, 0.2, 2 + 0.05 * dn], [0.6, 0.1, 2 - 0.05 * dn], [0.3, 0.6, 2 + 0.05 * up], [1.1, 0.4, 2 - 0.05 * up]]])
    cases.append(("inlier distance", [dist], 5, 200.0, [1]))
    # a point fl(0.05) below the plane z = 2^-5 (the subtraction is exact); the hypotheses are that plane only to rounding, so its flag is
    # left undecided and the refit is checked on whichever set the kernel returns
    cases.append(("inlier distance exactly 0.05", [np.vstack([grid(6, 4, z=2.0 ** -5), [0.0, 0.0, 2.0 ** -5 - 0.05]])], 5, 1e6, [1]))
    cnt = []
    for F, n_in, mi, exp in ((20, 17, 5, 1), (20, 16, 5, 0), (21, 17, 5, 1), (21, 16, 5, 0), (20, 19, 18, 1), (20, 18, 18, 0)):
        P = grid(5, 5)[:F].copy()
        P[n_in:, 2] += 0.3
        cnt.append((P, mi, exp))
    for P, mi, exp in cnt:
        cases.append(("count F %d thr %d inliers %d" % (len(P), max(mi, int(len(P) * 0.8)), int((P[:, 2] == 2.0).sum())), [P], mi, 200.0, [exp]))
    five = np.array([[0.0, 0.0, 2.0], [1.0, 0.0, 2.0], [0.0, 0.5, 2.0], [1.0, 1.0, 2.0], [0.25, 0.75, 2.0]])
    c0 = pr.fit_plane_ld(five, 1e9)["cond"]
    cases.append(("condition above", [five], 3, c0 * dn, [0]))
    cases.append(("condition below", [five], 3, c0 * up, [1]))
    cases.append(("cp above", [grid(5, 4, z=0.02 * up)], 5, 1e6, [1]))
    cases.append(("cp below", [grid(5, 4, z=0.02 * dn)], 5, 1e6, [0]))
    low = grid(6, 7, z=0.019)
    low[np.linspace(0, 41, 4).astype(int), 2] = 0.025  # hypotheses through the raised points pass |cp| > 0.02; the refit on all 42 does not
    cases.append(("hypotheses pass, refit fails", [low], 5, 1e6, [0]))
    rng = np.random.RandomState(9)
    cases.append(("cluster", [np.array([1.0, 2.0, 3.0]) + 0.004 * rng.randn(30, 3)], 5, 200.0, [0]))
    cases.append(("collinear", [np.array([[0.25 * k, 0.5, 2.0] for k in range(12)])], 5, 200.0, [0]))
    cases.append(("duplicated", [np.repeat(grid(4, 4), 2, axis=0)], 5, 200.0, [1]))
    cases.append(("through the origin", [np.array([[0.25 * i, 0.25 * j, 0.25 * i] for i in range(5) for j in range(4)])], 5, 200.0, [0]))
    trng = np.random.RandomState(21)
    tie = np.c_[trng.uniform(-1, 1, size=(40, 2)), 2.0 + 0.02 * trng.randn(40)]
    cases.append(("tie-break", [tie], 5, 200.0, [1]))  # the draws with the top count keep two different inlier sets
    return cases


@pytest.mark.parametrize("case", range(len(_planted_sets())))
def test_ransac_planted_thresholds(env, case):
    S, ctx, ch = env
    name, sets, mi, mc, expect = _planted_sets()[case]
    st, ab, inl = run_ransac(ctx, sets, mi, mc)
    check_ransac(name, sets, st, ab, inl, mi, mc, 0, expect=expect)
    ref = pr.ransac_ld(sets[0], mi, mc, perms_of(len(sets[0]), 0))
    if name == "hypotheses pass, refit fails":
        assert ref["winners"] and all(ref["draws"][h]["fit"]["cp_margin"] > ref["draws"][h]["fit"]["cp_bound"] for h in ref["winners"])
        assert -ref["refit"]["cp_margin"] > ref["refit"]["cp_bound"]
    if name == "tie-break":  # the mean error decides between different inlier sets, and the reversed rule returns another one
        top = [D for D in ref["draws"] if D["valid"] and D["count"] == ref["draws"][ref["winners"][0]]["count"]]
        assert len({tuple(D["inl"]) for D in top}) > 1 and ref["gap"] > ref["gap_bound"] and ref["inlier_decided"].all()
        rev = pr.ransac_ld(sets[0], mi, mc, perms_of(len(sets[0]), 0), mistake="tiebreak")
        assert not np.array_equal(rev["inlier"], ref["inlier"])


# ---- refinement ----------------------------------------------------------------------------------------------------------------------------
def plane_in_view(ctx, ch, F, seed, m=4, const_frac=0.1, noise=0.004, px=1.0, z0=3.0):
    """a consistent refinement problem: F points on a plane in front of the current camera, each observed by m of the clones that see all of
    them (spread over them, cycled) with px pixels of noise, a share without measurements, positions off by noise metres, the plane off by 0.2 % and 2 mm"""
    rng = np.random.RandomState(500 + seed)
    Rcur, pcur = (np.asarray(x, np.float64) for x in pr.current_camera_ld(ctx))
    nC = np.array([-0.2, 0.1, 1.0])
    nC /= np.linalg.norm(nC)
    xy = rng.uniform(-0.4, 0.4, size=(F, 2)) * z0
    z = (z0 * nC[2] - xy @ nC[:2]) / nC[2]
    ptrue = (np.c_[xy, z]) @ Rcur + pcur
    nG = Rcur.T @ nC
    dG = z0 * nC[2] + nG @ pcur
    cp = dG * nG
    calib = ctx.var_get(ctx.handle_calib())[0]
    poses = [tuple(np.asarray(x, np.float64) for x in pr.camera_pose_ld(ctx.var_get(h)[0], calib)) for h in ch]
    seeing = [j for j, (R, pc) in enumerate(poses) if ((ptrue - pc) @ R[2] > 0.5).all()]
    assert len(seeing) >= 3, len(seeing)
    mo, mc, uv = [0], [], []
    for f in range(F):
        mf = 0 if (f > 0 and rng.rand() < const_frac) else m
        for k in range(mf):
            j = seeing[(k * len(seeing) // min(m, len(seeing)) + k // len(seeing)) % len(seeing)]  # spread over the seeing clones
            R, pc = poses[j]
            c = R @ (ptrue[f] - pc)
            mc.append(ch[j])
            uv.append(c[:2] / c[2] + px / 458.0 * rng.randn(2))
        mo.append(mo[-1] + mf)
    return dict(mo=np.array(mo, np.int32), mc=np.array(mc, np.int32), uv=np.array(uv, np.float32).reshape(-1, 2),
                p0=ptrue + noise * rng.randn(F, 3), cp0=cp * (1 + 0.002 * rng.randn()) + 0.002 * rng.randn(3))


def run_refine(ctx, probs, fix, max_iter, sig_px=1.0 / 458.0, sig_c=0.01):
    fo = np.concatenate([[0], np.cumsum([len(q["p0"]) for q in probs])]).astype(np.int32)
    mo = np.concatenate([[0]] + [q["mo"][1:] + off for q, off in zip(probs, np.cumsum([0] + [q["mo"][-1] for q in probs[:-1]]))]).astype(np.int32)
    mc = np.concatenate([q["mc"] for q in probs]).astype(np.int32)
    uv = np.vstack([q["uv"] for q in probs]).astype(np.float32)
    p0, cp0 = np.vstack([q["p0"] for q in probs]), np.vstack([q["cp0"] for q in probs])
    fx = np.asarray(fix, np.int32)
    st, po, co, inl, info = ctx.optimize_plane(fo, mo, mc, uv, p0, cp0, fx, sig_px, sig_c, max_num_iterations=max_iter)
    Rcur, pcur = pr.current_camera_ld(ctx)
    for p, q in enumerate(probs):
        a, b = fo[p], fo[p + 1]
        F = b - a
        tag = "refine F %d m %s fix %d it %d plane %d" % (F, q["mo"][-1], fx[p], max_iter, p)
        if (not fx[p] and F < 4) or (fx[p] and F == 0):  # refused: nothing is touched
            assert st[p] == 0 and (info[p] == 0).all() and np.array_equal(co[p], cp0[p]) and np.array_equal(po[a:b], p0[a:b])
            continue
        prob = pr.RefineProblem(q["mo"], *_poses(ctx, q["mc"]), q["uv"], fx[p], sig_px, sig_c)
        e0 = prob.evaluate(p0[a:b], cp0[p])
        err = abs(info[p, 2] - float(e0["cost"]))
        assert err <= e0["bound"], (tag, info[p, 2], float(e0["cost"]), e0["bound"])
        _note("refine initial cost", err / e0["bound"] if e0["bound"] else 0.0)
        if info[p, 0] != 1:  # no CONVERGENCE: everything as it came in
            assert st[p] == 0 and (inl[a:b] == 0).all() and np.array_equal(co[p], cp0[p]) and np.array_equal(po[a:b], p0[a:b]), tag
            print("%s: not converged in %d iterations (reason %d)" % (tag, info[p, 1], info[p, 4]))
            continue
        assert info[p, 3] <= info[p, 2], tag
        if fx[p]:
            assert np.array_equal(co[p], cp0[p]), tag
        const = np.diff(q["mo"]) == 0
        keep = const | (inl[a:b] == 0)
        assert np.array_equal(po[a:b][keep], p0[a:b][keep]), tag
        rs = pr.refine_status_ld(p0[a:b], po[a:b], co[p], Rcur, pcur, fx[p])
        assert np.array_equal((inl[a:b] == 1)[rs["flag_decided"]], rs["inlier"][rs["flag_decided"]]), tag
        if rs["decided"]:
            assert st[p] == rs["status"], (tag, st[p], rs["status"])
        if inl[a:b].all():
            e1 = prob.evaluate(po[a:b], co[p])
            err = abs(info[p, 3] - float(e1["cost"]))
            assert err <= e1["bound"], (tag, info[p, 3], float(e1["cost"]), e1["bound"])
            _note("refine final cost", err / e1["bound"] if e1["bound"] else 0.0)
            if max_iter >= 100 and info[p, 4] in (1, 2, 3) and info[p, 3] > 1e-9 * info[p, 2]:
                # (a problem with as many residuals as parameters ends at cost ~ 0: the parameter tolerance stops it, and the decrement is ~ the cost)
                nd, cost = prob.newton_decrement(po[a:b], co[p])
                ratio = float(nd / cost)
                _note("refine Newton decrement / (1e-4 cost)", ratio / 1e-4)
                print("%s: %d iterations, reason %d, cost %.6g -> %.6g, Newton decrement / cost %.2e" % (tag, info[p, 1], info[p, 4], info[p, 2],
                                                                                                        info[p, 3], ratio))
                assert ratio <= 1e-4, tag
        else:
            print("%s: %d of %d features returned as inliers" % (tag, int(inl[a:b].sum()), F))
    return st, po, co, inl, info


def _poses(ctx, mc):
    calib = ctx.var_get(ctx.handle_calib())[0]
    cache = {}
    for h in set(int(x) for x in mc):
        cache[h] = pr.camera_pose_ld(ctx.var_get(h)[0], calib)
    return (np.array([cache[int(h)][0] for h in mc], dtype=LD).reshape(-1, 3, 3), np.array([cache[int(h)][1] for h in mc], dtype=LD).reshape(-1, 3))


@pytest.mark.parametrize("max_iter", [12, 100])
@pytest.mark.parametrize("F", [4, 8, 9, 255, 256, 257, 600])
def test_refine_sizes(env, F, max_iter):
    S, ctx, ch = env
    probs = [plane_in_view(ctx, ch, F, F, const_frac=0.0 if F == 4 else 0.1)]
    run_refine(ctx, probs, [0], max_iter)


@pytest.mark.parametrize("m,fix", [(1, 1), (2, 0), (2, 1), (32, 0), (32, 1), (33, 0), (33, 1), (64, 0), (64, 1)])
def test_refine_track_lengths(env, m, fix):
    # (one measurement per feature and a free plane has more parameters than residuals: only the fixed plane is a well-posed problem)
    S, ctx, ch = env
    run_refine(ctx, [plane_in_view(ctx, ch, 12, 70 + m, m=m)], [fix], 100)


def test_refine_batch(env):
    S, ctx, ch = env
    rng = np.random.RandomState(16)
    probs = [plane_in_view(ctx, ch, int(F), 200 + i, m=int(m)) for i, (F, m) in enumerate(zip(rng.choice([4, 9, 20, 40, 257], 16),
                                                                                                 rng.choice([2, 4, 33], 16)))]
    fix = (np.arange(16) % 3 == 0).astype(np.int32)
    for it in (12, 100):
        run_refine(ctx, probs, fix, it)


def _const_plane_case(ctx, depths, dists, zp):
    """constant features only, fixed plane (reason 4: nothing is free, every output is exact): features at the given depths in front of the
    current camera, the plane z_C = zp of the current camera, each feature moved dists metres along the normal"""
    Rcur, pcur = (np.asarray(x, np.float64) for x in pr.current_camera_ld(ctx))
    nG = Rcur[2].copy()
    d = zp + nG @ pcur
    if d < 0:
        nG, d = -nG, -d
    F = len(depths)
    pts = []
    for k in range(F):
        c = np.array([0.02 * (k - F / 2.0), 0.01 * k, depths[k]])
        pts.append(Rcur.T @ c + pcur + dists[k] * nG)
    return dict(mo=np.zeros(F + 1, np.int32), mc=np.zeros(0, np.int32), uv=np.zeros((0, 2), np.float32), p0=np.array(pts).reshape(-1, 3), cp0=d * nG)


def test_refine_planted_thresholds(env):
    S, ctx, ch = env
    up, dn = 1 + 1e-6, 1 - 1e-6
    cases = []  # (problem, expected inlier flags, expected status)
    # depth 0.1 m in front of the current camera: 8 of 10 pass (thr = 8: accepted), 7 of 10 (refused)
    for n_in in (8, 7):
        dep = [0.1 * up] * n_in + [0.1 * dn] * (10 - n_in)
        cases.append((_const_plane_case(ctx, dep, [0.0] * 10, 0.1), [True] * n_in + [False] * (10 - n_in), int(n_in >= 8)))
    # distance 0.03 m of the original position to the (fixed) plane, both sides
    for n_in in (8, 7):
        dist = [0.03 * dn * (-1) ** k for k in range(n_in)] + [0.03 * up * (-1) ** k for k in range(10 - n_in)]
        cases.append((_const_plane_case(ctx, [0.5] * 10, dist, 0.5), [True] * n_in + [False] * (10 - n_in), int(n_in >= 8)))
    # F = 1 against a fixed plane: one inlier (accepted), none (refused)
    cases.append((_const_plane_case(ctx, [0.5], [0.03 * dn], 0.5), [True], 1))
    cases.append((_const_plane_case(ctx, [0.5], [0.03 * up], 0.5), [False], 0))
    probs = [c[0] for c in cases]
    st, po, co, inl, info = run_refine(ctx, probs, [1] * len(probs), 12)
    off = 0
    Rcur, pcur = pr.current_camera_ld(ctx)
    for (q, flags, status), p in zip(cases, range(len(cases))):
        F = len(q["p0"])
        rs = pr.refine_status_ld(q["p0"], q["p0"], q["cp0"], Rcur, pcur, True)
        assert rs["decided"] and np.array_equal(rs["inlier"], flags) and rs["status"] == status  # the case is built so
        assert info[p, 0] == 1 and info[p, 4] == 4 and info[p, 2] == 0.0 and info[p, 3] == 0.0
        assert np.array_equal(inl[off:off + F] == 1, flags) and st[p] == status, (p, inl[off:off + F], st[p])
        assert np.array_equal(po[off:off + F], q["p0"]) and np.array_equal(co[p], q["cp0"])
        off += F
    # measured features against a fixed plane, original positions at 0.03 (1 -+ 1e-6) m: the flags follow the original positions
    q = plane_in_view(ctx, ch, 20, 31, const_frac=0.0, noise=0.0)
    cp = q["cp0"] = np.asarray(q["cp0"], np.float64)
    n = cp / np.linalg.norm(cp)
    base = q["p0"] - np.outer(q["p0"] @ n - np.linalg.norm(cp), n)
    sgn = np.where(np.arange(20) % 2 == 0, 1.0, -1.0)
    q["p0"] = base + np.outer(sgn * 0.03 * np.where(np.arange(20) < 17, dn, up), n)
    st, po, co, inl, info = run_refine(ctx, [q], [1], 100)
    assert info[0, 0] == 1 and np.array_equal(inl == 1, np.arange(20) < 17) and st[0] == 1
    # refused before anything is built: a fixed plane without features, a free plane with three
    e = plane_in_view(ctx, ch, 3, 33)
    empty = dict(mo=np.zeros(1, np.int32), mc=np.zeros(0, np.int32), uv=np.zeros((0, 2), np.float32), p0=np.zeros((0, 3)), cp0=e["cp0"])
    st, po, co, inl, info = run_refine(ctx, [empty, e], [1, 0], 12)
    assert (st == 0).all() and (info == 0).all()
