"""CPU checks of the long-double PlaneFitting references (tests/planefit_reference.py): the small solvers against NumPy, the plane fit and
the RANSAC loop against the double transcription and the oracle, the refinement cost against the oracle, its gradient against long-double
central differences, and planted mistakes that every check must catch."""
import ctypes as C

import numpy as np
import pytest

import oracle_backend
import planefit_cases
import planefit_reference as pr
from ov_plane_b200 import api, synth
from test_cpu_planefit import _fit_plane_np, _plane_fitting_py

LD = pr.LD


def setup_module():
    pr.require_long_double()


def shuffles(n, kind=0):
    out = np.zeros((pr.N_HYP, n), dtype=np.int32)
    assert api.load_library().ovp_plane_shuffle(n, pr.N_HYP, kind, out.ctypes.data_as(C.c_void_p)) == 0
    return out


def test_small_solvers_match_numpy():
    rng = np.random.RandomState(7)
    for _ in range(50):
        A = rng.randn(rng.randint(3, 40), 3) * rng.choice([1.0, 1e-3, 1e3], size=3)
        ev = pr.jacobi_eig3(A.T @ A)
        assert np.allclose(np.asarray(ev, np.float64), np.linalg.eigvalsh(A.T @ A)[::-1], rtol=1e-9, atol=1e-12 * ev[0])
        b = rng.randn(len(A))
        x, res = pr.lstsq3_ld(A, b)
        xn = np.linalg.lstsq(A, b, rcond=None)[0]
        assert np.abs(np.asarray(x, np.float64) - xn).max() <= 1e-8 * np.abs(xn).max()
        assert abs(float(res) - np.linalg.norm(A @ xn - b)) <= 1e-8 * (1 + np.linalg.norm(b))


def test_fit_plane_matches_numpy_and_the_oracle():
    rng = np.random.RandomState(3)
    L = oracle_backend.lib()
    n_ok = 0
    for trial in range(150):
        K = rng.choice([3, 5, 5, 12, 40])
        nrm = rng.randn(3)
        nrm /= np.linalg.norm(nrm)
        B = np.linalg.svd(nrm[None, :])[2][1:]
        P = np.ascontiguousarray((rng.uniform(-2, 2, size=(K, 2)) * rng.choice([1.0, 0.05])) @ B + rng.uniform(0.01, 4.0) * nrm + 0.003 * rng.randn(K, 3))
        thr = rng.choice([50.0, 200.0])
        f = pr.fit_plane_ld(P, thr)
        ok_np, abcd_np = _fit_plane_np(P, thr)
        abcd, ok = np.zeros(4), C.c_int(0)
        L.orc_fit_plane(int(K), P.ctypes.data_as(C.c_void_p), C.c_double(thr), 1, abcd.ctypes.data_as(C.c_void_p), C.byref(ok))
        if abs(f["cond_margin"]) <= f["cond_bound"] or (f["abcd"] is not None and abs(f["cp_margin"]) <= f["cp_bound"]):
            continue
        assert f["ok"] == bool(ok_np) == bool(ok.value), trial
        if f["ok"]:
            n_ok += 1
            # the oracle (Eigen in double) is within the bound the GPU is held to
            assert np.abs(abcd - np.asarray(f["abcd"], np.float64)).max() <= f["abcd_bound"], trial
            assert np.abs(abcd_np - np.asarray(f["abcd"], np.float64)).max() <= f["abcd_bound"], trial
    assert n_ok > 30


@pytest.mark.parametrize("name,seed", [("small_planes", 0), ("small_planes", 1)])
def test_ransac_matches_the_transcription_and_the_oracle(name, seed):
    S = synth.make_scenario(name, seed=seed)
    fo, pts = planefit_cases.plane_point_sets(S, seed=seed)
    orc = oracle_backend.OracleContext(S.options)
    st, ab, inl = orc.plane_fitting(fo, pts, 5, 200.0, shuffle_kind=0)
    for p in range(len(fo) - 1):
        P = pts[fo[p]:fo[p + 1]]
        perms = shuffles(len(P))
        ref = pr.ransac_ld(P, 5, 200.0, perms)
        ok, abcd, best = _plane_fitting_py(P, 5, 200.0, perms)
        assert ref["decided"], ref["undecided"]
        assert ref["status"] == int(bool(ok)) == st[p]
        assert np.array_equal(ref["inlier"].astype(np.int32), inl[fo[p]:fo[p + 1]])
        if ok:
            assert np.abs(ab[p] - np.asarray(ref["abcd"], np.float64)).max() <= ref["abcd_bound"]
            print("%s seed %d plane %d: %d of %d inliers, %d draws may win, gap to the runner-up %.3e (bound %.1e)" % (
                name, seed, p, ref["inlier"].sum(), len(P), len(ref["winners"]), ref["gap"], ref["gap_bound"]))


def _refine_setup():
    S = synth.make_scenario("small_planes", seed=2)
    orc = oracle_backend.OracleContext(S.options)
    ch = synth.load_scenario_into(orc, S)
    return S, orc, planefit_cases.refine_problem(S, ch, seed=2, consistent=True, slam_share=0.15, noise=0.006)


def _plane_problem(orc, q, p, fix, sig_px=1.0 / 458.0, sig_c=0.01):
    fo, mo = q["feat_offset"], q["meas_offset"]
    a, b = fo[p], fo[p + 1]
    lmo = mo[a:b + 1] - mo[a]
    mc, uv = q["meas_clone"][mo[a]:mo[b]], q["uv_norm"][mo[a]:mo[b]]
    return pr.problem_from_context(orc, lmo, mc, uv, fix, sig_px, sig_c), (lmo, mc, uv), (a, b)


@pytest.mark.parametrize("fix", [0, 1])
def test_refinement_cost_matches_the_oracle(fix):
    S, orc, q = _refine_setup()
    fx = np.full(len(q["feat_offset"]) - 1, fix, dtype=np.int32)
    st, po, co, inl, info = orc.optimize_plane(q["feat_offset"], q["meas_offset"], q["meas_clone"], q["uv_norm"], q["p_FinG"], q["cp_inG"], fx,
                                                1.0 / 458.0, 0.01, max_num_iterations=100)
    Rcur, pcur = pr.current_camera_ld(orc)
    for p in range(len(fx)):
        prob, (lmo, mc, uv), (a, b) = _plane_problem(orc, q, p, fix)
        e0 = prob.evaluate(q["p_FinG"][a:b], q["cp_inG"][p])
        assert abs(info[p, 2] - float(e0["cost"])) <= e0["bound"], (info[p, 2], float(e0["cost"]), e0["bound"])
        rs = pr.refine_status_ld(q["p_FinG"][a:b], po[a:b], co[p], Rcur, pcur, fix)
        if info[p, 0] == 1 and rs["decided"]:
            assert st[p] == rs["status"] and np.array_equal(inl[a:b] == 1, rs["inlier"])
        if info[p, 0] == 1 and inl[a:b].all():
            e1 = prob.evaluate(po[a:b], co[p])
            assert abs(info[p, 3] - float(e1["cost"])) <= e1["bound"]
            nd, cost = prob.newton_decrement(po[a:b], co[p])
            print("plane %d fix %d: cost %.6f -> %.6f, reason %d, Newton decrement / cost %.2e" % (p, fix, info[p, 2], info[p, 3], info[p, 4], nd / cost))
            assert nd <= 1e-4 * cost
        c = orc.optimize_plane_cost(lmo, mc, uv, q["p_FinG"][a:b], q["cp_inG"][p], fix, 1.0 / 458.0, 0.01)
        assert abs(c - float(e0["cost"])) <= e0["bound"]


@pytest.mark.parametrize("fix", [0, 1])
def test_gradient_matches_central_differences(fix):
    S, orc, q = _refine_setup()
    prob, _, (a, b) = _plane_problem(orc, q, 1, fix)
    p0, cp0 = q["p_FinG"][a:b].astype(LD), q["cp_inG"][1].astype(LD)
    g = prob.gradient(p0, cp0)
    free = np.nonzero(prob.m > 0)[0]
    h = LD(1e-7)
    num = []
    for f in free:
        for i in range(3):
            pp, pm = p0.copy(), p0.copy()
            pp[f, i] += h
            pm[f, i] -= h
            num.append((prob.evaluate(pp, cp0)["cost"] - prob.evaluate(pm, cp0)["cost"]) / (2 * h))
    if not fix:
        for i in range(3):
            cp_, cm_ = cp0.copy(), cp0.copy()
            cp_[i] += h
            cm_[i] -= h
            num.append((prob.evaluate(p0, cp_)["cost"] - prob.evaluate(p0, cm_)["cost"]) / (2 * h))
    num = np.array(num, dtype=LD)
    tol = 1e-6 * float(np.abs(num).max())
    err = float(np.abs(g - num).max())
    assert err <= tol, (err, tol)
    if not fix:  # the point-on-plane Jacobian without its -d n term: the plane's gradient moves by far more than the tolerance
        gm = prob.gradient(p0, cp0, mistake="jc_without_dn")
        assert float(np.abs(gm - num).max()) > 2 * tol


def test_planted_ransac_mistakes_are_caught():
    # points exactly 0.05 apart: the oracle's double distance is 0.05 (sqrt(fl(x^2)) = x), "<" keeps the point, "<=" drops it
    # (F = 5, min_inlier_num 3: every draw takes all five points, and "<=" leaves every draw short)
    P = np.array([[0.0, 0.0, 2.0], [0.05, 0.0, 2.0], [1.0, 0.0, 2.001], [0.0, 1.0, 1.999], [1.0, 1.0, 2.002]])
    perms = shuffles(len(P))
    ok = pr.ransac_ld(P, 3, 1e6, perms)
    bad = pr.ransac_ld(P, 3, 1e6, perms, mistake="sep<=")
    orc = oracle_backend.OracleContext(synth.make_scenario("tiny_planes").options)
    so = orc.plane_fitting([0, len(P)], P, 3, 1e6)[0][0]
    assert ok["status"] == so == 1 and bad["status"] == 0 and bad["short"]
    # the strict count: exactly thr inliers (F = 20, thr = 16) is not a valid set; ">=" accepts it
    rng = np.random.RandomState(1)
    xy = np.array([[i * 0.25, j * 0.25] for i in range(4) for j in range(5)])
    P = np.c_[xy, np.full(20, 2.0)]
    P[16:, 2] += 0.3
    P[:16, 2] += 0.002 * rng.randn(16)
    perms = shuffles(20)
    ok, bad = pr.ransac_ld(P, 5, 200.0, perms), pr.ransac_ld(P, 5, 200.0, perms, mistake="count>=")
    assert ok["decided"] and ok["status"] == 0 and bad["status"] == 1
    assert orc.plane_fitting([0, 20], P, 5, 200.0)[0][0] == 0
    # tie-break reversed: the draws with the top count keep two inlier sets, and the reversed rule returns the other one
    trng = np.random.RandomState(21)
    P = np.c_[trng.uniform(-1, 1, size=(40, 2)), 2.0 + 0.02 * trng.randn(40)]
    perms = shuffles(40)
    ok, bad = pr.ransac_ld(P, 5, 200.0, perms), pr.ransac_ld(P, 5, 200.0, perms, mistake="tiebreak")
    assert ok["decided"] and ok["inlier_decided"].all() and ok["status"] == bad["status"] == 1
    assert not np.array_equal(ok["inlier"], bad["inlier"])
    so, _, io = orc.plane_fitting([0, 40], P, 5, 200.0)
    assert so[0] == 1 and np.array_equal(io == 1, ok["inlier"])
    # the mean error over all points: 5 outliers 0.4 m off push it above 0.05, and no set is valid any more
    P = np.array([[i * 0.25, j * 0.25, 2.0] for i in range(6) for j in range(5)])
    P[25:, 2] += 0.4
    perms = shuffles(30)
    ok, bad = pr.ransac_ld(P, 5, 200.0, perms), pr.ransac_ld(P, 5, 200.0, perms, mistake="avg_all")
    assert ok["decided"] and ok["status"] == 1 and bad["status"] == 0
    assert orc.plane_fitting([0, 30], P, 5, 200.0)[0][0] == 1


def test_planted_refinement_mistakes_are_caught():
    S, orc, q = _refine_setup()
    prob, _, (a, b) = _plane_problem(orc, q, 0, 0)
    e = prob.evaluate(q["p_FinG"][a:b], q["cp_inG"][0])
    eb = prob.evaluate(q["p_FinG"][a:b], q["cp_inG"][0], mistake="one_copy_short")
    assert abs(float(e["cost"] - eb["cost"])) > 2 * e["bound"]
    # the 0.03 test on the refined position: a feature whose original position is 0.035 m off the plane and whose refined one is on it
    cp = np.array([0.0, 0.0, 2.0])
    p0 = np.array([[0.1 * i, 0.0, 2.0 + (0.035 if i == 0 else 0.001)] for i in range(6)])
    pa = p0.copy()
    pa[:, 2] = 2.0
    Rcur, pcur = np.diag([1.0, -1.0, -1.0]), np.array([0.0, 0.0, 5.0])
    ok = pr.refine_status_ld(p0, pa, cp, Rcur, pcur, True)
    bad = pr.refine_status_ld(p0, pa, cp, Rcur, pcur, True, mistake="refined_distance")
    assert ok["decided"] and bad["decided"] and not ok["inlier"][0] and bad["inlier"][0]
