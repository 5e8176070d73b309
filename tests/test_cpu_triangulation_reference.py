"""CPU checks of the long-double triangulation reference (tests/triangulation_reference.py): against the oracle's restatement (cofactor
inverse, Jacobi, plain double) on the synthetic scenarios, against an independent minimiser of the reprojection cost, its cond(A) against
NumPy's SVD, the generated cases against the paths they were built for, and planted mistakes that the generated cases must catch."""
import numpy as np
import pytest
from scipy.optimize import least_squares

import oracle_backend
import triangulation_reference as tr
from ov_plane_b200 import synth, vio_sim

LD = tr.LD


def setup_module():
    tr.require_long_double()


@pytest.fixture(scope="module")
def gen():
    S = tr.scenario()
    orc = oracle_backend.OracleContext(S.options)
    ch = synth.load_scenario_into(orc, S)
    ctx = tr.Context(orc, ch, S.intr_value[0])
    return ctx, tr.case_sets(ctx, n_random=600)


@pytest.mark.parametrize("name", ["cfg1_euroc_n96", "cfg2_n256_f200", "cfg3_n512_f600_p8"])
def test_reference_matches_the_oracle(name):
    S = synth.make_scenario(name, seed=1)
    orc = oracle_backend.OracleContext(S.options)
    ch = np.asarray(synth.load_scenario_into(orc, S), dtype=np.int32)
    uvn = np.array([vio_sim.undistort(S.intr_value, uv.astype(np.float64)) for uv in S.uv], dtype=np.float32)
    mc = ch[S.meas_clone_idx]
    po, so = orc.triangulate_features(S.meas_offset, mc, uvn)
    ctx = tr.Context(orc, ch, S.intr_value[0])
    n_dec, worst = 0, 0.0
    for f in range(S.F):
        a, b = S.meas_offset[f], S.meas_offset[f + 1]
        res = ctx.run(dict(track=mc[a:b], uvn=uvn[a:b]), tr.DEFAULTS)
        if not res["decided"]:
            continue
        n_dec += 1
        assert res["status"] == so[f], (f, res["reason"])
        if so[f]:
            # the oracle's double LM differs from the reference by its own rounding, amplified by the float32 residuals: a float ulp of the
            # reprojection moves a point a few metres out over a short baseline by up to ~1e-5 m (tests/test_gpu_triangulation.py)
            worst = max(worst, float(np.abs(po[f] - np.asarray(res["p_FinG"], np.float64)).max()))
    print("%s: %d of %d features decided, max |reference - oracle| %.2e m" % (name, n_dec, S.F, worst))
    assert n_dec >= 0.9 * S.F and worst < 5e-5


def _smooth_cost(g, uvn, s):
    a = np.array([s[0], s[1], 1.0])
    h = np.einsum("kij,j->ki", np.asarray(g.RAt, np.float64), a) + s[2] * np.asarray(g.pAC, np.float64)
    return (uvn.astype(np.float64) - h[:, :2] / h[:, 2:3]).ravel()


def test_converged_points_minimise_the_reprojection_cost(gen):
    """where the loop stopped on min_dcost, the reference's end point lies within what that rule allows of scipy's minimiser of the
    double-precision reprojection cost: cost(s) - cost(s*) <= min_dcost cost plus the float32 rounding of the residuals, so
    |s - s*|_{J^T J}^2 <= 4 (min_dcost cost + noise)"""
    ctx, cs = gen
    n = 0
    for c in cs["defaults"]["random"][:300]:
        res = ctx.run(c, tr.DEFAULTS)
        if res["status"] != 1 or not res["decided"] or res["stop"] != "min_dcost" or len(c["track"]) > 40:
            continue
        R, pc = ctx.pose_arrays(c["track"])
        g = tr._Geometry(R, pc, len(c["track"]) - 1)
        RA, pA = np.asarray(g.RA, np.float64), np.asarray(g.pA, np.float64)
        pfa = RA @ (np.asarray(res["p_FinG"], np.float64) - pA)
        s = np.array([pfa[0] / pfa[2], pfa[1] / pfa[2], 1 / pfa[2]])
        ls = least_squares(lambda x: _smooth_cost(g, c["uvn"], x), s, xtol=1e-15, ftol=1e-15, gtol=1e-15, method="lm")
        r = _smooth_cost(g, c["uvn"], s)
        cost = float(r @ r)
        J = ls.jac
        d = s - ls.x
        noise = float((4 * np.abs(r) * 6e-8 * np.maximum(np.abs(c["uvn"].ravel()), 1.0)).sum())
        q = float(d @ (J.T @ J) @ d)
        assert q <= 4 * (tr.DEFAULTS["min_dcost"] * cost + noise), (q, cost, noise)
        n += 1
    print("%d converged features checked against scipy" % n)
    assert n >= 50


def test_cond_matches_numpy_svd(gen):
    ctx, cs = gen
    n = 0
    for c in cs["defaults"]["random"][:200]:
        if len(c["track"]) < 2:
            continue
        res = ctx.run(c, tr.DEFAULTS)
        cc = tr.cmp_of(res, "cond")
        if cc is None:
            continue
        cond = cc["value"]
        if cond > 1e6:
            continue
        R, pc = ctx.pose_arrays(c["track"])
        g = tr._Geometry(R, pc, len(c["track"]) - 1)
        bv = np.einsum("kji,kj->ki", np.asarray(g.RAt, np.float64), np.c_[c["uvn"].astype(np.float64), np.ones(len(c["track"]))])
        bv /= np.linalg.norm(bv, axis=1)[:, None]
        A = sum(np.eye(3) - np.outer(b, b) for b in bv)
        sv = np.linalg.svd(A, compute_uv=False)
        assert abs(sv[0] / sv[-1] - cond) <= 1e-9 * cond, (sv[0] / sv[-1], cond)
        n += 1
    assert n >= 100


@pytest.mark.parametrize("opt_name", ["defaults", "non_default"])
def test_generated_cases_take_the_paths_they_were_built_for(gen, opt_name):
    ctx, cs = gen
    c = cs[opt_name]
    opt = c["opt"]
    rules = set()
    for case in c["pairs"]:
        res = ctx.run(case, opt)
        cc = tr.cmp_of(res, case["rule"])
        assert tr.REL_MIN <= abs(cc["margin"]) <= tr.REL_MAX and cc["decided"] and res["decided"]
        assert res["status"] == (1 if case["side"] == "in" else 0)
        assert case["side"] == "in" or res["reason"] == case["rule"]
        rules.add((case["rule"], case["side"]))
    assert rules == {(r, s) for r in ("cond", "lin_min", "lin_max", "fin_max", "baseline") for s in ("in", "out")}
    for case in c["degenerate"]:
        res = ctx.run(case, opt)
        assert res["status"] == 0 and res["decided"] and res["reason"] in (case["expect"], "lin_chol", "cond"), (case["name"], res["reason"])
    # a rejected step and the min_dcost break under both sets; max_runs, max_lamda and min_dx where the set reaches them (all three
    # are reached by the LM option sets, test_lm_option_sets_reach_their_exit)
    print(opt_name, "LM paths found:", sorted(c["lm"]))
    assert set(c["lm"]) >= {"reject", "min_dcost"}
    for path, case in c["lm"].items():
        res = ctx.run(case, opt)
        p = tr.path_of(res)
        assert p["rejected"] if path == "reject" else p["stop"] == path
    # no generated track meets a non-positive Cholesky pivot that ov_core's QR would step over (the forward-motion track is rejected by
    # cond(A) before the LM loop, where the rho column of the Jacobian would vanish)
    for case in c["pairs"] + c["degenerate"] + list(c["lm"].values()) + c["random"]:
        assert not ctx.run(case, opt)["finding"], case["name"]
    lengths = {len(x["track"]) for x in c["random"]}
    assert lengths >= {2, 3, 16, 32, 33, 64, 100}


@pytest.mark.parametrize("opt_name,path", [("max_lamda", "max_lamda"), ("max_runs_1", "max_runs"), ("big_min_dx", "min_dx")])
def test_lm_option_sets_reach_their_exit(gen, opt_name, path):
    ctx, cs = gen
    c = cs[opt_name]
    assert path in c["lm"], sorted(c["lm"])
    res = ctx.run(c["lm"][path], c["opt"])
    assert res["stop"] == path and res["decided"]
    if path == "max_lamda":
        assert tr.path_of(res)["rejected"]


@pytest.mark.parametrize("mistake", tr.MISTAKES)
def test_planted_mistakes_are_caught(gen, mistake):
    ctx, cs = gen
    for opt_name in ("defaults", "non_default", "max_lamda", "max_runs_1", "big_min_dx"):
        c = cs[opt_name]
        cases = c.get("pairs", []) + c.get("degenerate", []) + list(c["lm"].values()) + c.get("random", [])[:200]
        for case in cases:
            ok = ctx.run(case, c["opt"])
            if not ok["decided"]:
                continue
            bad = ctx.run(case, c["opt"], mistake)
            if tr.trace_signature(bad) != tr.trace_signature(ok):
                print("%s caught by %s (%s) under %s: status %d -> %d, reason %s -> %s" % (mistake, case["name"], case.get("side", ""), opt_name,
                                                                                        ok["status"], bad["status"], ok["reason"], bad["reason"]))
                return
    raise AssertionError("planted mistake %s changes no generated case" % mistake)
