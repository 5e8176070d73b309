"""CPU checks of the long-double reference of the triangulation modes (tests/triangulation_1d_reference.py): the 1-D depth against an
independent least-squares solve, its restated Gauss-Newton stage against triangulation_reference, a threshold pair on either side of every
rule of every mode, the collinear and clone-twice tracks, and planted mistakes that the generated cases must catch."""
import numpy as np
import pytest

import oracle_backend
import triangulation_1d_reference as t1
import triangulation_reference as tr
from ov_plane_b200 import synth

LD = tr.LD


def setup_module():
    tr.require_long_double()


@pytest.fixture(scope="module")
def gen():
    S = tr.scenario()
    orc = oracle_backend.OracleContext(S.options)
    ch = synth.load_scenario_into(orc, S)
    base = tr.Context(orc, ch, S.intr_value[0])
    ctxs = {mode: t1.ModeContext(base, mode) for mode in t1.MODES}
    pool = tr.random_cases(base, 300, 11)
    pairs = {(mode, o): t1.threshold_pairs(ctxs[mode], tr.OPTION_SETS[o]) for mode in ("3d_linear", "1d_linear", "1d_refine")
             for o in tr.OPTION_SETS}
    return base, ctxs, pool, pairs


def test_1d_depth_is_the_least_squares_minimiser(gen):
    """depth = argmin_d sum_k |skew(b_k) (d b_A - p_CkinA)|^2: numpy.linalg.lstsq on the stacked 3-row blocks, in double"""
    base, ctxs, pool, _ = gen
    n = 0
    for c in pool[:200] + t1.clone_twice_cases(base):
        R, pc = base.pose_arrays(c["track"])
        res = t1.linear_1d(R, pc, c["uvn"], tr.DEFAULTS)
        if "depth" not in res:
            continue
        m = len(c["track"])
        g = tr._Geometry(np.asarray(R, np.float64), np.asarray(pc, np.float64), m - 1)
        uv = np.c_[c["uvn"].astype(np.float64), np.ones(m)]
        bA = uv[-1] / np.linalg.norm(uv[-1])
        rows, rhs = [], []
        for k in range(m - 1):
            bk = g.RAt[k].T @ uv[k]
            bk /= np.linalg.norm(bk)
            rows.append(np.cross(bk, bA))
            rhs.append(np.cross(bk, g.pCA[k]))
        d = np.linalg.lstsq(np.concatenate(rows)[:, None], np.concatenate(rhs), rcond=None)[0][0]
        assert abs(d - float(res["depth"])) <= 1e-9 * max(1.0, abs(d)), (c["name"], d, float(res["depth"]))
        n += 1
    assert n >= 150


def test_refine_from_the_3d_start_reproduces_the_refined_reference(gen):
    """refine() is triangulation_reference's Gauss-Newton stage restated from any start: from the 3-D linear point it takes the same
    path and ends at the same point"""
    base, ctxs, pool, _ = gen
    n = 0
    for c in pool:
        R, pc = base.pose_arrays(c["track"])
        full = tr.triangulate(R, pc, c["uvn"], tr.DEFAULTS)
        lin = t1.linear_3d(R, pc, c["uvn"], tr.DEFAULTS)
        if lin["status"] != 1:
            continue
        res = t1.refine(R, pc, c["uvn"], tr.DEFAULTS, dict(lin, dp=0.0))
        assert tr.trace_signature(res) == tr.trace_signature(full), c["name"]
        if full["status"] == 1:
            assert float(np.abs(np.asarray(res["p_FinG"] - full["p_FinG"], np.float64)).max()) <= 1e-12
        n += 1
    assert n >= 100


@pytest.mark.parametrize("opt_name", sorted(tr.OPTION_SETS))
@pytest.mark.parametrize("mode", ["3d_linear", "1d_linear", "1d_refine"])
def test_every_rule_has_a_threshold_pair(gen, mode, opt_name):
    _, ctxs, _, pairs = gen
    opt = tr.OPTION_SETS[opt_name]
    seen = set()
    for case in pairs[(mode, opt_name)]:
        res = ctxs[mode].run(case, opt)
        cc = tr.cmp_of(res, case["rule"])
        assert tr.REL_MIN <= abs(cc["margin"]) <= tr.REL_MAX and cc["decided"] and res["decided"]
        assert res["status"] == (1 if case["side"] == "in" else 0)
        assert case["side"] == "in" or res["reason"] == case["rule"]
        seen.add((case["rule"], case["side"]))
    assert seen == {(r, s) for r in t1.RULES[mode] for s in ("in", "out")}


@pytest.mark.parametrize("opt_name", sorted(tr.OPTION_SETS))
def test_unrefined_3d_skips_the_baseline_rule(gen, opt_name):
    """the baseline pair of the refined reference: its outside case, rejected by the baseline rule alone, passes unrefined"""
    base, ctxs, _, _ = gen
    opt = tr.OPTION_SETS[opt_name]
    out = [c for c in tr.threshold_pairs(base, opt) if c["rule"] == "baseline" and c["side"] == "out"][0]
    assert base.run(out, opt)["reason"] == "baseline"
    res = ctxs["3d_linear"].run(out, opt)
    assert res["status"] == 1 and res["decided"]


def test_collinear_and_clone_twice_tracks(gen):
    base, ctxs, _, _ = gen
    for c in t1.collinear_cases(base):
        for mode in ("1d_linear", "1d_refine"):
            res = ctxs[mode].run(c, tr.DEFAULTS)
            assert res["status"] == 0 and res["decided"], (c["name"], mode, res["reason"])
            if c["name"] == "anchor_twice":
                assert res["reason"] == "lin1_zero"
    # an exact A = 0 is a NaN depth, which the NaN rule rejects
    R, pc = base.pose_arrays([base.handles[-1]] * 2)
    uvn = np.zeros((2, 2), np.float32)
    res = t1.linear_1d(np.array([np.eye(3)] * 2, dtype=LD), pc, uvn, tr.DEFAULTS)
    assert res["status"] == 0 and res["decided"] and res["A"] == 0
    # a second observation from the anchor's clone adds to A and not to b
    for c in t1.clone_twice_cases(base):
        R, pc = base.pose_arrays(c["track"])
        res = t1.linear_1d(R, pc, c["uvn"], tr.DEFAULTS)
        skip = t1.linear_1d(R, pc, c["uvn"], tr.DEFAULTS, "skip_anchor_clone")
        if c["track"].count(c["track"][-1]) > 1:
            assert res["A"] > skip["A"] and abs(res["b"] - skip["b"]) <= 1e-15 * abs(skip["b"])


@pytest.mark.parametrize("mistake", t1.MISTAKES)
def test_planted_mistakes_are_caught(gen, mistake):
    base, ctxs, pool, pairs = gen
    for (mode, opt_name), cases in sorted(pairs.items()):
        opt = tr.OPTION_SETS[opt_name]
        for case in cases + t1.clone_twice_cases(base) + t1.collinear_cases(base) + pool[:100]:
            ok = ctxs[mode].run(case, opt)
            if not ok["decided"]:
                continue
            bad = ctxs[mode].run(case, opt, mistake)
            if (bad["status"], bad["reason"]) != (ok["status"], ok["reason"]) or (
                    ok["status"] == 1 and float(np.abs(np.asarray(bad["p_FinG"] - ok["p_FinG"], np.float64)).max()) > 1e3 * ok["p_bound"]):
                print("%s caught by %s (%s) in %s under %s: status %d -> %d, reason %s -> %s" % (
                    mistake, case["name"], case.get("side", ""), mode, opt_name, ok["status"], bad["status"], ok["reason"], bad["reason"]))
                return
    raise AssertionError("planted mistake %s changes no generated case" % mistake)
