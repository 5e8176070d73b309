"""The MSCKF point update (the last plan of every ovp_msckf_update call) end to end against the long-double reference of
tests/msckf_point_reference.py, on gate_reference.correlated_cov and on its kappa = 1e10 variant (synth's P0 has diagonal clone blocks and
no calibration x clone covariance, on which a transposed clone block, a misplaced calibration column or a dropped cross term changes
nothing), along every route the update can take.

Per case: ovp_debug_msckf_gram gives the point plan's G (or, in the direct form, its raw rows), its columns and the features' statuses;
the zero pivots are decided at the smallest tolerance of 1e-11 ... 1e-6 that leaves every pivot 100 times from its threshold (another
scenario seed when there is none, its pivot gap printed); the reference is built once per (case, feature path).  On a fresh context
with the same state every route then runs the update, and each must give the hook's statuses, an Hx_order over the plan's columns and a
posterior within the same bound (update_reference.check_update: P+ element-wise and exactly symmetric, every value, FEJs bit-identical):
the default (the innovation system factored in the Gram factorisation's launch, M and S formed there, programmatic launches), the two
factorisations one after the other, M and S by two GEMM launches, the one-block-per-feature kernel and dense Gram matrix, launches
without programmatic dependence, a prepared batch replayed three times from its graph, and every system wider than 64, 128 or 192
columns factored in panels (ovp_debug_update_panel_width: chol_partial in panels, M and S by GEMMs, the innovation system in panels).

Cases: the direct form on a context of max_state 128 (Rcap = 192) at 1, 63, 64, 65, 127, 128, 129 and 192 rows, and 193 rows (the
same features, compressed); compressed systems with nc1 = ncx + 1 on and beside the 64-column tile edges (63, 127, 129, 193, 255);
tracks of 32 (the block-sparse path's longest) and of 33..39 (the one-block-per-feature kernel); the benchmark's point plans (cfg2, and
cfg3 with planeid zeroed: N = 512, 470 columns), one with sigma_pix and chi2_mult away from 1; cfg3 with its planes, whose point plan
must read P after the last plane's downdate on the side stream; and a batch with nothing accepted on an asymmetric P, in both forms,
which must leave P, values and FEJs bit-identical."""
import ctypes as C

import numpy as np
import pytest

import gate_reference as gr
import msckf_point_reference as mr
import plane_update_reference as pr
import update_reference as ur
from ov_plane_b200 import api, synth
from test_gpu_compression import _p
from test_gpu_slam_reference import _asymmetric, pick_tolerance, pivot_gap

pytestmark = pytest.mark.gpu

COVS = ("correlated", "kappa 1e10")
SEEDS = 6
TABLE_SCALE = 2.0
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for k, v in sorted(WORST.items()):
        print("MSCKF point update reference: worst %-34s %.3e" % (k, v))


def _note(k, v):
    WORST[k] = max(WORST.get(k, 0.0), v)


# ---- the library's hooks ------------------------------------------------------------------------------------------------------------
def set_panel_width(ctx, width):
    """ovp_debug_update_panel_width: every later factorisation wider than width columns runs in panels of width (0: off)"""
    ctx._ck(ctx.lib.ovp_debug_update_panel_width(ctx.h, int(width)))


def debug_gram(ctx, b, sigma_pix=1.0, chi2_mult=1.0, dense=False):
    """ovp_debug_msckf_gram on the point plan: G (None in the direct form), its layout, the statuses and the raw rows"""
    fb, keep = api.Context._batch_struct(b)
    uo = api.UpdaterOptions(sigma_pix, chi2_mult)
    F, M = fb.F, int(b["meas_offset"][-1])
    gcap = ctx.cov_rows() + 4
    G, info, cols = np.zeros(gcap * gcap), np.zeros(8, dtype=np.int32), np.zeros(gcap, dtype=np.int32)
    sel, fs, fc = np.zeros(F, dtype=np.int32), np.zeros(F, dtype=np.int32), np.zeros(F)
    raw = np.zeros(3 * gr.RAW_ROW * M)
    ctx._ck(ctx.lib.ovp_debug_force_dense_features(ctx.h, int(dense)))
    ctx._ck(ctx.lib.ovp_debug_msckf_gram(ctx.h, C.byref(fb), C.byref(uo), gcap, _p(G), _p(info), _p(cols), _p(sel), _p(fs), _p(fc), _p(raw)))
    ctx._ck(ctx.lib.ovp_debug_force_dense_features(ctx.h, 0))
    nc1, ncal, ncx, is_point = (int(v) for v in info[:4])
    assert is_point, "the first plan of the batch is not the point plan"
    return dict(G=G[:nc1 * nc1].reshape((nc1, nc1), order="F").copy() if nc1 else None, direct=nc1 == 0, ncal=ncal, ncx=ncx,
                cols=[int(c) for c in cols[:ncx]], status=fs.copy(), raw=raw.reshape(M, 3, gr.RAW_ROW))


# ---- states -------------------------------------------------------------------------------------------------------------------------
def kinds_of(ctx, S, chg):
    kinds = {ctx.handle_imu(): ur.IMU}
    if S.options["do_calib_camera_timeoffset"]:
        kinds[ctx.handle_dt()] = ur.VEC
    if S.options["do_calib_camera_pose"]:
        kinds[ctx.handle_calib()] = ur.POSE
    if S.options["do_calib_camera_intrinsics"]:
        kinds[ctx.handle_intrinsics()] = ur.VEC
    for h in chg:
        kinds[int(h)] = ur.POSE
    for pid, _, _ in S.planes:
        kinds[ctx.plane_handle(pid)] = ur.VEC
    for fid, _, _ in S.slam:
        kinds[ctx.slam_handle(fid)] = ur.LANDMARK
    return kinds


def snapshot(ctx, kinds):
    vals, fejs = {}, {}
    for h in kinds:
        vals[h], fejs[h] = ctx.var_get(h)
    return ctx.cov().copy(), vals, fejs


def same_state(a, b):
    return (np.array_equal(a[0].view(np.uint64), b[0].view(np.uint64)) and
            all(np.array_equal(a[1][h].view(np.uint64), b[1][h].view(np.uint64)) and np.array_equal(a[2][h].view(np.uint64), b[2][h].view(np.uint64))
                for h in a[1]))


class Case(object):
    pass


def new_ctx(cs, P=None, values=None):
    """a debug context with the case's scenario loaded, P (the case's covariance by default) and, when given, the values {handle:
    (value, fej)} uploaded; returns (ctx, clone handles, batch)"""
    S = cs.S
    ctx = api.Context(S.options, device=0, max_state=cs.max_state, max_meas_rows=60000, debug=True)
    ctx.set_chi2_table(cs.table)
    chg = synth.load_scenario_into(ctx, S)
    if values is not None:
        for h, (v, f) in values.items():
            ctx.var_set(h, v, f)
    ctx.cov_upload(cs.P if P is None else P)
    return ctx, chg, cs.batch_of(synth.feature_batch(S, chg))


# (name, ncal, rows of a cut batch or None, max_state or None (N), scenario)
def _direct(rows, ncal):
    return ("direct-rows%d" % rows, ncal, rows, 128, dict(n_clones=16, F=40, m_min=8, m_max=16))


def _edge(nc1, ncal):
    k = (nc1 - 1 - ncal) // 6
    assert ncal + 6 * k + 1 == nc1
    return ("compressed-nc1_%d" % nc1, ncal, None, None, dict(n_clones=k, F=max(60, 3 * k), m_min=6, m_max=min(k, 16)))


DIRECT = [_direct(r, n) for r, n in ((1, 0), (63, 14), (64, 6), (65, 8), (127, 0), (128, 8), (129, 8), (192, 14), (193, 14))]
EDGES = [_edge(n, c) for n, c in ((63, 14), (127, 0), (129, 8), (193, 6), (255, 14))]
KERNELS = [("tracks_of_32", 8, None, None, dict(n_clones=34, F=37, m_min=32, m_max=32, dtheta=0.006)),
           ("tracks_33_39", 6, None, None, dict(n_clones=40, F=23, m_min=33, m_max=39, dtheta=0.005))]
BENCH = [("cfg2_n256_f200", None, None, None, None), ("cfg3_n512_f600_p8", None, None, None, None),
         ("cfg2_n256_f200-sigma1.3-chi0.9", None, None, None, None)]
CASES = DIRECT + EDGES + KERNELS + BENCH

COMPRESSED_ROUTES = ("default", "sequential", "unfused", "dense", "pdl off", "graph", "panels 64", "panels 128", "panels 192")
DIRECT_ROUTES = ("default", "pdl off", "graph")


def routes_of(name, direct, rows):
    if name.startswith("cfg3"):
        return ("default", "panels 192")
    if "sigma" in name:
        return ("default", "panels 64")
    if direct:
        return DIRECT_ROUTES + (("panels 64",) if rows > 64 else ())
    return COMPRESSED_ROUTES


def make_case(case, cov, seed):
    name, ncal, rows, max_state, sc = case
    cs = Case()
    cs.name, cs.seed, cs.sigma_pix, cs.chi2_mult = name, seed, 1.0, 1.0
    if sc is None:  # the benchmark's point plans
        base = name.split("-")[0]
        cs.S = synth.make_scenario(base, seed=seed)
        if "sigma" in name:
            cs.sigma_pix, cs.chi2_mult = 1.3, 0.9
        cs.max_state = cs.S.N + 64
        cs.batch_of = lambda b: dict(b, planeid=np.zeros_like(b["planeid"]))
    else:
        sc = dict(sc)
        cs.S = mr.point_scenario(ncal, sc.pop("n_clones"), sc.pop("F"), sc.pop("m_min"), sc.pop("m_max"), seed=seed, **sc)
        cs.max_state = max_state or cs.S.N
        cs.batch_of = (lambda b: mr.cut_to_rows(b, rows)) if rows else (lambda b: b)
    # the scenarios' state errors are drawn from synth's P0, not from the correlated covariance, so their chi2 runs at 1 ... 3 times the
    # 95% threshold: with the table doubled most features pass and some are still rejected (their rows zero in G)
    cs.table = TABLE_SCALE * synth.chi2_table()
    cs.P = gr.correlated_cov(cs.S, cs.S.N, 41 + seed + (ncal or 0), cond=None if cov == "correlated" else 1e10)
    return cs


# ---- one route of the update --------------------------------------------------------------------------------------------------------
def run_route(ctx, route, b, cs):
    """the update of b on ctx (its state restored from the snapshot) through one route; returns the results of every run (three for the
    graph replay)"""
    set_ = {"sequential": ctx.lib.ovp_debug_sequential_factorisations, "unfused": ctx.lib.ovp_debug_unfused_update_products,
            "dense": ctx.lib.ovp_debug_force_dense_features}
    if route in set_:
        ctx._ck(set_[route](ctx.h, 1))
    if route == "pdl off":
        ctx._ck(ctx.lib.ovp_debug_programmatic_launches(ctx.h, 0))
    if route.startswith("panels"):
        set_panel_width(ctx, int(route.split()[1]))
    try:
        if route == "graph":
            ctx.msckf_prepare(b, cs.sigma_pix, cs.chi2_mult)
            for _ in range(3):
                ctx.restore()
                ctx.msckf_launch()
                yield ctx.msckf_finish()
        else:
            ctx.restore()
            yield ctx.msckf_update(b, cs.sigma_pix, cs.chi2_mult)
    finally:
        for fn in set_.values():
            ctx._ck(fn(ctx.h, 0))
        ctx._ck(ctx.lib.ovp_debug_programmatic_launches(ctx.h, 1))
        set_panel_width(ctx, 0)


def _id(case):
    return case[0] + ("-ncal%d" % case[1] if case[1] is not None else "")


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
@pytest.mark.parametrize("cov", COVS, ids=["correlated", "kappa1e10"])
def test_point_update_against_long_double(case, cov):
    ur.require_long_double()
    name, ncal, rows, _, _ = case
    for seed in range(SEEDS):
        cs = make_case(case, cov, seed)
        ctx, chg, b = new_ctx(cs)
        kinds = kinds_of(ctx, cs.S, chg)
        snap0 = snapshot(ctx, kinds)
        g = debug_gram(ctx, b, cs.sigma_pix, cs.chi2_mult)
        assert same_state(snap0, snapshot(ctx, kinds)), "ovp_debug_msckf_gram changed the state"
        direct = g["direct"]
        routes = routes_of(name, direct, rows or 0)
        gd = debug_gram(ctx, b, cs.sigma_pix, cs.chi2_mult, dense=True) if "dense" in routes else None
        calib = gr.calib_ids(ctx, cs.S.options)
        ids = {h: ctx.var_id(h) for h in kinds}
        var_id = {int(h): ctx.var_id(int(h)) for h in chg}.__getitem__  # clone handle -> state id, usable after close
        ctx.close()
        st = g["status"]
        tag = "%s %s seed %d: F %d, ncx %d, %s, accepted %d" % (_id(case), cov, seed, b["F"], g["ncx"], "direct" if direct else "nc1 %d" % (g["ncx"] + 1),
                                                               int((st == 1).sum()))
        if ncal is not None:
            assert g["ncal"] == ncal, tag
        if rows is not None:
            # the form: direct up to the innovation workspace (Rcap = max_state + 64 = 192), compressed one row beyond
            assert direct == (rows <= 192), tag
        if name.startswith("compressed") or name.startswith("tracks"):
            if g["ncx"] != ncal + 6 * cs.S.cfg["n_clones"]:
                print("%s: not every clone observed; next scenario" % tag)
                continue
        if gd is not None:
            assert np.array_equal(gd["status"], st), "%s: the dense feature path's statuses differ" % tag
        if direct:
            tol = pr.GRAM_TOL
            break
        Gs = [g["G"]] + ([gd["G"]] if gd is not None else [])
        tols = [pick_tolerance(G, g["ncx"]) for G in Gs]
        if all(t is not None for t in tols):
            tol = max(tols)
            if all(pick_tolerance_at(G, g["ncx"], tol) for G in Gs):
                break
        hi, lo = pivot_gap(g["G"], g["ncx"])
        print("%s: no tolerance in 1e-11 ... 1e-6 leaves every pivot 100x clear (at 1e-11: %.3g above, %.3g below); next scenario" % (tag, hi, lo))
    else:
        raise AssertionError("%s: no scenario of %d has a rank decision clear of rounding" % (_id(case), SEEDS))
    P = snap0[0]
    cols = g["cols"]
    assert (st == 1).any(), "%s: the gates accept no feature; the case checks nothing" % tag
    acc_cols = sorted(set(calib) | {var_id(int(b["meas_clone"][k])) + j for f in range(b["F"]) if st[f] == 1
                                    for k in range(int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])) for j in range(6)})
    assert set(acc_cols) <= set(cols), tag
    # the reference, once per feature path
    refs = {}
    if direct:
        X, Xb = mr.stacked_rows(mr.raw_features(g["raw"], b, st, g["ncal"], calib, var_id), cols)
        assert X.shape[0] == sum(2 * (int(b["meas_offset"][f + 1]) - int(b["meas_offset"][f])) - 3 for f in range(b["F"]) if st[f] == 1)
        refs["warp"] = refs["dense"] = mr.direct_reference(P, cols, X, Xb)
    else:
        refs["warp"] = mr.gram_reference(P, cols, g["G"], tol)
        refs["dense"] = mr.gram_reference(P, cols, gd["G"], tol) if gd is not None else None
    print("%s: tol %g" % (tag, tol))
    ctx, chg, b = new_ctx(cs)
    ctx.set_rank_tolerance(tol)
    ctx.snapshot()
    for route in routes:
        d = refs["dense" if route == "dense" else "warp"]
        for res in run_route(ctx, route, b, cs):
            assert np.array_equal(res["feat_status"], st), "%s, %s: statuses differ from the hook's" % (tag, route)
            got = snapshot(ctx, kinds)
            hx = sorted(i for h in res["hx_order"] for i in range(ctx.var_id(h), ctx.var_id(h) + ctx.var_size(h)))
            assert hx == acc_cols, "%s, %s: Hx_order does not map to the plan's columns of the accepted features" % (tag, route)
            qP, qv = ur.check_update(got[0], got[1], got[2], P, kinds, ids, snap0[1], snap0[2], d["ref"]["dx"], d["dxb"], d["dPb"],
                                     d["ref"]["P"])
            form = "direct" if direct else "compressed"
            _note("%s %s P+" % (form, route), qP)
            _note("%s %s values" % (form, route), qv)
            _note("%s P+" % cov, qP)
            print("%s, %s: worst error / bound P+ %.3e values %.3e" % (tag, route, qP, qv))
    ctx.close()


def pick_tolerance_at(G, npiv, tol):
    _, _, ratio = pr.ld_factor(G, npiv, tol)
    return bool(np.all((ratio >= pr.PIVOT_MARGIN) | (ratio <= 1.0 / pr.PIVOT_MARGIN)))


# ---- the benchmark's chain: planes, then the point plan -----------------------------------------------------------------------------
def _after_planes(cs, tol):
    """(kinds, state after an update of the plane features alone at tolerance tol, their plane statuses)"""
    ctx, chg, _ = new_ctx(cs)
    ctx.set_rank_tolerance(tol)
    kinds = kinds_of(ctx, cs.S, chg)
    r = ctx.msckf_update(synth.feature_batch(cs.S, chg, np.nonzero(cs.S.planeid != 0)[0]), 1.0, 1.0)
    s1 = snapshot(ctx, kinds)
    ctx.close()
    return kinds, s1, r["plane_status"]


def test_point_plan_reads_the_covariance_after_the_last_plane():
    """cfg3 with its 8 planes: the point plan's M = P[:, cols] L must read P after the last plane's downdate (on the side stream).  On
    a seed where every plane passes (no feature falls through to the point update): the state after a call with the plane features
    alone, the reference of the remaining features' point plan on that state, against one msckf_update of the whole batch."""
    ur.require_long_double()
    found = None
    for seed in range(SEEDS):
        cs = Case()
        cs.S = synth.make_scenario("cfg3_n512_f600_p8", seed=seed)
        # every plane (chi2 about twice its threshold on the correlated covariance) passes a table four times synth's
        cs.max_state, cs.table, cs.sigma_pix, cs.chi2_mult = cs.S.N + 64, 4.0 * synth.chi2_table(), 1.0, 1.0
        cs.P = gr.correlated_cov(cs.S, cs.S.N, 77 + seed)
        cs.batch_of = lambda bb: bb
        off = np.nonzero(cs.S.planeid == 0)[0]
        for tol in (1e-11, 1e-10, 1e-9, 1e-8, 1e-7, 1e-6):
            kinds, s1, ps = _after_planes(cs, tol)
            if not np.all(ps == 1):
                print("seed %d, tol %g: plane statuses %s; next" % (seed, tol, ps))
                continue
            # the point plan of the remaining features on that state
            ctx, chg, _ = new_ctx(cs, P=s1[0], values={h: (s1[1][h], s1[2][h]) for h in kinds})
            bp = synth.feature_batch(cs.S, chg, off)
            g = debug_gram(ctx, bp)
            ids = {h: ctx.var_id(h) for h in kinds}
            feats = mr.raw_features(g["raw"], bp, g["status"], g["ncal"], gr.calib_ids(ctx, cs.S.options), ctx.var_id)
            ctx.close()
            if pick_tolerance_at(g["G"], g["ncx"], tol):
                found = (seed, tol)
                break
        if found:
            break
    assert found, "no cfg3 seed of %d has every plane passing and a rank decision clear of rounding" % SEEDS
    seed, tol = found
    # G here and the G the whole batch's point plan factors are two launches over the same rows: their rounding enters the bound
    X, _ = mr.stacked_rows(feats, g["cols"])
    d = mr.gram_reference(s1[0], g["cols"], g["G"], tol, X=X)
    ctx, chg, b = new_ctx(cs)
    ctx.set_rank_tolerance(tol)
    r = ctx.msckf_update(b, 1.0, 1.0)
    got = snapshot(ctx, kinds)
    ctx.close()
    assert np.all(r["plane_status"] == 1)
    assert np.array_equal(r["feat_status"][off], g["status"]), "the point features' statuses differ from the hook's"
    qP, qv = ur.check_update(got[0], got[1], got[2], s1[0], kinds, ids, s1[1], s1[2], d["ref"]["dx"], d["dxb"], d["dPb"], d["ref"]["P"])
    _note("chain P+", qP)
    _note("chain values", qv)
    print("cfg3 seed %d, tol %g: %d point features accepted; worst error / bound P+ %.3e values %.3e" % (
        seed, tol, int((g["status"] == 1).sum()), qP, qv))


# ---- nothing accepted ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [_direct(129, 8), _edge(127, 0)], ids=["direct", "compressed"])
def test_nothing_accepted_leaves_the_state_bit_identical(case):
    """the chi2 table times 1e-3 rejects every feature; on an asymmetric P a mirrored downdate would show"""
    cs = make_case(case, "correlated", 0)
    cs.table = synth.chi2_table() * 1e-3
    ctx, chg, b = new_ctx(cs, P=_asymmetric(cs.P, 5))
    kinds = kinds_of(ctx, cs.S, chg)
    g = debug_gram(ctx, b)
    assert g["direct"] == (case[0].startswith("direct"))
    s0 = snapshot(ctx, kinds)
    ctx.snapshot()
    for route in ("default", "graph"):
        for res in run_route(ctx, route, b, cs):
            assert np.all(res["feat_status"] == 0), res["feat_status"]
            assert same_state(s0, snapshot(ctx, kinds)), "%s: nothing accepted, the state changed" % route
    ctx.close()


def test_panel_width_hook_refuses_bad_widths():
    S = mr.point_scenario(0, 8, 10, 3, 8)
    ctx = api.Context(S.options, device=0, max_state=128, max_meas_rows=4096, debug=True)
    for w in (-64, 32, 65, 100000):
        with pytest.raises(api.OvpError) as e:
            set_panel_width(ctx, w)
        assert e.value.status == 1, e.value  # OVP_ERR_BAD_ARGS
    for w in (64, 128, 0):
        set_panel_width(ctx, w)
    ctx.close()
