"""UpdaterSLAM::update on the device (slam_host.inc) and marginalize_slam against the long-double references of tests/slam_reference.py.

Every update case runs on gate_reference.correlated_cov and on its kappa = 1e10 variant (synth's P0 has no clone x calibration or plane x
landmark covariance, on which a transposed or misplaced block changes nothing), with 0, 6, 8 and 14 calibration columns.  Per case:
- G from ovp_debug_slam_gram against the long-double X^T X of the reference's stack (the accepted landmarks' raw rows), Jacobi-scaled,
  within the Gram kernel's rounding bound; its strictly upper part, the columns of every rejected landmark and the plane columns no
  accepted landmark reaches exactly zero; the same bits run to run, the state and its bookkeeping untouched;
- on a fresh context, ovp_slam_update against the reference: P+ element-wise within its a-priori bound and exactly symmetric, every value
  (quaternions through rotation matrices too) within its bound, FEJs bit-identical, statuses, should_marg and the landmark-to-plane map
  as the reference keeps them.
The zero pivots are decided at the smallest tolerance of 1e-11 (the default) ... 1e-6 that leaves every pivot 100 times from its
threshold; the pivot gap at the default is printed.  Then: a batch with no accepted landmark leaves P, values and FEJs bit-identical (on an
asymmetric P too, where a mirrored downdate shows); a rejected ArUco landmark is not flagged; the row capacity is refused one row beyond
it with nothing changed; marginalize_slam is bit-exact."""
import ctypes as C

import numpy as np
import pytest

import gate_reference as gr
import plane_update_reference as pr
import slam_reference as sr
import update_reference as ur
from ov_plane_b200 import api, synth
from test_gpu_compression import _p

pytestmark = pytest.mark.gpu

COVS = ("correlated", "kappa 1e10")
TOLS = (1e-11, 1e-10, 1e-9, 1e-8, 1e-7, 1e-6)
ARUCO_FEATID = 7
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for k, v in sorted(WORST.items()):
        print("SLAM update reference: worst %-26s %.3e" % (k, v))


def _note(k, v):
    WORST[k] = max(WORST.get(k, 0.0), v)


# ---- setup ---------------------------------------------------------------------------------------------------------------------------
class Case(object):
    pass


def make_case(ncal, cov, shape, seed=0):
    """shape: ("batch", use_plane) the 24-landmark batch of gate_reference.slam_update_batch (tracks of 1, 2, 15, 29, three landmarks on a
    wrong plane); ("single", m, plane) one landmark with its newest m measurements, on its plane or not; ("retry_only",) the wrong-plane
    landmarks alone (every accepted one has status 3); ("long",) every landmark with its whole track less one measurement (thousands of
    rows, several k splits of the Gram kernel)."""
    cs = Case()
    cs.S = gr.slam_scenario(ncal, seed=seed)
    cs.S.featid[1] = ARUCO_FEATID
    cs.ncal, cs.cov, cs.shape, cs.seed = ncal, cov, shape, seed
    cs.use_plane = shape[1] if shape[0] == "batch" else True
    return cs


def new_ctx(cs, table=None, max_meas_rows=60000):
    S = cs.S
    ctx = api.Context(S.options, device=0, max_state=S.N + 3 * S.F + 64, max_meas_rows=max_meas_rows, debug=True)
    ctx.set_chi2_table(synth.chi2_table())
    chg = synth.load_scenario_into(ctx, S)
    g = ctx.slam_delayed_init(synth.feature_batch(S, chg), 1.0, 1.0)
    keep = np.nonzero(g["feat_status"] > 0)[0]
    attached = {int(S.featid[f]) for f in keep if g["feat_status"][f] == 1 and S.planeid[f] != 0}
    if not hasattr(cs, "P"):
        cs.P = gr.correlated_cov(S, ctx.cov_rows(), 7 + cs.ncal + cs.seed, cond=None if cs.cov == "correlated" else 1e10)
    ctx.cov_upload(cs.P)
    if table is not None:
        ctx.set_chi2_table(table)
    b = gr.slam_update_batch(S, chg, keep, seed=cs.ncal, wrong_plane=3)
    b = select(cs, b, attached, S, chg, keep)
    return ctx, chg, b, attached


def _cut(b, sel, lengths=None):
    offs, mc, uv = [0], [], []
    for i, f in enumerate(sel):
        a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
        n = e - a if lengths is None else lengths[i]
        mc.append(b["meas_clone"][e - n:e])
        uv.append(b["uv"][e - n:e])
        offs.append(offs[-1] + n)
    out = dict(b)
    for k in ("p_FinG", "p_FinG_original", "featid", "planeid"):
        out[k] = np.ascontiguousarray(b[k][sel])
    out.update(F=len(sel), meas_offset=np.array(offs, dtype=np.int32), meas_clone=np.ascontiguousarray(np.concatenate(mc), dtype=np.int32),
               uv=np.ascontiguousarray(np.concatenate(uv), dtype=np.float32))
    return out


def select(cs, b, attached, S, chg, keep):
    kind = cs.shape[0]
    if kind == "batch":
        return b
    if kind == "short":  # every landmark with its newest two measurements: a wide, short batch
        return _cut(b, list(range(b["F"])), [min(2, int(b["meas_offset"][f + 1] - b["meas_offset"][f])) for f in range(b["F"])])
    if kind == "single":
        _, m, plane = cs.shape
        full = synth.feature_batch(S, chg, keep)
        lens = np.diff(full["meas_offset"])
        f = next(i for i in range(full["F"]) if (int(full["featid"][i]) in attached) == plane and lens[i] >= m and int(full["featid"][i]) != ARUCO_FEATID)
        return _cut(full, [f], [m])
    if kind == "retry_only":
        moved = [i for i in range(b["F"]) if int(b["featid"][i]) in attached][:3]
        return _cut(b, moved)
    if kind == "long":  # whole tracks less one measurement; one more dropped where that makes the row count a multiple of 16
        full = synth.feature_batch(S, chg, keep)
        lens = np.diff(full["meas_offset"]) - 1
        rows = sum((3 if int(full["featid"][i]) in attached else 2) * lens[i] for i in range(full["F"]))
        if rows % 16 == 0:
            lens[0] -= 1
        return _cut(full, list(range(full["F"])), [int(x) for x in lens])
    raise AssertionError(kind)


def kinds_of(ctx, cs, chg, b):
    S = cs.S
    kinds = {ctx.handle_imu(): ur.IMU}
    if S.options["do_calib_camera_timeoffset"]:
        kinds[ctx.handle_dt()] = ur.VEC
    if S.options["do_calib_camera_pose"]:
        kinds[ctx.handle_calib()] = ur.POSE
    if S.options["do_calib_camera_intrinsics"]:
        kinds[ctx.handle_intrinsics()] = ur.VEC
    for h in chg:
        kinds[int(h)] = ur.POSE
    for pid in S.plane_ids:
        kinds[ctx.plane_handle(int(pid))] = ur.VEC
    for fid in S.featid:
        h = ctx.slam_handle(int(fid))
        if h >= 0:
            kinds[h] = ur.LANDMARK
    return kinds


def snapshot(ctx, kinds, fids):
    vals, fejs = {}, {}
    for h in kinds:
        vals[h], fejs[h] = ctx.var_get(h)
    book = [(ctx.slam_should_marg(int(f)), ctx.slam_plane_of(int(f))) for f in fids]
    return ctx.cov().copy(), vals, fejs, book


def same_state(a, b):
    return (np.array_equal(a[0].view(np.uint64), b[0].view(np.uint64)) and a[3] == b[3] and
            all(np.array_equal(a[1][h].view(np.uint64), b[1][h].view(np.uint64)) and np.array_equal(a[2][h].view(np.uint64), b[2][h].view(np.uint64))
                for h in a[1]))


def state_diff(a, b):
    out = []
    bad = a[0].view(np.uint64) != b[0].view(np.uint64)
    if bad.any():
        i, j = np.argwhere(bad)[0]
        out.append("P: %d entries differ, first [%d, %d] %r -> %r" % (int(bad.sum()), i, j, a[0][i, j], b[0][i, j]))
    for h in a[1]:
        if not np.array_equal(a[1][h].view(np.uint64), b[1][h].view(np.uint64)):
            out.append("value of handle %d: %s" % (h, (b[1][h] - a[1][h]).tolist()))
        if not np.array_equal(a[2][h].view(np.uint64), b[2][h].view(np.uint64)):
            out.append("FEJ of handle %d" % h)
    if a[3] != b[3]:
        out.append("bookkeeping %s -> %s" % (a[3], b[3]))
    return "; ".join(out)


def debug_gram(ctx, b, use_plane, sigma_pix=1.0, chi2_mult=1.0):
    F, M = int(b["F"]), int(b["meas_offset"][-1])
    uo = api.UpdaterOptions(sigma_pix, chi2_mult)
    gcap = ctx.cov_rows() + 1
    G, info, cols = np.zeros(gcap * gcap), np.zeros(2, dtype=np.int32), np.zeros(gcap, dtype=np.int32)
    fs, fc, raw = np.zeros(F, dtype=np.int32), np.zeros(F), np.zeros(3 * gr.RAW_ROW * M)
    mo, mc = np.ascontiguousarray(b["meas_offset"], dtype=np.int32), np.ascontiguousarray(b["meas_clone"], dtype=np.int32)
    uv = np.ascontiguousarray(b["uv"], dtype=np.float32)
    fid, pid = np.ascontiguousarray(b["featid"], dtype=np.int64), np.ascontiguousarray(b["planeid"], dtype=np.int64)
    ctx._ck(ctx.lib.ovp_debug_slam_gram(ctx.h, F, _p(mo), _p(mc), _p(uv), _p(fid), _p(pid), C.byref(uo), int(bool(use_plane)), gcap, _p(G),
                                        _p(info), _p(cols), _p(fs), _p(fc), _p(raw)))
    nc1, rows = int(info[0]), int(info[1])
    return dict(G=G[:nc1 * nc1].reshape((nc1, nc1), order="F").copy(), cols=cols[:nc1 - 1].copy(), status=fs, chi2=fc, rows=rows,
                raw=raw.reshape(M, 3, gr.RAW_ROW))


def on_plane(ctx, b, f, use_plane):
    """the landmark's rows carry its plane (slam_plane_of in slam_host.inc): a plane id, the plane in the state, not detached"""
    pid = int(b["planeid"][f])
    return bool(use_plane) and pid != 0 and ctx.plane_handle(pid) >= 0 and ctx.slam_plane_of(int(b["featid"][f])) != 0


def stacked(ctx, cs, b, g, use_plane, **mistakes):
    """(X over the library's compact columns, per-landmark (state ids of its columns, status, on its plane))"""
    cal = gr.calib_ids(ctx, cs.S.options)
    parts, info = [], []
    for f in range(b["F"]):
        a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
        hp = on_plane(ctx, b, f, use_plane)
        Hf, Hx, r = gr.raw_block(g["raw"], a, e, len(cal), hp)
        ids = gr.block_ids(ctx, [ctx.slam_handle(int(b["featid"][f]))]) + cal + gr.block_ids(ctx, b["meas_clone"][a:e], 6)
        if hp:
            ids += gr.block_ids(ctx, [ctx.plane_handle(int(b["planeid"][f]))])
        info.append((ids, int(g["status"][f]), hp))
        out = sr.landmark_rows(Hf, Hx, r, int(g["status"][f]), hp, e - a, **mistakes)
        if out is not None:
            parts.append((out[0], out[1], ids[:out[0].shape[1]]))
    return sr.stack(parts, [int(s) for s in g["cols"]]), info


def pick_tolerance(G, nc):
    for tol in TOLS:
        _, _, ratio = pr.ld_factor(G, nc, tol)
        if np.all((ratio >= pr.PIVOT_MARGIN) | (ratio <= 1.0 / pr.PIVOT_MARGIN)):
            return tol
    return None


def pivot_gap(G, nc):
    """the pivot / threshold ratios at the default tolerance nearest to 1 from above and from below"""
    _, _, ratio = pr.ld_factor(G, nc, pr.GRAM_TOL)
    above, below = ratio[ratio > 1.0], ratio[ratio <= 1.0]
    return (float(above.min()) if len(above) else np.inf), (float(below.max()) if len(below) else 0.0)


# ---- the update ----------------------------------------------------------------------------------------------------------------------
SINGLES = [("single", m, p) for m in (1, 2, 29) for p in (True, False)]
SHAPES = [("batch", True), ("batch", False)] + SINGLES + [("retry_only",), ("long",)]
# one landmark puts nc1 = 3 + ncal + 6m (+ 3 with its plane) + 1 on and beside the 64- and 128-column tile edges: 63, 64 and 126, 127,
# 129 (65 and 128 are not 3 + ncal + 6m + 3p + 1 for any ncal in {0, 6, 8, 14})
EDGES = [(14, ("single", 7, True)), (0, ("single", 10, False)), (8, ("single", 19, False)), (0, ("single", 20, True)), (8, ("single", 19, True))]
CASES = [(n, s) for s in SHAPES for n in (0, 6, 8, 14)] + EDGES
SEEDS = 6


def _id(case):
    n, s = case
    return "ncal%d-%s" % (n, "-".join(str(x) for x in s))


def check_gram(cs, cov):
    """ovp_debug_slam_gram on the case: G against long double, its exact zeros, the same bits run to run, the state untouched.  Returns
    (ctx, chg, b, kinds, fids, snap0, g, X, info, tag)."""
    ctx, chg, b, attached = new_ctx(cs)
    kinds = kinds_of(ctx, cs, chg, b)
    fids = list(cs.S.featid)
    snap0 = snapshot(ctx, kinds, fids)
    g = debug_gram(ctx, b, cs.use_plane)
    again = debug_gram(ctx, b, cs.use_plane)
    assert np.array_equal(g["G"].view(np.uint64), again["G"].view(np.uint64)), "G differs run to run"
    now = snapshot(ctx, kinds, fids)
    assert same_state(snap0, now), "ovp_debug_slam_gram changed the state: %s" % state_diff(snap0, now)
    X, info = stacked(ctx, cs, b, g, cs.use_plane)
    nc = len(g["cols"])
    st = g["status"]
    shape = cs.shape
    tag = "%s %s seed %d: F %d, rows %d, nc1 %d, statuses %s" % (_id((cs.ncal, shape)), cov, cs.seed, b["F"], g["rows"], nc + 1,
                                                                 np.bincount(st, minlength=4).tolist())
    # the row offsets the update laid out: 3m on the plane, 2m without, whatever the status
    assert g["rows"] == sum(3 * (e - a) if hp else 2 * (e - a) for (ids, s, hp), a, e in zip(info, b["meas_offset"][:-1], b["meas_offset"][1:])), tag
    if shape[0] == "single":
        assert nc + 1 == 3 + cs.ncal + 6 * shape[1] + (3 if shape[2] else 0) + 1, tag
    if shape[0] == "long":
        assert g["rows"] >= 1500 and g["rows"] % 16 != 0, tag
    # G: exactly lower, zero where no accepted row reaches, element-wise against long double
    G = g["G"]
    assert not np.triu(G, 1).any(), "%s: G has non-zero entries above the diagonal" % tag
    col_of = {int(s): c for c, s in enumerate(g["cols"])}
    reached = np.zeros(nc + 1, dtype=bool)
    reached[nc] = True
    for ids, s, hp in info:
        if s == 1:
            reached[[col_of[i] for i in ids]] = True
        elif s == 3:
            reached[[col_of[i] for i in ids[:len(ids) - (3 if hp else 0)]]] = True
    assert not G[~reached, :].any() and not G[:, ~reached].any(), "%s: G non-zero in a column no accepted landmark reaches" % tag
    Gref = sr.gram_ld(X)
    dG = sr.gram_bound(X)
    low = np.tril(np.ones_like(G, dtype=bool))
    eG = np.abs(np.asarray(G - Gref, dtype=np.float64))[low]
    assert np.all(eG <= dG[low]), "%s: G error above the Gram bound" % tag
    qG = float((eG / np.where(dG[low] > 0, dG[low], 1.0)).max())
    _note("G", qG)
    return ctx, chg, b, kinds, fids, snap0, g, X, info, tag + " (G error / bound %.3e)" % qG


# nc1 = 129 (nc = 128: two full 64-column tiles, the residual alone in a third) misses its posterior bound by about 60x on both
# covariances, P+ off by 1.5e-2 of the prior's standard deviations, while nc1 = 126 and 127 meet theirs: an open defect at that edge
KNOWN = {(8, ("single", 19, True)): "nc1 = 129: the posterior misses its bound by ~60x (open defect at nc = 128)"}


def _param(c):
    return pytest.param(c, id=_id(c), marks=pytest.mark.xfail(strict=True, reason=KNOWN[c])) if c in KNOWN else pytest.param(c, id=_id(c))


@pytest.mark.parametrize("case", [_param(c) for c in CASES])
@pytest.mark.parametrize("cov", COVS, ids=["correlated", "kappa1e10"])
def test_slam_update_against_long_double(case, cov):
    ur.require_long_double()
    ncal, shape = case
    # G is checked on every scenario tried; the posterior on the first (seed 0, 1, ...) whose G leaves every pivot 100x clear of one
    # tolerance in 1e-11 ... 1e-6.  Where the weakest real direction lies within 1e4 of the rounding-level pivots of the unobservable
    # ones there is no such tolerance: the library's and any reference's rank decision is rounding's, and its pivot gap is printed.
    for seed in range(SEEDS):
        cs = make_case(ncal, cov, shape, seed)
        ctx, chg, b, kinds, fids, snap0, g, X, info, tag = check_gram(cs, cov)
        nc = len(g["cols"])
        gap_hi, gap_lo = pivot_gap(g["G"], nc)
        tol = pick_tolerance(g["G"], nc)
        fits = shape[0] != "retry_only" or bool(np.all(g["status"] == 3))
        if tol is not None and fits:
            break
        print("%s: %s; next scenario" % (tag, "not every landmark has status 3" if not fits else
                                         "no tolerance in 1e-11 ... 1e-6 leaves every pivot 100x clear (at 1e-11: %.3g above, %.3g below)"
                                         % (gap_hi, gap_lo)))
        ctx.close()
    else:
        # every scenario tried leaves the rank decision to rounding: G was checked on each, the posterior has no reference to meet
        print("%s: G checked on %d scenarios; none has a rank decision clear of rounding, the posterior is not compared" % (_id(case), SEEDS))
        _note("cases with G only", 1.0)
        return
    P = snap0[0]
    G, st = g["G"], g["status"]
    ref = sr.slam_update_reference(P, [int(s) for s in g["cols"]], X)
    print("%s: tol %g" % (tag, tol))
    ctx.close()
    # the update on a fresh context
    ctx, chg, b, attached = new_ctx(cs)
    ctx.set_rank_tolerance(tol)
    res = ctx.slam_update(b, 1.0, 1.0, cs.use_plane)
    assert np.array_equal(res["feat_status"], st), "%s: statuses %s, the Gram hook's %s" % (tag, res["feat_status"], st)
    got = snapshot(ctx, kinds, fids)
    ids = {h: ctx.var_id(h) for h in kinds}
    if ref is None:
        assert same_state(snap0, got), "%s: nothing accepted, the state changed: %s" % (tag, state_diff(snap0, got))
        qP = qv = 0.0
    else:
        dxb, dPb, fac = sr.slam_bounds(P, [int(s) for s in g["cols"]], X, G, ref, tol)
        qP, qv = ur.check_update(got[0], got[1], got[2], P, kinds, ids, snap0[1], snap0[2], ref["dx"], dxb, dPb, ref["P"])
    # bookkeeping: detached from the plane when it failed on it, flagged when rejected unless an ArUco tag
    for f in range(b["F"]):
        fid, s = int(b["featid"][f]), int(st[f])
        if info[f][2]:
            assert ctx.slam_plane_of(fid) == (int(b["planeid"][f]) if s == 1 else 0), (tag, f)
        assert ctx.slam_should_marg(fid) == (1 if s == 0 and fid >= cs.S.options["max_aruco_features"] else 0), (tag, f, fid, s)
    print("%s: tol %g, pivot gap at 1e-11: %.3g above, %.3g below; worst error / bound P+ %.3e values %.3e"
          % (tag, tol, gap_hi, gap_lo, qP, qv))
    _note("P+", qP)
    _note("values", qv)
    ctx.close()


# ---- nothing accepted, ArUco, capacity -----------------------------------------------------------------------------------------------
def _asymmetric(P, seed):
    d = np.sqrt(np.diag(P))
    A = np.random.default_rng(seed).uniform(-1.0, 1.0, P.shape)
    return P + 1e-9 * np.outer(d, d) * (A - A.T)


@pytest.mark.parametrize("prior", ["correlated", "asymmetric"])
@pytest.mark.parametrize("ncal", [0, 14])
def test_nothing_accepted_leaves_the_state_bit_identical(prior, ncal):
    """a table of zeros rejects every landmark (chi2 > 0): the reference stacks nothing and returns before EKFUpdate"""
    cs = make_case(ncal, "correlated", ("batch", True))
    ctx, chg, b, attached = new_ctx(cs)
    if prior == "asymmetric":
        ctx.cov_upload(_asymmetric(cs.P, 3 + ncal))
    ctx.set_chi2_table(np.zeros(len(synth.chi2_table())))
    kinds = kinds_of(ctx, cs, chg, b)
    fids = list(cs.S.featid)
    s0 = snapshot(ctx, kinds, fids)
    on = [on_plane(ctx, b, f, True) for f in range(b["F"])]
    res = ctx.slam_update(b, 1.0, 1.0, True)
    assert np.all(res["feat_status"] == 0), res["feat_status"]
    s1 = snapshot(ctx, kinds, fids)
    for a, c in ((s0[0], s1[0]),):
        assert np.array_equal(a.view(np.uint64), c.view(np.uint64)), "P changed: %s" % state_diff(s0, s1)
    for h in kinds:
        assert np.array_equal(s0[1][h].view(np.uint64), s1[1][h].view(np.uint64)), "value of handle %d changed: %s" % (h, state_diff(s0, s1))
        assert np.array_equal(s0[2][h].view(np.uint64), s1[2][h].view(np.uint64)), "FEJ of handle %d changed" % h
    for f in range(b["F"]):
        if on[f]:
            assert ctx.slam_plane_of(int(b["featid"][f])) == 0, f
    ctx.close()


def test_rejected_aruco_landmark_is_not_flagged():
    """UpdaterSLAM.cpp:600-605, 613-618: a rejected landmark is flagged for marginalisation unless its featid is below
    max_aruco_features"""
    cs = make_case(0, "correlated", ("batch", True))
    ctx, chg, b, attached = new_ctx(cs)
    ctx.set_chi2_table(np.zeros(len(synth.chi2_table())))
    assert ARUCO_FEATID in [int(x) for x in b["featid"]]
    res = ctx.slam_update(b, 1.0, 1.0, True)
    assert np.all(res["feat_status"] == 0), res["feat_status"]
    lim = cs.S.options["max_aruco_features"]
    got = {int(f): ctx.slam_should_marg(int(f)) for f in b["featid"]}
    want = {f: 0 if f < lim else 1 for f in got}
    assert got == want, "should_marg %s, expected %s" % ({f: v for f, v in got.items() if v != want[f]}, {f: want[f] for f in got if got[f] != want[f]})
    ctx.close()


def _run_update(cs, b_of, max_meas_rows=60000, max_state=None):
    """a fresh context of the case, ovp_slam_update on b_of(b); returns (statuses, snapshot after)"""
    ctx, chg, b, _ = new_ctx(cs, max_meas_rows=max_meas_rows)
    kinds = kinds_of(ctx, cs, chg, b)
    res = ctx.slam_update(b_of(b), 1.0, 1.0, True)
    out = snapshot(ctx, kinds, list(cs.S.featid))
    ctx.close()
    return res["feat_status"].copy(), out


def _refused_then_next(cs, limit_words, **ctx_kw):
    """the whole batch refused with OVP_ERR_CAPACITY and the state and bookkeeping bit-identical; the next call (the batch less its first
    landmark, and at most 24) then gives the bits a fresh context gives.  Returns the refusal's message."""
    ctx, chg, b, _ = new_ctx(cs, **ctx_kw)
    kinds = kinds_of(ctx, cs, chg, b)
    s0 = snapshot(ctx, kinds, list(cs.S.featid))
    with pytest.raises(api.OvpError) as e:
        ctx.slam_update(b, 1.0, 1.0, True)
    assert e.value.status == 7, e.value  # OVP_ERR_CAPACITY
    assert any(w in str(e.value) for w in limit_words), str(e.value)
    s1 = snapshot(ctx, kinds, list(cs.S.featid))
    assert same_state(s0, s1), "a refused SLAM update changed the state: %s" % state_diff(s0, s1)
    rest = lambda bb: _cut(bb, list(range(1, min(bb["F"], 25))))
    res = ctx.slam_update(rest(b), 1.0, 1.0, True)
    after = snapshot(ctx, kinds, list(cs.S.featid))
    ctx.close()
    want_st, want = _run_update(cs, rest)
    assert np.array_equal(res["feat_status"], want_st) and same_state(want, after), "the call after the refusal: %s" % state_diff(want, after)
    return str(e.value)


def test_row_capacity_is_refused_one_row_beyond_and_leaves_the_state():
    """stacked rows at the context's row capacity: the same bits as with ample capacity; one row beyond it: refused"""
    cs = make_case(8, "correlated", ("batch", True))
    ctx, chg, b, attached = new_ctx(cs)
    rows = debug_gram(ctx, b, True)["rows"]
    ctx.close()
    st_cap, at_cap = _run_update(cs, lambda bb: bb, max_meas_rows=rows)
    st_big, big = _run_update(cs, lambda bb: bb)
    assert np.array_equal(st_cap, st_big) and np.count_nonzero(st_cap) > 0
    assert same_state(big, at_cap), "the update at the row capacity differs from one with room to spare: %s" % state_diff(big, at_cap)
    msg = _refused_then_next(cs, ["max_meas_rows"], max_meas_rows=rows - 1)
    print("row capacity %d: refused at %d: %s" % (rows, rows - 1, msg))


def test_batch_wider_than_the_co_resident_factorisation_is_refused():
    """A batch whose nc1 needs more co-resident factorisation CTAs than the device holds (T (T + 1) / 2 tiles of 64 columns, one per SM,
    as tests/test_gpu_cholfused.py derives it) is refused with OVP_ERR_CAPACITY before anything is launched; the context's column
    capacity (Rcap) may bind first, and the test names the limit the call reached."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    T = 1
    while (T + 1) * (T + 2) // 2 <= sms:
        T += 1
    width = 64 * T  # the widest nc1 the device factors in one launch
    cs = Case()
    cs.S = gr.slam_scenario(0, seed=0, F=(width + 64) // 3)
    cs.ncal, cs.cov, cs.shape, cs.seed, cs.use_plane = 0, "correlated", ("short",), 0, True
    ctx, chg, b, attached = new_ctx(cs)
    nc1 = 3 * b["F"] + 6 * len(set(b["meas_clone"].tolist())) + 3 * len({int(p) for p in b["planeid"] if p}) + 1
    ctx.close()
    assert nc1 > width, (nc1, width)
    msg = _refused_then_next(cs, ["co-resident", "columns, capacity"])
    print("nc1 %d against a co-resident width of %d columns (%d SMs): refused: %s" % (nc1, width, sms, msg))


# ---- marginalize_slam ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prior", ["symmetric", "asymmetric"])
def test_marginalize_slam_bit_exact(prior):
    """landmarks flagged first, in the middle and last of the landmark block (and enough more that N - 3k crosses a multiple of 64), one
    at featid 4 max_aruco_features (kept) and one at 4 max_aruco_features + 1 (marginalised)"""
    cs = make_case(14, "correlated", ("batch", True))
    lim = 4 * cs.S.options["max_aruco_features"]
    cs.S.featid[2] = lim
    ctx, chg, b, attached = new_ctx(cs)
    lm_fids = sorted((ctx.var_id(ctx.slam_handle(int(f))), int(f)) for f in cs.S.featid if ctx.slam_handle(int(f)) >= 0)
    N = ctx.cov_rows()
    order = [f for _, f in lm_fids]
    want = {order[0], order[len(order) // 2], order[-1], lim, lim + 1 if lim + 1 in order else order[1]}
    k_need = (N % 64) // 3 + 1
    for f in order:
        if len([x for x in want if x > lim]) >= k_need:
            break
        want.add(f)
    want.discard(ARUCO_FEATID)
    sel = [i for i in range(b["F"]) if int(b["featid"][i]) in want]
    ctx.set_chi2_table(np.zeros(len(synth.chi2_table())))
    ctx.slam_update(_cut(b, sel), 1.0, 1.0, True)  # rejected: flagged
    flagged = {f for f in order if ctx.slam_should_marg(f) == 1}
    assert lim in flagged and len(flagged) == len(sel), (flagged, want)
    P = cs.P if prior == "symmetric" else _asymmetric(cs.P, 11)
    ctx.cov_upload(P)
    P = ctx.cov().copy()
    lms = {f: (ctx.var_id(ctx.slam_handle(f)), f in flagged) for f in order}
    ref, removed = sr.marginalize_slam(P, lms, cs.S.options["max_aruco_features"])
    assert lim not in removed and order[0] in removed and order[-1] in removed
    assert (N // 64) != ((N - 3 * len(removed)) // 64) or (N - 3 * len(removed)) % 64 == 0, (N, len(removed))
    ctx.marginalize_slam()
    got = ctx.cov()
    assert got.shape == ref.shape
    bad = got.view(np.uint64) != ref.view(np.uint64)
    assert not bad.any(), "marginalize_slam: %d entries differ from the reference, first %s" % (int(bad.sum()), np.argwhere(bad)[0])
    for f in order:
        assert (ctx.slam_handle(f) < 0) == (f in removed), f
    print("marginalize_slam %s: N %d -> %d, removed %d landmarks (featid %d kept)" % (prior, N, got.shape[0], len(removed), lim))
    ctx.close()
