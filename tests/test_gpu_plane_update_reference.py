"""The per-plane stacked system of the MSCKF update (the code after the feature kernel in msckf_launch_body) and ovp_plane_init, against
the long-double references of tests/plane_update_reference.py, on both sides of the compression boundary.

Each case is one plane's features cut to chosen track lengths, so that rows = sum(3 m - 3) sits at a chosen distance from ncx (the
plan's x columns): -3, -2, 0, +1, +3 and well above, for a plane in the state (direct form when rows <= ncx, compressed above) and a
plane that is not (Gram factor over ncx + 3 columns when rows <= ncx, over ncx above).  Two more put the plane system's nc1 = ncx + 4 on
either side of the 64-column tile edge: 64, and 66 (ncx = 6 clones + ncal with ncal in {0, 6, 8, 14} is 0 or 2 mod 6, so nc1 = 65 does
not exist).  Every case runs on gate_reference.correlated_cov and on its kappa = 1e10 variant: synth's P0 has no plane x clone
covariance and isotropic plane blocks, on which a transposed or misplaced plane column changes nothing.

Per case: the library's G (or, for the direct form, its raw rows) from ovp_debug_msckf_gram, bit-identical from run to run, the state
untouched by the call; the update on a fresh context against the reference built on them (P+ element-wise and exactly symmetric, every
value, FEJs bit-identical, the plane chi2 within its bound and within the bound of the well-defined part of the reference's own chi2
from the raw rows, with what a factor over every Jacobian column drops equal to the residual on the rows without Jacobian); the same bits with
graphs off and through prepared replays; which chi2 table entry the gate reads; the decision five bounds on either side of the reference
chi2, a rejected plane leaving the state bit-identical.  The zero pivots are decided by the same rule in the library and the reference,
at the smallest tolerance of 1e-11 (the default) ... 1e-6 that leaves every pivot of the case at least 100 times from its threshold:
the unobservable directions of these systems come out of G at 1e-13 .. 3e-10 of their diagonal, within 100 times of the default, so
there the decision is rounding's.  A plane's features that its gate rejects fall through to the point update (UpdaterMSCKF.cpp:640-659);
the tables here are zero at every point dof 2m - 3, so that update rejects them all and the state is the plane's alone.  Not in the
state, the same batch through ovp_plane_init against update_reference.initialize on the reference's W: the table entry its gate reads,
and its decision on either side, with const_init_chi2 = 2.5.  Last, three planes in one batch with the middle one rejected, against
the chained reference (the third plane linearised at the first plane's posterior)."""
import ctypes as C

import numpy as np
import pytest

import gate_reference as gr
import plane_update_reference as pr
import update_reference as ur
from ov_plane_b200 import api, synth
from test_gpu_compression import _p

pytestmark = pytest.mark.gpu

RAW_ROW = 24
COVS = ("correlated", "kappa 1e10")
BIG = 1e300
CONST_INIT_CHI2 = 2.5
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for k, v in sorted(WORST.items()):
        print("plane update reference: worst %-26s %.3e" % (k, v))


def _note(k, v):
    WORST[k] = max(WORST.get(k, 0.0), v)


# ---- cases ---------------------------------------------------------------------------------------------------------------------------
# (in the state, rows - ncx or "above", ncal, nc1 wanted or None)
CASES = ([(True, d, n, None) for d, n in ((-3, 0), (-2, 8), (0, 6), (1, 14), (3, 0), ("above", 14))] +
         [(False, d, n, None) for d, n in ((-3, 0), (-2, 8), (0, 6), (1, 14), (3, 0), ("above", 14))] +
         [(True, 3, 0, 64), (False, -2, 8, 66)])


def _scenario(ncal, seed):
    cal = {0: (0, 0), 6: (1, 0), 8: (0, 1), 14: (1, 1)}[ncal]
    return synth.make_scenario("tiny_planes", seed=seed, n_clones=14, F=40, m_min=3, m_max=9, n_planes=1, plane_frac=1.0, n_slam=0,
                               calib_pose=cal[0], calib_intr=cal[1], dtheta=0.03)


def _pick(S, ncal, delta, nc1, in_state, seed):
    """(features, lengths): each feature cut to its newest `length` measurements, rows - ncx = delta (nc1 = ncx + 4 when given)."""
    m = np.diff(S.meas_offset)
    if delta == "above":
        return np.arange(S.F), m.copy()
    rng = np.random.default_rng(seed)
    kmin = 3 if in_state else 4  # a plane not in the state needs at least 4 features (features_host.inc, msckf_prepare)
    for _ in range(200000):
        k = int(rng.integers(kmin, 9))
        sel = np.sort(rng.choice(S.F, size=k, replace=False))
        ln = np.array([int(rng.integers(2, m[f] + 1)) for f in sel])
        U = set()
        for f, n in zip(sel, ln):
            e = S.meas_offset[f + 1]
            U.update(S.meas_clone_idx[e - n:e].tolist())
        ncx = ncal + 6 * len(U)
        rows = int(np.sum(3 * ln - 3))
        if rows - ncx == delta and (nc1 is None or ncx + 4 == nc1):
            return sel, ln
    raise AssertionError("no track cut reaches rows - ncx = %s" % delta)


def _cut(b, sel, ln):
    offs, mc, uv = [0], [], []
    for f, n in zip(sel, ln):
        e = int(b["meas_offset"][f + 1])
        mc.append(b["meas_clone"][e - n:e])
        uv.append(b["uv"][e - n:e])
        offs.append(offs[-1] + int(n))
    out = dict(b)
    for k in ("p_FinG", "p_FinG_original", "featid", "planeid"):
        out[k] = np.ascontiguousarray(b[k][sel])
    out.update(F=len(sel), meas_offset=np.array(offs, dtype=np.int32), meas_clone=np.ascontiguousarray(np.concatenate(mc), dtype=np.int32),
               uv=np.ascontiguousarray(np.concatenate(uv), dtype=np.float32))
    return out


class Case(object):
    pass


def make_case(in_state, delta, ncal, nc1, cov, attempt=0):
    seed = 17 + ncal + (0 if in_state else 100) + (nc1 or 0) + 1000 * attempt
    S = _scenario(ncal, seed)
    sel, ln = _pick(S, ncal, delta, nc1, in_state, seed)
    cs = Case()
    cs.planes = None if in_state else synth.drop_planes_from_state(S)
    cs.S, cs.sel, cs.ln, cs.in_state, cs.delta = S, sel, ln, in_state, delta
    cs.P = gr.correlated_cov(S, S.N, 500 + seed, cond=None if cov == "correlated" else 1e10)
    cs.point_dofs = sorted({int(2 * n - 3) for n in ln})
    cs.rows = int(np.sum(3 * ln - 3))
    cs.tol = pr.GRAM_TOL
    S.options["const_init_chi2"] = CONST_INIT_CHI2  # ovp_plane_init's gate multiplier; not 1, so that a missing multiplier shows
    return cs


def new_ctx(cs, table):
    S = cs.S
    ctx = api.Context(S.options, device=0, max_state=S.N + 64, max_meas_rows=8192, debug=True)
    ctx.set_chi2_table(table)
    chg = synth.load_scenario_into(ctx, S)
    ctx.cov_upload(cs.P)
    b = _cut(synth.feature_batch(S, chg), cs.sel, cs.ln)
    if cs.planes is not None:
        b["plane_ids"] = np.array([p[0] for p in cs.planes], dtype=np.int64)
        b["plane_cp"] = np.ascontiguousarray([p[1] for p in cs.planes], dtype=np.float64)
    return ctx, chg, b


def handles_of(ctx, cs, chg):
    """{handle: kind} of every variable with covariance rows"""
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
    for pid, _, _ in S.planes:
        kinds[ctx.plane_handle(pid)] = ur.VEC
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


def state_diff(a, b):
    """what differs between two snapshots, for a failure message"""
    out = []
    d = np.abs(a[0] - b[0])
    if d.max() > 0 or not np.array_equal(a[0].view(np.uint64), b[0].view(np.uint64)):
        i, j = np.unravel_index(np.argmax(d), d.shape)
        out.append("P: %d entries, largest %.3e at [%d, %d]" % (int((a[0].view(np.uint64) != b[0].view(np.uint64)).sum()), d[i, j], i, j))
    for h in a[1]:
        if not np.array_equal(a[1][h].view(np.uint64), b[1][h].view(np.uint64)):
            out.append("value of handle %d: %s" % (h, (a[1][h] - b[1][h]).tolist()))
        if not np.array_equal(a[2][h].view(np.uint64), b[2][h].view(np.uint64)):
            out.append("FEJ of handle %d" % h)
    return "; ".join(out)


def pick_tolerance(G, npiv):
    """the smallest zero-pivot tolerance of 1e-11 (the default) ... 1e-6 with every pivot of G at least PIVOT_MARGIN times from its
    threshold, on one side or the other; the decisions of a pivot closer than that are left to rounding"""
    for tol in (1e-11, 1e-10, 1e-9, 1e-8, 1e-7, 1e-6):
        _, _, ratio = pr.ld_factor(G, npiv, tol)
        if np.all((ratio >= pr.PIVOT_MARGIN) | (ratio <= 1.0 / pr.PIVOT_MARGIN)):
            return tol, ratio
    return None


def restore(ctx, P, snap):
    for h in snap[1]:
        ctx.var_set(h, snap[1][h], snap[2][h])
    ctx.cov_upload(P)


def debug_gram(ctx, b):
    fb, keep = api.Context._batch_struct(b)
    uo = api.UpdaterOptions(1.0, 1.0)
    F, M = fb.F, int(b["meas_offset"][-1])
    gcap = ctx.cov_rows() + 4
    G = np.zeros(gcap * gcap)
    info = np.zeros(8, dtype=np.int32)
    cols = np.zeros(gcap, dtype=np.int32)
    sel = np.zeros(F, dtype=np.int32)
    fs, fc = np.zeros(F, dtype=np.int32), np.zeros(F)
    raw = np.zeros(3 * RAW_ROW * M)
    ctx._ck(ctx.lib.ovp_debug_msckf_gram(ctx.h, C.byref(fb), C.byref(uo), gcap, _p(G), _p(info), _p(cols), _p(sel), _p(fs), _p(fc), _p(raw)))
    nc1, ncal, ncx, is_point, nsel = (int(v) for v in info[:5])
    assert not is_point, "the first plan of a plane batch is its plane"
    return dict(G=G[:nc1 * nc1].reshape((nc1, nc1), order="F").copy() if nc1 else None, direct=nc1 == 0, ncal=ncal, ncx=ncx,
                cols=cols[:ncx].copy(), sel=sel[:nsel].copy(), raw=raw.reshape(M, 3, RAW_ROW), in_state=bool(info[7]))


def table_for(cs, plane_value, n):
    """zero at every point dof (the point update rejects every feature), plane_value elsewhere"""
    t = np.full(n, float(plane_value)) if np.isscalar(plane_value) else np.array(plane_value, dtype=np.float64)[:n].copy()
    t[cs.point_dofs] = 0.0
    return t


# ---- the test ------------------------------------------------------------------------------------------------------------------------
def _ids(case):
    ins, d, n, nc1 = case
    return "%s-%s-ncal%d%s" % ("in_state" if ins else "not_in_state", d if d == "above" else "%+d" % d, n, "-nc1_%d" % nc1 if nc1 else "")


@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
@pytest.mark.parametrize("cov", COVS, ids=["correlated", "kappa1e10"])
def test_plane_update_against_long_double(case, cov, chi2_table):
    ur.require_long_double()
    in_state, delta, ncal, nc1 = case
    # a cut whose G leaves every pivot 100x clear of one tolerance in 1e-11 ... 1e-6 (a cut whose weakest real direction lies within
    # 1e4 of the rounding-level pivots of its unobservable ones has no such tolerance, and its decisions are left to rounding: the next
    # cut is taken)
    for attempt in range(6):
        cs = make_case(in_state, delta, ncal, nc1, cov, attempt)
        ntab = len(chi2_table)
        T_open = table_for(cs, BIG, ntab)
        ctx, chg, b = new_ctx(cs, T_open)
        kinds = handles_of(ctx, cs, chg)
        snap0 = snapshot(ctx, kinds)
        g = debug_gram(ctx, b)
        form, npiv, dof, rows_ref = pr.form_of(in_state, cs.rows, g["ncx"])
        if g["direct"] or form == "direct" or pick_tolerance(g["G"], npiv) is not None:  # a form mismatch is reported below
            break
        ctx.close()
    else:
        raise AssertionError("no cut of six has a G whose pivots all lie 100x from one tolerance")
    S = cs.S
    ncx = g["ncx"]
    assert g["ncal"] == ncal and g["in_state"] == in_state
    if delta != "above":
        assert cs.rows - ncx == delta, (cs.rows, ncx)
    else:
        assert cs.rows > ncx + 3
    if nc1 is not None:
        assert ncx + 4 == nc1
    assert g["direct"] == (form == "direct"), "the plan's form is not the one rows %d against ncx %d selects" % (cs.rows, ncx)
    assert dof not in cs.point_dofs
    again = debug_gram(ctx, b)
    if g["direct"]:
        assert np.array_equal(g["raw"].view(np.uint64), again["raw"].view(np.uint64)), "raw rows differ run to run"
    else:
        assert np.array_equal(g["G"].view(np.uint64), again["G"].view(np.uint64)), "G differs run to run"
    now = snapshot(ctx, kinds)
    assert same_state(snap0, now), "ovp_debug_msckf_gram changed the state: %s" % state_diff(snap0, now)
    P = snap0[0]
    col_of = {int(s): c for c, s in enumerate(g["cols"])}
    x_ids = [int(s) for s in g["cols"]]
    plane_ids = list(range(ctx.var_id(ctx.plane_handle(S.planes[0][0])), ctx.var_id(ctx.plane_handle(S.planes[0][0])) + 3)) if in_state else None
    X, Xb, _ = pr.stacked_rows(g["raw"], b, g["sel"], ncal, ncx, col_of, ctx.var_id)
    assert X.shape[0] == cs.rows
    if form == "direct":
        rf = pr.plane_reference(P, x_ids, plane_ids, ncx, form, X=X, Xb=Xb)
    else:
        tol, _ = pick_tolerance(g["G"], npiv)
        ctx.set_rank_tolerance(tol)
        rf = pr.plane_reference(P, x_ids, plane_ids, ncx, form, G=g["G"], npiv=npiv, tol=tol)
        cs.tol = tol
    # the update on a fresh context, with an open plane gate
    ctx.close()
    ctx, chg, b = new_ctx(cs, T_open)
    ctx.set_rank_tolerance(cs.tol)
    assert same_state(snap0, snapshot(ctx, kinds))
    res = ctx.msckf_update(b, 1.0, 1.0)
    assert res["plane_status"][0] == 1, "the plane gate rejected with an open table"
    assert np.all(res["feat_status"] == 2), "every feature is consumed by the plane update: %s" % res["feat_status"]
    got = snapshot(ctx, kinds)
    ids = {h: ctx.var_id(h) for h in kinds}
    qP, qv = ur.check_update(got[0], got[1], got[2], P, kinds, ids, snap0[1], snap0[2], rf["dx"], rf["dxb"], rf["dPb"], rf["ref"]["P"])
    chi = float(res["plane_chi2"][0])
    echi = abs(chi - float(rf["chi2"]))
    assert echi <= rf["chi2b"], "plane chi2 %.17g, reference %.17g: error %.3e above the bound %.3e" % (chi, float(rf["chi2"]), echi, rf["chi2b"])
    tag = "%s %s rows %d ncx %d form %s npiv %s dof %d tol %g" % (_ids(case), cov, cs.rows, ncx, form, npiv, dof, cs.tol)
    # the reference's own chi2 from the raw rows (no compression when rows <= ncx, the top ncx rows of a QR when rows > ncx)
    own, own_rows = pr.reference_chi2(X, ncx, P, x_ids, plane_ids)
    if form == "direct":  # the same rows, nothing dropped
        eown = abs(chi - float(own))
        assert eown <= rf["chi2b"], "%s: chi2 %.17g, the reference's own %.17g" % (tag, chi, float(own))
        note = "the reference's own chi2 %.6g, error / bound %.3e" % (float(own), eown / rf["chi2b"])
    else:
        # its well-defined part: the rows whose Jacobian lies outside the numerical null space of [H_x (H_cp)], rank by the same rule
        wd, dropped, zero_raw, ratio_raw, rest = pr.reference_chi2_well_defined(X, ncx, npiv, P, x_ids, plane_ids, cs.tol)
        assert zero_raw == rf["zero"], "%s: the raw rows' QR skips %s, the factor of G %s" % (tag, zero_raw, rf["zero"])
        assert np.all((ratio_raw >= pr.PIVOT_MARGIN) | (ratio_raw <= 1.0 / pr.PIVOT_MARGIN)), tag
        bwd = rf["chi2b"] + pr.raw_chi2_bound(rf, g["G"], X, Xb, cs.tol)
        ewd = abs(chi - float(wd))
        assert ewd <= bwd, "%s: chi2 %.17g, the well-defined part of the reference's own %.17g: error %.3e above %.3e" % (tag, chi, float(wd),
                                                                                                                       ewd, bwd)
        note = "the reference's own chi2 %.6g (%d rows), its well-defined part %.6g (error / bound %.3e)" % (float(own), own_rows, float(wd),
                                                                                                          ewd / bwd)
        if not in_state and cs.rows <= ncx:
            # every Jacobian column pivoted: what the factor drops is the residual on the rows without Jacobian, and nothing else;
            # the reference keeps those rows (S = I there), so its chi2 is the library's plus that share
            brest = pr.info_effects(rf["A"], rf["xhat"], pr.rest_dK(rest))[2]
            edrop = abs(float(own) - float(wd) - float(dropped))
            brest += 64 * cs.rows * float(np.finfo(ur.LD).eps) * float(own)  # the long-double rounding of the two chi2
            assert edrop <= brest, "%s: the reference's chi2 %.17g is not its well-defined part %.17g plus the dropped %.17g (%.3e above %.3e)" % (
                tag, float(own), float(wd), float(dropped), edrop, brest)
            assert abs(float(own) - chi - float(dropped)) <= bwd + brest, tag
            note += "; the factor over ncx + 3 columns drops %.6g of the residual (%.2f%% of the reference's chi2), the share on the rows " \
                    "without Jacobian" % (float(dropped), 100.0 * float(dropped) / float(own))
    print("%s: worst error / bound P+ %.3e values %.3e chi2 %.3e (chi2 %.6g); %s; zero pivots %s"
          % (tag, qP, qv, echi / rf["chi2b"], chi, note, rf["zero"]))
    _note("P+ " + form, qP)
    _note("values " + form, qv)
    _note("chi2 " + form, echi / rf["chi2b"])
    # graphs off, and the prepared plan replayed (second launch captures the graph, third replays it): the same bits
    for _ in range(2):
        restore(ctx, P, snap0)
        ctx.msckf_update(b, 1.0, 1.0)
        assert same_state(got, snapshot(ctx, kinds)), "a prepared replay gives other bits"
    ctx.set_use_graphs(False)
    restore(ctx, P, snap0)
    ctx.msckf_update(b, 1.0, 1.0)
    assert same_state(got, snapshot(ctx, kinds)), "the update without graphs gives other bits"
    ctx.set_use_graphs(True)
    # which table entry the gate reads: accepted exactly when the one non-zero entry is the form's dof
    for i in sorted({cs.rows, ncx, cs.rows - 3, ncx - 3, rows_ref, rows_ref - 3, cs.rows + 3} - set(cs.point_dofs)):
        if not 0 <= i < ntab:
            continue
        t = np.zeros(ntab)
        t[i] = BIG
        ctx.set_chi2_table(t)
        restore(ctx, P, snap0)
        q = ctx.msckf_update(b, 1.0, 1.0)
        assert (q["plane_status"][0] == 1) == (i == dof), "%s: table non-zero at %d, plane status %d (dof %d)" % (tag, i, q["plane_status"][0], dof)
    # the decision a few bounds on either side of the reference chi2; a rejected plane leaves the state as it was
    tab = table_for(cs, chi2_table, ntab)
    ctx.set_chi2_table(tab)
    assert float(rf["chi2"]) > 5.0 * rf["chi2b"], "%s: the bound %.3e is too wide to place a threshold below chi2 %.6g" % (tag, rf["chi2b"],
                                                                                                                       float(rf["chi2"]))
    for s, want in ((5.0, 1), (-5.0, 0)):
        mult = (float(rf["chi2"]) + s * rf["chi2b"]) / tab[dof]
        restore(ctx, P, snap0)
        q = ctx.msckf_update(b, 1.0, mult)
        assert q["plane_status"][0] == want, "%s: status %d with the threshold %+g bounds from the reference chi2" % (tag, q["plane_status"][0], s)
        if want:
            assert same_state(got, snapshot(ctx, kinds)), "an accepted plane at a finite threshold gives other bits"
        else:
            now = snapshot(ctx, kinds)
            assert same_state(snap0, now), "a rejected plane changed the state: %s (statuses %s)" % (state_diff(snap0, now), q["feat_status"])
    ctx.close()
    if not in_state:
        _check_plane_init(cs, P, g, rf, x_ids, ncx, npiv, rows_ref, chi2_table, tag)


def _check_plane_init(cs, P, g, rf, x_ids, ncx, npiv, rows_ref, chi2_table, tag):
    """ovp_plane_init on the same batch: update_reference.initialize on H_L = W's cp columns, H_R = its x columns, r = z, with W from
    the long-double factor of the library's G; the gate reads table[rows_ref] (a table non-zero at one entry), times const_init_chi2
    (2.5 here), five bounds on either side."""
    W = np.asarray(rf["sys"]["W"])
    H_L, H_R, r = W[:, :3], W[:, 3:3 + ncx], W[:, 3 + ncx]
    ref = ur.initialize(P, x_ids, H_R.astype(ur.LD), H_L.astype(ur.LD), r.astype(ur.LD), 1.0)
    N = P.shape[0]
    ntab = len(chi2_table)
    for i in sorted({rows_ref, npiv, rows_ref - 3, cs.rows, ncx, ncx + 3} - set(cs.point_dofs)):
        t = np.zeros(ntab)
        t[i] = BIG
        ctx, chg, b = new_ctx(cs, t)
        ctx.set_rank_tolerance(cs.tol)
        out = ctx.plane_init(b)
        assert (out["plane_status"][0] == 1) == (i == rows_ref), "%s: plane_init with the table non-zero at %d: status %d (rows_ref %d)" % (
            tag, i, out["plane_status"][0], rows_ref)
        ctx.close()
    assert float(ref["chi2"]) > 5.0 * rf["chi2b"], tag
    for s, want in ((5.0, 1), (-5.0, 0)):
        # the gate's chi2 is the projected system's, the one the update above gated (its bound carries over); threshold
        # const_init_chi2 * table[rows_ref]
        t = table_for(cs, chi2_table, ntab)
        t[rows_ref] = (float(ref["chi2"]) + s * rf["chi2b"]) / CONST_INIT_CHI2
        ctx, chg, b = new_ctx(cs, t)
        ctx.set_rank_tolerance(cs.tol)
        kinds = handles_of(ctx, cs, chg)
        snap0 = snapshot(ctx, kinds)
        out = ctx.plane_init(b)
        assert out["plane_status"][0] == want, "%s: plane_init status %d, threshold %+g bounds from the reference chi2 %.6g" % (
            tag, out["plane_status"][0], s, float(ref["chi2"]))
        if not want:
            now = snapshot(ctx, kinds)
            assert same_state(snap0, now) and ctx.cov_rows() == N, "a rejected plane initialisation changed the state: %s" % state_diff(snap0, now)
            ctx.close()
            continue
        nh = int(out["new_handles"][0])
        assert ctx.var_id(nh) == N and ctx.cov_rows() == N + 3
        got = snapshot(ctx, kinds)
        vals_got, fejs_got = dict(got[1]), dict(got[2])
        vals_got[nh], fejs_got[nh] = ctx.var_get(nh)
        cp = np.asarray(b["plane_cp"][0])
        kinds2, ids2 = {**kinds, nh: ur.VEC}, {**{h: ctx.var_id(h) for h in kinds}, nh: N}
        vals2 = {**snap0[1], nh: cp.astype(ur.LD) + ref["dxn"]}
        fejs2 = {**snap0[2], nh: cp}
        sv = np.linalg.svd(np.asarray(H_L, dtype=np.float64), compute_uv=False)
        kR = sv[0] / sv[-1]
        rows = W.shape[0]
        e_init = ur.BOUND_C * (rows + ncx + 2) * ur.EPS * kR * kR
        e_dxn = ur.BOUND_C * (rows + 2) * ur.EPS * kR * float(np.linalg.norm(np.asarray(r, dtype=np.float64))) / sv[-1]
        if ref["upd"] is None:
            P_ref, dx = ref["P_init"], np.zeros(N + 3, dtype=ur.LD)
            dxb, dPb = np.zeros(N + 3), np.zeros((N + 3, N + 3))
        else:
            P_ref, dx = ref["upd"]["P"], ref["upd"]["dx"]
            dxb, dPb, _ = ur.kalman_bounds(ref["P_init"], x_ids, ref["H2"], ref["upd"])
        dPb[N:, :] += e_init
        dPb[:, N:] += e_init
        dxb[N:] += e_dxn
        # the factor's error: the grown posterior is the joint (state, cp) posterior, A its columns of the system's unknowns
        Pg = np.asarray(P_ref, dtype=np.float64)
        A = Pg[:, list(x_ids) + [N, N + 1, N + 2]]
        xhat = np.concatenate([np.asarray(dx, dtype=np.float64)[x_ids], np.asarray(ref["dxn"] + dx[N:], dtype=np.float64)])
        dPi, ddx, _ = pr.info_effects(A, xhat, rf["dK"])
        sd = np.sqrt(np.diag(np.asarray(ref["P_init"], dtype=np.float64)))
        dPb = dPb + dPi / np.outer(sd, sd)
        dxb = dxb + ddx
        qP, qv = ur.check_update(got[0], vals_got, fejs_got, ref["P_init"], kinds2, ids2, vals2, fejs2, dx, dxb, dPb, P_ref)
        print("%s plane_init: rows_ref %d, chi2 %.6g, worst error / bound P+ %.3e values %.3e" % (tag, rows_ref, float(ref["chi2"]), qP, qv))
        _note("plane_init P+", qP)
        _note("plane_init values", qv)
        ctx.close()


# ---- three planes in one batch, the middle one rejected -------------------------------------------------------------------------------
CHAIN_MULT = 4.0  # chi2 multiplier of the chain: planes 1 and 3 pass it by far, plane 2 (an outlier in every feature) fails it by far


def _chain_case(in_state, cov, seed):
    S = synth.make_scenario("tiny_planes", seed=seed, n_clones=14, F=45, m_min=4, m_max=9, n_planes=3, plane_frac=1.0, n_slam=0,
                            calib_pose=1, calib_intr=1, dtheta=0.03)
    for f in np.nonzero(S.planeid == 2)[0]:  # 30 px on one measurement of every feature of plane 2
        k = (S.meas_offset[f] + S.meas_offset[f + 1]) // 2
        S.uv[k] += np.float32(30.0) * np.array([1.0, -1.0], dtype=np.float32)
    cs = Case()
    cs.planes = None if in_state else synth.drop_planes_from_state(S)
    cs.S, cs.in_state = S, in_state
    cs.sel, cs.ln = np.arange(S.F), np.diff(S.meas_offset)
    cs.P = gr.correlated_cov(S, S.N, 900 + seed, cond=None if cov == "correlated" else 1e10)
    cs.point_dofs = sorted({int(2 * n - 3) for n in cs.ln})
    cs.rows = None
    cs.tol = pr.GRAM_TOL
    return cs


def _planes_only(b, pids):
    """the batch restricted to the features of the planes pids, the plane list in the order 3, 1, 2 (the slots differ from the launch
    order, which is ascending id)"""
    sel = np.nonzero(np.isin(b["planeid"], pids))[0]
    out = _cut(b, sel, np.diff(b["meas_offset"])[sel])
    order = [list(b["plane_ids"]).index(p) for p in (3, 1, 2)]
    out["plane_ids"] = np.ascontiguousarray(b["plane_ids"][order])
    out["plane_cp"] = np.ascontiguousarray(b["plane_cp"][order])
    return out


def _plane_ref(ctx, cs, g, P, pid, in_state, tol):
    ncx = g["ncx"]
    x_ids = [int(s) for s in g["cols"]]
    plane_ids = list(range(ctx.var_id(ctx.plane_handle(pid)), ctx.var_id(ctx.plane_handle(pid)) + 3)) if in_state else None
    form, npiv, dof, _ = pr.form_of(in_state, int(np.sum(3 * np.diff(g["b"]["meas_offset"]) - 3)), ncx)
    assert form != "direct"
    rf = pr.plane_reference(P, x_ids, plane_ids, ncx, form, G=g["G"], npiv=npiv, tol=tol)
    assert np.all((rf["ratio"] >= pr.PIVOT_MARGIN) | (rf["ratio"] <= 1.0 / pr.PIVOT_MARGIN))
    return rf, dof


@pytest.mark.parametrize("in_state", [True, False], ids=["in_state", "not_in_state"])
@pytest.mark.parametrize("cov", COVS, ids=["correlated", "kappa1e10"])
def test_three_planes_middle_rejected_against_the_chained_reference(in_state, cov, chi2_table):
    """Planes 1, 2, 3 in one batch, plane 2 rejected by its gate: plane 1 against the reference at the prior, plane 3 against the
    reference linearised at plane 1's posterior (taken from a plane-1-only update: the rejected plane must leave nothing behind), each
    plane's status and chi2 in its own slot of a plane list that is not in launch order."""
    ur.require_long_double()
    ntab = len(chi2_table)
    for seed in range(5, 11):  # a scenario whose two Gram matrices leave every pivot 100x clear of one tolerance
        cs = _chain_case(in_state, cov, seed)
        table = table_for(cs, chi2_table, ntab)
        ctx, chg, b = new_ctx(cs, table)
        b1, b3 = _planes_only(b, [1]), _planes_only(b, [3])
        g1, g3 = debug_gram(ctx, b1), debug_gram(ctx, b3)
        ctx.close()

        def clean(g, t):  # every plane of the chain keeps more rows than columns: its factor pivots on the ncx x columns
            r = pr.ld_factor(g["G"], g["ncx"], t)[2]
            return np.all((r >= pr.PIVOT_MARGIN) | (r <= 1.0 / pr.PIVOT_MARGIN))

        tols = [t for t in (1e-11, 1e-10, 1e-9, 1e-8, 1e-7, 1e-6) if clean(g1, t) and clean(g3, t)]
        if tols:
            break
    else:
        raise AssertionError("no scenario with a clean pivot tolerance for both planes")
    # the reference chain: plane 1 at the prior, then plane 3's G at plane 1's posterior (its calibration columns move with the state,
    # so its pivots are checked there); the first tolerance clean for both
    for tol in tols:
        ctx, chg, b = new_ctx(cs, table)
        ctx.set_rank_tolerance(tol)
        kinds = handles_of(ctx, cs, chg)
        s0 = snapshot(ctx, kinds)
        b1, b3 = _planes_only(b, [1]), _planes_only(b, [3])
        g1 = debug_gram(ctx, b1)
        g1["b"] = b1
        rf1, dof1 = _plane_ref(ctx, cs, g1, s0[0], 1, in_state, tol)
        r1 = ctx.msckf_update(b1, 1.0, CHAIN_MULT)
        s1 = snapshot(ctx, kinds)
        g3 = debug_gram(ctx, b3)
        g3["b"] = b3
        if clean(g3, tol):
            break
        ctx.close()
    else:
        raise AssertionError("no tolerance leaves plane 3's pivots at plane 1's posterior 100x clear")
    cs.tol = tol
    tag = "three planes %s %s tol %g" % ("in the state" if in_state else "not in the state", cov, cs.tol)
    assert same_state(s1, snapshot(ctx, kinds))
    ids = {h: ctx.var_id(h) for h in kinds}
    q1 = ur.check_update(s1[0], s1[1], s1[2], s0[0], kinds, ids, s0[1], s0[2], rf1["dx"], rf1["dxb"], rf1["dPb"], rf1["ref"]["P"])
    rf3, dof3 = _plane_ref(ctx, cs, g3, s1[0], 3, in_state, cs.tol)
    ctx.close()
    # the chain, on a fresh context
    ctx, chg, b = new_ctx(cs, table)
    ctx.set_rank_tolerance(cs.tol)
    ball = _planes_only(b, [1, 2, 3])
    res = ctx.msckf_update(ball, 1.0, CHAIN_MULT)
    chain = snapshot(ctx, kinds)
    slot = {int(p): i for i, p in enumerate(ball["plane_ids"])}
    assert [int(res["plane_status"][slot[p]]) for p in (1, 2, 3)] == [1, 0, 1], "plane statuses %s for the slots of %s" % (
        res["plane_status"], ball["plane_ids"])
    on2 = ball["planeid"] == 2
    assert np.all(res["feat_status"][on2] == 0) and np.all(res["feat_status"][~on2] == 2), res["feat_status"]
    ctx.close()
    thr1 = CHAIN_MULT * table[dof1]
    for chi in (float(res["plane_chi2"][slot[1]]), float(r1["plane_chi2"][slot[1]])):
        assert abs(chi - float(rf1["chi2"])) <= rf1["chi2b"], (tag, chi, float(rf1["chi2"]), rf1["chi2b"])
    assert float(rf1["chi2"]) + 5 * rf1["chi2b"] < thr1
    # ... plane 2 fails its gate far from the threshold ...
    assert float(res["plane_chi2"][slot[2]]) > 5 * CHAIN_MULT * chi2_table[:cs.S.N].max(), (tag, res["plane_chi2"])
    # ... and the chain's state is plane 3's update linearised at plane 1's posterior
    q3 = ur.check_update(chain[0], chain[1], chain[2], s1[0], kinds, ids, s1[1], s1[2], rf3["dx"], rf3["dxb"], rf3["dPb"], rf3["ref"]["P"])
    chi3 = float(res["plane_chi2"][slot[3]])
    assert abs(chi3 - float(rf3["chi2"])) <= rf3["chi2b"], (tag, chi3, float(rf3["chi2"]), rf3["chi2b"])
    assert float(rf3["chi2"]) + 5 * rf3["chi2b"] < CHAIN_MULT * table[dof3]
    print("%s: plane 1 worst error / bound P+ %.3e values %.3e; plane 2 chi2 %.4g rejected; plane 3 (at plane 1's posterior) P+ %.3e "
          "values %.3e" % (tag, q1[0], q1[1], float(res["plane_chi2"][slot[2]]), q3[0], q3[1]))
    _note("P+ three-plane chain", max(q1[0], q3[0]))
    _note("values three-plane chain", max(q1[1], q3[1]))
