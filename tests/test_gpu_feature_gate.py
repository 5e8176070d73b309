"""The per-feature chi2 gates of the MSCKF point and SLAM feature kernels against the long-double references of tests/gate_reference.py,
on synth's P0 and on two correlated covariances (well conditioned, and kappa(P) = 1e10):

- point gate of the warp-per-feature kernel (msckf_warp.inc) and of the CTA-per-feature kernel (features.cu feature_kernel, mode 0),
  through ovp_debug_msckf_gram: chi2 within the first-order bound of gate_reference.gate_bound, statuses the reference's decision, the
  two kernels within the sum of their bounds with identical statuses, bit-identical from run to run, the covariance untouched;
- SLAM gate (feature_kernel, mode 2) through ovp_debug_slam_update, with the plane row and on the retry without it (status 3);
- the decision at its threshold: accepted when chi2_mult * table[dof] equals chi2 (or is the nearest product above it), rejected one
  product below; and on either side of the reference's chi2 by 100 times the bound;
- which table entry each gate reads (points 2m - 3; SLAM 3m with the plane, 2m on the retry), and the refusal of a table too short
  for the batch.

synth's P0 has diagonal clone blocks and no calibration x clone covariance: on it a transposed clone block or a dropped cross term
changes nothing, so every case also runs on the correlated covariances."""
import ctypes as C

import numpy as np
import pytest

import gate_reference as gr
from ov_plane_b200 import api, synth
from test_gpu_compression import _p, _scenario, add_outliers, debug_pair, run_gram
from test_gpu_parity import relerr

pytestmark = pytest.mark.gpu

COVS = ("P0", "correlated", "kappa 1e10")
WORST = {}  # (kernel, covariance) -> worst error / bound over the module, printed at the end


def _note(kernel, cov, ratio):
    WORST[(kernel, cov)] = max(WORST.get((kernel, cov), 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for (kernel, cov), v in sorted(WORST.items()):
        print("feature gate: %-10s %-11s worst chi2 error / bound %.3e" % (kernel, cov, v))


def _cov(S, N, which, seed):
    return {"P0": None, "correlated": lambda: gr.correlated_cov(S, N, seed), "kappa 1e10": lambda: gr.correlated_cov(S, N, seed, cond=1e10)}[which]


def _upload(be, S, which, seed):
    make = _cov(S, be.cov_rows(), which, seed)
    if make is not None:
        be.cov_upload(make())
    return be.cov()


def _reverse_tracks(b):
    """every track's measurements in reverse clone order"""
    for f in range(b["F"]):
        a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
        b["meas_clone"][a:e] = b["meas_clone"][a:e][::-1].copy()
        b["uv"][a:e] = b["uv"][a:e][::-1].copy()
    return b


def _check_raw(orc, b, f, raw, ids, ncal, cho_of, pf, pff, pid, cp, cpf, sigma_pix, sigma_c):
    """raw rows of feature f against the oracle's feature_jacobian_full, columns matched by state index"""
    a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
    Hf, Hx, r = gr.raw_block(raw, a, e, ncal, pid != 0)
    of, ox, orr, xo = orc.feature_jacobian_full([cho_of[int(h)] for h in b["meas_clone"][a:e]], b["uv"][a:e], pf, pff, pid, cp, cpf, sigma_pix,
                                                sigma_c)
    oid = gr.block_ids(orc, xo)
    assert sorted(oid) == sorted(ids), (oid, ids)
    pos = {s: i for i, s in enumerate(oid)}
    Hxo = np.zeros_like(ox)
    for j, s in enumerate(ids):
        Hxo[:, j] = ox[:, pos[s]]
    for k, (got, ref) in enumerate(((Hf, of), (Hx, Hxo), (r, orr))):
        assert relerr(np.asarray(got, dtype=np.float64), ref) < 1e-11, "raw block of feature %d, part %d: %.3e" % (f, k, relerr(np.asarray(got, dtype=np.float64), ref))


# ---------------------------------------------------------------------------------------------------------------------------------
# MSCKF point gate
# ---------------------------------------------------------------------------------------------------------------------------------
def _point_scenario(kind, L, ncal):
    cal = {0: (0, 0), 6: (1, 0), 8: (0, 1), 14: (1, 1)}[ncal]
    if kind == "len":  # every track L long; enough features that the plan compresses in a context of max_state = N + 8
        nclones = L + 3
        N = 16 + ncal + 6 * nclones
        F = max(24, int(np.ceil((2 * (N + 8) + 64) / (2 * L - 3))))
        S = synth.make_scenario("tiny_points", seed=10 + L, n_clones=nclones, F=F, m_min=L, m_max=L, dtheta=0.2 / nclones,
                                calib_pose=cal[0], calib_intr=cal[1])
        add_outliers(S, [1, F - 2])
        return S
    if kind == "33-39":
        return _scenario(("tracks_33_39", ncal))
    return _scenario(("points", ncal))


def point_gate_refs(ctx, S, b, r, P):
    """{feature: (chi2, bound, dof)} of the plan's features from the kernel's own raw rows"""
    cal = gr.calib_ids(ctx, S.options)
    out = {}
    for f in r["sel"]:
        a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
        Hf, Hx, rr = gr.raw_block(r["raw"], a, e, r["ncal"], False)
        ids = cal + gr.block_ids(ctx, b["meas_clone"][a:e], 6)
        out[int(f)] = gr.point_gate(Hf, Hx, rr, P[np.ix_(ids, ids)])
    return out


def check_gate(tag, status, chi2, refs, table, mult, accept_status=1):
    """chi2 within the bound, the status the reference's decision (where the reference is further than the bound from the threshold);
    returns the worst error / bound"""
    worst = 0.0
    for f, (ref, bound, dof) in refs.items():
        err = abs(float(chi2[f]) - float(ref))
        assert err <= bound, "%s feature %d: chi2 %.17g, reference %.17g, error %.3e above the bound %.3e" % (tag, f, chi2[f], float(ref), err,
                                                                                                           bound)
        worst = max(worst, err / bound)
        thr = mult * table[dof]
        if abs(float(ref) - thr) > bound:
            assert (status[f] == accept_status) == (float(ref) <= thr), "%s feature %d: status %d, reference %.6g, threshold %.6g" % (
                tag, f, status[f], float(ref), thr)
    return worst


POINT_CASES = ([("len", L, n, k) for L, n in ((2, 0), (2, 14), (3, 6), (16, 8), (31, 0), (32, 0), (32, 14)) for k in ("both",)] +
               [("33-39", None, 6, "cta")] + [("mixed", None, n, "both") for n in (0, 6, 8, 14)] +
               [("mixed reversed", None, 14, "both"), ("mixed sigma 0.5", None, 8, "both")])


@pytest.mark.parametrize("kind,L,ncal,kernels", POINT_CASES, ids=["%s%s-ncal%d" % (c[0].replace(" ", "_"), "" if c[1] is None else c[1], c[2])
                                                                 for c in POINT_CASES])
def test_point_gate_against_long_double_reference(kind, L, ncal, kernels, chi2_table):
    gr.require_long_double()
    S = _point_scenario(kind, L, ncal)
    sigma = 0.5 if "sigma" in kind else 1.0
    for ci, which in enumerate(COVS):
        ctx, orc, chg, cho = debug_pair(S, chi2_table, S.N + 8)
        b = synth.feature_batch(S, chg)
        bo = synth.feature_batch(S, cho)
        if "reversed" in kind:
            _reverse_tracks(b)
            _reverse_tracks(bo)
        P = _upload(ctx, S, which, 100 + ncal + ci)
        got = {}
        for dense in ((0, 1) if kernels == "both" else (1,)):
            name = "CTA" if dense else "warp"
            r = run_gram(ctx, b, dense, sigma, 1.0)
            assert r["is_point"] and r["ncal"] == ncal and len(r["sel"]) == S.F
            again = run_gram(ctx, b, dense, sigma, 1.0)
            assert np.array_equal(r["status"], again["status"]) and np.array_equal(r["chi2"].view(np.uint64), again["chi2"].view(np.uint64)), \
                "%s: statuses or chi2 differ from run to run" % name
            assert np.array_equal(P.view(np.uint64), ctx.cov().view(np.uint64)), "%s: the gate changed the covariance" % name
            refs = point_gate_refs(ctx, S, b, r, P)
            tag = "%s %s ncal=%d %s %s" % (kind, L, ncal, which, name)
            w = check_gate(tag, r["status"], r["chi2"], refs, chi2_table, 1.0)
            _note(name, which, w)
            print("%s: accepted %d of %d, worst chi2 error / bound %.3e" % (tag, int((r["status"][r["sel"]] == 1).sum()), len(r["sel"]), w))
            got[name] = (r, refs)
            if ci == 0:  # the raw rows the references start from are the oracle's (columns matched by state index)
                cal = gr.calib_ids(ctx, S.options)
                cho_of = {int(h): int(o) for h, o in zip(chg, cho)}
                for f in list(r["sel"][:3]) + list(r["sel"][-1:]):
                    a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
                    pf = b["p_FinG_original"][f]
                    _check_raw(orc, b, f, r["raw"], cal + gr.block_ids(ctx, b["meas_clone"][a:e], 6), ncal, cho_of, pf, pf, 0, None, None, sigma,
                               S.options["sigma_constraint"])
        if len(got) == 2:
            (rw, refw), (rc, _) = got["warp"], got["CTA"]
            assert np.array_equal(rw["status"], rc["status"]), "the two kernels' statuses differ"
            for f, (_, bound, _) in refw.items():
                assert abs(rw["chi2"][f] - rc["chi2"][f]) <= 2 * bound, (f, rw["chi2"][f], rc["chi2"][f], bound)
        if kind == "mixed" and ci == 0:
            assert (got["warp"][0]["status"] == 0).sum() >= 2, "the outliers should be rejected"
        ctx.close()
        orc.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# SLAM gate
# ---------------------------------------------------------------------------------------------------------------------------------
def slam_update_raw(ctx, b, sigma_pix=1.0, chi2_mult=1.0, use_plane=True):
    F, M = int(b["F"]), int(b["meas_offset"][-1])
    uo = api.UpdaterOptions(sigma_pix, chi2_mult)
    fs, fc, raw = np.zeros(F, dtype=np.int32), np.zeros(F), np.zeros(3 * gr.RAW_ROW * M)
    mo, mc = np.ascontiguousarray(b["meas_offset"], dtype=np.int32), np.ascontiguousarray(b["meas_clone"], dtype=np.int32)
    uv = np.ascontiguousarray(b["uv"], dtype=np.float32)
    fid, pid = np.ascontiguousarray(b["featid"], dtype=np.int64), np.ascontiguousarray(b["planeid"], dtype=np.int64)
    ctx._ck(ctx.lib.ovp_debug_slam_update(ctx.h, F, _p(mo), _p(mc), _p(uv), _p(fid), _p(pid), C.byref(uo), int(bool(use_plane)), _p(fs), _p(fc),
                                          _p(raw)))
    return fs, fc, raw.reshape(M, 3, gr.RAW_ROW)


def slam_setup(ncal, which, chi2_table, table=None, seed=0):
    """context with the landmarks of gr.slam_scenario initialised (delayed_init) and the covariance `which` uploaded; the update batch
    (tracks of 1, 2, 15 and 29, 3 features on a wrong plane), the featids attached to their plane, and P"""
    S = gr.slam_scenario(ncal, seed=seed)
    ctx, orc, chg, cho = debug_pair(S, chi2_table, S.N + 3 * S.F + 64)
    g = ctx.slam_delayed_init(synth.feature_batch(S, chg), 1.0, 1.0)
    keep = np.nonzero(g["feat_status"] > 0)[0]
    attached = {int(S.featid[f]) for f in keep if g["feat_status"][f] == 1 and S.planeid[f] != 0}
    assert len(keep) >= 16 and len(attached) >= 6, (len(keep), len(attached))
    P = _upload(ctx, S, which, 7 + ncal)
    if table is not None:
        ctx.set_chi2_table(table)
    b = gr.slam_update_batch(S, chg, keep, seed=ncal, wrong_plane=3)
    return S, ctx, orc, chg, cho, b, attached, P


def slam_refs(ctx, S, b, raw, statuses, attached, P, use_plane=True):
    """{feature: (chi2, bound, dof)} of the gate each reported status implies, from the kernel's raw rows"""
    cal = gr.calib_ids(ctx, S.options)
    out = {}
    for f in range(b["F"]):
        a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
        has_plane = use_plane and int(b["featid"][f]) in attached
        with_plane = has_plane and statuses[f] == 1
        Hf, Hx, rr = gr.raw_block(raw, a, e, len(cal), has_plane)
        lm = ctx.slam_handle(int(b["featid"][f]))
        ids = gr.block_ids(ctx, [lm]) + cal + gr.block_ids(ctx, b["meas_clone"][a:e], 6)
        H = np.hstack([Hf, Hx])
        if with_plane:
            ids += gr.block_ids(ctx, [ctx.plane_handle(int(b["planeid"][f]))])
        else:
            H, rr = H[:2 * (e - a), :H.shape[1] - (3 if has_plane else 0)], rr[:2 * (e - a)]
        out[f] = gr.slam_gate(H, rr, P[np.ix_(ids, ids)])
    return out


SLAM_CASES = [(n, use) for n in (0, 14) for use in (True, False)]


@pytest.mark.parametrize("ncal,use_plane", SLAM_CASES, ids=["ncal%d-%s" % (n, "plane" if u else "no_plane_constraint") for n, u in SLAM_CASES])
def test_slam_gate_against_long_double_reference(ncal, use_plane, chi2_table):
    gr.require_long_double()
    for which in COVS:
        S, ctx, orc, chg, cho, b, attached, P = slam_setup(ncal, which, chi2_table)
        # the values the kernel linearises at, read before the update moves them; the oracle takes the clones, calibration and planes
        lmv = {int(fid): ctx.var_get(ctx.slam_handle(int(fid))) for fid in b["featid"]}
        pairs = list(zip(chg, cho)) + [(ctx.handle_calib(), orc.handle_calib()), (ctx.handle_intrinsics(), orc.handle_intrinsics())]
        pairs += [(ctx.plane_handle(int(pid)), orc.plane_handle(int(pid))) for pid in S.plane_ids]
        for hg, ho in pairs:
            orc.var_set(int(ho), *ctx.var_get(int(hg)))
        fs, fc, raw = slam_update_raw(ctx, b, use_plane=use_plane)
        refs = slam_refs(ctx, S, b, raw, fs, attached, P, use_plane)
        w = 0.0
        for f, (ref, bound, dof) in refs.items():
            has_plane = use_plane and int(b["featid"][f]) in attached
            assert fs[f] in ((0, 1, 3) if has_plane else (0, 1))
            w = max(w, check_gate("SLAM ncal=%d %s" % (ncal, which), fs, fc, {f: refs[f]}, chi2_table, 1.0, 3 if has_plane and fs[f] != 1 else 1))
        _note("SLAM", which, w)
        counts = np.bincount(fs, minlength=4)
        print("SLAM ncal=%d plane=%d %s: statuses %s, worst chi2 error / bound %.3e" % (ncal, use_plane, which, counts.tolist(), w))
        assert counts[1] >= 8
        if use_plane:
            assert counts[3] >= 1, "the landmarks on a wrong plane should be accepted without it"
        # raw rows against the oracle (landmark as p_FinG), the partial last covariance panel is in the cases: ncs = 3 + ncal + 6m (+3)
        if which == "P0":
            cho_of = {int(h): int(o) for h, o in zip(chg, cho)}
            cal = gr.calib_ids(ctx, S.options)
            for f in range(min(8, b["F"])):
                a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
                val, fej = lmv[int(b["featid"][f])]
                pid, cp, cpf = 0, None, None
                ids = cal + gr.block_ids(ctx, b["meas_clone"][a:e], 6)
                if use_plane and int(b["featid"][f]) in attached:
                    pid = int(b["planeid"][f])
                    cp, cpf = orc.var_get(orc.plane_handle(pid))
                    ids += gr.block_ids(ctx, [ctx.plane_handle(pid)])
                _check_raw(orc, b, f, raw, ids, ncal, cho_of, val, fej, pid, cp, cpf, 1.0, S.options["sigma_constraint"])
        ctx.close()
        orc.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# decisions at the threshold, table entries, table length
# ---------------------------------------------------------------------------------------------------------------------------------
def mults_around(chi, t):
    """(hi, lo): hi the smallest multiplier with fl(hi * t) >= chi (= chi when such a product exists), lo the next smaller double, whose
    product lies below chi"""
    m = chi / t
    while m * t < chi:
        m = np.nextafter(m, np.inf)
    while np.nextafter(m, 0.0) * t >= chi:
        m = np.nextafter(m, 0.0)
    lo = np.nextafter(m, 0.0)
    assert lo * t < chi <= m * t
    return float(m), float(lo)


@pytest.mark.parametrize("dense", [0, 1], ids=["warp", "CTA"])
def test_point_gate_decision_at_its_threshold(dense, chi2_table):
    S = _point_scenario("mixed", None, 14)
    ctx, orc, chg, cho = debug_pair(S, chi2_table, S.N + 8)
    b = synth.feature_batch(S, chg)
    P = _upload(ctx, S, "correlated", 114)
    r = run_gram(ctx, b, dense)
    refs = point_gate_refs(ctx, S, b, r, P)
    picks = [f for f in r["sel"] if r["status"][f] == 1][:2] + [f for f in r["sel"] if r["status"][f] == 0][:1]
    for f in picks:
        chi = float(r["chi2"][f])
        ref, bound, dof = refs[int(f)]
        t = chi2_table[dof]
        hi, lo = mults_around(chi, t)
        for mult, want in ((hi, 1), (lo, 0)):
            q = run_gram(ctx, b, dense, 1.0, mult)
            assert q["chi2"][f] == chi, "chi2 depends on the multiplier"
            assert q["status"][f] == want, "feature %d: status %d with threshold %r for chi2 %r" % (f, q["status"][f], mult * t, chi)
        for s, want in ((1.0, 1), (-1.0, 0)):
            mult = float(ref) / t * (1.0 + s * 100.0 * bound / float(ref))
            q = run_gram(ctx, b, dense, 1.0, mult)
            assert q["status"][f] == want, "feature %d: status %d with the reference %s 100 bounds from the threshold" % (f, q["status"][f],
                                                                                                                      "within" if want else "beyond")
    ctx.close()
    orc.close()


def test_slam_gate_decision_at_its_threshold(chi2_table):
    S, ctx, orc, chg, cho, b, attached, P = slam_setup(14, "correlated", chi2_table)
    fs, fc, raw = slam_update_raw(ctx, b)
    refs = slam_refs(ctx, S, b, raw, fs, attached, P)
    ctx.close()
    orc.close()
    plane = [f for f in range(b["F"]) if fs[f] == 1 and int(b["featid"][f]) in attached][:2]
    retry = [f for f in range(b["F"]) if fs[f] == 3][:1]
    assert plane and retry
    for f in plane + retry:
        chi = float(fc[f])
        ref, bound, dof = refs[f]
        t = chi2_table[dof]
        hi, lo = mults_around(chi, t)
        accept = 1 if f in plane else 3
        cases = [(hi, lambda s: s == accept), (lo, (lambda s: s != 1) if accept == 1 else (lambda s: s == 0))]
        for s in (1.0, -1.0):
            mult = float(ref) / t * (1.0 + s * 100.0 * bound / float(ref))
            cases.append((mult, (lambda st: st == accept) if s > 0 else ((lambda st: st != 1) if accept == 1 else (lambda st: st == 0))))
        for mult, ok in cases:
            _, ctx, orc, _, _, b2, _, _ = slam_setup(14, "correlated", chi2_table)
            q, qc, _ = slam_update_raw(ctx, b2, 1.0, mult)
            ctx.close()
            orc.close()
            if mult in (hi, lo):
                assert qc[f] == chi or q[f] != accept, "chi2 depends on the multiplier"
            assert ok(q[f]), "landmark %d (%s): status %d with multiplier %r (chi2 %r, table %r)" % (f, "plane" if accept == 1 else "retry", q[f],
                                                                                                 mult, chi, t)


def test_point_gate_reads_table_entry_2m_minus_3(chi2_table):
    S = _point_scenario("mixed", None, 0)
    m = np.diff(S.meas_offset)
    n = 3 * int(m.max()) + 1
    for dense in (0, 1):
        ctx, orc, chg, cho = debug_pair(S, chi2_table, S.N + 8)
        b = synth.feature_batch(S, chg)
        for i in sorted({int(2 * x - 3) for x in m} | {int(2 * x - 2) for x in m[:3]} | {int(2 * x) for x in m[:3]}):
            table = np.zeros(n)
            table[i] = 1e300
            ctx.set_chi2_table(table)
            r = run_gram(ctx, b, dense)
            assert np.array_equal(r["status"] == 1, 2 * m - 3 == i), "%s kernel, table non-zero at %d: accepted %s" % (
                "CTA" if dense else "warp", i, sorted(set(m[r["status"] == 1].tolist())))
        ctx.close()
        orc.close()


def test_slam_gate_reads_table_entries_3m_then_2m(chi2_table):
    n = 3 * 30 + 1
    for i in (3, 2, 6, 4, 45, 30, 87, 58):
        table = np.zeros(n)
        table[i] = 1e300
        S, ctx, orc, chg, cho, b, attached, P = slam_setup(0, "correlated", chi2_table, table=table)
        fs, _, _ = slam_update_raw(ctx, b)
        ctx.close()
        orc.close()
        for f in range(b["F"]):
            m = int(b["meas_offset"][f + 1] - b["meas_offset"][f])
            if int(b["featid"][f]) in attached:
                want = 1 if 3 * m == i else (3 if 2 * m == i else 0)
            else:
                want = 1 if 2 * m == i else 0
            assert fs[f] == want, "table non-zero at %d: landmark %d (m = %d, plane %d) has status %d, expected %d" % (
                i, f, m, int(b["featid"][f]) in attached, fs[f], want)


def _state(ctx, handles):
    return [ctx.cov().copy()] + [np.concatenate(ctx.var_get(int(h))) for h in handles]


def _same(a, b):
    return all(np.array_equal(x.view(np.uint64), y.view(np.uint64)) for x, y in zip(a, b))


def test_chi2_table_length_is_checked(chi2_table):
    S = _point_scenario("mixed", None, 8)
    ctx, orc, chg, cho = debug_pair(S, chi2_table, S.N + 64)
    mmax = int(np.diff(S.meas_offset).max())
    b = synth.feature_batch(S, chg)
    hs = list(chg) + [ctx.handle_imu(), ctx.handle_calib(), ctx.handle_intrinsics()]
    before = _state(ctx, hs)
    ctx.set_chi2_table(chi2_table[:3 * mmax])
    with pytest.raises(api.OvpError) as e:
        ctx.msckf_update(b)
    assert e.value.status == 1  # OVP_ERR_BAD_ARGS
    assert _same(before, _state(ctx, hs)), "a refused MSCKF update changed the state"
    ctx.set_chi2_table(chi2_table[:3 * mmax + 1])
    ctx.msckf_update(b)
    ctx.close()
    orc.close()

    S, ctx, orc, chg, cho, b, attached, P = slam_setup(0, "P0", chi2_table)
    mmax = int(np.diff(b["meas_offset"]).max())
    hs = list(chg) + [ctx.slam_handle(int(fid)) for fid in b["featid"]]
    before = _state(ctx, hs)
    ctx.set_chi2_table(chi2_table[:3 * mmax])
    with pytest.raises(api.OvpError) as e:
        ctx.slam_update(b)
    assert e.value.status == 1
    assert _same(before, _state(ctx, hs)), "a refused SLAM update changed the state"
    ctx.set_chi2_table(chi2_table[:3 * mmax + 1])
    ctx.slam_update(b)
    ctx.close()
    orc.close()
