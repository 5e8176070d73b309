"""The raw rows of every device path that builds feature Jacobians, entry by entry against the long-double measurement model of
tests/feature_jacobian_reference.py (H_f, the clone, extrinsic and intrinsic blocks, the residual and the point-on-plane row, each within
its bound C u mag):

- the MSCKF feature CTA (msckf_warp.inc, tracks of at most 32) and the dense feature kernel (features.cu, forced, and for tracks of 33-39),
  points and planes, through ovp_debug_msckf_gram;
- the SLAM feature kernel (features.cu mode 2, the landmark's value and first estimate from the state) through ovp_debug_slam_gram, and
  the same rows from ovp_debug_slam_update;
- ovp_feature_jacobian_full (jacobian_only_kernel) and ovp_feature_jacobian_full_rep (representation_chain_kernel after it).

Each path also keeps its column layout, its structural zeros exactly 0.0, the same bits from run to run and the state untouched.  The
plausible wrong models of feature_jacobian_reference.MUTATIONS lie outside the bound from the kernels' rows.  The geometry is explicit
(tests/test_cpu_feature_jacobian_reference.py): first estimates of the clones 1e-2 rad and up to 5 cm from their values, landmark and
plane first estimates apart from theirs."""
import ctypes as C

import numpy as np
import pytest

import feature_jacobian_reference as fr
import gate_reference as gr
import test_cpu_feature_jacobian_reference as cr
from ov_plane_b200 import api, jpl
from test_gpu_compression import _p
from test_gpu_feature_gate import slam_update_raw

pytestmark = pytest.mark.gpu

WORST = {}  # (path, part) -> worst error / bound over the module
ULPS = {}  # (path, path) -> largest ulp distance of the same feature's rows


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for (path, part), v in sorted(WORST.items()):
        print("feature Jacobians: %-14s %-11s worst error / bound %.3e" % (path, part, v))
    for (a, b), v in sorted(ULPS.items()):
        print("feature Jacobians: %s vs %s: largest ulp difference %d" % (a, b, v))


def _note(path, w):
    for part, v in w.items():
        WORST[(path, part)] = max(WORST.get((path, part), 0.0), v)
        assert v <= 1.0, "%s: %s outside its bound (worst error / bound %.3e)" % (path, part, v)


def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float64).view(np.uint64)


def _state(ctx, handles):
    return [_bits(ctx.cov())] + [_bits(np.concatenate(ctx.var_get(int(h)))) for h in handles]


def _context(S, chi2_table, max_state):
    """a context on libovp_debug.so with the layout of S (load_case fills it in)"""
    ctx = api.Context(S.options, device=0, max_state=max_state, max_meas_rows=60000, debug=True)
    ctx.set_chi2_table(chi2_table)
    return ctx


def _same_state(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


# ---------------------------------------------------------------------------------------------------------------------------------
# batches
# ---------------------------------------------------------------------------------------------------------------------------------
def _project_uv(clones, track, pf, cam, rng, noise=0.5):
    uv = []
    for i, k in enumerate(track):
        pc = cr.R_ItoC @ (jpl.quat_2_Rot(clones[k][0][:4]) @ (pf - clones[k][0][4:])) + cr.P_IinC
        u, v = jpl.radtan_distort(cr.CAMS[cam], pc[0] / pc[2], pc[1] / pc[2])
        e = rng.normal(0.0, noise, 2) if i % 3 else np.zeros(2)
        uv.append((u + e[0], v + e[1]))
    return np.array(uv, dtype=np.float32)


def features_around(case, F, seed):
    """clones, the track, and F features: the case's own first, then points within 1e-3 Z of it (each with its own pixels)"""
    L, radius, depth, cam, order = case["L"], case["radius"], case["depth"], case["cam"], case["order"]
    clones, track, pf, pff, uv = cr.geometry(L, radius, depth, cam, seed=seed, order=order)
    rng = np.random.default_rng(seed + 77)
    Z = cr.DEPTHS[depth]
    pts, uvs = [pf], [uv]
    for _ in range(F - 1):
        p = pf + 1e-3 * Z * rng.normal(0.0, 1.0, 3)
        pts.append(p)
        uvs.append(_project_uv(clones, track, p, cam, rng))
    return clones, track, np.array(pts), uvs


def msckf_batch(ch, track, pts, uvs, planeid, plane_cp):
    F, m = len(pts), len(track)
    return dict(F=F, meas_offset=np.arange(F + 1, dtype=np.int32) * m, meas_clone=np.ascontiguousarray(np.tile([ch[k] for k in track], F), dtype=np.int32),
                uv=np.ascontiguousarray(np.concatenate(uvs), dtype=np.float32), p_FinG=np.ascontiguousarray(pts), p_FinG_original=np.ascontiguousarray(pts),
                featid=np.arange(F, dtype=np.int64) + 4097, planeid=np.full(F, planeid, dtype=np.int64),
                plane_ids=np.array([planeid] if planeid else [], dtype=np.int64),
                plane_cp=np.ascontiguousarray(np.asarray(plane_cp, dtype=np.float64).reshape(-1, 3)) if planeid else np.zeros((0, 3)))


def gram_raw(ctx, batch, dense, sigma_pix):
    """ovp_debug_msckf_gram: (raw M x 3 x 24, info, statuses)"""
    fb, keep = api.Context._batch_struct(batch)
    uo = api.UpdaterOptions(sigma_pix, 1.0)
    F, M = fb.F, int(batch["meas_offset"][-1])
    gcap = ctx.cov_rows() + 4
    G, info, cols = np.zeros(gcap * gcap), np.zeros(8, dtype=np.int32), np.zeros(gcap, dtype=np.int32)
    sel, fs, fc = np.zeros(F, dtype=np.int32), np.zeros(F, dtype=np.int32), np.zeros(F)
    raw = np.zeros(3 * gr.RAW_ROW * M)
    ctx._ck(ctx.lib.ovp_debug_force_dense_features(ctx.h, int(dense)))
    ctx._ck(ctx.lib.ovp_debug_msckf_gram(ctx.h, C.byref(fb), C.byref(uo), gcap, _p(G), _p(info), _p(cols), _p(sel), _p(fs), _p(fc), _p(raw)))
    ctx._ck(ctx.lib.ovp_debug_force_dense_features(ctx.h, 0))
    return raw.reshape(M, 3, gr.RAW_ROW), info, fs


def slam_gram_raw(ctx, b, sigma_pix):
    """ovp_debug_slam_gram without the plane constraint: the raw rows, the state left as it was"""
    F, M = int(b["F"]), int(b["meas_offset"][-1])
    uo = api.UpdaterOptions(sigma_pix, 1.0)
    gcap = ctx.cov_rows() + 4
    G, info, cols = np.zeros(gcap * gcap), np.zeros(2, dtype=np.int32), np.zeros(gcap, dtype=np.int32)
    fs, fc, raw = np.zeros(F, dtype=np.int32), np.zeros(F), np.zeros(3 * gr.RAW_ROW * M)
    arr = [np.ascontiguousarray(b[k], dtype=t) for k, t in (("meas_offset", np.int32), ("meas_clone", np.int32), ("uv", np.float32),
                                                              ("featid", np.int64), ("planeid", np.int64))]
    ctx._ck(ctx.lib.ovp_debug_slam_gram(ctx.h, F, *[_p(a) for a in arr], C.byref(uo), 0, gcap, _p(G), _p(info), _p(cols), _p(fs), _p(fc),
                                        _p(raw)))
    return raw.reshape(M, 3, gr.RAW_ROW)


def check_raw(path, be, raw, a, track_handles, pf, pff, uv, sigma_pix, do_fej, ncal, plane=None):
    """raw rows of the measurements [a, a + m) against the reference in the raw_block layout; returns the per-part ratios"""
    m = len(track_handles)
    Hf, Hx, r = gr.raw_block(raw, a, a + m, ncal, plane is not None)
    I = cr.inputs(be, track_handles, pf, pff, uv, sigma_pix, do_fej)
    ref, mag, part = cr.dense_reference(I, ncal, plane, True)
    return cr.entry_ratios({"Hf": Hf, "Hx": Hx, "res": r}, ref, mag, part), I, (Hf, Hx, r), plane


# ---------------------------------------------------------------------------------------------------------------------------------
# MSCKF: the feature CTA and the dense kernel
# ---------------------------------------------------------------------------------------------------------------------------------
def _case(L, radius, depth, cam, do_fej, ncal, sigma, order, paths, plane=None):
    return dict(L=L, radius=radius, depth=depth, cam=cam, do_fej=do_fej, ncal=ncal, sigma=sigma, order=order, paths=paths, plane=plane)


MSCKF_CASES = [_case(2, "centre", "near", "tangential", 1, 14, 1.0, "forward", "both"),
               _case(3, "x axis", "far", "euroc", 1, 6, 0.37, "reversed", "both"),
               _case(31, "wide", "near", "tangential", 0, 8, 4.0, "gaps", "both"),
               _case(32, "y axis", "far", "tangential", 1, 0, 1.0, "forward", "both"),
               _case(33, "wide", "far", "euroc", 1, 14, 1.0, "reversed", "dense"),
               _case(39, "centre", "near", "tangential", 1, 6, 0.37, "forward", "dense"),
               _case(37, "wide", "near", "tangential", 1, 14, 1.0, "forward", "dense", plane="in"),
               _case(3, "x axis", "far", "euroc", 1, 8, 4.0, "gaps", "both", plane="out"),
               _case(4, "centre", "near", "tangential", 1, 0, 0.37, "reversed", "both", plane="in")]
PLANE_ID = 7


def msckf_setup(c, chi2_table, seed):
    L = c["L"]
    if c["plane"] is None:  # enough features that the point plan compresses in a context of max_state = N + 8 (it then has a Gram matrix)
        n_cl = 2 * L + 1 if c["order"] == "gaps" else L + 1
        N = 16 + c["ncal"] + 6 * n_cl
        F = max(24, int(np.ceil((2 * (N + 8) + 64) / (2 * L - 3)))) if L > 1 else 24
    else:
        F = 24
    clones, track, pts, uvs = features_around(c, F, seed)
    cp = cpf = None
    planes = ()
    if c["plane"] is not None:
        cp, cpf = cr.plane_for(pts[0], seed, Z=cr.DEPTHS[c["depth"]])
        if c["plane"] == "in":
            planes = ((PLANE_ID, cp, cpf),)
        else:
            cpf = cp  # a plane outside the state is linearised at the batch's cp
    S = cr.scenario(c["ncal"], len(clones), c["do_fej"], planes)
    ctx = _context(S, chi2_table, S.N + 8)
    ch = cr.load_case(ctx, S, clones, c["cam"])
    b = msckf_batch(ch, track, pts, uvs, PLANE_ID if c["plane"] else 0, cp)
    return ctx, ch, track, b, pts, (cp, cpf)


@pytest.mark.parametrize("c", MSCKF_CASES, ids=["L%d-%s-%s-%s-fej%d-ncal%d-sigma%g-%s-%s-plane_%s" % (
    c["L"], c["radius"].replace(" ", "_"), c["depth"], c["cam"], c["do_fej"], c["ncal"], c["sigma"], c["order"], c["paths"], c["plane"])
    for c in MSCKF_CASES])
def test_msckf_feature_rows_against_the_reference(c, chi2_table):
    fr.require_long_double()
    ctx, ch, track, b, pts, (cp, cpf) = msckf_setup(c, chi2_table, seed=c["L"] + c["ncal"])
    hs = [ch[k] for k in track]
    watch = list(ch) + [ctx.handle_calib(), ctx.handle_intrinsics()] + ([ctx.plane_handle(PLANE_ID)] if c["plane"] == "in" else [])
    before = _state(ctx, watch)
    m = c["L"]
    got = {}
    for dense in ((0, 1) if c["paths"] == "both" else (1,)):
        path = ("dense" if dense else "feature CTA") + (" plane" if c["plane"] else "")
        raw, info, fs = gram_raw(ctx, b, dense, c["sigma"])
        assert int(info[3]) == (c["plane"] is None) and int(info[1]) == c["ncal"]
        if not dense:
            assert info[5] == 1, "the batch did not take the feature CTA"
        if c["plane"] is not None:
            assert int(info[7]) == (c["plane"] == "in")
        again, _, _ = gram_raw(ctx, b, dense, c["sigma"])
        assert np.array_equal(_bits(raw), _bits(again)), "%s: the raw rows differ from run to run" % path
        assert _same_state(before, _state(ctx, watch)), "%s: the state changed" % path
        checked = 0
        for f in range(b["F"]):
            if fs[f] == 2:
                continue
            plane = (cp, cpf, cr.SIGMA_C) if c["plane"] else None
            w, *_ = check_raw(path, ctx, raw, f * m, hs, pts[f], pts[f], b["uv"][f * m:(f + 1) * m], c["sigma"], c["do_fej"], c["ncal"], plane)
            _note(path, w)
            checked += 1
        assert checked >= b["F"] // 2, (checked, b["F"])
        got[dense] = raw
    sfx = " plane" if c["plane"] else ""
    if len(got) == 2:
        key = ("feature CTA" + sfx, "dense" + sfx)
        ULPS[key] = max(ULPS.get(key, 0), fr.ulp_diff(got[0], got[1]))
    if c["plane"] is None:  # the same feature through the public entry point
        o = ctx.feature_jacobian_full(hs, b["uv"][:m], pts[0], pts[0], 0, None, None, c["sigma"], cr.SIGMA_C)
        for dense, raw in got.items():
            Hf, Hx, r = gr.raw_block(raw, 0, m, c["ncal"], False)
            key = ("dense" if dense else "feature CTA", "public")
            ULPS[key] = max(ULPS.get(key, 0), max(fr.ulp_diff(np.asarray(x, dtype=np.float64), y) for x, y in ((Hf, o[0]), (Hx, o[1]), (r, o[2]))))
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# SLAM: the landmark's value and first estimate from the state
# ---------------------------------------------------------------------------------------------------------------------------------
SLAM_CASES = [(14, 1, "wide", "near", "tangential", 1.0), (0, 1, "centre", "far", "euroc", 0.37), (6, 0, "x axis", "near", "tangential", 4.0)]


@pytest.mark.parametrize("ncal,do_fej,radius,depth,cam,sigma", SLAM_CASES, ids=["ncal%d-fej%d-%s-%s-%s-sigma%g" % (n, d, r.replace(" ", "_"), z, k, s)
                                                                               for n, d, r, z, k, s in SLAM_CASES])
def test_slam_feature_rows_against_the_reference(ncal, do_fej, radius, depth, cam, sigma, chi2_table):
    fr.require_long_double()
    L = 29
    c = dict(L=L, radius=radius, depth=depth, cam=cam, order="reversed")
    clones, track, pts, _ = features_around(c, 6, seed=ncal + 3)
    Z = cr.DEPTHS[depth]
    rng = np.random.default_rng(ncal)
    fej = pts + 1e-3 * Z * rng.normal(0.0, 1.0, pts.shape)  # the landmarks' first estimates apart from their values
    S = cr.scenario(ncal, len(clones), do_fej)
    S.slam = [(9000 + i, pts[i], fej[i]) for i in range(len(pts))]
    N = S.N + 3 * len(pts)
    P0 = np.eye(N) * 1e-4
    P0[:S.N, :S.N] = S.P0
    S.P0, S.N = P0, N
    ctx = _context(S, chi2_table, S.N + 8)
    ch = cr.load_case(ctx, S, clones, cam)
    lengths = [1, 2, 29, 1, 2, 29]
    mo, mc, uv = [0], [], []
    for i, m in enumerate(lengths):
        tr = track[-m:] if i % 2 else track[:m]
        mc += [ch[k] for k in tr]
        uv.append(_project_uv(clones, tr, pts[i], cam, rng))
        mo.append(mo[-1] + m)
    b = dict(F=len(lengths), meas_offset=np.array(mo, dtype=np.int32), meas_clone=np.array(mc, dtype=np.int32),
             uv=np.ascontiguousarray(np.concatenate(uv), dtype=np.float32), featid=np.array([s[0] for s in S.slam], dtype=np.int64),
             planeid=np.zeros(len(lengths), dtype=np.int64))
    watch = list(ch) + [ctx.handle_calib(), ctx.handle_intrinsics()] + [ctx.slam_handle(s[0]) for s in S.slam]
    before = _state(ctx, watch)
    raw = slam_gram_raw(ctx, b, sigma)
    assert np.array_equal(_bits(raw), _bits(slam_gram_raw(ctx, b, sigma))), "the SLAM rows differ from run to run"
    assert _same_state(before, _state(ctx, watch)), "ovp_debug_slam_gram changed the state"
    for i in range(b["F"]):
        a, e = int(mo[i]), int(mo[i + 1])
        val, fe = ctx.var_get(ctx.slam_handle(int(b["featid"][i])))
        w, *_ = check_raw("SLAM", ctx, raw, a, mc[a:e], val, fe, b["uv"][a:e], sigma, do_fej, ncal)
        _note("SLAM", w)
    # the update's own hook builds the same rows (before it moves the state)
    _, _, raw_u = slam_update_raw(ctx, b, sigma, 1.0, use_plane=False)
    assert np.array_equal(_bits(raw), _bits(raw_u)), "ovp_debug_slam_update's rows differ from ovp_debug_slam_gram's"
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# the public entry points
# ---------------------------------------------------------------------------------------------------------------------------------
def _public_setup(chi2_table, m, do_fej, ncal, cam, radius, depth, seed):
    clones, track, pf, pff, uv = cr.geometry(m, radius, depth, cam, seed=seed, order="reversed")
    cp, cpf = cr.plane_for(pf, seed, Z=cr.DEPTHS[depth])
    S = cr.scenario(ncal, len(clones), do_fej, ((PLANE_ID, cp, cpf),))
    ctx = _context(S, chi2_table, S.N + 16)
    ch = cr.load_case(ctx, S, clones, cam)
    return ctx, ch, [ch[k] for k in track], pf, pff, uv, (cp, cpf)


def public_rows(ctx, hs, uv, pf, pff, planeid, cp, cpf, sigma, ncal, do_fej):
    """ovp_feature_jacobian_full against the reference in the dense layout; returns (ratios, rows, reference inputs)"""
    o = ctx.feature_jacobian_full(hs, uv, pf, pff, planeid, cp, cpf, sigma, cr.SIGMA_C)
    want = ([ctx.handle_calib()] if cr.NCAL[ncal][0] else []) + ([ctx.handle_intrinsics()] if cr.NCAL[ncal][1] else []) + list(hs)
    in_state = planeid != 0 and ctx.plane_handle(planeid) >= 0
    want += [ctx.plane_handle(planeid)] if in_state else []
    assert o[3] == want, (o[3], want)
    m = len(hs)
    assert o[1].shape == ((3 if planeid else 2) * m, ncal + 6 * m + (3 if in_state else 0)), o[1].shape
    I = cr.inputs(ctx, hs, pf, pff, uv, sigma, do_fej)
    ref, mag, part = cr.dense_reference(I, ncal, (cp, cpf, cr.SIGMA_C) if planeid else None, in_state)
    got = {"Hf": o[0], "Hx": o[1], "res": o[2]}
    # structural zeros: exactly 0.0 wherever the reference has an exact zero
    for key in ("Hf", "Hx"):
        z = ref[key] == 0
        assert (got[key][z] == 0.0).all(), "%s: a structural zero is not 0.0" % key
    return cr.entry_ratios(got, ref, mag, part), o, I, (ref, mag, part)


PUBLIC_CASES = [(1, 14, "tangential", "wide", "near", 0.37), (1, 6, "euroc", "centre", "far", 4.0), (0, 8, "tangential", "x axis", "near", 1.0),
                (1, 0, "euroc", "y axis", "far", 1.0)]


@pytest.mark.parametrize("do_fej,ncal,cam,radius,depth,sigma", PUBLIC_CASES, ids=["fej%d-ncal%d-%s-%s-%s-sigma%g" % (d, n, k, r.replace(" ", "_"), z, s)
                                                                               for d, n, k, r, z, s in PUBLIC_CASES])
def test_feature_jacobian_full_against_the_reference(do_fej, ncal, cam, radius, depth, sigma, chi2_table):
    """the longest track one launch takes (64 measurements, one thread block) with the plane in the state, then shorter tracks in the
    same context: without a plane, with a plane outside the state; the landmark's first estimate apart from its value"""
    fr.require_long_double()
    ctx, ch, hs, pf, pff, uv, (cp, cpf) = _public_setup(chi2_table, 64, do_fej, ncal, cam, radius, depth, seed=ncal + do_fej)
    watch = list(ch) + [ctx.handle_calib(), ctx.handle_intrinsics(), ctx.plane_handle(PLANE_ID)]
    before = _state(ctx, watch)
    w, o, _, _ = public_rows(ctx, hs, uv, pf, pff, PLANE_ID, cp, cpf, sigma, ncal, do_fej)
    _note("public", w)
    again = ctx.feature_jacobian_full(hs, uv, pf, pff, PLANE_ID, cp, cpf, sigma, cr.SIGMA_C)
    assert all(np.array_equal(_bits(x), _bits(y)) for x, y in zip(o[:3], again[:3])), "the rows differ from run to run"
    for sub, planeid in ((slice(3, 8), 0), (slice(10, 12), 0), (slice(0, 5), 99)):
        w, *_ = public_rows(ctx, hs[sub], uv[sub], pf, pff, planeid, cp if planeid else None, cpf if planeid else None, sigma, ncal, do_fej)
        _note("public", w)
    with pytest.raises(api.OvpError):
        ctx.feature_jacobian_full(list(hs) + [hs[0]], np.vstack([uv, uv[:1]]), pf, pff, 0, None, None, sigma, cr.SIGMA_C)
    assert _same_state(before, _state(ctx, watch)), "ovp_feature_jacobian_full changed the state"
    ctx.close()


C_REP = fr.C_PART["clone"] + 3 + 8


@pytest.mark.parametrize("do_fej", [0, 1])
def test_feature_jacobian_full_rep_against_the_reference(do_fej, chi2_table):
    fr.require_long_double()
    m, ncal = 6, 14
    ctx, ch, hs, pG, pGf, uv, _ = _public_setup(chi2_table, m, do_fej, ncal, "tangential", "wide", "near", seed=40 + do_fej)
    outside = [h for h in ch if h not in hs]
    assert outside
    cal = ctx.var_get(ctx.handle_calib())[0]
    for rep in range(6):
        for anchor in ([hs[2], outside[0]] if rep >= 2 else [-1]):
            if rep >= 2:
                pF = np.asarray(fr.global_to_anchor(fr.ld(ctx.var_get(anchor)[0]), fr.ld(cal), fr.ld(pG)), dtype=np.float64)
                pFf = pF
            else:
                pF, pFf = pG, pGf
            o = ctx.feature_jacobian_full_rep(hs, uv, rep, anchor, pF, pFf, 1.0)
            Hf, Hx, res, order, mags = cr.rep_reference(ctx, hs, uv, rep, anchor, pF, pFf, 1.0, do_fej, ncal, mags=True)
            assert o[3] == order, (rep, o[3], order)
            assert o[0].shape == Hf.shape and o[1].shape == Hx.shape
            assert (o[1][Hx == 0] == 0.0).all(), "rep %d: a structural zero of H_x is not 0.0" % rep
            # the bearing rows' bound, and the chain's 3-term products (3) after d p_FinG / d . (trigonometry and the anchor
            # transform on the host, depth at most 8): C_REP
            for key, got, want, mg, c in (("Hf", o[0], Hf, mags[0], C_REP), ("Hx", o[1], Hx, mags[1], C_REP), ("res", o[2], res, mags[2], None)):
                e = fr.ratio(got, want, mg, "res") if c is None else fr.ratio(got, want, mg, "clone") * fr.C_PART["clone"] / c
                v = float(e.max())
                WORST[("public rep", key)] = max(WORST.get(("public rep", key), 0.0), v)
                assert v <= 1.0, "rep %d anchor %d: %s outside its bound (worst error / bound %.3e)" % (rep, anchor, key, v)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# the wrong models lie outside the bound from the kernels' rows
# ---------------------------------------------------------------------------------------------------------------------------------
def test_wrong_models_lie_outside_the_bound_from_the_kernel_rows(chi2_table):
    fr.require_long_double()
    found = {}
    for do_fej, ncal, cam, radius, depth, sigma in PUBLIC_CASES:
        ctx, ch, hs, pf, pff, uv, (cp, cpf) = _public_setup(chi2_table, 8, do_fej, ncal, cam, radius, depth, seed=5 + ncal)
        for planeid in (PLANE_ID, 0):
            w, o, I, (ref, mag, part) = public_rows(ctx, hs, uv, pf, pff, planeid, cp, cpf, sigma, ncal, do_fej)
            assert max(w.values()) <= 1.0
            got = {"Hf": o[0], "Hx": o[1], "res": o[2]}
            for mu in fr.MUTATIONS:
                bad, _, _ = cr.dense_reference(I, ncal, (cp, cpf, cr.SIGMA_C) if planeid else None, True, mu)
                r = max(cr.entry_ratios(got, bad, mag, part).values())
                if r > 1.0:
                    found.setdefault(mu, []).append(r)
        ctx.close()
    # the feature CTA's rows as well
    c = MSCKF_CASES[0]
    ctx, ch, track, b, pts, _ = msckf_setup(c, chi2_table, seed=2)
    raw, _, _ = gram_raw(ctx, b, 0, c["sigma"])
    hs = [ch[k] for k in track]
    for f in range(3):
        w, I, got, _ = check_raw("feature CTA", ctx, raw, f * c["L"], hs, pts[f], pts[f], b["uv"][f * c["L"]:(f + 1) * c["L"]], c["sigma"],
                                 c["do_fej"], c["ncal"])
        _, mag, part = cr.dense_reference(I, c["ncal"], None, True)
        for mu in fr.MUTATIONS[:5]:
            bad, _, _ = cr.dense_reference(I, c["ncal"], None, True, mu)
            r = max(cr.entry_ratios({"Hf": got[0], "Hx": got[1], "res": got[2]}, bad, mag, part).values())
            if r > 1.0:
                found.setdefault(mu + " (feature CTA)", []).append(r)
    ctx.close()
    for mu, v in sorted(found.items()):
        print("wrong model '%s': outside the bound on %d cases (largest error / bound %.2e)" % (mu, len(v), max(v)))
    assert set(fr.MUTATIONS) <= set(found), "not caught: %s" % sorted(set(fr.MUTATIONS) - set(found))
