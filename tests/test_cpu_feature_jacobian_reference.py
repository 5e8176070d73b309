"""The long-double measurement model of tests/feature_jacobian_reference.py pinned to the reference project's behaviour (the CPU oracle's
get_feature_jacobian_full and its anchored form, at the oracle's own normwise precision), to the complex step of the whole chain where
no first estimate differs from its value, and to its power to tell plausible wrong models from the right one.

The cases are built explicitly: clones placed around a feature chosen as (xn, yn, Z) in one clone's camera (centre, on an axis, wide;
near and far), values and first estimates set apart by var_set, EuRoC-like and strongly tangential intrinsics.  They are shared with
tests/test_gpu_feature_jacobian_reference.py."""
import numpy as np
import pytest

import feature_jacobian_reference as fr
import oracle_backend
from ov_plane_b200 import jpl, synth

CAMS = {"euroc": synth.EUROC_CAM.copy(),
        "tangential": np.array([458.654, 457.296, 367.215, 248.375, -0.28340811, 0.07395907, -0.02, 0.015])}
RADII = {"centre": (4e-4, -7e-4), "x axis": (0.3, 0.0), "y axis": (0.0, -0.25), "wide": (0.8, -0.62)}
DEPTHS = {"near": 0.12, "far": 3000.0}
NCAL = {0: (0, 0), 6: (1, 0), 8: (0, 1), 14: (1, 1)}
R_ItoC = jpl.exp_so3(np.array([0.02, -0.01, 0.015]))
P_IinC = np.array([0.02, -0.04, 0.01])


def pose7(R_GtoI, p):
    return np.concatenate([jpl.rot_2_quat(R_GtoI), p])


def geometry(m, radius="centre", depth="near", cam="euroc", seed=0, n_clones=None, order="forward", fej=True, noise=0.5):
    """A feature seen by m clones: (clones [(value7, fej7)] for n_clones clones, track (clone indices of the m measurements, in
    measurement order), p_FinG, p_FinG_fej, uv (m x 2 float32)).  The feature is at (xn, yn, Z) = RADII[radius] x DEPTHS[depth] in
    the camera of the track's middle clone; the other clones step sideways by 0.3 Z / m each and turn by about 0.01 rad.  fej: clone
    first estimates 1e-2 rad and min(5 cm, Z / 5) away from the values, the feature's 1e-3 Z away.  order: 'forward', 'reversed'
    (measurements in reversed clone order) or 'gaps' (every other clone)."""
    rng = np.random.default_rng(seed)
    n_clones = n_clones or (2 * m + 1 if order == "gaps" else m + 1)
    xn, yn = RADII[radius]
    Z = DEPTHS[depth]
    track = list(range(0, 2 * m, 2)) if order == "gaps" else list(range(m))
    assert track[-1] < n_clones
    mid = track[len(track) // 2]
    R0 = jpl.exp_so3(rng.normal(0.0, 0.5, 3))  # R_GtoC of the middle clone
    c0 = rng.normal(0.0, 2.0, 3)
    side = R0.T @ np.array([1.0, 0.4, 0.0])
    pf = c0 + R0.T @ (Z * np.array([xn, yn, 1.0]))
    clones = []
    for k in range(n_clones):
        R_GtoC = jpl.exp_so3(rng.normal(0.0, 0.01, 3)) @ R0 if k != mid else R0
        c = c0 + (k - mid) * (0.3 * Z / m) * side
        R_GtoI = R_ItoC.T @ R_GtoC
        p_IinG = c - R_GtoI.T @ (R_ItoC.T @ P_IinC)
        val = pose7(R_GtoI, p_IinG)
        f = val.copy()
        if fej:
            f[:4] = jpl.quat_left_update(val[:4], rng.normal(0.0, 1e-2 / np.sqrt(3), 3))
            f[4:] = val[4:] + min(0.05, 0.2 * Z) * rng.normal(0.0, 1.0 / np.sqrt(3), 3)
        clones.append((val, f))
    if order == "reversed":
        track = track[::-1]
    pf_fej = pf + (1e-3 * Z * rng.normal(0.0, 1.0, 3) if fej else 0.0)
    uv = []
    for i, k in enumerate(track):
        R_GtoI = jpl.quat_2_Rot(clones[k][0][:4])
        pc = R_ItoC @ (R_GtoI @ (pf - clones[k][0][4:])) + P_IinC
        u, v = jpl.radtan_distort(CAMS[cam], pc[0] / pc[2], pc[1] / pc[2])
        e = rng.normal(0.0, noise, 2) if i % 3 else np.zeros(2)  # every third pixel exact to float32: a residual near zero
        uv.append((u + e[0], v + e[1]))
    return clones, track, pf, pf_fej, np.array(uv, dtype=np.float32)


def plane_for(pf, seed, fej=True, Z=1.0):
    """a closest point cp whose plane passes within 1e-3 Z of pf, and its first estimate"""
    rng = np.random.default_rng(1000 + seed)
    n = rng.normal(0.0, 1.0, 3)
    n /= np.linalg.norm(n)
    if n @ pf < 0:
        n = -n
    d = n @ pf + 1e-3 * Z
    cp = n * d
    return cp, cp + (1e-3 * rng.normal(0.0, 1.0, 3) if fej else 0.0)


def scenario(ncal, n_clones, do_fej, planes=()):
    """a synth state of n_clones clones with the calibration blocks of ncal (the values are overwritten by load_case)"""
    S = synth.make_scenario("tiny_points", seed=0, n_clones=n_clones, F=1, m_min=2, m_max=2, calib_pose=NCAL[ncal][0],
                            calib_intr=NCAL[ncal][1])
    S.options = dict(S.options, do_fej=do_fej, sigma_constraint=SIGMA_C)
    S.planes = list(planes)
    if planes:  # planes in the state: their rows / columns after the clones
        N = S.N + 3 * len(planes)
        P0 = np.eye(N) * 1e-4
        P0[:S.N, :S.N] = S.P0
        S.P0, S.N = P0, N
    return S


def load_case(be, S, clones, cam):
    """var_set the explicit geometry into a backend loaded with S: clone values and first estimates, extrinsics, intrinsics"""
    ch = synth.load_scenario_into(be, S)
    for h, (v, f) in zip(ch, clones):
        be.var_set(h, v, f)
    be.var_set(be.handle_calib(), pose7(R_ItoC, P_IinC), pose7(R_ItoC, P_IinC))
    be.var_set(be.handle_intrinsics(), CAMS[cam], CAMS[cam])
    return ch


def inputs(be, handles, pf, pf_fej, uv, sigma_pix, do_fej):
    cv = np.array([be.var_get(int(h))[0] for h in handles])
    cf = np.array([be.var_get(int(h))[1] for h in handles])
    return fr.Inputs(cv, cf, be.var_get(be.handle_calib())[0], be.var_get(be.handle_intrinsics())[0], pf, pf_fej, uv, sigma_pix, do_fej)


def dense_reference(I, ncal, plane=None, plane_in_state=False, mutate=None):
    """(H_f, H_x, res, magnitudes of each, part name of each H_x column / H_f column / row) in the reference's dense layout:
    H_x = [extrinsics 6 | intrinsics 8 | 6 per measurement's clone | cp 3 when the plane is in the state], bearing rows, then one
    point-on-plane row per measurement (plane = (cp, cp_fej, sigma_c)); a plane not in the state puts H_cp in H_f's columns 3..5."""
    pose, intr = NCAL[ncal]
    B, M = fr.bearing_rows(I, mutate), fr.bearing_mags(I)
    m = I.m
    rows = 3 * m if plane is not None else 2 * m
    hfc = 6 if (plane is not None and not plane_in_state) else 3
    hxc = ncal + 6 * m + (3 if plane is not None and plane_in_state else 0)
    out = {k: np.zeros(s, dtype=fr.LD) for k, s in (("Hf", (rows, hfc)), ("Hx", (rows, hxc)), ("res", rows))}
    mag = {k: np.zeros_like(v) for k, v in out.items()}
    part = {"Hf": np.full((rows, hfc), "Hf", dtype=object), "Hx": np.full((rows, hxc), "clone", dtype=object),
            "res": np.full(rows, "res", dtype=object)}
    for src, (key, c0, c1, nm) in (("extrinsics", ("Hx", 0, 6 * pose, "extrinsics")), ("intrinsics", ("Hx", 6 * pose, ncal, "intrinsics"))):
        if c1 > c0:
            out["Hx"][:2 * m, c0:c1] = B[src].reshape(2 * m, -1)
            mag["Hx"][:2 * m, c0:c1] = M[src].reshape(2 * m, -1)
            part["Hx"][:, c0:c1] = nm
    for k in range(m):
        out["Hx"][2 * k:2 * k + 2, ncal + 6 * k:ncal + 6 * k + 6] = B["clone"][k]
        mag["Hx"][2 * k:2 * k + 2, ncal + 6 * k:ncal + 6 * k + 6] = M["clone"][k]
    out["Hf"][:2 * m, :3], mag["Hf"][:2 * m, :3] = B["Hf"].reshape(2 * m, 3), M["Hf"].reshape(2 * m, 3)
    out["res"][:2 * m], mag["res"][:2 * m] = B["res"].reshape(-1), M["res"].reshape(-1)
    if plane is not None:
        cp, cpf, sc = plane
        r, hf, hcp, pm = fr.plane_row(I.pf, I.pff, cp, cpf, sc, I.do_fej, mutate)
        out["Hf"][2 * m:, :3], mag["Hf"][2 * m:, :3] = hf, pm["Hf"]
        out["res"][2 * m:], mag["res"][2 * m:] = r, pm["res"]
        part["Hf"][2 * m:, :] = "plane"
        part["res"][2 * m:] = "plane"
        if plane_in_state:
            out["Hx"][2 * m:, -3:], mag["Hx"][2 * m:, -3:] = hcp, pm["Hcp"]
            part["Hx"][2 * m:, -3:] = "plane"
        else:
            out["Hf"][2 * m:, 3:], mag["Hf"][2 * m:, 3:] = hcp, pm["Hcp"]
    return out, mag, part


def entry_ratios(got, ref, mag, part):
    """{part: worst |got - ref| / (C u mag)} over H_f, H_x and res"""
    w = {}
    for key in ("Hf", "Hx", "res"):
        for p in set(part[key].ravel().tolist()):
            sel = part[key] == p
            w[p] = max(w.get(p, 0.0), fr.worst(np.asarray(got[key])[sel], ref[key][sel], mag[key][sel], p))
    return w


def relerr(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


# (radius, depth, cam, m, do_fej, ncal, plane: None / "in" / "out", order, sigma_pix)
ORACLE_CASES = [("centre", "near", "euroc", 3, 1, 14, None, "forward", 1.0), ("x axis", "far", "tangential", 5, 1, 6, "in", "reversed", 0.37),
                ("y axis", "near", "tangential", 4, 0, 8, "out", "gaps", 4.0), ("wide", "far", "euroc", 7, 1, 0, "out", "forward", 1.0),
                ("wide", "near", "tangential", 6, 1, 14, "in", "gaps", 1.0), ("centre", "far", "tangential", 2, 0, 14, "in", "forward", 0.37),
                ("wide", "near", "euroc", 9, 0, 6, None, "reversed", 4.0), ("x axis", "near", "euroc", 3, 1, 8, None, "forward", 1.0)]
SIGMA_C = 0.004  # a non-default sigma_constraint


def oracle_case(case, seed=0, mutate=None):
    """the oracle's get_feature_jacobian_full of one case and the reference in its layout"""
    radius, depth, cam, m, do_fej, ncal, plane, order, sp = case
    clones, track, pf, pff, uv = geometry(m, radius, depth, cam, seed=seed, order=order)
    cp = cpf = None
    planes = ()
    if plane is not None:
        cp, cpf = plane_for(pf, seed, Z=DEPTHS[depth])
        if plane == "in":
            planes = ((7, cp, cpf),)
    S = scenario(ncal, len(clones), do_fej, planes)
    orc = oracle_backend.OracleContext(S.options)
    ch = load_case(orc, S, clones, cam)
    hs = [ch[k] for k in track]
    o = orc.feature_jacobian_full(hs, uv, pf, pff, 7 if plane else 0, cp, cpf, sp, SIGMA_C)
    I = inputs(orc, hs, pf, pff, uv, sp, do_fej)
    ref = dense_reference(I, ncal, (cp, cpf, SIGMA_C) if plane else None, plane == "in", mutate)
    want = ([orc.handle_calib()] if NCAL[ncal][0] else []) + ([orc.handle_intrinsics()] if NCAL[ncal][1] else []) + hs
    want += [orc.plane_handle(7)] if plane == "in" else []
    assert o[3] == want, (o[3], want)
    orc.close()
    return o, ref


@pytest.mark.parametrize("case", ORACLE_CASES, ids=["%s-%s-%s-m%d-fej%d-ncal%d-plane_%s-%s-sigma%g" % c for c in ORACLE_CASES])
def test_reference_matches_the_oracle(case):
    fr.require_long_double()
    o, (ref, mag, part) = oracle_case(case)
    for k, (got, key) in enumerate(zip(o[:3], ("Hf", "Hx", "res"))):
        assert got.shape == ref[key].shape, (key, got.shape, ref[key].shape)
        assert relerr(got, ref[key]) < 1e-11, "%s: %.3e" % (key, relerr(got, ref[key]))
    w = entry_ratios({"Hf": o[0], "Hx": o[1], "res": o[2]}, ref, mag, part)
    print("oracle rows within the entrywise bound: worst error / bound %s" % ", ".join("%s %.2e" % kv for kv in sorted(w.items())))


@pytest.mark.parametrize("rep", range(6))
@pytest.mark.parametrize("do_fej", [0, 1])
def test_representations_match_the_oracle(rep, do_fej):
    fr.require_long_double()
    m = 5
    for anchor_in in ((True, False) if rep >= 2 else (None,)):
        clones, track, pG, pGf, uv = geometry(m, "wide", "near", "tangential", seed=rep, n_clones=m + 2, order="reversed")
        S = scenario(14, len(clones), do_fej)
        orc = oracle_backend.OracleContext(S.options)
        ch = load_case(orc, S, clones, "tangential")
        hs = [ch[k] for k in track]
        anchor = -1 if rep < 2 else (hs[1] if anchor_in else ch[-1])
        cal = orc.var_get(orc.handle_calib())[0]
        if rep >= 2:
            av, af = orc.var_get(anchor)
            pF = np.asarray(fr.global_to_anchor(fr.ld(av), fr.ld(cal), fr.ld(pG)), dtype=np.float64)
            pFf = pF
        else:
            pF, pFf = pG, pGf
        o = orc.feature_jacobian_full_rep(hs, uv, rep, anchor, pF, pFf, 1.0)
        ref = rep_reference(orc, hs, uv, rep, anchor, pF, pFf, 1.0, do_fej, 14)
        assert o[3] == ref[3], (o[3], ref[3])
        for got, want in zip(o[:3], ref[:3]):
            assert got.shape == want.shape and relerr(got, want) < 1e-11, (rep, anchor_in, relerr(got, want))
        orc.close()


def rep_reference(be, hs, uv, rep, anchor, pF, pFf, sigma_pix, do_fej, ncal, mags=False):
    """(H_f, H_x, res, x_order) of get_feature_jacobian_full with a representation: the bearing rows at the global point the
    representation stands for, chained with d p_FinG / d (lambda, anchor, extrinsics).  mags: also the magnitudes of the three, the
    bearing rows' magnitudes through |d p_FinG / d .|"""
    cal = be.var_get(be.handle_calib())[0]
    av, af = be.var_get(anchor) if rep >= 2 else (None, None)
    pG, pGf, L, Ha, Hc = fr.representation_jacobians(rep, do_fej, pF, pFf, av, af, cal)
    I = inputs(be, hs, np.asarray(pG, dtype=np.float64), np.asarray(pGf, dtype=np.float64), uv, sigma_pix, do_fej)
    ref, mag, _ = dense_reference(I, ncal)
    raw, mraw = ref["Hf"], mag["Hf"]
    Hf, mHf = raw @ L, mraw @ abs(L)
    Hx, mHx = ref["Hx"], mag["Hx"]
    order = ([be.handle_calib()] if NCAL[ncal][0] else []) + ([be.handle_intrinsics()] if NCAL[ncal][1] else []) + list(hs)
    if rep >= 2:
        if anchor not in hs:
            Hx = np.hstack([Hx, np.zeros((Hx.shape[0], 6), dtype=fr.LD)])
            mHx = np.hstack([mHx, np.zeros((Hx.shape[0], 6), dtype=fr.LD)])
            order.append(anchor)
        a = ncal + 6 * list(hs).index(anchor) if anchor in hs else Hx.shape[1] - 6
        Hx[:, a:a + 6] += raw @ Ha
        mHx[:, a:a + 6] += mraw @ abs(Ha)
        if NCAL[ncal][0]:
            Hx[:, 0:6] += raw @ Hc
            mHx[:, 0:6] += mraw @ abs(Hc)
    if mags:
        return Hf, Hx, ref["res"], order, (mHf, mHx, mag["res"])
    return Hf, Hx, ref["res"], order


def test_factors_equal_the_whole_chain():
    """the FEJ composition with nothing to first-estimate is the derivative of the whole measurement function"""
    fr.require_long_double()
    for radius in RADII:
        for depth in DEPTHS:
            for fej, do_fej in ((True, 0), (False, 1)):
                clones, track, pf, pff, uv = geometry(4, radius, depth, "tangential", seed=3, fej=fej)
                cv = np.array([clones[k][0] for k in track])
                cf = np.array([clones[k][1] for k in track])
                cam = CAMS["tangential"]
                I = fr.Inputs(cv, cf, pose7(R_ItoC, P_IinC), cam, pf, pff, uv, 0.37, do_fej)
                a, b, mag = fr.bearing_rows(I), fr.whole_chain(I), fr.bearing_mags(I)
                for p in ("res", "Hf", "clone", "extrinsics", "intrinsics"):
                    err = abs(a[p] - b[p])
                    # long-double rounding of the two evaluations: far inside the double-precision bound
                    assert (err <= 2.0 ** -56 * mag[p]).all(), (radius, depth, do_fej, p, float((err / mag[p]).max()))


def caught(ref_good, ref_bad, got, mag, part):
    """True when the wrong model lies outside the bound from rows the right model accepts"""
    ok = entry_ratios(got, ref_good, mag, part)
    bad = entry_ratios(got, ref_bad, mag, part)
    return max(ok.values()) <= 1.0 and max(bad.values()) > 1.0


MUTATION_CASES = ORACLE_CASES


def test_wrong_models_lie_outside_the_bound():
    """every plausible wrong model lies outside the entrywise bound from the oracle's rows on at least one case"""
    fr.require_long_double()
    found = {}
    for case in MUTATION_CASES:
        o, (ref, mag, part) = oracle_case(case)
        got = {"Hf": o[0], "Hx": o[1], "res": o[2]}
        for mu in fr.MUTATIONS:
            bad, _, _ = oracle_case(case, mutate=mu)[1]
            bad_ratio = max(entry_ratios(got, bad, mag, part).values())
            if bad_ratio > 1.0:
                found.setdefault(mu, []).append(bad_ratio)
    for mu in fr.MUTATIONS:
        print("wrong model '%s': outside the bound on %d of %d cases (largest error / bound %.2e)" % (
            mu, len(found.get(mu, [])), len(MUTATION_CASES), max(found.get(mu, [0.0]))))
    assert set(found) == set(fr.MUTATIONS), "not caught: %s" % sorted(set(fr.MUTATIONS) - set(found))
