"""SLAM landmarks in the MSCKF update of planes that are not in the state (use_plane_constraint_slamu, UpdaterMSCKF.cpp:231-254,
454-560, 626-639), through ovp_msckf_update_landmarks.

The reference is the branch restated on the oracle's own primitives: feature_jacobian_full + the plane nullspace projection per batch
feature, one point-on-plane row per member with its landmark as state columns, the compression, the projection of the plane columns,
the chi2 gate and StateHelper::EKFUpdate.  The compression keeps the range of the stacked x Jacobian.  A member's block has rank 1,
so each member leaves two columns without information; the reference's Givens compression keeps two rows per member from outside that
range (which ones depends on its rotation order), the library drops them as it drops the gauge rows (DESIGN §1)."""
import ctypes as C

import numpy as np
import pytest

from ov_plane_b200 import api, synth
from test_gpu_parity import compare_states

pytestmark = pytest.mark.gpu

LM0 = 1000000  # featids of the added landmarks


def _pair(S, chi2, debug=False):
    import oracle_backend
    ctx = api.Context(S.options, device=0, max_state=max(128, S.N + 64), max_meas_rows=60000, debug=debug)
    ctx.set_chi2_table(chi2)
    orc = oracle_backend.OracleContext(S.options)
    orc.set_chi2_table(chi2)
    return ctx, orc, synth.load_scenario_into(ctx, S), synth.load_scenario_into(orc, S)


def _add_landmarks(S, planes, per_plane, rng, off=0.004):
    """per_plane[pid] landmarks on (near) plane pid, near the plane's features; their 3x3 prior blocks are appended to P0.  Returns
    the (featid, planeid) list."""
    cps = {pid: np.asarray(cp) for pid, cp, _ in planes}
    mem = []
    for pid, k in per_plane.items():
        cp = cps[pid]
        d = np.linalg.norm(cp)
        n = cp / d
        pts = S.p_FinG[S.planeid == pid]
        for i in range(k):
            p = pts[i % len(pts)] + 0.05 * rng.randn(3)
            p = p - (n @ p - d) * n + off * rng.randn() * n
            fid = LM0 + 100 * pid + i
            S.slam.append((fid, p, p + 1e-3 * rng.randn(3)))
            mem.append((fid, pid))
    L = 3 * len(mem)
    P0 = np.zeros((S.N + L, S.N + L))
    P0[:S.N, :S.N] = S.P0
    A = 0.01 * rng.randn(L, L)
    P0[S.N:, S.N:] = A @ A.T + 1e-4 * np.eye(L)
    S.P0, S.N = P0, S.N + L
    return mem


def _case(name, seed, chi2, per_plane, do_fej=1, debug=False, off=0.004, in_state=False):
    S = synth.make_scenario(name, seed=seed)
    S.options["do_fej"] = do_fej
    planes = list(S.planes) if in_state else synth.drop_planes_from_state(S)
    mem = _add_landmarks(S, planes, per_plane, np.random.RandomState(100 + seed), off)
    ctx, orc, chg, cho = _pair(S, chi2, debug)
    return S, planes, mem, ctx, orc, chg, cho


def _plane_batch(S, ch, planes, pid, nfeat=None):
    sel = np.nonzero(S.planeid == pid)[0]
    if nfeat is not None:
        sel = sel[:nfeat]
    b = synth.feature_batch(S, ch, sel)
    cp = [p[1] for p in planes if p[0] == pid][0]
    b["plane_ids"] = np.array([pid], dtype=np.int64)
    b["plane_cp"] = np.ascontiguousarray([cp], dtype=np.float64)
    return b


def _mem_arrays(mem):
    return np.array([m[0] for m in mem], dtype=np.int64), np.array([m[1] for m in mem], dtype=np.int64)


def reference_plane_update(orc, S, bo, pid, members, chi2, mult=1.0, tol=1e-9):
    """The plane branch with landmark members on the oracle: returns (passed, chi2, dof); on a pass the update is applied.  Also checks that
    chi2 equals the well-defined part of the reference's Givens path (its chi2 less the share on rows without Jacobian)."""
    sig_c, do_fej = S.options["sigma_constraint"], S.options["do_fej"]
    cp = np.asarray(bo["plane_cp"][0])
    blocks = []
    for f in range(bo["F"]):
        a, b = bo["meas_offset"][f], bo["meas_offset"][f + 1]
        Hf, Hx, r, xo = orc.feature_jacobian_full(bo["meas_clone"][a:b], bo["uv"][a:b], bo["p_FinG"][f], bo["p_FinG"][f], pid, cp, cp, 1.0, sig_c)
        Hx, Hcp, r = orc.nullspace_project_inplace(Hf[:, :3], Hx, r, Hf[:, 3:])
        blocks.append((xo, Hx, Hcp, r))
    for fid in members:  # the oracle's get_feature_jacobian_full of a feature without measurements: one row (UpdaterHelper.cpp:313-315)
        h = orc.slam_handle(fid)
        v, fe = orc.var_get(h)
        Hf, _, r, _ = orc.feature_jacobian_full([], np.zeros((0, 2)), v, fe, pid, cp, cp, 1.0, sig_c)
        assert Hf.shape == (1, 6)
        blocks.append(([h], Hf[:, :3], Hf[:, 3:], r))
    handles = []
    for xo, _, _, _ in blocks:
        handles += [h for h in xo if h not in handles]
    off = np.cumsum([0] + [orc.var_size(h) for h in handles])
    col = dict(zip(handles, off[:-1]))
    rows = sum(len(bl[3]) for bl in blocks)
    H, C, z = np.zeros((rows, off[-1])), np.zeros((rows, 3)), np.zeros(rows)
    i = 0
    for xo, Hx, Hcp, r in blocks:
        k = 0
        for h in xo:
            s = orc.var_size(h)
            H[i:i + len(r), col[h]:col[h] + s] = Hx[:, k:k + s]
            k += s
        C[i:i + len(r)], z[i:i + len(r)] = Hcp, r
        i += len(r)
    ncx = H.shape[1]
    # the reference's own numbers beside: its Givens compression, the plane projection, chi2 and the part carried by rows whose Jacobian
    # part is zero (the GaugeProbe split of test_gpu_parity.oracle_msckf_update)
    Hg, Cg, zg = orc.measurement_compress_inplace(H, z, C)
    Hg, zg = orc.nullspace_project_inplace(Cg, Hg, zg)
    Pm = orc.get_marginal_covariance(handles)
    chi_ref = float(zg @ np.linalg.solve(Hg @ Pm @ Hg.T + np.eye(len(zg)), zg))
    Ug, sg, _ = np.linalg.svd(Hg, full_matrices=True)
    zn = Ug[:, int((sg > 1e-7 * sg[0]).sum()):].T @ zg
    chi_wd = chi_ref - float(zn @ zn)
    print("reference Givens path: chi2 %.6f, of it on rows without Jacobian %.6f, well-defined %.6f" % (chi_ref, zn @ zn, chi_wd))
    if rows > ncx:  # UpdaterPlane::measurement_compress_inplace keeps the range of H (see the module docstring)
        U, sv, _ = np.linalg.svd(H, full_matrices=False)
        Q = U[:, :int((sv > tol * sv[0]).sum())]
        H, C, z = Q.T @ H, Q.T @ C, Q.T @ z
    U2 = np.linalg.svd(C, full_matrices=True)[0][:, 3:]
    H, z = U2.T @ H, U2.T @ z
    dof = min(rows, ncx) - 3
    chi = float(z @ np.linalg.solve(H @ Pm @ H.T + np.eye(len(z)), z))
    assert abs(chi / chi_wd - 1) < 1e-6, (chi, chi_wd)
    passed = chi <= mult * chi2[dof]
    if passed:
        orc.ekf_update(handles, H, z)
    return passed, chi, dof


def _check_landmarks(ctx, orc, mem, tol=1e-6):
    for fid, _ in mem:
        vg, vo = ctx.var_get(ctx.slam_handle(fid))[0], orc.var_get(orc.slam_handle(fid))[0]
        assert np.abs(vg - vo).max() < tol * max(1.0, np.abs(vo).max()), fid


@pytest.mark.parametrize("name,seed,per,do_fej,dense", [
    ("small_planes", 0, 1, 1, 0), ("small_planes", 2, 6, 1, 0), ("small_planes", 3, 6, 0, 0), ("small_planes", 0, 6, 1, 1),
    ("tiny_planes", 1, 3, 0, 1)])
def test_members_against_reference(name, seed, per, do_fej, dense, chi2_table):
    S, planes, mem, ctx, orc, chg, cho = _case(name, seed, chi2_table, {p[0]: per for p in S_planes(name, seed)}, do_fej, debug=True)
    ctx._ck(ctx.lib.ovp_debug_force_dense_features(ctx.h, dense))  # 1: the one-CTA-per-feature kernel and the dense Gram
    pid = planes[0][0]
    bg, bo = _plane_batch(S, chg, planes, pid), _plane_batch(S, cho, planes, pid)
    fids, pids = _mem_arrays(mem)
    g = ctx.msckf_update_landmarks(bg, fids, pids)
    passed, chi, dof = reference_plane_update(orc, S, bo, pid, [f for f, p in mem if p == pid], chi2_table)
    print(name, seed, per, do_fej, dense, "plane", g["plane_status"], passed, "chi2", g["plane_chi2"], chi, "dof", dof)
    assert passed and g["plane_status"][0] == 1
    assert np.all(g["feat_status"] == 2)
    assert abs(g["plane_chi2"][0] / chi - 1) < 1e-5
    compare_states(ctx, orc, S, chg, cho)
    _check_landmarks(ctx, orc, mem)
    for fid, p in mem:  # members of the other planes (not in the batch) are left alone
        assert ctx.slam_plane_of(fid) == (pid if p == pid else -1)


def S_planes(name, seed):
    return synth.make_scenario(name, seed=seed).planes


def test_member_completes_four_feature_rule(chi2_table):
    """Three batch features and one member: the plane qualifies only with its member (UpdaterMSCKF.cpp:396)."""
    S, planes, mem, ctx, orc, chg, cho = _case("small_planes", 0, chi2_table, {1: 1})
    bg, bo = _plane_batch(S, chg, planes, 1, 3), _plane_batch(S, cho, planes, 1, 3)
    fids, pids = _mem_arrays(mem)
    g0 = ctx.msckf_update(bg)  # without the member the plane is not visited
    assert g0["plane_status"][0] == -1
    S2, planes2, mem2, ctx2, orc2, chg2, cho2 = _case("small_planes", 0, chi2_table, {1: 1})
    g = ctx2.msckf_update_landmarks(_plane_batch(S2, chg2, planes2, 1, 3), fids, pids)
    passed, chi, _ = reference_plane_update(orc2, S2, _plane_batch(S2, cho2, planes2, 1, 3), 1, [mem2[0][0]], chi2_table)
    assert g["plane_status"][0] == int(passed) == 1
    assert abs(g["plane_chi2"][0] / chi - 1) < 1e-5
    compare_states(ctx2, orc2, S2, chg2, cho2)
    _check_landmarks(ctx2, orc2, mem2)
    assert ctx2.slam_plane_of(mem2[0][0]) == 1


def _bitwise_same(a, b):
    assert np.array_equal(a.cov(), b.cov())
    assert a.variable_order() == b.variable_order()
    for h in a.variable_order():
        assert np.array_equal(a.var_get(h)[0], b.var_get(h)[0])


def test_ignored_members_are_bit_identical_to_the_plain_update(chi2_table):
    """Members only on planes without batch features, on in-state planes, or with _features_SLAM_to_PLANE == 0 change nothing."""
    # a plane whose only features are members: skipped
    S, planes, mem, ctx, orc, chg, cho = _case("small_planes", 2, chi2_table, {2: 5})
    S2, _, _, ctx2, _, chg2, _ = _case("small_planes", 2, chi2_table, {2: 5})
    b = _plane_batch(S, chg, planes, 1)
    b["plane_ids"] = np.array([1, 2], dtype=np.int64)
    b["plane_cp"] = np.ascontiguousarray([planes[0][1], planes[1][1]], dtype=np.float64)
    b2 = dict(_plane_batch(S2, chg2, planes, 1), plane_ids=b["plane_ids"], plane_cp=b["plane_cp"])
    fids, pids = _mem_arrays(mem)
    g = ctx.msckf_update_landmarks(b, fids, pids)
    g2 = ctx2.msckf_update(b2)
    assert g["plane_status"][1] == -1 and np.array_equal(g["plane_status"], g2["plane_status"])
    _bitwise_same(ctx, ctx2)
    assert all(ctx.slam_plane_of(f) == -1 for f in fids)
    # in-state planes: left to UpdaterSLAM
    S, planes, mem, ctx, orc, chg, cho = _case("small_planes", 0, chi2_table, {1: 4}, in_state=True)
    S2, _, _, ctx2, _, chg2, _ = _case("small_planes", 0, chi2_table, {1: 4}, in_state=True)
    fids, pids = _mem_arrays(mem)
    g = ctx.msckf_update_landmarks(synth.feature_batch(S, chg), fids, pids)
    g2 = ctx2.msckf_update(synth.feature_batch(S2, chg2))
    assert np.array_equal(g["plane_status"], g2["plane_status"]) and np.array_equal(g["feat_status"], g2["feat_status"])
    _bitwise_same(ctx, ctx2)
    assert all(ctx.slam_plane_of(f) == -1 for f in fids)


def test_failing_plane_detaches_members(chi2_table):
    """Members far off the plane make it fail its gate: members -> 0, the batch features go to the point update, and a later call
    ignores the detached members (bit-identical to the plain update)."""
    S, planes, mem, ctx, orc, chg, cho = _case("small_planes", 0, chi2_table, {1: 4}, off=0.5)
    bg, bo = _plane_batch(S, chg, planes, 1), _plane_batch(S, cho, planes, 1)
    fids, pids = _mem_arrays(mem)
    g = ctx.msckf_update_landmarks(bg, fids, pids)
    assert g["plane_status"][0] == 0
    assert all(ctx.slam_plane_of(f) == 0 for f in fids)
    bo_pts = dict(bo, plane_ids=np.zeros(0, dtype=np.int64), plane_cp=np.zeros((0, 3)))
    o = orc.msckf_update(bo_pts)
    assert np.array_equal(g["feat_status"], o["feat_status"])
    compare_states(ctx, orc, S, chg, cho)
    # detached: a repeat is the plain update
    S2, planes2, _, ctx2, _, chg2, _ = _case("small_planes", 0, chi2_table, {1: 4}, off=0.5)
    ctx2.msckf_update_landmarks(_plane_batch(S2, chg2, planes2, 1), fids, pids)
    g1 = ctx.msckf_update_landmarks(bg, fids, pids)
    g2 = ctx2.msckf_update(_plane_batch(S2, chg2, planes2, 1))
    assert np.array_equal(g1["plane_status"], g2["plane_status"])
    _bitwise_same(ctx, ctx2)


def test_refusals_leave_the_state_untouched(chi2_table):
    S, planes, mem, ctx, orc, chg, cho = _case("small_planes", 0, chi2_table, {1: 3})
    bg = _plane_batch(S, chg, planes, 1)
    fids, pids = _mem_arrays(mem)
    P0, v0 = ctx.cov(), [ctx.var_get(h)[0] for h in ctx.variable_order()]
    cases = [(np.r_[fids, fids[:1]], np.r_[pids, pids[:1]]),             # listed twice
             (np.r_[fids, bg["featid"][:1]], np.r_[pids, [1]])]          # also a feature of the batch
    for f, p in cases:
        with pytest.raises(api.OvpError) as e:
            ctx.msckf_update_landmarks(bg, f, p)
        assert "landmark" in str(e.value)
    ctx.slam_set_representation(int(fids[0]), 1, -1)  # not GLOBAL_3D
    with pytest.raises(api.OvpError) as e:
        ctx.msckf_update_landmarks(bg, fids, pids)
    assert "GLOBAL_3D" in str(e.value)
    assert np.array_equal(ctx.cov(), P0)
    assert all(np.array_equal(ctx.var_get(h)[0], v) for h, v in zip(ctx.variable_order(), v0))
    assert all(ctx.slam_plane_of(f) == -1 for f in fids)


def test_prepared_replay_equals_one_shot(chi2_table):
    """prepare -> launch -> finish, then new measurement values through the same plan, equals two one-shot calls."""
    runs = []
    for split in (True, False):
        S, planes, mem, ctx, orc, chg, cho = _case("small_planes", 2, chi2_table, {1: 5})
        fids, pids = _mem_arrays(mem)
        b = _plane_batch(S, chg, planes, 1)
        b2 = dict(b, uv=np.ascontiguousarray(b["uv"] + np.float32(0.3)))
        out = []
        for bb in (b, b2):
            if split:
                ctx.msckf_prepare_landmarks(bb, fids, pids)
                ctx.msckf_launch()
                out.append(ctx.msckf_finish())
            else:
                out.append(ctx.msckf_update_landmarks(bb, fids, pids))
        runs.append((ctx, out, [ctx.slam_plane_of(f) for f in fids]))
    (c1, o1, s1), (c2, o2, s2) = runs
    for a, b in zip(o1, o2):
        assert np.array_equal(a["plane_status"], b["plane_status"]) and np.array_equal(a["plane_chi2"], b["plane_chi2"])
    assert s1 == s2
    _bitwise_same(c1, c2)


def test_empty_list_is_bit_identical_on_cfg3(chi2_table):
    out = []
    for with_list in (True, False):
        S = synth.make_scenario("cfg3_n512_f600_p8", seed=0)
        ctx, orc, chg, cho = _pair(S, chi2_table)
        b = synth.feature_batch(S, chg)
        g = ctx.msckf_update_landmarks(b, [], []) if with_list else ctx.msckf_update(b)
        out.append((ctx, g))
    (c1, g1), (c2, g2) = out
    for k in ("feat_status", "feat_chi2", "plane_status", "plane_chi2"):
        assert np.array_equal(g1[k], g2[k], equal_nan=True) if g1[k].dtype.kind == "f" else np.array_equal(g1[k], g2[k])
    assert g1["hx_order"] == g2["hx_order"]
    _bitwise_same(c1, c2)


def _gram(ctx, b, fids, pids):
    """ovp_debug_msckf_gram_landmarks: G of the batch's first plan, with its members' rows"""
    fb, keep = api.Context._batch_struct(b)
    lm, keep_lm = api.Context._landmarks_struct(fids, pids)
    uo = api.UpdaterOptions(1.0, 1.0)
    F, gcap = fb.F, ctx.cov_rows() + 4
    G, info, cols = np.zeros(gcap * gcap), np.zeros(8, dtype=np.int32), np.zeros(gcap, dtype=np.int32)
    sel, fs, fc = np.zeros(F, dtype=np.int32), np.zeros(F, dtype=np.int32), np.zeros(F)
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    ctx._ck(ctx.lib.ovp_debug_msckf_gram_landmarks(ctx.h, C.byref(fb), C.byref(lm), C.byref(uo), gcap, P(G), P(info), P(cols), P(sel), P(fs),
                                                   P(fc), None))
    nc1, ncx = int(info[0]), int(info[2])
    return G[:nc1 * nc1].reshape((nc1, nc1), order="F").copy(), ncx, cols[:ncx].copy()


def _zero_pivots(G, npiv, tol=1e-11):
    """the zero-pivot rule of the Gram factorisation (chol_fused_kernel) on the host: a pivot <= tol x its column's original diagonal is
    zeroed with its column"""
    A = np.tril(G).astype(np.longdouble)
    A = A + np.tril(A, -1).T
    d0, zero = np.diag(A).copy(), []
    for j in range(npiv):
        if not A[j, j] > tol * d0[j]:
            zero.append(j)
            A[j:, j] = 0.0
            A[j, j:] = 0.0
            continue
        A[j:, j] /= np.sqrt(A[j, j])
        A[j + 1:, j + 1:] -= np.outer(A[j + 1:, j], A[j + 1:, j])
    return zero


@pytest.mark.parametrize("dense", [0, 1])
def test_gram_with_members_two_zero_pivots_each_and_bit_identical(dense, chi2_table):
    """The kernel's G with members: rows/columns of every member block as the oracle's member row gives them, exactly two zero pivots
    per member (rank-1 block), and the same bits on a second run."""
    S, planes, mem, ctx, orc, chg, cho = _case("small_planes", 2, chi2_table, {1: 5}, debug=True)
    ctx._ck(ctx.lib.ovp_debug_force_dense_features(ctx.h, dense))
    b = _plane_batch(S, chg, planes, 1)
    fids, pids = _mem_arrays(mem)
    G0, ncx0, _ = _gram(ctx, b, [], [])
    G, ncx, cols = _gram(ctx, b, fids, pids)
    G2, _, _ = _gram(ctx, b, fids, pids)
    assert np.array_equal(G, G2)
    L = len(mem)
    assert ncx == ncx0 + 3 * L
    assert np.array_equal(G[:ncx0, :ncx0], G0[:ncx0, :ncx0])  # the batch features' part is untouched
    # member rows from the oracle (same state values on both sides)
    cp = np.asarray(b["plane_cp"][0])
    rows = []
    for k, fid in enumerate(fids):
        v, fe = orc.var_get(orc.slam_handle(int(fid)))
        Hf, _, r, _ = orc.feature_jacobian_full([], np.zeros((0, 2)), v, fe, 1, cp, cp, 1.0, S.options["sigma_constraint"])
        assert list(cols[ncx0 + 3 * k:ncx0 + 3 * k + 3]) == [ctx.var_id(ctx.slam_handle(int(fid))) + j for j in range(3)]
        rows.append(np.r_[Hf[0], r])
    R = np.array(rows)  # per member: H_f(3), H_cp(3), r
    Gl = G[ncx0:ncx, ncx0:ncx]
    for k in range(L):
        blk = Gl[3 * k:3 * k + 3, 3 * k:3 * k + 3]
        ref = np.outer(R[k, :3], R[k, :3])
        assert np.abs(np.tril(blk) - np.tril(ref)).max() <= 1e-12 * np.abs(ref).max()
        assert np.abs(G[ncx:, ncx0 + 3 * k:ncx0 + 3 * k + 3] - np.outer(R[k, 3:], R[k, :3])).max() <= 1e-12 * np.abs(R[k]).max() ** 2
    dense_ref = np.tril(G0[ncx0:, ncx0:] + R[:, 3:].T @ R[:, 3:])
    assert np.abs(np.tril(G[ncx:, ncx:]) - dense_ref).max() <= 1e-12 * np.abs(dense_ref).max()
    assert np.abs(G[ncx0:ncx, :ncx0]).max() == 0.0 and np.abs(np.triu(G, 1)).max() == 0.0
    z = _zero_pivots(G, ncx)
    z0 = _zero_pivots(G0, ncx0)
    assert [j for j in z if j < ncx0] == z0
    for k in range(L):
        assert len([j for j in z if ncx0 + 3 * k <= j < ncx0 + 3 * k + 3]) == 2, (k, z)


def test_members_on_cfg3(chi2_table):
    """A cfg3-sized state (N = 512 + members) with two out-of-state planes carrying landmarks."""
    S, planes, mem, ctx, orc, chg, cho = _case("cfg3_n512_f600_p8", 0, chi2_table, {1: 8, 2: 8})
    fids, pids = _mem_arrays(mem)
    for pid in (1, 2):
        bg, bo = _plane_batch(S, chg, planes, pid), _plane_batch(S, cho, planes, pid)
        g = ctx.msckf_update_landmarks(bg, fids, pids)
        passed, chi, dof = reference_plane_update(orc, S, bo, pid, [f for f, p in mem if p == pid], chi2_table)
        print("cfg3 plane", pid, g["plane_status"], passed, g["plane_chi2"], chi, dof)
        assert g["plane_status"][0] == int(passed) == 1
        assert abs(g["plane_chi2"][0] / chi - 1) < 1e-5
        compare_states(ctx, orc, S, chg, cho)
        _check_landmarks(ctx, orc, mem)
    assert all(ctx.slam_plane_of(f) == p for f, p in mem)


def test_optimize_plane_with_measurement_free_features(chi2_table):
    """Landmark members enter the plane refinement as features without measurements (ovp_optimize_plane, PlaneFitting.cpp:274-277): half of
    every plane's features here, against the oracle."""
    import planefit_cases
    from conftest import make_pair
    S = synth.make_scenario("small_planes", seed=2)
    ctx, orc, chg, cho = make_pair(S, chi2_table)
    pr = planefit_cases.refine_problem(S, chg, seed=2, consistent=True, noise=0.006, slam_share=0.5)
    mo = pr["meas_offset"]
    assert (np.diff(mo) == 0).sum() > 10
    fx = np.zeros(len(pr["feat_offset"]) - 1, dtype=np.int32)
    args = (pr["feat_offset"], mo, pr["meas_clone"], pr["uv_norm"], pr["p_FinG"], pr["cp_inG"], fx, 1.0 / 458.0, 0.01)
    sg, pg, cg, ig, ng = ctx.optimize_plane(*args)
    so, po, co, io, no = orc.optimize_plane(*args)
    assert np.array_equal(sg, so) and np.array_equal(ig, io) and np.array_equal(ng[:, 1], no[:, 1])
    assert np.abs(pg - po).max() < 1e-7 and np.abs(cg - co).max() < 1e-7
    free = np.nonzero(np.diff(mo) == 0)[0]
    assert np.array_equal(pg[free][ig[free] == 1], pr["p_FinG"][free][ig[free] == 1])  # constant in the refinement
