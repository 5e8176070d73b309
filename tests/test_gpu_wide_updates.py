"""Updates wider than one co-resident launch of the fused Cholesky (csrc/cholpanel.cu, DESIGN.md 4.1): the panelled factorisation on its
own against NumPy at forced panel widths, the default width refusing exactly as before, and ovp_ekf_update, ovp_slam_update and
ovp_msckf_update past 960 columns with the width declared, against float64 restatements and the oracle.  Systems within the
co-resident width give the same bits whatever width is declared."""
import ctypes as C

import numpy as np
import pytest
from scipy.linalg import solve_triangular

import update_reference as ur
from ov_plane_b200 import api, synth
from conftest import make_pair
from test_gpu_parity import _check_msckf, oracle_msckf_update

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _coresident_width():
    """64 T with T (T + 1) / 2 tile CTAs within the device, one per SM (tests/test_gpu_cholfused.py)"""
    T = 1
    while (T + 1) * (T + 2) // 2 <= _sms():
        T += 1
    return 64 * T


@pytest.fixture(scope="module")
def ctx():
    S = synth.make_scenario("tiny_points")
    c = api.Context(S.options, device=0, max_state=640, max_meas_rows=4096, debug=True)  # libovp_debug.so: ovp_debug_chol_panels
    yield c
    c.close()


def _panels(ctx, panel, A, npiv, tol, M=None, z=None, gate=-1.0):
    """ovp_debug_chol_panels (panel > 0) or ovp_debug_chol_solve_gated (panel = 0): (L, Y, w, chi2, gate flag)"""
    n = A.shape[0]
    A = np.asfortranarray(np.tril(A))
    L = np.zeros((n, n), order="F")
    Y = w = None
    pM = pz = pY = pw = None
    mrows = 0
    chi2, flag = C.c_double(-1.0), C.c_int(-1)
    if M is not None:
        M, z = np.asfortranarray(M), np.ascontiguousarray(z)
        mrows = M.shape[0]
        Y, w = np.zeros((mrows, npiv), order="F"), np.zeros(npiv)
        pM, pz, pY, pw = (x.ctypes.data_as(C.c_void_p) for x in (M, z, Y, w))
    args = (A.ctypes.data_as(C.c_void_p), n, npiv, C.c_double(tol), pM, mrows, pz, 1, C.c_double(gate), L.ctypes.data_as(C.c_void_p), pY, pw,
            C.byref(chi2), C.byref(flag))
    if panel:
        ctx._ck(ctx.lib.ovp_debug_chol_panels(ctx.h, panel, *args))
    else:
        ctx._ck(ctx.lib.ovp_debug_chol_solve_gated(ctx.h, *args))
    return np.tril(L), Y, w, chi2.value, flag.value


# ---- 1. the panelled factorisation against NumPy, at the tolerances of tests/test_gpu_cholfused.py -------------------------------------
CASES = [(n, npiv, p) for p in (64, 128, 192) for n, npiv in ((65, 65), (200, 200), (200, 130), (333, 333), (333, 300), (600, 600),
                                                               (600, 471))]


@pytest.mark.parametrize("n,npiv,panel", CASES)
def test_panels_factor_and_solve(ctx, n, npiv, panel):
    rng = np.random.default_rng(n + npiv + panel)
    B = rng.normal(size=(n + 8, n))
    A = B.T @ B + 0.5 * np.eye(n)
    L, _, _, _, _ = _panels(ctx, panel, A, npiv, 0.0)
    L11 = np.linalg.cholesky(A[:npiv, :npiv])
    L21 = np.linalg.solve(L11, A[npiv:, :npiv].T).T
    assert np.abs(L[:npiv, :npiv] - L11).max() < 1e-11 * np.abs(L11).max() * n
    if npiv < n:
        assert np.abs(L[npiv:, :npiv] - L21).max() < 1e-10 * np.abs(L21).max() * n
    assert np.array_equal(L[:, npiv:], np.tril(A)[:, npiv:]), "columns past the pivots were written"
    if npiv == n:  # with a right-hand side: Y = M L^-T, w = L^-1 z, chi2 and the gate on both sides of the threshold
        M = rng.normal(size=(37 + n % 29, n))
        z = rng.normal(size=n)
        chi2_ref = float(np.sum(np.linalg.solve(L11, z) ** 2))
        for gate, want in ((chi2_ref * (1 + 1e-6), 1), (chi2_ref * (1 - 1e-6), 0), (-1.0, 1)):
            L, Y, w, chi2, flag = _panels(ctx, panel, A, n, 0.0, M, z, gate)
            assert np.abs(Y - np.linalg.solve(L11, M.T).T).max() < 1e-9 * np.abs(M).max() * n
            assert np.abs(w - np.linalg.solve(L11, z)).max() < 1e-9 * np.abs(z).max() * n
            assert abs(chi2 - chi2_ref) < 1e-9 * chi2_ref, (chi2, chi2_ref)
            assert flag == want, (gate, chi2, flag)


@pytest.mark.parametrize("panel", [64, 128])
def test_panels_zero_pivot_rule_against_the_original_diagonal(ctx, panel):
    """A rank-deficient Gram matrix whose dropped directions fall in a later panel: the same count of zero columns as the fused launch,
    in the later panels, and L L^T reproduces G."""
    rng = np.random.default_rng(7)
    n, r = 300, 250
    H = rng.normal(size=(600, r)) @ rng.normal(size=(r, n))  # rank r < n: the last n - r columns depend on the first r
    G = H.T @ H
    L, _, _, _, _ = _panels(ctx, panel, G, n, 1e-11)
    Lf, _, _, _, _ = _panels(ctx, 0, G, n, 1e-11)
    assert np.isfinite(L).all()
    zero_cols = np.where(np.abs(np.diag(L)) == 0.0)[0]
    assert len(zero_cols) == n - r == len(np.where(np.abs(np.diag(Lf)) == 0.0)[0])
    assert zero_cols.min() >= panel, zero_cols  # every dropped direction lies past the first panel
    assert np.abs(L[:, zero_cols]).max() == 0.0
    assert np.abs(L @ L.T - G).max() < 1e-8 * np.abs(G).max()


@pytest.mark.parametrize("panel", [64, 128])
def test_panels_report_an_indefinite_pivot_in_a_later_panel(ctx, panel):
    A = np.eye(300)
    A[250, 250] = -1.0
    for p in (0, panel):
        with pytest.raises(api.OvpError) as e:
            _panels(ctx, p, A, 300, 0.0)
        assert e.value.status == 9  # OVP_ERR_NOT_POSITIVE_DEFINITE, as the fused launch reports it
    L, _, _, _, _ = _panels(ctx, panel, np.eye(300), 300, 0.0)  # and the flag is cleared
    assert np.array_equal(L, np.eye(300))


def test_panel_width_out_of_range_is_refused(ctx):
    A = np.eye(100)
    for p in (32, 100, _coresident_width() + 64):
        with pytest.raises(api.OvpError) as e:
            _panels(ctx, p, A, 100, 0.0)
        assert e.value.status == 1


# ---- 2. the default width -------------------------------------------------------------------------------------------------------------
def _wide_state(max_state=2048, seed=0):
    """A context with max_state columns and a state of IMU, calibration and landmarks filling it to within 2 columns, with a correlated
    covariance: (ctx, kinds, ids, vals, fejs, P)."""
    ctx = api.Context(ur.STATE_OPTIONS, device=0, max_state=max_state, max_meas_rows=4096)
    rng = np.random.default_rng(seed)
    kinds = {ctx.handle_imu(): ur.IMU, ctx.handle_dt(): ur.VEC, ctx.handle_calib(): ur.POSE, ctx.handle_intrinsics(): ur.VEC}
    for i in range((max_state - ctx.cov_rows()) // 3):
        p = 3.0 * rng.standard_normal(3)
        kinds[ctx.add_slam_raw(5000000 + i, p, p)] = ur.LANDMARK
    N = ctx.cov_rows()
    ids = {h: ctx.var_id(h) for h in kinds}
    vals, fejs = {}, {}
    for h in kinds:
        vals[h], fejs[h] = ctx.var_get(h)
    d = np.exp(rng.uniform(-2.0, 0.0, N))
    P = ur.correlated(d, seed)
    ctx.cov_upload(P)
    return ctx, kinds, ids, vals, fejs, ctx.cov().copy()


def _landmark_handles(kinds, ids, ncols):
    hs = sorted((h for h in kinds if kinds[h] == ur.LANDMARK), key=lambda h: ids[h])
    hs = hs[:(ncols + 2) // 3]
    return hs, [ids[h] + k for h in hs for k in range(3)]


def test_default_width_refuses_as_before_and_the_setter_checks_its_range():
    ctx, kinds, ids, _, _, P = _wide_state()
    cw = _coresident_width()
    assert ctx.max_update_width() == (cw, cw)
    rows = 1000
    hs, cols = _landmark_handles(kinds, ids, 300)
    H = np.random.default_rng(1).normal(size=(rows, len(cols)))
    r = np.zeros(rows)
    T = (rows + 63) // 64
    if T * (T + 1) // 2 > _sms():
        with pytest.raises(api.OvpError) as e:
            ctx.ekf_update(hs, H, r)
        assert e.value.status == 7
        assert "chol_fused: a %d-wide system needs %d co-resident tile CTAs, the device holds %d" % (rows, T * (T + 1) // 2, _sms()) in str(e.value)
        assert np.array_equal(ctx.cov(), P), "a refused update changed the covariance"
    cap = 2048 + 64  # max_state rounded up to 64, plus 64
    for bad in (-1, cw - 64, cap + 1):
        with pytest.raises(api.OvpError) as e:
            ctx.set_max_update_width(bad)
        assert e.value.status == 1
        assert ctx.max_update_width() == (cw, cw)
    ctx.set_max_update_width(cap)
    assert ctx.max_update_width() == (cap, cw)
    with pytest.raises(api.OvpError):
        ctx.set_max_update_width(cap + 64)
    assert ctx.max_update_width() == (cap, cw)
    ctx.set_max_update_width(0)
    assert ctx.max_update_width() == (cw, cw)
    ctx.close()


# ---- 3. ovp_ekf_update past the co-resident width ---------------------------------------------------------------------------------------
def kalman64(P, cols, H, r, R):
    """EKFUpdate in float64 (NumPy / SciPy): S = H P_cc H^T + R, L = chol(S), Y = P H^T L^-T, w = L^-1 r, P+ = P - Y Y^T, dx = Y w."""
    M = P[:, cols] @ H.T
    S = H @ M[cols, :] + np.diag(np.ones(H.shape[0]) if R is None else R)
    L = np.linalg.cholesky(S)
    w = solve_triangular(L, r, lower=True)
    Y = solve_triangular(L, M.T, lower=True).T
    return dict(P=P - Y @ Y.T, dx=Y @ w, w=w, S=S, Y=Y, M=M)


@pytest.mark.parametrize("rows", [961, 1024, 1500, 2000])
@pytest.mark.parametrize("rdiag", [None, "diag"])
def test_ekf_update_wider_than_one_launch(rows, rdiag):
    """n = rows innovation system over about as many landmark columns of an N = 2048 state.  Error bound: each of the library and the
    float64 restatement is within the first-order bound of update_reference.kalman_bounds of the exact update - it scales with
    kappa(S) = lambda_max / lambda_min and the sizes - so the two are held to twice that bound."""
    ctx, kinds, ids, vals, fejs, P = _wide_state(seed=rows)
    cw = _coresident_width()
    ctx.set_max_update_width(2048 + 64)
    hs, cols = _landmark_handles(kinds, ids, rows)
    rng = np.random.default_rng(rows)
    sd = np.sqrt(np.diag(P)[cols])
    H = rng.normal(size=(rows, len(cols))) / (sd[None, :] * np.sqrt(len(cols)))
    R = None if rdiag is None else np.exp(rng.uniform(-1.0, 1.0, rows))
    r = rng.normal(size=rows) * (1.0 if R is None else np.sqrt(R))
    assert rows > cw
    ctx.ekf_update(hs, H, r, R)
    P_got = ctx.cov()
    vals_got = {h: ctx.var_get(h)[0] for h in kinds}
    fejs_got = {h: ctx.var_get(h)[1] for h in kinds}
    ref = kalman64(P, cols, H, r, R)
    dxb, dPb, kS = ur.kalman_bounds(P, cols, H, ref)
    qP, qv = ur.check_update(P_got, vals_got, fejs_got, P, kinds, ids, vals, fejs, ref["dx"], 2 * dxb, 2 * dPb, ref["P"])
    print("ekf_update N %d rows %d cols %d R %s: kappa(S) %.2e, worst error / bound P+ %.3e values %.3e" % (
        P.shape[0], rows, len(cols), rdiag, kS, qP, qv))
    ctx.close()


# ---- 4. ovp_slam_update past the co-resident width --------------------------------------------------------------------------------------
def test_slam_update_wider_than_one_launch():
    """The scenario of test_gpu_slam_reference.py::test_batch_wider_than_the_co_resident_factorisation_is_refused with the width declared:
    accepted, statuses those of the library's per-landmark gates (the Gram hook, which the SLAM parity tests check against long double),
    and the posterior against a float64 restatement of EKFUpdate over the stacked rows (long double is too slow at this size), within
    twice the first-order bound of update_reference.kalman_bounds."""
    import gate_reference as gr
    import test_gpu_slam_reference as tsr
    width = _coresident_width()
    cs = tsr.Case()
    cs.S = gr.slam_scenario(0, seed=0, F=(width + 64) // 3)
    cs.ncal, cs.cov, cs.shape, cs.seed, cs.use_plane = 0, "correlated", ("short",), 0, True
    ctx, chg, b, attached = tsr.new_ctx(cs)
    kinds = tsr.kinds_of(ctx, cs, chg, b)
    ctx.set_max_update_width((cs.S.N + 3 * cs.S.F + 64 + 63) // 64 * 64 + 64)  # new_ctx's max_state, rounded up to 64, plus 64
    snap0 = tsr.snapshot(ctx, kinds, list(cs.S.featid))
    g = tsr.debug_gram(ctx, b, True)
    nc = len(g["cols"])
    assert nc + 1 > width, (nc + 1, width)
    X, info = tsr.stacked(ctx, cs, b, g, True)
    res = ctx.slam_update(b, 1.0, 1.0, True)
    assert np.array_equal(res["feat_status"], g["status"])
    got = tsr.snapshot(ctx, kinds, list(cs.S.featid))
    P = np.asarray(snap0[0], dtype=np.float64)
    cols = [int(s) for s in g["cols"]]
    X = np.asarray(X, dtype=np.float64)
    ref = kalman64(P, cols, X[:, :nc], X[:, nc], None)
    dxb, dPb, kS = ur.kalman_bounds(P, cols, X[:, :nc], ref)
    ids = {h: ctx.var_id(h) for h in kinds}
    qP, qv = ur.check_update(got[0], got[1], got[2], P, kinds, ids, snap0[1], snap0[2], ref["dx"], 2 * dxb, 2 * dPb, ref["P"])
    print("slam_update F %d, rows %d, nc1 %d (co-resident width %d): kappa(S) %.2e, worst error / bound P+ %.3e values %.3e" % (
        b["F"], X.shape[0], nc + 1, width, kS, qP, qv))
    ctx.close()


# ---- 5. MSCKF point and in-state plane updates past the co-resident width ---------------------------------------------------------------
def test_msckf_update_wider_than_one_launch(chi2_table):
    """170 clones: the point update and the in-state plane updates compress to more than 960 columns.  Statuses, Hx_order and the
    covariance against the oracle (1e-6 relative); a prepared batch replayed three times from its graph gives the eager run's bits."""
    S = synth.make_scenario("small_planes", seed=0, n_clones=170, F=700, m_min=12, m_max=20)
    ctx, orc, chg, cho = make_pair(S, chi2_table)
    cap = (max(128, S.N + 64) + 63) // 64 * 64 + 64  # make_pair's max_state, rounded up to 64, plus 64
    ctx.set_max_update_width(cap)
    ctx.set_use_graphs(False)
    P0 = ctx.cov().copy()
    g = ctx.msckf_update(synth.feature_batch(S, chg), 1.0, 1.0)
    o = oracle_msckf_update(orc, synth.feature_batch(S, cho), 1.0, 1.0)
    e = _check_msckf(S, ctx, orc, chg, cho, g, o, chi_tol=1e-6)
    assert 6 * len(g["hx_order"]) > _coresident_width(), len(g["hx_order"])  # Hx_order: the point update's clones (and calibration)
    eager = ctx.cov().copy()
    print("msckf_update: %d clones in the point update, cov rel err %.2e" % (len(g["hx_order"]), e))
    ctx.close()
    ctx, orc, chg, cho = make_pair(S, chi2_table)
    ctx.set_max_update_width(cap)
    assert np.array_equal(ctx.cov(), P0)
    ctx.snapshot()
    ctx.msckf_prepare(synth.feature_batch(S, chg), 1.0, 1.0)
    for _ in range(3):
        ctx.restore()
        ctx.msckf_launch()
        f = ctx.msckf_finish()
        assert np.array_equal(f["feat_status"], g["feat_status"]) and f["hx_order"] == g["hx_order"]
        assert np.array_equal(ctx.cov().view(np.uint64), eager.view(np.uint64)), "graph replay differs from the eager run"
    ctx.close()


# ---- 6. bit identity below the width ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cfg2_n256_f200", "cfg3_n512_f600_p8"])
def test_declared_width_changes_nothing_within_one_launch(name, chi2_table):
    """The same context size twice (column capacity 1088, above the co-resident width), once with the default width and once with its
    full column capacity declared: the same bits and the same launch count."""
    S = synth.make_scenario(name, seed=0)
    out = []
    for declare in (False, True):
        ctx = api.Context(S.options, device=0, max_state=1024, max_meas_rows=60000)
        ctx.set_chi2_table(chi2_table)
        chg = synth.load_scenario_into(ctx, S)
        if declare:
            ctx.set_max_update_width(1024 + 64)
            assert ctx.max_update_width()[0] > ctx.max_update_width()[1]
        l0 = ctx.launch_count()
        g = ctx.msckf_update(synth.feature_batch(S, chg), 1.0, 1.0)
        out.append((ctx.cov().copy(), g, ctx.launch_count() - l0))
        ctx.close()
    (P0, g0, n0), (P1, g1, n1) = out
    assert np.array_equal(P0.view(np.uint64), P1.view(np.uint64))
    assert np.array_equal(g0["feat_status"], g1["feat_status"]) and g0["hx_order"] == g1["hx_order"]
    assert n0 == n1, (n0, n1)
