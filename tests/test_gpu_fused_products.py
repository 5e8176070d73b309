"""The update products formed inside the factorisation of the compression's Gram matrix (chol_fused_kernel, cholfused.cu): with L = rows
[0, nc) of the factor, M = P[:, cols] L and S = L^T M[cols, :] + I, through the ovp_debug_chol_products hook of libovp_debug.so, against a
NumPy long-double reference with the element-wise bound of tests/test_gpu_gemm.py:

    |C - C_ref| <= 2 (K + 2) 2^-53 (|A| |B| + |diag|)

M is checked against P[:, cols] L of the returned factor, S against L^T M[cols, :] + I of the returned M (lower triangle).  The factor
itself must carry the same bits as the factorisation without products (ovp_debug_chol_solve).  End to end, the benchmarked workload runs
with the products formed inside the factorisation and with the two GEMM launches (ovp_debug_unfused_update_products); both must match
each other and the oracle."""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle_backend
from ov_plane_b200 import api, synth
from test_gpu_parity import oracle_msckf_update, _check_msckf

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -53
TOL = 1e-11


def _ctx():
    S = synth.make_scenario("tiny_points")
    return api.Context(S.options, device=0, max_state=1024, max_meas_rows=4096, debug=True)


@pytest.fixture(scope="module")
def ctx():
    c = _ctx()
    yield c
    c.close()


def _p(x):
    return x.ctypes.data_as(C.c_void_p)


def make_system(seed, nc, npiv, N, zero_cols=()):
    """Gram matrix of a random stacked system [H | z] (H's zero_cols exactly zero: exact zero pivots), an SPD covariance P and nc
    sorted distinct column ids into it."""
    rng = np.random.default_rng(seed)
    H = rng.standard_normal((nc + 24, nc + 1))
    H[:, list(zero_cols)] = 0.0
    G = np.asfortranarray(np.tril(H.T @ H))
    A = rng.standard_normal((N, N))
    P = np.asfortranarray(A @ A.T / N + np.eye(N))
    cols = np.ascontiguousarray(np.sort(rng.choice(N, size=nc, replace=False)), dtype=np.int32)
    return G, P, cols


def run_products(ctx, G, nc, npiv, P, cols):
    N = P.shape[0]
    L = np.zeros((nc + 1, npiv), order="F")
    M = np.zeros((N, npiv), order="F")
    S = np.full((npiv, npiv), np.nan, order="F")
    ctx._ck(ctx.lib.ovp_debug_chol_products(ctx.h, _p(G), nc, npiv, C.c_double(TOL), _p(P), N, _p(cols), _p(L), _p(M), _p(S)))
    return L, M, S


def factor_only(ctx, G, npiv):
    n = G.shape[0]
    L = np.zeros((n, n), order="F")
    ctx._ck(ctx.lib.ovp_debug_chol_solve(ctx.h, _p(G), n, npiv, C.c_double(TOL), None, 0, None, _p(L), None, None))
    return L[:, :npiv]


def check_bound(tag, got, exp, mag, K):
    err = np.abs(got.astype(np.longdouble) - exp).astype(np.float64)
    bnd = 2.0 * (K + 2) * EPS * mag
    assert np.all(np.isfinite(got)), "%s: non-finite result" % tag
    ratio = float((err / np.maximum(bnd, 1e-300)).max())
    assert np.all(err <= bnd), "%s: error %.3e above its bound (worst error / bound = %.2f)" % (tag, err.max(), ratio)
    return ratio


def check_products(ctx, tag, G, nc, npiv, P, cols):
    L, M, S = run_products(ctx, G, nc, npiv, P, cols)
    assert np.array_equal(L.view(np.uint64), factor_only(ctx, G, npiv).view(np.uint64)), "%s: the factor differs from the factorisation alone" % tag
    ld = np.longdouble
    Lk = L[:nc, :]  # row nc is z: not part of the products
    Pc = P[:, cols]
    rM = check_bound(tag + " M", M, Pc.astype(ld) @ Lk.astype(ld), np.abs(Pc) @ np.abs(Lk), nc)
    Mg = M[cols, :]
    low = np.tril(np.ones((npiv, npiv), dtype=bool))
    Sref = Lk.T.astype(ld) @ Mg.astype(ld) + np.eye(npiv, dtype=ld)
    mag = np.abs(Lk.T) @ np.abs(Mg) + np.eye(npiv)
    rS = check_bound(tag + " S", S[low], Sref[low], mag[low], nc)
    print("%s: worst error / bound  M %.3f  S %.3f" % (tag, rM, rS))
    return L, M, S


@pytest.mark.parametrize("form,nc,npiv", [("plane", 473, 470), ("point", 470, 470)])
@pytest.mark.parametrize("N", [512, 1000])
def test_products_at_update_shapes(ctx, form, nc, npiv, N):
    """The benchmark's plane (474 columns with z, 470 pivots) and point (471, 470) systems with exact zero pivots, at N = 512 and at
    N = 1000 (16 row blocks of M)."""
    G, P, cols = make_system(N + nc, nc, npiv, N, zero_cols=(5, 130, 300))
    check_products(ctx, "%s N=%d" % (form, N), G, nc, npiv, P, cols)


@pytest.mark.parametrize("nc,npiv,N", [(40, 40, 100), (63, 60, 64), (129, 129, 200), (129, 126, 300)])
def test_products_small_and_ragged(ctx, nc, npiv, N):
    """One tile (the spine alone: a product-only CTA forms them) and systems whose size is not a multiple of 64."""
    G, P, cols = make_system(nc * 7 + N, nc, npiv, N, zero_cols=(3,))
    check_products(ctx, "nc=%d npiv=%d N=%d" % (nc, npiv, N), G, nc, npiv, P, cols)


def test_products_bit_identical_run_to_run(ctx):
    G, P, cols = make_system(7, 473, 470, 512, zero_cols=(11,))
    first = run_products(ctx, G, 473, 470, P, cols)
    for _ in range(3):
        again = run_products(ctx, G, 473, 470, P, cols)
        for a, b in zip(first, again):
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


def test_two_filters_concurrently(ctx):
    """Two contexts' fused launches at the same time (each its own stream, flags and queue counters) give their solo results."""
    other = _ctx()
    try:
        sys_a = make_system(21, 473, 470, 512, zero_cols=(9,))
        sys_b = make_system(22, 470, 470, 512)
        solo_a = run_products(ctx, sys_a[0], 473, 470, sys_a[1], sys_a[2])
        solo_b = run_products(other, sys_b[0], 470, 470, sys_b[1], sys_b[2])
        res = {}

        def work(key, c, s, nc):
            res[key] = [run_products(c, s[0], nc, 470, s[1], s[2]) for _ in range(4)]

        th = [threading.Thread(target=work, args=("a", ctx, sys_a, 473)), threading.Thread(target=work, args=("b", other, sys_b, 470))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        for key, solo in (("a", solo_a), ("b", solo_b)):
            for r in res[key]:
                for x, y in zip(solo, r):
                    assert np.array_equal(x.view(np.uint64), y.view(np.uint64)), key
    finally:
        other.close()


def test_cfg3_fused_and_unfused_products(chi2_table):
    """The benchmarked workload (8 plane updates + the point update) with M and S formed inside the Gram factorisation and with the two
    GEMM launches: same gates and Hx order, state and covariance equal to round-off, both at the oracle's tolerances."""
    S = synth.make_scenario("cfg3_n512_f600_p8", seed=0)
    runs = {}
    for unfused in (0, 1):
        ctx = api.Context(S.options, device=0, max_state=S.N + 64, max_meas_rows=60000, debug=True)
        ctx.set_chi2_table(chi2_table)
        orc = oracle_backend.OracleContext(S.options)
        orc.set_chi2_table(chi2_table)
        chg, cho = synth.load_scenario_into(ctx, S), synth.load_scenario_into(orc, S)
        ctx._ck(ctx.lib.ovp_debug_unfused_update_products(ctx.h, unfused))
        l0 = ctx.launch_count()
        g = ctx.msckf_update(synth.feature_batch(S, chg), 1.0, 1.0)
        launches = ctx.launch_count() - l0
        o = oracle_msckf_update(orc, synth.feature_batch(S, cho), 1.0, 1.0)
        e = _check_msckf(S, ctx, orc, chg, cho, g, o, chi_tol=1e-6)
        runs[unfused] = (g, ctx.cov(), launches, e)
        ctx.close()
    (g0, P0, l0, e0), (g1, P1, l1, e1) = runs[0], runs[1]
    for k in ("feat_status", "plane_status", "hx_order"):
        assert np.array_equal(g0[k], g1[k]), k
    d = np.abs(P0 - P1).max() / np.abs(P1).max()  # the summation order of M and S changes: round-off of the reordered sums
    print("cfg3 fused vs unfused: cov max diff / max |P| %.2e; vs oracle %.2e / %.2e; launches %d vs %d" % (d, e0, e1, l0, l1))
    assert d < 1e-9
    assert l1 - l0 == 2 * 9  # two GEMM launches per compressed update
