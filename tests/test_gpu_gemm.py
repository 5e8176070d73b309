"""The DMMA GEMM (gemm.cuh, launch_gemm in linalg.cu) against a NumPy long-double reference, one GemmProblem at a time through the
ovp_debug_gemm hook of libovp_debug.so.

Covered: both tile widths (32 and 64, forced, and the automatic choice), TRI_FULL / TRI_LOWER / TRI_LOWER_MIRROR, k-gathers on A and
on B (sorted distinct indices, as the update's column lists are), transposed and k-contiguous operand layouts, diag_add / diag_const,
the downdate form (alpha = -1, beta = 1), sizes around the tile edges and the three products of ekf_update_core at the benchmark's
shapes.  Every element the mode writes must satisfy

    |C - C_ref| <= 2 (K + 2) 2^-53 (|alpha| |A| |B| + |beta| |C0| + |diag|)

and every element it does not write must keep its bits (NaN sentinels included)."""
import ctypes as C

import numpy as np
import pytest

from ov_plane_b200 import api, synth

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -53
SIZES = (1, 7, 8, 17, 31, 32, 33, 64, 65, 130)
TRI_FULL, TRI_LOWER, TRI_LOWER_MIRROR = 0, 1, 2


@pytest.fixture(scope="module")
def ctx():
    S = synth.make_scenario("tiny_points")
    c = api.Context(S.options, device=0, max_state=128, max_meas_rows=1024, debug=True)
    yield c
    c.close()


class Op(object):
    """One operand: a physical column-major matrix, read transposed or not, with an optional gather of the contraction index."""

    def __init__(self, phys, trans, kidx):
        self.phys = np.asfortranarray(phys, dtype=np.float64)
        self.trans = int(trans)
        self.kidx = None if kidx is None else np.ascontiguousarray(kidx, dtype=np.int32)


def logical_A(op):  # M x K
    P = op.phys.T if op.trans else op.phys
    return P if op.kidx is None else P[:, op.kidx]


def logical_B(op):  # K x N
    P = op.phys.T if op.trans else op.phys
    return P if op.kidx is None else P[op.kidx, :]


def make_A(rng, M, K, trans, gather, scale=1.0):
    Kp = K + 5 if gather else K
    kidx = np.sort(rng.choice(Kp, size=K, replace=False)) if gather else None
    phys = rng.standard_normal((Kp, M) if trans else (M, Kp)) * scale
    return Op(phys, trans, kidx)


def make_B(rng, K, N, trans, gather, scale=1.0):
    Kp = K + 5 if gather else K
    kidx = np.sort(rng.choice(Kp, size=K, replace=False)) if gather else None
    phys = rng.standard_normal((N, Kp) if trans else (Kp, N)) * scale
    return Op(phys, trans, kidx)


def run_gemm(ctx, M, N, K, A, B, C0, alpha=1.0, beta=0.0, diag_add=None, diag_const=0.0, tri=TRI_FULL, ktri=0, flag=-1, tile=0):
    Cw = np.asfortranarray(C0, dtype=np.float64).copy(order="F")
    ldc = Cw.shape[0]
    info = np.zeros(2, dtype=np.int32)
    d = None if diag_add is None else np.ascontiguousarray(diag_add, dtype=np.float64)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    st = ctx.lib.ovp_debug_gemm(ctx.h, M, N, K, p(A.phys), A.phys.shape[0], A.phys.shape[1], A.trans, p(A.kidx), p(B.phys), B.phys.shape[0],
                                B.phys.shape[1], B.trans, p(B.kidx), p(Cw), ldc, C.c_double(alpha), C.c_double(beta), p(d), C.c_double(diag_const),
                                tri, ktri, flag, tile, p(info))
    ctx._ck(st)
    return Cw, int(info[0]), int(info[1])


def reference(M, N, A, B, C0, alpha, beta, diag_add, diag_const, tri):
    """(expected C, per-element bound, mask of the written elements)"""
    Al, Bl = logical_A(A), logical_B(B)
    K = Al.shape[1]
    ld = np.longdouble
    v = ld(alpha) * (Al.astype(ld) @ Bl.astype(ld)) if K else np.zeros((M, N), dtype=ld)
    mag = abs(alpha) * (np.abs(Al) @ np.abs(Bl)) if K else np.zeros((M, N))
    c0 = C0[:M, :N]
    if beta != 0.0:
        v = v + ld(beta) * c0.astype(ld)
        mag = mag + abs(beta) * np.abs(c0)
    dg = np.zeros(min(M, N)) + (diag_add if diag_add is not None else diag_const)
    i = np.arange(min(M, N))
    v[i, i] += dg.astype(ld)
    mag[i, i] += np.abs(dg)
    bound = 2.0 * (K + 2) * EPS * mag
    exp = C0.astype(ld).copy()
    bnd = np.zeros(C0.shape)
    wrote = np.zeros(C0.shape, dtype=bool)
    ii, jj = np.meshgrid(np.arange(M), np.arange(N), indexing="ij")
    low = np.ones((M, N), dtype=bool) if tri == TRI_FULL else (ii >= jj)
    exp[:M, :N][low] = v[low]
    bnd[:M, :N][low] = bound[low]
    wrote[:M, :N] |= low
    if tri == TRI_LOWER_MIRROR:  # C(j, i) = value (i, j) for i > j, i < N, j < M
        mi, mj = np.nonzero((ii > jj) & (ii < N) & (jj < M))
        exp[mj, mi] = v[mi, mj]
        bnd[mj, mi] = bound[mi, mj]
        wrote[mj, mi] = True
    return exp, bnd, wrote


def check(tag, Cg, exp, bnd, wrote, C0):
    assert np.all(np.isfinite(Cg[wrote])), "%s: non-finite result in the written region" % tag
    err = np.abs(Cg[wrote].astype(np.longdouble) - exp[wrote]).astype(np.float64)
    ratio = float((err / np.maximum(bnd[wrote], 1e-300)).max()) if err.size else 0.0
    assert np.all(err <= bnd[wrote]), "%s: error %.3e above its bound (worst error / bound = %.2f)" % (tag, err.max(), ratio)
    untouched = ~wrote
    assert np.array_equal(Cg[untouched].view(np.uint64), C0[untouched].view(np.uint64)), "%s: an element outside the written region changed" % tag
    return ratio


def _case(ctx, rng, M, N, K, tile, tri, beta=None, tag=""):
    a_trans, b_trans = int(rng.integers(2)), int(rng.integers(2))
    ga = bool(rng.integers(2))
    gb = bool(rng.integers(2))
    A = make_A(rng, M, K, a_trans, ga)
    B = make_B(rng, K, N, b_trans, gb)
    beta = float(rng.choice([0.0, 0.75])) if beta is None else beta
    alpha = float(rng.choice([1.0, -1.0, 0.3]))
    diag_add = rng.standard_normal(min(M, N)) if rng.integers(3) == 0 else None
    diag_const = float(rng.choice([0.0, 1.0]))
    ldc = M + int(rng.integers(0, 3))
    C0 = np.full((ldc, N), np.nan, order="F")
    if beta != 0.0:
        C0[:M, :] = rng.standard_normal((M, N))  # padding rows stay NaN sentinels
    Cg, used, _ = run_gemm(ctx, M, N, K, A, B, C0, alpha, beta, diag_add, diag_const, tri, 0, -1, tile)
    assert used == tile
    exp, bnd, wrote = reference(M, N, A, B, C0, alpha, beta, diag_add, diag_const, tri)
    return check("%s M=%d N=%d K=%d tile=%d tri=%d aT=%d bT=%d gA=%d gB=%d beta=%g" % (tag, M, N, K, tile, tri, a_trans, b_trans, ga, gb, beta),
                 Cg, exp, bnd, wrote, C0)


@pytest.mark.parametrize("tri", [TRI_FULL, TRI_LOWER, TRI_LOWER_MIRROR])
@pytest.mark.parametrize("tile", [32, 64])
def test_gemm_sizes_layouts_modes(ctx, tile, tri):
    """Every M and N of SIZES against a rotating K, layout, gather, beta and diagonal term."""
    rng = np.random.default_rng(100 * tile + tri)
    worst = 0.0
    n = 0
    for M in SIZES:
        for N in SIZES:
            K = SIZES[(3 * n + tri) % len(SIZES)]
            n += 1
            worst = max(worst, _case(ctx, rng, M, N, K, tile, tri))
    for M, N, K in ((130, 130, 130), (1, 1, 1), (65, 130, 33), (130, 7, 64)):
        for beta in (0.0, 1.0):
            worst = max(worst, _case(ctx, rng, M, N, K, tile, tri, beta))
    print("tile %d tri %d: %d products, worst error / bound = %.3f" % (tile, tri, n + 8, worst))


@pytest.mark.parametrize("tile", [32, 64])
@pytest.mark.parametrize("K", [1, 17, 33, 64, 65, 130])
def test_ktri_skips_only_structural_zeros(ctx, tile, K):
    """ktri = 1 (B lower trapezoidal, gather on A) and ktri = 2 (A = L^T, gather on B) are bit-identical to ktri = 0."""
    rng = np.random.default_rng(7 + K + tile)
    M, N = 130, 97
    # ktri = 1: B(k, j) == 0 for k < j, as the Cholesky factor L used as H^T in M = P[:, ids] L
    A = make_A(rng, M, K, 0, True)
    B = Op(np.tril(rng.standard_normal((K, N))), 0, None)
    C0 = np.full((M, N), np.nan, order="F")
    c0, _, _ = run_gemm(ctx, M, N, K, A, B, C0, ktri=0, tile=tile)
    c1, _, _ = run_gemm(ctx, M, N, K, A, B, C0, ktri=1, tile=tile)
    assert np.array_equal(c0, c1)
    exp, bnd, wrote = reference(M, N, A, B, C0, 1.0, 0.0, None, 0.0, TRI_FULL)
    check("ktri=1", c1, exp, bnd, wrote, C0)
    # ktri = 2: A(i, k) == 0 for k < i, as L^T in S = L^T M[ids, :] (lower tiles, + I)
    Mq = 90
    A = Op(np.tril(rng.standard_normal((K, Mq))), 1, None)
    B = make_B(rng, K, Mq, 0, True)
    C0 = np.full((Mq, Mq), np.nan, order="F")
    c0, _, _ = run_gemm(ctx, Mq, Mq, K, A, B, C0, diag_const=1.0, tri=TRI_LOWER, ktri=0, tile=tile)
    c2, _, _ = run_gemm(ctx, Mq, Mq, K, A, B, C0, diag_const=1.0, tri=TRI_LOWER, ktri=2, tile=tile)
    assert np.array_equal(c0, c2, equal_nan=True)
    exp, bnd, wrote = reference(Mq, Mq, A, B, C0, 1.0, 0.0, None, 1.0, TRI_LOWER)
    check("ktri=2", c2, exp, bnd, wrote, C0)


@pytest.mark.parametrize("tile", [32, 64])
def test_flag_zero_leaves_C_untouched(ctx, tile):
    rng = np.random.default_rng(3)
    M, N, K = 65, 65, 33
    A, B = make_A(rng, M, K, 0, False), make_B(rng, K, N, 1, False)
    C0 = np.asfortranarray(rng.standard_normal((M + 1, N)))
    C0[M, :] = np.nan
    c, _, _ = run_gemm(ctx, M, N, K, A, B, C0, -1.0, 1.0, tri=TRI_LOWER_MIRROR, flag=0, tile=tile)
    assert np.array_equal(c.view(np.uint64), C0.view(np.uint64))
    c, _, _ = run_gemm(ctx, M, N, K, A, B, C0, -1.0, 1.0, tri=TRI_LOWER_MIRROR, flag=1, tile=tile)
    exp, bnd, wrote = reference(M, N, A, B, C0, -1.0, 1.0, None, 0.0, TRI_LOWER_MIRROR)
    check("flag=1", c, exp, bnd, wrote, C0)


def test_automatic_tile_choice(ctx):
    """The launcher takes 64-wide tiles when the product has at least one 64-tile per SM, and the result is then bit-identical to a
    forced 64 (below that, to a forced 32)."""
    rng = np.random.default_rng(11)
    for M, N, K, tri in ((130, 130, 64, TRI_FULL), (1040, 1040, 40, TRI_FULL), (1024, 1024, 40, TRI_LOWER_MIRROR), (1000, 1000, 40, TRI_LOWER),
                         (576, 576, 40, TRI_LOWER_MIRROR)):
        A = make_A(rng, M, K, 0, False)
        B = make_B(rng, K, N, 1, False)
        C0 = np.asfortranarray(rng.standard_normal((M, N)))
        ca, used, sms = run_gemm(ctx, M, N, K, A, B, C0, -1.0, 1.0, tri=tri, tile=0)
        t = (M + 63) // 64
        tiles64 = t * t if tri == TRI_FULL else t * (t + 1) // 2
        want = 64 if tiles64 >= sms else 32
        print("M=N=%d tri=%d: %d 64-tiles on %d SMs -> %d-wide tiles" % (M, tri, tiles64, sms, used))
        assert used == want
        cf, _, _ = run_gemm(ctx, M, N, K, A, B, C0, -1.0, 1.0, tri=tri, tile=want)
        assert np.array_equal(ca, cf)
        exp, bnd, wrote = reference(M, N, A, B, C0, -1.0, 1.0, None, 0.0, tri)
        check("auto M=%d" % M, ca, exp, bnd, wrote, C0)


@pytest.mark.parametrize("N,rr", [(512, 470), (1000, 470)])  # the benchmark's state, and a state near max_state = 1024
def test_ekf_update_core_products(ctx, N, rr):
    """The three products of ekf_update_core with the compressed point system of the benchmark: M = P[:, ids] L (gather on A, ktri 1),
    S = L^T M[ids, :] + I (lower tiles, gather on B, ktri 2) and the downdate P -= Y Y^T (lower tiles mirrored), each with both tile
    widths and the automatic choice."""
    rng = np.random.default_rng(N)
    nc = rr
    ids = np.sort(rng.choice(N, size=nc, replace=False)).astype(np.int32)
    G = rng.standard_normal((N, N)) / np.sqrt(N)
    P = np.asfortranarray(G @ G.T + np.eye(N))
    L = np.tril(rng.standard_normal((nc, rr)))
    L[np.arange(rr), np.arange(rr)] = 3.0 + np.abs(L[np.arange(rr), np.arange(rr)])
    worst = {}
    for tile in (32, 64, 0):
        A, B = Op(P, 0, ids), Op(L, 0, None)
        C0 = np.full((N, rr), np.nan, order="F")
        Mg, _, _ = run_gemm(ctx, N, rr, nc, A, B, C0, ktri=1, tile=tile)
        exp, bnd, wrote = reference(N, rr, A, B, C0, 1.0, 0.0, None, 0.0, TRI_FULL)
        r1 = check("M = P[:, ids] L tile %d" % tile, Mg, exp, bnd, wrote, C0)
        A, B = Op(L, 1, None), Op(Mg, 0, ids)
        C0 = np.full((rr, rr), np.nan, order="F")
        Sg, _, _ = run_gemm(ctx, rr, rr, nc, A, B, C0, diag_const=1.0, tri=TRI_LOWER, ktri=2, tile=tile)
        exp, bnd, wrote = reference(rr, rr, A, B, C0, 1.0, 0.0, None, 1.0, TRI_LOWER)
        r2 = check("S = L^T M[ids, :] + I tile %d" % tile, Sg, exp, bnd, wrote, C0)
        Y = rng.standard_normal((N, rr)) * 0.05
        A, B = Op(Y, 0, None), Op(Y, 1, None)
        Pg, used, sms = run_gemm(ctx, N, N, rr, A, B, P, -1.0, 1.0, tri=TRI_LOWER_MIRROR, flag=1, tile=tile)
        exp, bnd, wrote = reference(N, N, A, B, P, -1.0, 1.0, None, 0.0, TRI_LOWER_MIRROR)
        r3 = check("P -= Y Y^T tile %d" % tile, Pg, exp, bnd, wrote, P)
        worst[tile if tile else "auto(%d)" % used] = (round(r1, 3), round(r2, 3), round(r3, 3))
    print("N=%d rr=%d worst error / bound (M, S, downdate):" % (N, rr), worst)
