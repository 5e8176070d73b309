"""The DMMA GEMM's split k (gemm.cuh, gemm_plan / launch_gemm in linalg.cu): a launch cuts K into chunks at fixed boundaries
c * kc, one CTA per chunk and output tile, and the CTAs of a tile reduce their partial tiles in chunk order inside one thread-block
cluster.  test_gpu_gemm.py checks the products; this file checks what only a split launch does, asking the launcher through the
ovp_debug_gemm_split hook which split it takes:

- several chunks, with K not a multiple of kc, so the last chunk ends inside a 16-wide k-step;
- ktri products whose leading chunks are entirely structural zeros (not computed), bit-identical to ktri = 0;
- K below one chunk (the unsplit walk);
- the three products of ekf_update_core at N = 512 and 1000 with rr = 470;
- two identical calls giving identical bits.

Every case uses the long-double bound of test_gpu_gemm.py."""
import ctypes as C

import numpy as np
import pytest

from ov_plane_b200 import api, synth
from test_gpu_gemm import TRI_FULL, TRI_LOWER, TRI_LOWER_MIRROR, Op, check, make_A, make_B, reference, run_gemm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    S = synth.make_scenario("tiny_points")
    c = api.Context(S.options, device=0, max_state=128, max_meas_rows=1024, debug=True)
    yield c
    c.close()


def plan(ctx, M, N, K, tri=TRI_FULL, ktri=0, tile=0):
    """(tile width, chunk count, chunk length) the launcher takes for this product"""
    info = np.zeros(3, dtype=np.int32)
    ctx._ck(ctx.lib.ovp_debug_gemm_split(ctx.h, M, N, K, tri, ktri, tile, info.ctypes.data_as(C.c_void_p)))
    return int(info[0]), int(info[1]), int(info[2])


def check_layout(K, n, kc):
    assert kc % 16 == 0 and kc >= 16
    assert 1 <= n <= 8
    assert (n - 1) * kc < K <= n * kc or (K == 0 and n == 1)


@pytest.mark.parametrize("tri", [TRI_FULL, TRI_LOWER, TRI_LOWER_MIRROR])
@pytest.mark.parametrize("tile", [32, 64])
def test_split_chunks_end_inside_a_k_step(ctx, tile, tri):
    """K of 2 to 8 chunks, none a multiple of kc or of 16, against every layout, gather, beta and diagonal term."""
    rng = np.random.default_rng(31 * tile + tri)
    worst = 0.0
    for M, N, K in ((97, 97, 333), (70, 45, 131), (130, 97, 470), (33, 65, 201), (64, 64, 515)):
        _, n, kc = plan(ctx, M, N, K, tri, 0, tile)
        check_layout(K, n, kc)
        assert n > 1 and K % kc != 0, (M, N, K, n, kc)
        for rep in range(2):
            a_trans, b_trans, ga, gb = (int(x) for x in rng.integers(2, size=4))
            A, B = make_A(rng, M, K, a_trans, ga), make_B(rng, K, N, b_trans, gb)
            beta = (0.0, 0.75)[rep]
            alpha = float(rng.choice([1.0, -1.0, 0.3]))
            diag_add = rng.standard_normal(min(M, N)) if rep == 0 else None
            ldc = M + int(rng.integers(0, 3))
            C0 = np.full((ldc, N), np.nan, order="F")
            if beta != 0.0:
                C0[:M, :] = rng.standard_normal((M, N))
            Cg, used, _ = run_gemm(ctx, M, N, K, A, B, C0, alpha, beta, diag_add, 1.0, tri, 0, -1, tile)
            assert used == tile
            exp, bnd, wrote = reference(M, N, A, B, C0, alpha, beta, diag_add, 1.0, tri)
            worst = max(worst, check("M=%d N=%d K=%d chunks %d x %d aT=%d bT=%d gA=%d gB=%d" % (M, N, K, n, kc, a_trans, b_trans, ga, gb),
                                     Cg, exp, bnd, wrote, C0))
    print("tile %d tri %d: worst error / bound = %.3f" % (tile, tri, worst))


@pytest.mark.parametrize("tile", [32, 64])
def test_split_ktri_dead_leading_chunks(ctx, tile):
    """ktri = 1 / 2 with tiles whose first chunks lie wholly in the structural zeros: bit-identical to ktri = 0."""
    rng = np.random.default_rng(5 + tile)
    M, N, K = 200, 300, 300
    _, n, kc = plan(ctx, M, N, K, TRI_FULL, 1, tile)
    check_layout(K, n, kc)
    assert n > 1 and (N - 1) // tile * tile >= 2 * kc  # the last tile column skips at least two chunks
    A = make_A(rng, M, K, 0, True)
    B = Op(np.tril(rng.standard_normal((K, N))), 0, None)
    C0 = np.full((M, N), np.nan, order="F")
    c0, _, _ = run_gemm(ctx, M, N, K, A, B, C0, ktri=0, tile=tile)
    c1, _, _ = run_gemm(ctx, M, N, K, A, B, C0, ktri=1, tile=tile)
    assert np.array_equal(c0, c1)
    exp, bnd, wrote = reference(M, N, A, B, C0, 1.0, 0.0, None, 0.0, TRI_FULL)
    check("ktri=1", c1, exp, bnd, wrote, C0)
    Mq = 300
    _, n, kc = plan(ctx, Mq, Mq, K, TRI_LOWER, 2, tile)
    assert n > 1
    A = Op(np.tril(rng.standard_normal((K, Mq))), 1, None)
    B = make_B(rng, K, Mq, 0, True)
    C0 = np.full((Mq, Mq), np.nan, order="F")
    c0, _, _ = run_gemm(ctx, Mq, Mq, K, A, B, C0, diag_const=1.0, tri=TRI_LOWER, ktri=0, tile=tile)
    c2, _, _ = run_gemm(ctx, Mq, Mq, K, A, B, C0, diag_const=1.0, tri=TRI_LOWER, ktri=2, tile=tile)
    assert np.array_equal(c0, c2, equal_nan=True)
    exp, bnd, wrote = reference(Mq, Mq, A, B, C0, 1.0, 0.0, None, 1.0, TRI_LOWER)
    check("ktri=2", c2, exp, bnd, wrote, C0)


@pytest.mark.parametrize("K", [1, 15, 16, 40, 64, 100, 128])
def test_k_below_one_chunk(ctx, K):
    rng = np.random.default_rng(K)
    M, N = 97, 70
    for tile in (32, 64):
        _, n, kc = plan(ctx, M, N, K, TRI_FULL, 0, tile)
        check_layout(K, n, kc)
        assert n == 1
        A, B = make_A(rng, M, K, 1, True), make_B(rng, K, N, 0, True)
        C0 = np.asfortranarray(rng.standard_normal((M, N)))
        Cg, _, _ = run_gemm(ctx, M, N, K, A, B, C0, -1.0, 1.0, tile=tile)
        exp, bnd, wrote = reference(M, N, A, B, C0, -1.0, 1.0, None, 0.0, TRI_FULL)
        check("K=%d tile %d" % (K, tile), Cg, exp, bnd, wrote, C0)


@pytest.mark.parametrize("N,rr", [(512, 470), (1000, 470)])
def test_ekf_update_core_products_split(ctx, N, rr):
    """M = P[:, ids] L (ktri 1), S = L^T M[ids, :] + I (lower, ktri 2) and P -= Y Y^T (lower mirrored) with the launcher's own
    choice of tile and split, each run twice: within the bound, and the same bits both times."""
    rng = np.random.default_rng(N + 1)
    nc = rr
    ids = np.sort(rng.choice(N, size=nc, replace=False)).astype(np.int32)
    G = rng.standard_normal((N, N)) / np.sqrt(N)
    P = np.asfortranarray(G @ G.T + np.eye(N))
    L = np.tril(rng.standard_normal((nc, rr)))
    L[np.arange(rr), np.arange(rr)] = 3.0 + np.abs(L[np.arange(rr), np.arange(rr)])
    Y = rng.standard_normal((N, rr)) * 0.05
    plans = {"M": plan(ctx, N, rr, nc, TRI_FULL, 1), "S": plan(ctx, rr, rr, nc, TRI_LOWER, 2), "downdate": plan(ctx, N, N, rr, TRI_LOWER_MIRROR, 0)}
    for t, n, kc in plans.values():
        check_layout(nc, n, kc)
    if N == 512:  # the benchmark's shapes are below two waves of tiles: M and S split
        assert plans["M"][1] > 1 and plans["S"][1] > 1
    ratios = []

    def twice(*args, **kw):
        a, _, _ = run_gemm(ctx, *args, **kw)
        b, _, _ = run_gemm(ctx, *args, **kw)
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), "two identical calls differ"
        return a

    A, B = Op(P, 0, ids), Op(L, 0, None)
    C0 = np.full((N, rr), np.nan, order="F")
    Mg = twice(N, rr, nc, A, B, C0, ktri=1)
    exp, bnd, wrote = reference(N, rr, A, B, C0, 1.0, 0.0, None, 0.0, TRI_FULL)
    ratios.append(check("M = P[:, ids] L", Mg, exp, bnd, wrote, C0))
    A, B = Op(L, 1, None), Op(Mg, 0, ids)
    C0 = np.full((rr, rr), np.nan, order="F")
    Sg = twice(rr, rr, nc, A, B, C0, diag_const=1.0, tri=TRI_LOWER, ktri=2)
    exp, bnd, wrote = reference(rr, rr, A, B, C0, 1.0, 0.0, None, 1.0, TRI_LOWER)
    ratios.append(check("S = L^T M[ids, :] + I", Sg, exp, bnd, wrote, C0))
    A, B = Op(Y, 0, None), Op(Y, 1, None)
    Pg = twice(N, N, rr, A, B, P, -1.0, 1.0, tri=TRI_LOWER_MIRROR, flag=1)
    exp, bnd, wrote = reference(N, N, A, B, P, -1.0, 1.0, None, 0.0, TRI_LOWER_MIRROR)
    ratios.append(check("P -= Y Y^T", Pg, exp, bnd, wrote, P))
    print("N=%d rr=%d plans (tile, chunks, kc) %s, worst error / bound (M, S, downdate) %s" % (N, rr, plans, [round(r, 3) for r in ratios]))
