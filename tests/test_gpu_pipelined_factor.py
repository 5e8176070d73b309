"""The paired factorisation of a compressed update (chol_fused_pair, cholfused.cu): the Gram matrix's factorisation with the update
products and the innovation system's factorisation in ONE cooperative launch, each S tile starting once its product item is stored, and
the innovation system's row blocks (Y, w, chi2 and the gate) in a second launch that starts while the first runs.  Every tile, item and row block does the same arithmetic in the same order as in the two launches, so every
output must carry the same bits as with ovp_debug_sequential_factorisations(1): the factors, M, Y, w, chi2 and the gate through the
ovp_debug_chol_pair hook of libovp_debug.so, and P+, every variable value, the chi2 values and the gates of the benchmarked step and of the
SLAM update end to end."""
import ctypes as C
import threading

import numpy as np
import pytest

from ov_plane_b200 import api, synth

pytestmark = pytest.mark.gpu

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


def run_pair(ctx, G, nc, npiv, P, cols, sequential, gate_thresh=-1.0, timeline=None):
    """Both factorisations of one compressed update: (outputs, paired)."""
    N = P.shape[0]
    ctx._ck(ctx.lib.ovp_debug_sequential_factorisations(ctx.h, 1 if sequential else 0))
    L = np.zeros((nc + 1, npiv), order="F")
    M = np.zeros((N, npiv), order="F")
    LS = np.full((npiv, npiv), np.nan, order="F")
    Y = np.zeros((N, npiv), order="F")
    w = np.zeros(npiv)
    chi2 = C.c_double(0.0)
    gate = C.c_int(-1)
    info = np.zeros(1, dtype=np.int32)
    ctx._ck(ctx.lib.ovp_debug_chol_pair(ctx.h, _p(G), nc, npiv, C.c_double(TOL), _p(P), N, _p(cols), C.c_double(gate_thresh), _p(L), _p(M),
                                        _p(LS), _p(Y), _p(w), C.byref(chi2), C.byref(gate), _p(info),
                                        None if timeline is None else _p(timeline)))
    ctx._ck(ctx.lib.ovp_debug_sequential_factorisations(ctx.h, 0))
    return (L, M, LS, Y, w, np.array([chi2.value]), np.array([gate.value])), bool(info[0])


def same_bits(a, b, tag):
    for name, x, y in zip(("L", "M", "L_S", "Y", "w", "chi2", "gate"), a, b):
        assert np.array_equal(np.ascontiguousarray(x).view(np.uint8), np.ascontiguousarray(y).view(np.uint8)), "%s: %s differs" % (tag, name)


# 1, 2, 7 and 8 block columns; ragged last blocks, a z row alone in its block row (nc = 128), fewer pivots than columns, zero pivots
@pytest.mark.parametrize("nc,npiv,N,zero_cols", [(40, 40, 100, (3,)), (63, 60, 64, ()), (100, 97, 200, (7,)), (128, 128, 130, (64,)),
                                                 (420, 417, 512, (5, 300)), (473, 470, 512, (5, 130, 300)), (470, 470, 512, ())])
def test_pair_matches_two_launches(ctx, nc, npiv, N, zero_cols):
    G, P, cols = make_system(nc * 3 + N, nc, npiv, N, zero_cols)
    seq, paired_seq = run_pair(ctx, G, nc, npiv, P, cols, True)
    assert not paired_seq
    # one gate each way: above and below the update's chi2
    for thresh in (2.0 * seq[5][0], 0.5 * seq[5][0]):
        ref, _ = run_pair(ctx, G, nc, npiv, P, cols, True, thresh)
        got, paired = run_pair(ctx, G, nc, npiv, P, cols, False, thresh)
        assert paired, "a %d-column system with %d rows of M fits a pair on this device" % (nc + 1, N)
        same_bits(ref, got, "nc=%d npiv=%d N=%d thresh=%g" % (nc, npiv, N, thresh))
    assert got[6][0] == 0 and ref[6][0] == 0


def test_wide_pair_takes_two_launches(ctx):
    """691 columns: 66 + 66 tiles leave no SM of an H100 for the product-only CTAs of a pair, so the update runs the two
    factorisations one after the other (and still gives their bits)."""
    G, P, cols = make_system(3, 690, 690, 700, zero_cols=(17,))
    ref, _ = run_pair(ctx, G, 690, 690, P, cols, True)
    got, paired = run_pair(ctx, G, 690, 690, P, cols, False)
    assert not paired
    same_bits(ref, got, "wide")


def test_two_filters_pair_concurrently(ctx):
    """Two contexts' pairs at the same time (each its own stream, workspaces and counters) give their solo results."""
    other = _ctx()
    try:
        sys_a = make_system(21, 473, 470, 512, zero_cols=(9,))
        sys_b = make_system(22, 470, 470, 512)
        solo_a, pa = run_pair(ctx, sys_a[0], 473, 470, sys_a[1], sys_a[2], False)
        solo_b, pb = run_pair(other, sys_b[0], 470, 470, sys_b[1], sys_b[2], False)
        assert pa and pb
        res = {}

        def work(key, c, s, nc):
            res[key] = [run_pair(c, s[0], nc, 470, s[1], s[2], False)[0] for _ in range(4)]

        th = [threading.Thread(target=work, args=("a", ctx, sys_a, 473)), threading.Thread(target=work, args=("b", other, sys_b, 470))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        for key, solo in (("a", solo_a), ("b", solo_b)):
            for r in res[key]:
                same_bits(solo, r, key)
    finally:
        other.close()


def _state(ctx):
    vals = [ctx.var_get(int(h)) for h in ctx.variable_order()]
    return ctx.cov(), np.concatenate([np.concatenate([v, f]) for v, f in vals])


def _bits_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def test_cfg3_step_paired_and_sequential(chi2_table):
    """The benchmarked step (8 plane updates + the point update) paired and in two launches per update: P+, every variable value, the
    chi2 values and the gates carry the same bits, with as many launches."""
    S = synth.make_scenario("cfg3_n512_f600_p8", seed=0)
    runs = {}
    for seq in (1, 0):
        ctx = api.Context(S.options, device=0, max_state=S.N + 64, max_meas_rows=60000, debug=True)
        ctx.set_chi2_table(chi2_table)
        ch = synth.load_scenario_into(ctx, S)
        ctx._ck(ctx.lib.ovp_debug_sequential_factorisations(ctx.h, seq))
        l0 = ctx.launch_count()
        g = ctx.msckf_update(synth.feature_batch(S, ch), 1.0, 1.0)
        runs[seq] = (g, _state(ctx), ctx.launch_count() - l0)
        ctx.close()
    (g0, s0, l0), (g1, s1, l1) = runs[0], runs[1]
    for k in g0:
        assert _bits_equal(g0[k], g1[k]), k
    assert _bits_equal(s0[0], s1[0]) and _bits_equal(s0[1], s1[1])
    assert l1 == l0


def test_slam_update_paired_and_sequential(chi2_table):
    """UpdaterSLAM's delayed initialisation and update of 20 landmarks on the benchmark's state, paired and in two launches per
    compressed update: the same bits everywhere."""
    S = synth.make_scenario("cfg3_n512_f600_p8", seed=0)
    out = {}
    for seq in (1, 0):
        ctx = api.Context(S.options, device=0, max_state=S.N + 3 * 20 + 64, max_meas_rows=60000, debug=True)
        ctx.set_chi2_table(chi2_table)
        ch = synth.load_scenario_into(ctx, S)
        ctx._ck(ctx.lib.ovp_debug_sequential_factorisations(ctx.h, seq))
        g = ctx.slam_delayed_init(synth.feature_batch(S, ch, np.arange(20)), 1.0, 1.0)
        keep = np.nonzero(g["feat_status"] > 0)[0]
        ub = synth.feature_batch(S, ch, keep)
        ub["uv"] = ub["uv"] + np.random.default_rng(7).normal(0.0, 0.5, ub["uv"].shape).astype(np.float32)
        g2 = ctx.slam_update(ub, 1.0, 1.0)
        out[seq] = (g, g2, _state(ctx))
        ctx.close()
    (a0, b0, s0), (a1, b1, s1) = out[0], out[1]
    assert (b0["feat_status"] == 1).any()
    for x, y in ((a0, a1), (b0, b1)):
        for k in x:
            assert _bits_equal(x[k], y[k]), k
    assert _bits_equal(s0[0], s1[0]) and _bits_equal(s0[1], s1[1])
