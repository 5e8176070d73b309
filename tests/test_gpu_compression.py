"""The three stages of a compressed update, element by element against long-double NumPy references:

1. the Gram matrix G = [H_o r_o]^T [H_o r_o] of the nullspace-projected system (block-sparse path: msckf_feature_warp_kernel,
   gram_dpart_kernel, gram_kernel, gram_reduce_sparse_kernel; dense path: feature_kernel, gram_kernel, gram_reduce_kernel), through
   ovp_debug_msckf_gram.  The reference starts from the raw whitened blocks the feature kernel itself built (a one-ulp change of H_f moves
   the projected dense entries by more than the accuracy checked here), projects each accepted feature's block onto the left null space
   of its H_f with a 3-reflector Householder QR in long double, and sums (P_N X)^T (P_N X) over the feature's own columns.  The error is
   Jacobi-scaled, |G - G_ref|_ij / sqrt(G_ref,ii G_ref,jj), and bounded per class of columns: clone x clone, dense x clone and dense x
   dense (dense: calibration, H_cp and the residual);
2. the zero-pivot rule of the Gram factorisation (chol_fused_kernel): a pivot is zeroed when it is <= tol times the column's ORIGINAL
   diagonal.  The planted columns sit at the 16-column panel and 64-column tile boundaries, and pivots of 0.5x and 2x the threshold;
3. the innovation launch: S = L L^T, Y = M L^-T, w = L^-1 z with z read in place at the compressed update's stride, chi2 = |w|^2 and the
   gate flag, with element-wise backward-error bounds.

End to end, the point and in-state plane updates with 0 and 8 calibration columns are compared with the oracle."""
import ctypes as C

import numpy as np
import pytest

from conftest import make_pair
from ov_plane_b200 import api, synth
from gate_reference import householder_q3
from test_gpu_parity import _check_msckf, oracle_msckf_update, relerr

pytestmark = pytest.mark.gpu

LD = np.longdouble
EPS = 2.0 ** -53
RAW_ROW = 24  # OVP_RAW_ROW (features.cu): doubles per raw row, 3 rows per measurement
# Bounds of the Jacobi-scaled error of G per column class: the worst error measured over the cases below on an H100 80GB HBM3 (700 W),
# times 3 to 10 (DESIGN.md §6).  Measured: 1.5e-15, 9.7e-15 and 1.0e-14; with tracks of 2 (one projected row per feature: P_N removes
# three of the four rows, so G's diagonal is small next to |x|^2) 2.5e-14, 2.9e-14 and 5.8e-15.  Forming the dense entries by the
# subtractive x_d^T x_e - y_d^T y_e instead costs (|x| / |P_N x|)^2 in accuracy (2.7e-13 at the benchmark's sizes, DESIGN.md §4.2).
GRAM_TOL = {"clone x clone": 1.5e-14, "dense x clone": 5e-14, "dense x dense": 5e-14}
GRAM_TOL_ONE_ROW = {"clone x clone": 1e-13, "dense x clone": 1e-13, "dense x dense": 3e-14}


def _p(x):
    return None if x is None else x.ctypes.data_as(C.c_void_p)


def _require_long_double():
    assert np.finfo(np.longdouble).eps < 1e-18, "the references need an extended-precision long double"


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. Gram matrix
# ---------------------------------------------------------------------------------------------------------------------------------
def run_gram(ctx, batch, dense, sigma_pix=1.0, chi2_mult=1.0):
    """ovp_debug_msckf_gram on one batch: G, the plan's layout, statuses and the raw rows of every measurement."""
    fb, keep = api.Context._batch_struct(batch)
    uo = api.UpdaterOptions(sigma_pix, chi2_mult)
    F, M = fb.F, int(batch["meas_offset"][-1])
    gcap = ctx.cov_rows() + 4
    G = np.zeros(gcap * gcap)
    info = np.zeros(8, dtype=np.int32)
    cols = np.zeros(gcap, dtype=np.int32)
    sel = np.zeros(F, dtype=np.int32)
    fs, fc = np.zeros(F, dtype=np.int32), np.zeros(F)
    raw = np.zeros(3 * RAW_ROW * M)
    ctx._ck(ctx.lib.ovp_debug_force_dense_features(ctx.h, int(dense)))
    ctx._ck(ctx.lib.ovp_debug_msckf_gram(ctx.h, C.byref(fb), C.byref(uo), gcap, _p(G), _p(info), _p(cols), _p(sel), _p(fs), _p(fc), _p(raw)))
    nc1, ncal, ncx, is_point, nsel, fast, plane_slot, in_state = (int(v) for v in info)
    assert bool(fast) == (not dense), "the batch did not take the path asked for"
    return dict(G=G[:nc1 * nc1].reshape((nc1, nc1), order="F").copy(), nc1=nc1, ncal=ncal, ncx=ncx, is_point=bool(is_point),
                sel=sel[:nsel].copy(), status=fs, chi2=fc, raw=raw.reshape(M, 3, RAW_ROW), plane_slot=plane_slot, in_state=bool(in_state),
                cols=cols[:ncx].copy())


def feature_block(r, batch, f):
    """The kernel's raw rows of feature f as [H_f | calibration | 6 per measurement's clone | H_cp (plane) | r], in long double."""
    a, b = int(batch["meas_offset"][f]), int(batch["meas_offset"][f + 1])
    m, ncal, plane = b - a, r["ncal"], not r["is_point"]
    ncol = 3 + ncal + 6 * m + (3 if plane else 0) + 1
    X = np.zeros((3 * m if plane else 2 * m, ncol), dtype=LD)
    for k in range(m):
        for i in range(2):
            row = r["raw"][a + k, i]
            X[2 * k + i, :3] = row[:3]
            X[2 * k + i, 3:3 + ncal] = row[9:9 + ncal]
            X[2 * k + i, 3 + ncal + 6 * k:3 + ncal + 6 * k + 6] = row[3:9]
            X[2 * k + i, -1] = row[RAW_ROW - 1]
        if plane:
            row = r["raw"][a + k, 2]
            X[2 * m + k, :3] = row[:3]
            X[2 * m + k, -4:-1] = row[9:12]
            X[2 * m + k, -1] = row[RAW_ROW - 1]
    return X


def gram_reference(r, batch, var_id):
    """sum over the plan's accepted features of (P_N X)^T (P_N X), scattered to the compact columns (long double)."""
    nc1, ncal, ncx = r["nc1"], r["ncal"], r["ncx"]
    col_of = {int(s): c for c, s in enumerate(r["cols"])}  # state index -> compact column
    Gr = np.zeros((nc1, nc1), dtype=LD)
    for f in r["sel"]:
        if r["is_point"] and r["status"][f] != 1:
            continue
        X = feature_block(r, batch, f)
        a, b = int(batch["meas_offset"][f]), int(batch["meas_offset"][f + 1])
        Q = householder_q3(X[:, :3])
        Y = X[:, 3:]
        Z = Y - Q @ (Q.T @ Y)
        idx = list(range(ncal))
        for k in range(a, b):
            c0 = col_of[var_id(int(batch["meas_clone"][k]))]
            idx += list(range(c0, c0 + 6))
        if not r["is_point"]:
            idx += [ncx, ncx + 1, ncx + 2]
        idx.append(nc1 - 1)
        Gr[np.ix_(idx, idx)] += Z.T @ Z
    return Gr


def column_classes(r):
    nc1, ncal, ncx = r["nc1"], r["ncal"], r["ncx"]
    dense = np.ones(nc1, dtype=bool)
    dense[ncal:ncx] = False
    return dense


def check_gram(tag, r, Gr, tol):
    G = r["G"]
    assert np.all(np.isfinite(G)), tag
    assert np.all(np.triu(G, 1) == 0.0), "%s: strictly upper part of G not zero" % tag
    d = np.sqrt(np.maximum(np.diag(Gr).astype(np.float64), 0.0))
    den = np.outer(d, d)
    err = np.abs(G.astype(LD) - Gr).astype(np.float64)
    low = np.tril(np.ones_like(G, dtype=bool))
    zero = den == 0.0
    assert np.all(err[low & zero] == 0.0), "%s: an entry of a column no accepted feature touches is not zero" % tag
    scaled = np.where(zero, 0.0, err / np.where(zero, 1.0, den))
    dense = column_classes(r)
    cls = {"clone x clone": np.outer(~dense, ~dense), "dense x clone": np.outer(dense, ~dense) | np.outer(~dense, dense),
           "dense x dense": np.outer(dense, dense)}
    worst = {}
    for name, mask in cls.items():
        m = mask & low
        worst[name] = float(scaled[m].max()) if m.any() else 0.0
    print("%s: nc1 %d ncal %d, worst Jacobi-scaled error of G: %s" % (tag, r["nc1"], r["ncal"],
                                                                       ", ".join("%s %.2e (/ bound %.3f)" % (k, v, v / tol[k])
                                                                                 for k, v in worst.items())))
    for name, v in worst.items():
        assert v <= tol[name], "%s: %s error %.3e above %.1e" % (tag, name, v, tol[name])
    return worst


def check_raw_against_oracle(r, batch, S, orc, cho, chg, nfeat=4):
    """The raw rows against the oracle's feature_jacobian_full (test_gpu_parity.py::test_feature_jacobian_full's tolerance)."""
    handle_of = {h: cho[i] for i, h in enumerate(chg)}
    pf_all = batch["p_FinG_original"] if r["is_point"] else batch["p_FinG"]
    for f in list(r["sel"][:nfeat]) + list(r["sel"][-1:]):
        if r["is_point"] and r["status"][f] == 2:
            continue
        a, b = int(batch["meas_offset"][f]), int(batch["meas_offset"][f + 1])
        X = feature_block(r, batch, f).astype(np.float64)
        pid, cp, cpf = 0, None, None
        if not r["is_point"] and r["in_state"]:
            pid = int(batch["plane_ids"][r["plane_slot"]])
            cp, cpf = orc.var_get(orc.plane_handle(pid))
        o = orc.feature_jacobian_full([handle_of[int(h)] for h in batch["meas_clone"][a:b]], batch["uv"][a:b], pf_all[f], pf_all[f], pid,
                                      cp, cpf, 1.0, S.options["sigma_constraint"])
        rows = o[0].shape[0]
        if pid == 0:  # the bearing rows alone: [H_f | calibration | clones | r]
            X = np.hstack([X[:2 * (b - a), :3 + r["ncal"] + 6 * (b - a)], X[:2 * (b - a), -1:]])
        assert X.shape[0] == rows and X.shape[1] == 3 + o[1].shape[1] + 1, (X.shape, [x.shape for x in o[:3]])
        for k, (got, ref) in enumerate(((X[:, :3], o[0]), (X[:, 3:-1], o[1]), (X[:, -1], o[2]))):
            assert relerr(got, ref) < 1e-11, ("raw block of feature %d, part %d: %.3e" % (f, k, relerr(got, ref)))


def debug_pair(S, chi2, max_state):
    """make_pair with the GPU context on libovp_debug.so"""
    import oracle_backend
    ctx = api.Context(S.options, device=0, max_state=max_state, max_meas_rows=60000, debug=True)
    ctx.set_chi2_table(chi2)
    orc = oracle_backend.OracleContext(S.options)
    orc.set_chi2_table(chi2)
    return ctx, orc, synth.load_scenario_into(ctx, S), synth.load_scenario_into(orc, S)


def add_outliers(S, feats, px=30.0):
    """one measurement of each feature moved by px pixels: the gate rejects the feature"""
    for f in feats:
        k = (S.meas_offset[f] + S.meas_offset[f + 1]) // 2
        S.uv[k] += np.float32(px) * np.array([1.0, -1.0], dtype=np.float32)


def _scenario(case):
    """Scenarios of the Gram cases; rows of every compressed plan exceed the innovation workspace of a context of max_state = N + 8,
    so every plan forms its Gram matrix."""
    kind, ncal = case
    cal = {0: (0, 0), 6: (1, 0), 8: (0, 1), 14: (1, 1)}[ncal]
    ov = dict(calib_pose=cal[0], calib_intr=cal[1])
    if kind == "points":  # 61 features (not a multiple of 4 or 32), some rejected by the gate
        S = synth.make_scenario("tiny_points", seed=1, n_clones=14, F=61, m_min=3, m_max=14, dtheta=0.02, **ov)
        add_outliers(S, [3, 17, 40, 60])
    elif kind == "plane_in_state":
        S = synth.make_scenario("tiny_planes", seed=1, F=70, **ov)
    elif kind == "plane_not_in_state":
        S = synth.make_scenario("tiny_planes", seed=1, F=70, **ov)
        synth.drop_planes_from_state(S)
    elif kind == "tracks_of_2":  # one projected row per feature
        S = synth.make_scenario("tiny_points", seed=2, n_clones=10, F=197, m_min=2, m_max=2, dtheta=0.02, **ov)
    elif kind == "tracks_of_32":
        S = synth.make_scenario("tiny_points", seed=3, n_clones=34, F=37, m_min=32, m_max=32, dtheta=0.006, **ov)
    elif kind == "tracks_33_39":  # longer than a warp: the one-CTA-per-feature kernel
        S = synth.make_scenario("tiny_points", seed=4, n_clones=40, F=23, m_min=33, m_max=39, dtheta=0.005, **ov)
    elif kind == "cfg3_points":  # the benchmark's point plan: gram_kernel splits k, Dddp has 19 chunks
        S = synth.make_scenario("cfg3_n512_f600_p8", seed=0)
        S.planeid[:] = 0
    return S


GRAM_CASES = ([(("points", n), d) for n in (0, 6, 8, 14) for d in (0, 1)] +
              [((k, n), d) for k in ("plane_in_state", "plane_not_in_state") for n in (0, 14) for d in (0, 1)] +
              [(("tracks_of_2", 14), d) for d in (0, 1)] + [(("tracks_of_32", 8), d) for d in (0, 1)] + [(("tracks_33_39", 6), 1)] +
              [(("cfg3_points", 14), d) for d in (0, 1)])


@pytest.mark.parametrize("case,dense", GRAM_CASES, ids=["%s-ncal%d-%s" % (c[0], c[1], "dense" if d else "warp") for c, d in GRAM_CASES])
def test_gram_matrix_against_long_double_reference(case, dense, chi2_table):
    _require_long_double()
    S = _scenario(case)
    big = case[0] == "cfg3_points"
    ctx, orc, chg, cho = debug_pair(S, chi2_table, S.N + (64 if big else 8))
    batch = synth.feature_batch(S, chg)
    P0 = ctx.cov()
    r = run_gram(ctx, batch, dense)
    assert r["is_point"] == (case[0] not in ("plane_in_state", "plane_not_in_state"))
    assert r["ncal"] == case[1]
    if case[0] == "points":
        assert (r["status"][r["sel"]] == 0).sum() >= 2 and (r["status"][r["sel"]] == 1).sum() > 30, "the gate should reject a few features"
    if case[0].startswith("plane"):
        assert r["in_state"] == (case[0] == "plane_in_state")
    check_raw_against_oracle(r, batch, S, orc, cho, chg)
    Gr = gram_reference(r, batch, ctx.var_id)
    check_gram("%s ncal=%d %s" % (case[0], case[1], "dense" if dense else "warp"), r, Gr,
               GRAM_TOL_ONE_ROW if case[0] == "tracks_of_2" else GRAM_TOL)
    again = run_gram(ctx, batch, dense)
    assert np.array_equal(r["G"].view(np.uint64), again["G"].view(np.uint64)), "G differs run to run"
    assert np.array_equal(P0.view(np.uint64), ctx.cov().view(np.uint64)), "forming G changed the covariance"
    # the state is untouched: a full update afterwards still matches the oracle
    if case[0] == "points":
        ctx._ck(ctx.lib.ovp_debug_force_dense_features(ctx.h, 0))
        g = ctx.msckf_update(batch, 1.0, 1.0)
        o = oracle_msckf_update(orc, synth.feature_batch(S, cho), 1.0, 1.0)
        _check_msckf(S, ctx, orc, chg, cho, g, o)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. zero-pivot rule
# ---------------------------------------------------------------------------------------------------------------------------------
ZTOL = 1e-8  # large enough that the round-off of G (~1e-13 of a diagonal) cannot move a planted pivot across the threshold


def _ctx(max_state=1024):
    S = synth.make_scenario("tiny_points")
    return api.Context(S.options, device=0, max_state=max_state, max_meas_rows=4096, debug=True)


@pytest.fixture(scope="module")
def ctx():
    c = _ctx()
    yield c
    c.close()


def planted_gram(n, seed):
    """G = H^T H with exactly dependent columns at the panel / tile boundaries and the last pivoted column (n - 2; column n - 1 is the
    right-hand-side row of the compressed update), and columns whose pivot is 0.5x (zeroed) or 2x (kept) tol times their diagonal, in
    block columns >= 1."""
    rng = np.random.default_rng(seed)
    npiv = n - 1
    m = 2 * n + 8
    H = rng.standard_normal((m, n))
    dep = sorted(j for j in {0, 15, 16, 63, 64, 127, 128, npiv - 1} if j < npiv)
    near = {j: f for j, f in zip((70, 100, 143, 200, 381, 700, 901), (0.5, 2.0, 0.5, 2.0, 0.5, 2.0, 0.5)) if j < npiv - 1 and j not in dep}
    for j in range(npiv):
        if j in dep or j in near:
            acc = [k for k in range(j) if k not in dep and near.get(k, 2.0) != 0.5]
            c = np.zeros(j)
            if acc:
                pick = rng.choice(acc, size=min(3, len(acc)), replace=False)
                c[pick] = rng.choice([0.5, -1.25, 1.0, 2.0], size=len(pick))
            h = H[:, :j] @ c if j else np.zeros(m)
            if j in near:
                q = rng.standard_normal(m)
                B = H[:, :j]
                for _ in range(2):
                    q -= B @ np.linalg.lstsq(B, q, rcond=None)[0]
                q /= np.linalg.norm(q)
                s = h @ h
                p = near[j] * ZTOL * s / (1.0 - near[j] * ZTOL)
                h = h + np.sqrt(p) * q
            H[:, j] = h
    G = H.T @ H
    zero = sorted(dep + [j for j, f in near.items() if f == 0.5])
    return G, npiv, zero, near


def ld_factor(G, npiv, tol):
    """Right-looking Cholesky in long double with the zero-pivot rule (pivot <= tol * original diagonal -> zero column); returns the zeroed
    columns and each pivot over its threshold."""
    A = np.tril(G).astype(LD)
    A = A + np.tril(A, -1).T
    d0 = np.diag(G).astype(LD).copy()
    zero, ratio = [], {}
    for j in range(npiv):
        d = A[j, j]
        ratio[j] = float(d / (tol * d0[j])) if d0[j] > 0 else 0.0
        if not d > tol * d0[j]:
            zero.append(j)
            continue
        l = A[j:, j] / np.sqrt(d)
        A[j:, j:] -= np.outer(l, l)
    return zero, ratio


def check_factor(tag, G, L, npiv, zero, n):
    """Exactly the planted columns zeroed (every row), and |G - L L^T| <= 2 (n + 1) eps |L| |L^T| element-wise on the kept columns."""
    Lp = L[:, :npiv]
    got = [j for j in range(npiv) if Lp[j, j] == 0.0]
    assert got == zero, "%s: zeroed columns %s, expected %s" % (tag, got, zero)
    assert np.all(Lp[:, zero] == 0.0), "%s: a zeroed column has a non-zero entry" % tag
    keep = np.ones(npiv, dtype=bool)
    keep[zero] = False
    Lk = Lp.astype(LD)
    R = np.abs(np.tril(G)[:, :npiv].astype(LD) - Lk @ Lk[:npiv].T).astype(np.float64)
    bnd = 2.0 * (n + 1) * EPS * (np.abs(Lp) @ np.abs(Lp[:npiv]).T)
    mask = np.tril(np.ones((n, npiv), dtype=bool)) & keep[None, :]
    ratio = float((R[mask] / np.maximum(bnd[mask], 1e-300)).max())
    assert np.all(R[mask] <= bnd[mask]), "%s: |G - L L^T| above its element-wise bound (worst ratio %.2f)" % (tag, ratio)
    return ratio


def chol_solve(c, A, npiv, tol, M=None, z=None, zstride=0, thresh=-1.0):
    n = A.shape[0]
    A = np.asfortranarray(np.tril(A))
    L = np.zeros((n, n), order="F")
    Y = w = None
    mrows = 0
    chi2, gate = np.zeros(1), np.full(1, -7, dtype=np.int32)
    if M is not None:
        M = np.asfortranarray(M)
        z = np.ascontiguousarray(z)
        mrows = M.shape[0]
        Y, w = np.zeros((mrows, npiv), order="F"), np.zeros(npiv)
    c._ck(c.lib.ovp_debug_chol_solve_gated(c.h, _p(A), n, npiv, C.c_double(tol), _p(M), mrows, _p(z), zstride, C.c_double(thresh), _p(L),
                                           _p(Y), _p(w), _p(chi2) if M is not None else None, _p(gate) if M is not None else None))
    return np.tril(L), Y, w, chi2[0], int(gate[0])


def _planted(n, seed):
    _require_long_double()
    G, npiv, zero, near = planted_gram(n, seed)
    ref_zero, ratio = ld_factor(G, npiv, ZTOL)
    assert ref_zero == zero, "planted system: the long-double factorisation zeroes %s, planted %s" % (ref_zero, zero)
    for j, f in near.items():  # the planted pivots sit where they were put (G's round-off is far below the threshold)
        assert abs(ratio[j] / f - 1.0) < 0.01, (j, f, ratio[j])
    return G, npiv, zero


@pytest.mark.parametrize("n", [150, 300, 960])
def test_zero_pivot_rule_on_planted_columns(ctx, n):
    """Single launch (n = 150, 300) and the two-launch fallback (n = 960: 959 pivoted columns with 700 right-hand-side rows need more
    CTAs than an H100 holds at once); with a right-hand side the zeroed columns of Y and w are exactly zero."""
    G, npiv, zero = _planted(n, n)
    rng = np.random.default_rng(n + 1)
    M = rng.standard_normal((700 if n > 900 else 90, npiv))
    z = rng.standard_normal(npiv)
    L, Y, w, _, _ = chol_solve(ctx, G, npiv, ZTOL, M, z)
    ratio = check_factor("n=%d" % n, G, L, npiv, zero, n)
    assert np.all(Y[:, zero] == 0.0) and np.all(w[zero] == 0.0)
    print("zero-pivot rule n=%d: zeroed %s, worst |G - LL^T| / bound %.3f" % (n, zero, ratio))


def test_zero_pivot_rule_does_not_read_a_stale_diagonal(ctx):
    """The original diagonal of block columns >= 1 reaches the spine through a buffer that is not cleared between launches: a second
    system with a very different diagonal right after the first, on the same context, must take the same decisions.  (D G D keeps
    every pivot's ratio to its diagonal.)"""
    G, npiv, zero = _planted(300, 11)
    n = G.shape[0]
    rng = np.random.default_rng(12)
    d = np.where(rng.random(n) < 0.5, 1e-3, 1e3) * (1.0 + rng.random(n))
    G2 = G * np.outer(d, d)
    assert ld_factor(G2, npiv, ZTOL)[0] == zero
    for A in (G, G2, G, G2):
        L, _, _, _, _ = chol_solve(ctx, A, npiv, ZTOL)
        check_factor("scaled" if A is G2 else "plain", A, L, npiv, zero, n)


def test_zero_pivot_rule_in_the_launch_that_forms_the_update_products(ctx):
    """ovp_debug_chol_products: the factorisation that also forms M and S takes the same decisions."""
    G, npiv, zero = _planted(300, 21)
    nc = G.shape[0] - 1
    N = 400
    rng = np.random.default_rng(22)
    A = rng.standard_normal((N, N))
    P = np.asfortranarray(A @ A.T / N + np.eye(N))
    cols = np.ascontiguousarray(np.sort(rng.choice(N, size=nc, replace=False)), dtype=np.int32)
    L = np.zeros((nc + 1, npiv), order="F")
    Mo = np.zeros((N, npiv), order="F")
    So = np.zeros((npiv, npiv), order="F")
    Gf = np.asfortranarray(np.tril(G))
    ctx._ck(ctx.lib.ovp_debug_chol_products(ctx.h, _p(Gf), nc, npiv, C.c_double(ZTOL), _p(P), N, _p(cols), _p(L), _p(Mo), _p(So)))
    check_factor("products", G, L, npiv, zero, nc + 1)
    assert np.all(Mo[:, zero] == 0.0)


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. innovation launch
# ---------------------------------------------------------------------------------------------------------------------------------
def _elementwise(tag, resid, bound):
    ratio = float((resid / np.maximum(bound, 1e-300)).max())
    assert np.all(resid <= bound), "%s: worst residual / bound %.2f" % (tag, ratio)
    return ratio


@pytest.mark.parametrize("n", [1, 16, 17, 64, 65, 470, 960])
def test_innovation_launch_backward_errors_chi2_and_gate(ctx, n):
    """S = L L^T, Y = M L^-T and w = L^-1 z with z read at the compressed update's stride, element-wise backward errors
    (c = 2: |S - L L^T| <= 2 (n + 1) eps |L| |L^T| and likewise for M^T = L Y^T and z = L w), chi2 = |w|^2 to n eps, and the gate
    flag exact at thresholds below, at and just above chi2 and without a gate.  n = 960 with 700 rows runs as two launches."""
    _require_long_double()
    rng = np.random.default_rng(1000 + n)
    B = rng.standard_normal((n + 8, n)) * rng.uniform(0.1, 10.0, size=n)
    Sm = B.T @ B + np.eye(n)
    mrows = 700 if n == 960 else 37 + n % 29
    M = rng.standard_normal((mrows, n))
    z = rng.standard_normal(n) * 3.0
    L, Y, w, chi2, gate = chol_solve(ctx, Sm, n, 0.0, M, z, zstride=0)
    assert gate == 1
    c = 2.0 * (n + 1) * EPS
    Ll = L.astype(LD)
    low = np.tril(np.ones((n, n), dtype=bool))
    rS = _elementwise("S", np.abs(np.tril(Sm).astype(LD) - Ll @ Ll.T).astype(np.float64)[low], (c * (np.abs(L) @ np.abs(L).T))[low])
    rM = _elementwise("M", np.abs(M.T.astype(LD) - Ll @ Y.T.astype(LD)).astype(np.float64), c * (np.abs(L) @ np.abs(Y).T))
    rz = _elementwise("z", np.abs(z.astype(LD) - Ll @ w.astype(LD)).astype(np.float64), c * (np.abs(L) @ np.abs(w)))
    ww = (w.astype(LD) ** 2).sum()
    assert abs(LD(chi2) - ww) <= n * EPS * ww, (chi2, float(ww))
    # the strided read must agree with the contiguous one bit for bit
    L1, Y1, w1, chi21, _ = chol_solve(ctx, Sm, n, 0.0, M, z, zstride=1)
    assert np.array_equal(w1.view(np.uint64), w.view(np.uint64)) and chi21 == chi2
    for thr, want in ((np.nextafter(chi2, 0.0), 0), (chi2, 1), (np.nextafter(chi2, np.inf), 1), (-1.0, 1), (0.5 * chi2, 0)):
        _, _, _, c2, g = chol_solve(ctx, Sm, n, 0.0, M, z, zstride=0, thresh=thr)
        assert c2 == chi2, "chi2 differs run to run"
        assert g == want, "gate flag %d at threshold %r for chi2 %r, expected %d" % (g, thr, chi2, want)
    print("innovation n=%d: worst residual / bound  S %.3f  M %.3f  z %.3f" % (n, rS, rM, rz))


# ---------------------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,ncal", [("cfg2_n256_f200", 0), ("cfg2_n256_f200", 8), ("small_planes", 0), ("small_planes", 8)])
def test_msckf_update_without_and_with_intrinsics_only_calibration(name, ncal, chi2_table):
    """Points (compressed: 200 features) and in-state planes with no calibration columns and with the 8 intrinsics alone, against the
    oracle at the tolerances of test_gpu_parity.py."""
    S = synth.make_scenario(name, seed=0, calib_pose=0, calib_intr=1 if ncal == 8 else 0)
    ctx, orc, chg, cho = make_pair(S, chi2_table)
    g = ctx.msckf_update(synth.feature_batch(S, chg), 1.0, 1.0)
    o = oracle_msckf_update(orc, synth.feature_batch(S, cho), 1.0, 1.0)
    e = _check_msckf(S, ctx, orc, chg, cho, g, o, chi_tol=1e-6 if S.cfg["n_planes"] else 1e-7)
    print("%s ncal=%d: cov rel err %.2e, accepted %d of %d" % (name, ncal, e, int((g["feat_status"] == 1).sum()), S.F))
    ctx.close()
