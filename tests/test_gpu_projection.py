"""householder_cols_kernel through ovp_nullspace_project_inplace / ovp_plane_nullspace_project_inplace, against a long-double Householder
QR with the kernel's sign convention (tests/update_reference.py).  With that convention the reflectors of a full-column-rank H_f are
unique, so the returned rows are compared element by element with rows [k:] of H_k ... H_1 [H_f | H_x (| H_cp) | r], each column j
within c rows eps kappa(H_f) |X_j|_2.

Shapes: H_f of 1, 2 and 3 columns; rows = hf_cols (nothing returned); rows around the 32-lane norm loop (31 .. 65); 255, 256 and 257
columns in all (the 256-thread column loop); 6142, 6143 and 20000 rows (a kernel that kept the reflector in dynamic shared memory had
its launch refused from 6142 rows on and returned the rows unprojected); every shape with and without the plane's H_cp columns.  A zero column of H_f is skipped (identity reflector); a column parallel
to another leaves a reflector set by round-off, so that case checks the invariants instead of the rows."""
import numpy as np
import pytest

import update_reference as ur
from ov_plane_b200 import api

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = api.Context(ur.STATE_OPTIONS, device=0, max_state=64, max_meas_rows=1024)
    yield c
    c.close()


def system(rows, hf, hx, plane, seed):
    rng = np.random.default_rng(seed)
    Hf = rng.standard_normal((rows, hf))
    Hx = rng.standard_normal((rows, hx)) * np.exp(rng.uniform(-3, 3, hx))  # columns of different scales: the bound is per column
    Hcp = rng.standard_normal((rows, 3)) if plane else None
    r = rng.standard_normal(rows)
    return Hf, Hx, Hcp, r


def project(ctx, Hf, Hx, Hcp, r):
    """The library's projection as one matrix [H_x (| H_cp) | r] of rows - hf_cols rows."""
    if Hcp is None:
        ox, orr = ctx.nullspace_project_inplace(Hf, Hx, r)
        return np.column_stack([ox, orr])
    ox, ocp, orr = ctx.nullspace_project_inplace(Hf, Hx, r, Hcp)
    return np.column_stack([ox, ocp, orr])


def check_rows(ctx, Hf, Hx, Hcp, r, bound_cols=None):
    k = Hf.shape[1]
    X = np.column_stack([Hx] + ([Hcp] if Hcp is not None else []) + [r])
    got = project(ctx, Hf, Hx, Hcp, r)
    assert got.shape == (Hf.shape[0] - k, X.shape[1])
    ref = ur.householder_project(np.column_stack([Hf, X]), k)[k:, k:]
    bound = ur.projection_bound(Hf if bound_cols is None else Hf[:, bound_cols], X)
    err = np.abs(got.astype(ur.LD) - ref).max(axis=0).astype(np.float64) if got.size else np.zeros(X.shape[1])
    assert np.all(err <= bound), "worst column error / bound %.3e (rows %d, hf_cols %d)" % ((err / bound).max(), Hf.shape[0], k)
    return float((err / bound).max()) if got.size else 0.0


SHAPES = [(hf, rows, 12) for hf in (1, 2, 3) for rows in sorted({hf, 31, 32, 33, 63, 64, 65})]
SHAPES += [(3, 300, total - 4) for total in (255, 256, 257)]  # [H_f | H_x | r] of 255 .. 257 columns (the plane variant: + 3)
SHAPES += [(3, rows, 20) for rows in (6142, 6143, 20000)]


@pytest.mark.parametrize("plane", [False, True], ids=["plain", "plane"])
@pytest.mark.parametrize("hf,rows,hx", SHAPES)
def test_projection_against_long_double(ctx, hf, rows, hx, plane):
    ur.require_long_double()
    if plane and hx > 12 and rows == 300:
        hx -= 3  # the same 255 .. 257 columns in all
    Hf, Hx, Hcp, r = system(rows, hf, hx, plane, seed=rows * 10 + hf)
    q = check_rows(ctx, Hf, Hx, Hcp, r)
    print("hf_cols %d rows %d columns %d %s: worst error / bound %.3e" % (hf, rows, hf + hx + (3 if plane else 0) + 1,
                                                                          "plane" if plane else "plain", q))


@pytest.mark.parametrize("plane", [False, True], ids=["plain", "plane"])
@pytest.mark.parametrize("rows", [3, 33, 65])
def test_projection_zero_column_skips_its_reflector(ctx, rows, plane):
    ur.require_long_double()
    Hf, Hx, Hcp, r = system(rows, 3, 10, plane, seed=rows)
    Hf[:, 1] = 0.0
    check_rows(ctx, Hf, Hx, Hcp, r, bound_cols=[0, 2])


@pytest.mark.parametrize("plane", [False, True], ids=["plain", "plane"])
@pytest.mark.parametrize("rows", [33, 65, 6143])
def test_projection_parallel_column_invariants(ctx, rows, plane):
    """H_f = [a | b | 2 a]: the third reflector is set by round-off, so the returned rows O (rows - 3 of them) are O = N^T X for some
    orthonormal N whose columns are orthogonal to range(H_f), which has rank 2.  Hence G - O^T O, G = X^T (I - Q_1 Q_1^T) X, is positive
    semi-definite of rank <= 1: checked on its Jacobi-scaled eigenvalues."""
    ur.require_long_double()
    Hf, Hx, Hcp, r = system(rows, 3, 10, plane, seed=rows + 1)
    Hf[:, 2] = 2.0 * Hf[:, 0]
    X = np.column_stack([Hx] + ([Hcp] if Hcp is not None else []) + [r])
    O = project(ctx, Hf, Hx, Hcp, r)
    assert O.shape == (rows - 3, X.shape[1])
    G = ur.left_null_gram(Hf[:, :2], X)
    D = np.asarray(G - O.astype(ur.LD).T @ O.astype(ur.LD), dtype=np.float64)
    d = 1.0 / np.sqrt(np.diag(np.asarray(G, dtype=np.float64)))
    lam = np.linalg.eigvalsh(d[:, None] * D * d[None, :])
    sv = np.linalg.svd(Hf[:, :2], compute_uv=False)
    tol = ur.BOUND_C * rows * ur.EPS * (sv[0] / sv[-1]) * X.shape[1]
    assert lam[0] >= -tol and lam[-2] <= tol, (lam[0], lam[-2], lam[-1], tol)
