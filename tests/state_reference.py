"""References of the covariance operations between updates: StateHelper::EKFPropagation in long double with an element-wise bound, exact
numpy restatements of clone, marginalize, get_marginal_covariance and set_initial_covariance, the time-offset terms of augment_clone in
long double with their bound, and an asymmetric covariance to run them on.  Used by tests/test_gpu_state_ops.py, pinned against numpy
and the oracle, planted mistakes included, by tests/test_cpu_state_references.py.

The copies are defined exactly by the reference (StateHelper.cpp:302-318, :376-378, :204-229, :241-254), so the library must reproduce
them bit for bit.  They differ only where P is not exactly symmetric, and the reference's EKFPropagation leaves it so every frame
(Cov_PhiT and Phi_Cov_PhiT are written as computed, :103-105): `asymmetric` makes that visible far above one ulp.  The bounds reuse the
GEMM bound of tests/update_reference.py: an inner dimension K is exact for |dA| <= (K + 2) eps |A| (|B|).  Nothing here is measured."""
import numpy as np

from update_reference import BOUND_C, EPS, LD, correlated

ASYM = 1e-9  # relative size of the antisymmetric part of `asymmetric`


def asymmetric(d, seed, cond=None):
    """correlated(d, seed, cond) plus an antisymmetric perturbation of ASYM sqrt(P_ii P_jj): P_ij - P_ji is about 1e-9 of the entry, far
    above one ulp, and the diagonal is unchanged."""
    P = correlated(d, seed, cond)
    A = np.random.default_rng(seed + 7919).uniform(-1.0, 1.0, P.shape)
    d = np.asarray(d, dtype=np.float64)
    return P + ASYM * np.outer(d, d) * (A - A.T)


def covariance(kind, d, seed):
    """The three covariances of the state tests: "corr" (correlated), "cond" (correlated, kappa(C) ~ 1e10) and "asym" (asymmetric)."""
    return {"corr": lambda: correlated(d, seed), "cond": lambda: correlated(d, seed, 1e10), "asym": lambda: asymmetric(d, seed)}[kind]()


def upper_sym(Q):
    """Q.selfadjointView<Upper>(): the upper triangle mirrored, the lower one ignored."""
    Q = np.asarray(Q)
    return np.triu(Q) + np.triu(Q, 1).T


# ---- EKFPropagation ---------------------------------------------------------------------------------------------------------------
def propagate(P, new, old, Phi, Q, lower=False):
    """StateHelper::EKFPropagation (StateHelper.cpp:83-105) in long double: C = P[:, old] Phi^T, D = Qsym + Phi C[old, :], then
    P[new, :] = C^T, P[:, new] = C, P[new, new] = D (new: the contiguous state indices of the NEW variables, old: those of the OLD ones in
    Phi's column order).  Returns (P+, bound) with the element-wise bound BOUND_C ((K + 2) eps |P[:, old]| |Phi^T|) of C (K = len(old))
    and BOUND_C ((K + 2) eps (|Phi| |C[old, :]| + |Qsym|) + |Phi| |dC[old, :]|) of D; zero outside the new rows and columns.
    lower: take Q's lower triangle instead (a planted mistake)."""
    P64, F64 = np.asarray(P, dtype=np.float64), np.asarray(Phi, dtype=np.float64)
    Qs = upper_sym(np.asarray(Q).T).T if lower else upper_sym(Q)
    Pl, F = np.asarray(P, dtype=LD), np.asarray(Phi, dtype=LD)
    C = Pl[:, old] @ F.T
    D = np.asarray(Qs, dtype=LD) + F @ C[old, :]
    out = Pl.copy()
    out[new, :] = C.T
    out[:, new] = C
    out[np.ix_(new, new)] = D
    K = len(old)
    bC = (K + 2) * EPS * (np.abs(P64[:, old]) @ np.abs(F64).T)
    C64 = np.asarray(C, dtype=np.float64)
    bD = (K + 2) * EPS * (np.abs(F64) @ np.abs(C64[old, :]) + np.abs(Qs)) + np.abs(F64) @ bC[old, :]
    B = np.zeros(P64.shape)
    B[new, :] = bC.T
    B[:, new] = bC
    B[np.ix_(new, new)] = bD
    return out, BOUND_C * B


# ---- exact copies -----------------------------------------------------------------------------------------------------------------
def clone(P, old, s, rows_from_cols=False):
    """StateHelper::clone (StateHelper.cpp:376-378): the variable at [old, old + s) appended at N: the new x new block from the old x old
    block, the new column block from the old columns, the new row block from the old rows.  rows_from_cols: the row block taken from the
    old columns (a planted mistake)."""
    P = np.asarray(P)
    N = P.shape[0]
    out = np.zeros((N + s, N + s), dtype=P.dtype)
    out[:N, :N] = P
    out[N:, N:] = P[old:old + s, old:old + s]
    out[:N, N:] = P[:, old:old + s]
    out[N:, :N] = P[:, old:old + s].T if rows_from_cols else P[old:old + s, :]
    return out


def marginalize(P, mid, ms, copy_x2x1=False, shift=0):
    """StateHelper::marginalize (StateHelper.cpp:302-318): x1 = [0, mid), x2 = [mid + ms, N); x1x1, x1x2 and x2x2 copied, x2x1 set to
    the transpose of the new x1x2 block.  copy_x2x1: x2x1 copied as stored; shift: x2 read `shift` rows / columns late (planted
    mistakes)."""
    P = np.asarray(P)
    N = P.shape[0]
    n = N - ms
    out = np.zeros((n, n), dtype=P.dtype)
    a = mid + ms + shift
    x2 = np.minimum(np.arange(a, a + n - mid), N - 1)
    out[:mid, :mid] = P[:mid, :mid]
    out[:mid, mid:] = P[:mid][:, x2]
    out[mid:, :mid] = P[x2][:, :mid] if copy_x2x1 else out[:mid, mid:].T
    out[mid:, mid:] = P[np.ix_(x2, x2)]
    return out


def marginal(P, ids):
    """StateHelper::get_marginal_covariance (StateHelper.cpp:241-254): the blocks of the variables in the order given."""
    return np.asarray(P)[np.ix_(ids, ids)]


def set_initial(P, cov, ids):
    """StateHelper::set_initial_covariance (StateHelper.cpp:216-228): cov scattered block by block to the variables' indices, then the
    whole P made symmetric from its upper triangle."""
    out = np.array(P, copy=True)
    out[np.ix_(ids, ids)] = cov
    return upper_sym(out)


# ---- augment_clone's time-offset terms --------------------------------------------------------------------------------------------
def augment_dt(P, new, dt, d, stale_row=False):
    """StateHelper::augment_clone (StateHelper.cpp:620-623) on the cloned P in long double: P[:, new:new+6] += P[:, dt] d^T, then
    P[new:new+6, :] += d P[dt, :], the second pass reading the dt row the first one updated (it carries d d^T P_dt,dt in the new x new
    block).  Returns (P+, bound) with the element-wise bound BOUND_C eps (|P| + |P[:, dt]| |d|^T + |d| |P[dt, :]| + |d| |d|^T |P_dt,dt|)
    on the new rows and columns, zero elsewhere.  stale_row: the second pass reads the dt row as it was before the first (a planted
    mistake)."""
    P64, d64 = np.asarray(P, dtype=np.float64), np.asarray(d, dtype=np.float64)
    Pl, dl = np.asarray(P, dtype=LD), np.asarray(d, dtype=LD)
    row0 = Pl[dt, :].copy()
    out = Pl.copy()
    out[:, new:new + 6] += np.outer(out[:, dt], dl)
    out[new:new + 6, :] += np.outer(dl, row0 if stale_row else out[dt, :])
    ad = np.abs(d64)
    B = np.zeros(P64.shape)
    B[:, new:new + 6] = np.abs(P64[:, new:new + 6]) + np.outer(np.abs(P64[:, dt]), ad)
    B[new:new + 6, :] = np.maximum(B[new:new + 6, :], np.abs(P64[new:new + 6, :])) + np.outer(ad, np.abs(P64[dt, :]))
    B[new:new + 6, new:new + 6] += np.outer(ad, ad) * abs(P64[dt, dt])
    return out, BOUND_C * EPS * B


# ---- checks -------------------------------------------------------------------------------------------------------------------------
def within(got, ref, bound, what):
    """Element-wise |got - ref| <= bound; returns the worst error / bound (entries with a zero bound must be exact)."""
    e = np.abs(np.asarray(np.asarray(got, dtype=LD) - ref, dtype=np.float64))
    r = e / np.where(bound > 0, bound, 1.0)
    i, j = np.unravel_index(np.argmax(r), r.shape)
    assert np.all(e <= bound), "%s[%d, %d]: error %.3e above the bound %.3e" % (what, i, j, e[i, j], bound[i, j])
    return float(r.max())


def exceed(bad, ref, bound):
    """How far `bad` fails `within`, in units of the bound (inf where a zero-bound entry differs)."""
    e = np.abs(np.asarray(np.asarray(bad, dtype=LD) - ref, dtype=np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bound > 0, e / np.where(bound > 0, bound, 1.0), np.where(e > 0, np.inf, 0.0))
    return float(r.max())


def bits(got, ref, what):
    """Bit-exact equality; reports the first mismatching entry and the number of mismatches."""
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, "%s: shape %s, expected %s" % (what, got.shape, ref.shape)
    bad = np.argwhere(got.view(np.uint64) != ref.view(np.uint64))
    if len(bad):
        i, j = bad[0]
        raise AssertionError("%s: %d entries differ, first [%d, %d]: %r != %r" % (what, len(bad), i, j, got[i, j], ref[i, j]))
