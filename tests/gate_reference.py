"""Long-double references of the per-feature Mahalanobis gate chi2 = r_o^T (H_o P_m H_o^T + I)^-1 r_o of the MSCKF point and SLAM
feature kernels, its first-order error bound, and correlated covariances to run them on (tests/test_gpu_feature_gate.py,
tests/test_cpu_feature_gate.py).

synth.make_scenario's P0 has diagonal 6 x 6 clone blocks and no covariance between the calibration, plane and landmark blocks and the
clones, so a gate that reads a clone block transposed, drops a calibration x clone term or gathers the wrong covariance column gives the
same chi2 on it.  correlated_cov keeps P0's variances and correlates everything with everything."""
import numpy as np

LD = np.longdouble
EPS = 2.0 ** -53
RAW_ROW = 24  # OVP_RAW_ROW (features.cu): doubles per raw row, 3 rows per measurement
BOUND_C = 2.0  # the constant c of the bound (gate_bound)


def require_long_double():
    assert np.finfo(np.longdouble).eps < 1e-18, "the references need an extended-precision long double"


def householder_q3(Hf, null_basis=False):
    """First three columns of Q of Hf = Q R (3 Householder reflectors, long double).  null_basis: also an orthonormal basis N
    (rows x (rows - 3)) of the left null space of Hf, the remaining columns of the same Q."""
    A = Hf.astype(LD)
    n = A.shape[0]
    vs = []
    for j in range(3):
        x = A[j:, j].copy()
        nrm = np.sqrt((x * x).sum())
        alpha = -nrm if x[0] > 0 else nrm
        v = x.copy()
        v[0] -= alpha
        vtv = (v * v).sum()
        beta = 2 / vtv if vtv > 0 else LD(0)
        A[j:, :] -= beta * np.outer(v, v @ A[j:, :])
        vs.append((j, v, beta))
    Q = np.eye(n, dtype=LD) if null_basis else np.zeros((n, 3), dtype=LD)
    if not null_basis:
        Q[:3, :3] = np.eye(3, dtype=LD)
    for j, v, beta in reversed(vs):
        Q[j:, :] -= beta * np.outer(v, v @ Q[j:, :])
    return (Q[:, :3].copy(), Q[:, 3:].copy()) if null_basis else Q


def ld_chi2(H, r, Pm):
    """r^T (H Pm H^T + I)^-1 r by a long-double Cholesky and forward substitution; returns (chi2, S)."""
    H, r, Pm = H.astype(LD), r.astype(LD), Pm.astype(LD)
    S = H @ Pm @ H.T + np.eye(H.shape[0], dtype=LD)
    n = S.shape[0]
    L = np.zeros_like(S)
    for j in range(n):
        d = S[j, j] - (L[j, :j] * L[j, :j]).sum()
        assert d > 0, "S = H P H^T + I is not positive definite: P is not a covariance"
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (S[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    y = np.zeros(n, dtype=LD)
    for i in range(n):
        y[i] = (r[i] - L[i, :i] @ y[:i]) / L[i, i]
    return (y * y).sum(), S


def gate_bound(chi2, S, Hx, r, Pm, kappa_f, k):
    """First-order a-priori bound of |chi2_computed - chi2| (w = S^-1 r_o, S >= I gives |w|^2 <= chi2):
    |d chi2| <= 2 sqrt(chi2) |d r_o| + chi2 |dS|_2, with |d r_o| <= c k eps kappa(H_f) |r| and
    |dS|_2 <= c k eps (|S|_2 + kappa(H_f) |H_x|_2^2 |P_m|_2).  k = rows + columns of the feature block (the longest inner products),
    kappa(H_f) = 1 without a projection (the kernel's reflectors are exact for a nearby H_f + dH_f)."""
    c = BOUND_C * k * EPS
    nS = float(np.linalg.norm(np.asarray(S, dtype=np.float64), 2))
    nH = float(np.linalg.norm(np.asarray(Hx, dtype=np.float64), 2)) if Hx.size else 0.0
    nP = float(np.linalg.norm(np.asarray(Pm, dtype=np.float64), 2)) if Pm.size else 0.0
    dr = c * kappa_f * float(np.linalg.norm(np.asarray(r, dtype=np.float64)))
    dS = c * (nS + kappa_f * nH * nH * nP)
    x = max(float(chi2), 0.0)
    return 2.0 * np.sqrt(x) * dr + x * dS


def point_gate(Hf, Hx, r, Pm):
    """MSCKF point gate: H_o = N^T H_x, r_o = N^T r with N a long-double basis of the left null space of H_f.  Returns (chi2, bound,
    dof).  chi2 does not depend on the basis, so this is the reference of the kernels' reflectors and of the oracle's Givens rotations."""
    _, N = householder_q3(Hf, null_basis=True)
    chi2, S = ld_chi2(N.T @ Hx.astype(LD), N.T @ r.astype(LD), Pm)
    sv = np.linalg.svd(np.asarray(Hf, dtype=np.float64), compute_uv=False)
    kf = float(sv[0] / sv[-1])
    return chi2, gate_bound(chi2, S, Hx, r, Pm, kf, Hx.shape[0] + Hx.shape[1] + 3), N.shape[1]


def slam_gate(H, r, Pm):
    """SLAM gate: no projection; H = [landmark 3 | calibration | clones (| H_cp 3)] on the 3m rows with the plane, or on the 2m bearing
    rows.  Returns (chi2, bound, dof)."""
    chi2, S = ld_chi2(H, r, Pm)
    return chi2, gate_bound(chi2, S, H, r, Pm, 1.0, H.shape[0] + H.shape[1]), H.shape[0]


def raw_block(raw, a, b, ncal, plane):
    """The raw rows of the measurements [a, b) (raw: M x 3 x RAW_ROW, the layout of ovp_debug_msckf_gram / ovp_debug_slam_update) as
    (H_f, H_x, r) in long double: H_x = [calibration | 6 per measurement's clone (| H_cp 3)], bearing rows first, then (plane) the m
    point-on-plane rows."""
    m = b - a
    nx = ncal + 6 * m + (3 if plane else 0)
    rows = 3 * m if plane else 2 * m
    Hf, Hx, r = np.zeros((rows, 3), dtype=LD), np.zeros((rows, nx), dtype=LD), np.zeros(rows, dtype=LD)
    for k in range(m):
        for i in range(2):
            row = raw[a + k, i]
            Hf[2 * k + i] = row[:3]
            Hx[2 * k + i, :ncal] = row[9:9 + ncal]
            Hx[2 * k + i, ncal + 6 * k:ncal + 6 * k + 6] = row[3:9]
            r[2 * k + i] = row[RAW_ROW - 1]
        if plane:
            row = raw[a + k, 2]
            Hf[2 * m + k] = row[:3]
            Hx[2 * m + k, -3:] = row[9:12]
            r[2 * m + k] = row[RAW_ROW - 1]
    return Hf, Hx, r


def calib_ids(be, options):
    """State indices of the calibration columns of a backend (Context or the oracle mirror) with these state options: camera pose, then
    intrinsics."""
    ids = []
    if options["do_calib_camera_pose"]:
        ids += list(range(be.var_id(be.handle_calib()), be.var_id(be.handle_calib()) + 6))
    if options["do_calib_camera_intrinsics"]:
        ids += list(range(be.var_id(be.handle_intrinsics()), be.var_id(be.handle_intrinsics()) + 8))
    return ids


def block_ids(be, handles, sizes=None):
    """State indices of the variables `handles` (each var_size wide), concatenated."""
    ids = []
    for h in handles:
        i0 = be.var_id(int(h))
        ids += list(range(i0, i0 + (be.var_size(int(h)) if sizes is None else sizes)))
    return ids


SLAM_LENGTHS = (1, 2, 15, 29)


def slam_scenario(ncal, seed=0, F=24):
    """Landmarks tracked over 29-30 of 30 clones, half of them on one of 4 in-state planes."""
    from ov_plane_b200 import synth
    cal = {0: (0, 0), 6: (1, 0), 8: (0, 1), 14: (1, 1)}[ncal]
    return synth.make_scenario("small_planes", seed=seed, n_clones=30, F=F, m_min=29, m_max=30, dtheta=0.01, calib_pose=cal[0],
                               calib_intr=cal[1])


def slam_update_batch(S, handles, keep, seed, wrong_plane=0):
    """The update batch of the landmarks `keep` (initialised from their whole tracks): their newest 1, 2, 15 and 29 measurements in
    turn, with 0.5 px of noise; the first `wrong_plane` features on a plane are attached to another in-state plane, so that their gate
    with the plane row fails and the retry without it decides."""
    from ov_plane_b200 import synth
    b = synth.feature_batch(S, handles, keep)
    rng = np.random.default_rng(seed)
    mo, mc, uv = [0], [], []
    for i in range(b["F"]):
        a, e = int(b["meas_offset"][i]), int(b["meas_offset"][i + 1])
        m = min(SLAM_LENGTHS[i % len(SLAM_LENGTHS)], e - a)
        mc.append(b["meas_clone"][e - m:e])
        uv.append(b["uv"][e - m:e] + rng.normal(0.0, 0.5, (m, 2)).astype(np.float32))
        mo.append(mo[-1] + m)
    b["meas_offset"] = np.array(mo, dtype=np.int32)
    b["meas_clone"] = np.ascontiguousarray(np.concatenate(mc), dtype=np.int32)
    b["uv"] = np.ascontiguousarray(np.concatenate(uv), dtype=np.float32)
    ids = [int(p) for p in S.plane_ids]
    moved = 0
    for i in range(b["F"]):
        if moved < wrong_plane and b["planeid"][i] != 0:
            b["planeid"][i] = ids[(ids.index(int(b["planeid"][i])) + 1) % len(ids)]
            moved += 1
    return b


def correlated_cov(S, N, seed, cond=None, tail_var=0.05 ** 2):
    """P = D C D: D = the square roots of the diagonal of S.P0 (of tail_var for the state indices S.N .. N - 1, e.g. landmarks added
    after the scenario was loaded), C a random correlation matrix with strong off-diagonal entries everywhere (a rank-4 factor plus
    0.3 I, normalised: correlations of a few tenths, every block with every block).  cond: the 6 smallest eigenvalues of C are lowered
    to the one value that makes kappa_2(P) = cond within a factor of 2, as a filter's covariance is after it has observed a few
    directions very well; the other directions keep their variance, so the gates see residuals of the size they expect."""
    rng = np.random.default_rng(seed)
    d = np.sqrt(np.concatenate([np.diag(S.P0), np.full(N - S.N, tail_var)]))
    F = rng.standard_normal((N, 4))
    A = F @ F.T / 4.0 + 0.3 * np.eye(N)
    s = 1.0 / np.sqrt(np.diag(A))
    C = s[:, None] * A * s[None, :]

    def scaled(C):
        P = d[:, None] * C * d[None, :]
        return 0.5 * (P + P.T)

    if cond is None:
        return scaled(C)
    lam, V = np.linalg.eigh(C)

    def make(low):
        return scaled((V * np.concatenate([np.full(6, low), lam[6:]])) @ V.T)

    def kappa(P):
        w = np.linalg.eigvalsh(P)
        return w[-1] / w[0] if w[0] > 0 else np.inf

    lo, hi = 1e-30, float(lam[6])  # kappa decreases as the lowered eigenvalues grow
    for _ in range(100):
        mid = np.sqrt(lo * hi)
        if kappa(make(mid)) > cond:
            lo = mid
        else:
            hi = mid
    P = make(hi)
    assert cond / 2 <= kappa(P) <= 2 * cond, kappa(P)
    return P
