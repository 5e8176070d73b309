"""Long-double references of the left-nullspace projection (householder_cols_kernel), of the EKF update's tail (dx = P H^T S^-1 r, the
manifold update of every variable kind, the downdate) and of StateHelper::initialize, with their error bounds.  Used by
tests/test_gpu_projection.py and tests/test_gpu_update_tail.py, and pinned against numpy / the oracle, planted mistakes included, by
tests/test_cpu_update_references.py.

Bounds are first-order, built from the element bounds the suite already uses: a GEMM of inner dimension K is exact for |dA| <=
(K + 2) eps |A| (|B|), a Cholesky factorisation of S for |dS| <= (n + 2) eps |L||L^T| <= (n + 2) eps n |S|_2.  Nothing here is measured."""
import numpy as np

LD = np.longdouble
EPS = 2.0 ** -53
BOUND_C = 4.0  # the constant c of every bound below
VEC, POSE, IMU, LANDMARK = 0, 1, 2, 3  # OVP_KIND_*
DX_SPLIT = 8  # OVP_DX_SPLIT: dx = Y w is summed in 8 fixed chunks of w


def require_long_double():
    assert np.finfo(np.longdouble).eps < 1e-18, "the references need an extended-precision long double"


# ---- projection --------------------------------------------------------------------------------------------------------------------
def householder_project(X, k):
    """H_k ... H_1 X in long double with the kernel's reflectors: column j of X gives v = x - alpha e_1, alpha = -|x| for x_0 > 0 and
    +|x| otherwise (x = X[j:, j] after the first j reflectors); a zero x gives no reflector (identity)."""
    A = np.array(X, dtype=LD)
    for j in range(k):
        x = A[j:, j].copy()
        nrm = np.sqrt((x * x).sum())
        if nrm == 0:
            continue
        alpha = -nrm if x[0] > 0 else nrm
        v = x.copy()
        v[0] -= alpha
        vtv = (v * v).sum()
        if vtv > 0:
            A[j:, j + 1:] -= (2 / vtv) * np.outer(v, v @ A[j:, j + 1:])
        A[j:, j] = 0
        A[j, j] = alpha
    return A


def projection_bound(Hf, X):
    """Per-column bound c rows eps kappa(H_f) |X_j|_2 of the projected rows (X = the columns after H_f)."""
    sv = np.linalg.svd(np.asarray(Hf, dtype=np.float64), compute_uv=False)
    kappa = float(sv[0] / sv[-1]) if sv[-1] > 0 else np.inf
    rows = Hf.shape[0]
    return BOUND_C * rows * EPS * kappa * np.linalg.norm(np.asarray(X, dtype=np.float64), axis=0)


def left_null_gram(B, X):
    """X^T (I - Q_1 Q_1^T) X in long double, Q_1 an orthonormal basis of range(B); B has full column rank (for a rank-deficient H_f:
    its independent columns)."""
    r = B.shape[1]
    Q1 = _apply_reflectors_transposed(np.asarray(B, dtype=LD), r, np.eye(B.shape[0], dtype=LD))[:, :r]
    Xl = np.asarray(X, dtype=LD)
    return Xl.T @ (Xl - Q1 @ (Q1.T @ Xl))


def _apply_reflectors_transposed(A, k, Q):
    """Q H_1 ... H_k: the first k columns of the result are an orthonormal basis of range(A[:, :k]) (long double)."""
    A = A.copy()
    vs = []
    for j in range(k):
        x = A[j:, j].copy()
        nrm = np.sqrt((x * x).sum())
        alpha = -nrm if x[0] > 0 else nrm
        v = x.copy()
        v[0] -= alpha
        vtv = (v * v).sum()
        beta = 2 / vtv if vtv > 0 else LD(0)
        A[j:, j:] -= beta * np.outer(v, v @ A[j:, j:])
        vs.append((j, v, beta))
    for j, v, beta in vs:
        Q[:, j:] -= beta * np.outer(Q[:, j:] @ v, v)
    return Q


# ---- Kalman update -----------------------------------------------------------------------------------------------------------------
def ld_cholesky(S):
    n = S.shape[0]
    L = np.zeros_like(S)
    for j in range(n):
        d = S[j, j] - (L[j, :j] * L[j, :j]).sum()
        assert d > 0, "S is not positive definite"
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (S[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def ld_solve_lower(L, B):
    X = np.array(B, dtype=LD)
    for i in range(L.shape[0]):
        X[i] = (X[i] - L[i, :i] @ X[:i]) / L[i, i]
    return X


def kalman(P, ids, H, r, R):
    """S = H P_ids H^T + diag(R), P+ = P - P H^T S^-1 H P, dx = P H^T S^-1 r in long double (R: vector or None = ones).  Returns a dict
    with P+, dx, w = L^-1 r (|w|^2 = chi2), S, Y = M L^-T and the bound inputs."""
    P, H, r = np.asarray(P, dtype=LD), np.asarray(H, dtype=LD), np.asarray(r, dtype=LD)
    Rv = np.ones(H.shape[0], dtype=LD) if R is None else np.asarray(R, dtype=LD)
    M = P[:, ids] @ H.T
    S = H @ M[ids, :] + np.diag(Rv)
    L = ld_cholesky(S)
    w = ld_solve_lower(L, r)
    Y = ld_solve_lower(L, M.T).T
    return dict(P=P - Y @ Y.T, dx=Y @ w, w=w, S=S, Y=Y, M=M)


def kalman_bounds(P, ids, H, ref):
    """First-order bounds of the computed dx and P+ (Jacobi-scaled: |dP+_ij| / sqrt(P_ii P_jj)).  dS collects the GEMM error of S
    ((n_c + 2) eps |H||P||H^T|) and the Cholesky's backward error ((rr + 2) eps rr |S|_2); dM_i the GEMM error of row i of M = P H^T.
    With |w| = sqrt(chi2), |Y_i| <= sqrt(P_ii) and lambda = lambda_min(S):
        |d dx_i| <= |dM_i| |w| / sqrt(lambda) + sqrt(P_ii) |w| (|dS| / lambda + rr + 2) eps-scaled,
        |d P+_ij| <= (|dM_i| sqrt(P_jj) + |dM_j| sqrt(P_ii)) / sqrt(lambda) + sqrt(P_ii P_jj) (|dS| / lambda + rr + 2) eps."""
    P64, H64 = np.asarray(P, dtype=np.float64), np.asarray(H, dtype=np.float64)
    rr, nc = H64.shape
    S64 = np.asarray(ref["S"], dtype=np.float64)
    lam = np.linalg.eigvalsh(S64)
    lmin, lmax = float(lam[0]), float(lam[-1])
    aH = np.abs(H64)
    absPH = np.abs(P64[:, ids]) @ aH.T  # |P||H^T|, N x rr
    dS = (nc + 2) * EPS * float(np.linalg.norm(aH @ absPH[ids, :], 2)) + (rr + 2) * rr * EPS * lmax
    dM = (nc + 2) * EPS * np.linalg.norm(absPH, axis=1)
    sd = np.sqrt(np.diag(P64))
    wn = float(np.sqrt(np.sum(np.asarray(ref["w"], dtype=np.float64) ** 2)))
    rel = dS / lmin + (rr + 2) * EPS
    dx = BOUND_C * (dM * wn / np.sqrt(lmin) + sd * wn * rel)
    dP = BOUND_C * ((dM[:, None] * sd[None, :] + sd[:, None] * dM[None, :]) / np.sqrt(lmin) + np.outer(sd, sd) * rel)
    scale = np.outer(sd, sd)
    return dx, dP / scale, lmax / lmin


# ---- the manifold update of ov_type (written from the JPL definitions, independently of ov_plane_b200.jpl) -------------------------
def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]], dtype=LD)


def rot(q):
    """Rotation matrix of the JPL quaternion q = [q_v; q_4] (Trawny & Roumeliotis eq. 78): (2 q4^2 - 1) I - 2 q4 [q_v x] + 2 q_v q_v^T."""
    q = np.asarray(q, dtype=LD)
    v, q4 = q[:3], q[3]
    return (2 * q4 * q4 - 1) * np.eye(3, dtype=LD) - 2 * q4 * skew(v) + 2 * np.outer(v, v)


def jpl_product(a, b):
    """a (x) b in JPL convention, R(a (x) b) = R(a) R(b) (Trawny & Roumeliotis eq. 9)."""
    a, b = np.asarray(a, dtype=LD), np.asarray(b, dtype=LD)
    av, a4, bv, b4 = a[:3], a[3], b[:3], b[3]
    return np.concatenate([a4 * bv + b4 * av - np.cross(av, bv), [a4 * b4 - av @ bv]])


def dq_of(dth, normalise=True):
    dq = np.concatenate([np.asarray(dth, dtype=LD) / 2, [LD(1)]])
    return dq / np.sqrt((dq * dq).sum()) if normalise else dq


def quat_update(q, dth, order="left", normalise=True, flip=True):
    """q+ = dq (x) q with dq = normalise([dth / 2; 1]) and the sign chosen so that q4 >= 0 (ov_type::JPLQuat::update); the keyword
    arguments plant the mistakes the tests must catch."""
    dq = dq_of(dth, normalise)
    p = jpl_product(dq, q) if order == "left" else jpl_product(q, dq)
    if flip and p[3] < 0:
        p = -p
    return p


def apply_dx(kinds, values, ids, dx, quat=quat_update):
    """ov_type::*::update of every variable: {handle: new value} from {handle: value}, kinds {handle: kind} and ids {handle: state id}."""
    out = {}
    for h, v in values.items():
        v = np.asarray(v, dtype=LD)
        d = np.asarray(dx[ids[h]:ids[h] + {IMU: 15, POSE: 6}.get(kinds[h], len(v))], dtype=LD)
        if kinds[h] in (VEC, LANDMARK):
            out[h] = v + d
        else:
            nv = v.copy()
            nv[:4] = quat(v[:4], d[:3])
            nv[4:] = v[4:] + d[3:]
            out[h] = nv
    return out


def value_bounds(kinds, values, ids, dx_bound):
    """Bound of every value element: dx's bound plus one rounding of the sum; a quaternion element moves by at most half the norm of
    its dtheta error, plus a few roundings of the product and the normalisations."""
    out = {}
    for h, v in values.items():
        v = np.abs(np.asarray(v, dtype=np.float64))
        n = {IMU: 15, POSE: 6}.get(kinds[h], len(v))
        d = dx_bound[ids[h]:ids[h] + n]
        if kinds[h] in (VEC, LANDMARK):
            out[h] = d + 2 * EPS * v
        else:
            b = np.empty(len(v))
            b[:4] = 0.5 * np.linalg.norm(d[:3]) + 16 * EPS
            b[4:] = d[3:] + 2 * EPS * v[4:]
            out[h] = b
    return out


def check_update(P_got, vals_got, fejs_got, P0, kinds, ids, vals, fejs, dx, dx_bound, dP_bound, P_ref):
    """Everything the EKF update wrote, against the long-double reference: P+ element-wise (Jacobi-scaled by the prior P) and exactly
    symmetric; every variable's value, the ones outside H included; every quaternion through rotation matrices (R(q+) = R(dq) R(q)),
    q4 >= 0 and unit norm; every FEJ bit-identical.  Returns the worst error / bound of P+ and of the values."""
    assert np.array_equal(P_got, P_got.T), "P+ is not exactly symmetric"
    sd = np.sqrt(np.diag(np.asarray(P0, dtype=np.float64)))
    eP = np.abs(np.asarray(P_got - P_ref, dtype=np.float64)) / np.outer(sd, sd)
    rP = eP / np.where(dP_bound > 0, dP_bound, 1.0)  # a zero bound (an entry nothing may change) holds a zero error
    i, j = np.unravel_index(np.argmax(rP), eP.shape)
    assert np.all(eP <= dP_bound), "P+[%d, %d]: scaled error %.3e above the bound %.3e" % (i, j, eP[i, j], dP_bound[i, j])
    ref = apply_dx(kinds, vals, ids, dx)
    vb = value_bounds(kinds, vals, ids, dx_bound)
    worst = 0.0
    for h in kinds:
        g = np.asarray(vals_got[h], dtype=LD)
        e = np.abs(np.asarray(g - ref[h], dtype=np.float64))
        assert np.all(e <= vb[h]), "handle %d (kind %d, id %d): error %s above %s" % (h, kinds[h], ids[h], e, vb[h])
        worst = max(worst, float((e / vb[h]).max()))
        assert np.array_equal(fejs_got[h], fejs[h]), "handle %d: the FEJ changed" % h
        if kinds[h] in (POSE, IMU):
            q = np.asarray(vals_got[h][:4], dtype=np.float64)
            assert q[3] >= 0, "handle %d: q4 = %.3e < 0" % (h, q[3])
            assert abs(np.linalg.norm(q.astype(LD)) - 1) <= 8 * EPS,"handle %d: |q| - 1 = %.3e" % (h, float(np.linalg.norm(q.astype(LD)) - 1))
            dth = np.asarray(dx[ids[h]:ids[h] + 3], dtype=LD)
            eR = np.abs(np.asarray(rot(g[:4]) - rot(dq_of(dth)) @ rot(vals[h][:4]), dtype=np.float64)).max()
            bR = 2 * np.linalg.norm(dx_bound[ids[h]:ids[h] + 3]) + 64 * EPS
            assert eR <= bR, "handle %d: R(q+) - R(dq) R(q) = %.3e above %.3e" % (h, eR, bR)
    return float(rP.max()), worst


def flipped(kinds, vals, ids, dx):
    """Handles whose dq (x) q has a negative scalar part (the sign-flip branch of the update)."""
    return [h for h in kinds if kinds[h] in (POSE, IMU) and jpl_product(dq_of(dx[ids[h]:ids[h] + 3]), vals[h][:4])[3] < 0]


# ---- StateHelper::initialize -------------------------------------------------------------------------------------------------------
def initialize(P, ids, H_R, H_L, r, sigma2):
    """StateHelper::initialize without the gate decision, in long double, independent of the rotation that splits the system:
    with H_L = [Q_1 Q_2] [R_1; 0]: chi2 of Q_2^T [H_R r] against P (R = sigma2 I), the new variable's value offset R_1^-1 Q_1^T r,
    P_LL, the cross terms, then the EKF update of the grown state with the remaining rows.  Returns dict(chi2, dxn, P_init (grown, before
    the update), upd (kalman() of the update or None), H2, r2)."""
    P, H_R, H_L, r = (np.asarray(a, dtype=LD) for a in (P, H_R, H_L, r))
    rows, s = H_L.shape
    Q = _apply_reflectors_transposed(H_L.copy(), s, np.eye(rows, dtype=LD))
    Q1, Q2 = Q[:, :s], Q[:, s:]
    R1 = Q1.T @ H_L
    Rinv = np.linalg.inv(np.asarray(R1, dtype=np.float64)).astype(LD)
    for _ in range(2):  # refine the float64 inverse to long double
        Rinv = Rinv + Rinv @ (np.eye(s, dtype=LD) - R1 @ Rinv)
    H1, r1 = Q1.T @ H_R, Q1.T @ r
    H2, r2 = Q2.T @ H_R, Q2.T @ r
    chi2 = LD(0)
    if rows > s:
        S2 = H2 @ P[np.ix_(ids, ids)] @ H2.T + sigma2 * np.eye(rows - s, dtype=LD)
        w = ld_solve_lower(ld_cholesky(S2), r2)
        chi2 = (w * w).sum()
    N = P.shape[0]
    Mm = H1 @ P[np.ix_(ids, ids)] @ H1.T + sigma2 * np.eye(s, dtype=LD)
    Pg = np.zeros((N + s, N + s), dtype=LD)
    Pg[:N, :N] = P
    cross = -(P[:, ids] @ H1.T) @ Rinv.T
    Pg[:N, N:] = cross
    Pg[N:, :N] = cross.T
    Pg[N:, N:] = Rinv @ Mm @ Rinv.T
    upd = None
    if rows > s:
        upd = kalman(Pg, ids, H2, r2, np.full(rows - s, sigma2, dtype=LD))
    return dict(chi2=chi2, dxn=Rinv @ r1, P_init=Pg, upd=upd, H2=H2, r2=r2)


# ---- states -----------------------------------------------------------------------------------------------------------------------
# time offset, extrinsics and intrinsics calibrated: dt and both calibration variables have covariance rows
STATE_OPTIONS = dict(do_fej=1, imu_avg=0, use_rk4_integration=1, do_calib_camera_pose=1, do_calib_camera_intrinsics=1,
                     do_calib_camera_timeoffset=1, max_clone_size=64, max_aruco_features=1024, sigma_constraint=0.01, const_init_multi=1.0,
                     const_init_chi2=1.0, sigma_plane_merge=0.01, plane_merge_chi2=0.75, plane_merge_deg_max=1.0)
# standard deviations of the state rows of each kind
SIGMA = {IMU: [3e-3] * 3 + [1e-2] * 6 + [1e-3] * 6, POSE: [3e-3] * 3 + [1e-2] * 3, "dt": [1e-3], "intr": [1.0] * 4 + [1e-3] * 4,
         "plane": [1e-2] * 3, "lm": [5e-2] * 3}
REUSE_LAG = 64  # OVP_HANDLE_REUSE_LAG


def _unit_quat(rng, small_q4=False):
    q = rng.standard_normal(4)
    if small_q4:  # close to a half turn: dq (x) q can have a negative scalar part
        q[3] = 0.0
        q = q / np.linalg.norm(q)
        q[3] = 2e-4
    q = q / np.linalg.norm(q)
    return q if q[3] >= 0 else -q


def build_state(be, extra_landmarks, seed):
    """Every variable kind in one state on a backend (api.Context or the oracle mirror): IMU, dt, extrinsics, intrinsics, 12 clones
    (the first four close to a half turn), 3 planes, landmarks.  REUSE_LAG + 6 landmarks are added and marginalised first, so that the
    GPU hands their slots out again to clones, planes and landmarks; two clones and two landmarks are marginalised in the middle, so ids
    shift and the handle table has holes.  N = 123 + 3 extra_landmarks.  Returns (kinds, sigma, handles) with {handle: kind},
    {handle: standard deviations of its rows} and named handle lists."""
    rng = np.random.default_rng(seed)
    imu = np.concatenate([_unit_quat(rng), rng.standard_normal(12)])
    be.var_set(be.handle_imu(), imu, imu + 1e-3 * rng.standard_normal(16))
    be.var_set(be.handle_dt(), [0.004], [0.003])
    cal = np.concatenate([_unit_quat(rng), 0.05 * rng.standard_normal(3)])
    be.var_set(be.handle_calib(), cal, cal)
    intr = np.array([458.6, 457.3, 367.2, 248.4, -0.28, 0.074, 2e-4, 1.8e-5])
    be.var_set(be.handle_intrinsics(), intr, intr)
    kinds = {be.handle_imu(): IMU, be.handle_dt(): VEC, be.handle_calib(): POSE, be.handle_intrinsics(): VEC}
    sig = {be.handle_imu(): SIGMA[IMU], be.handle_dt(): SIGMA["dt"], be.handle_calib(): SIGMA[POSE], be.handle_intrinsics(): SIGMA["intr"]}
    tmp = [be.add_slam_raw(9000000 + i, rng.standard_normal(3), rng.standard_normal(3)) for i in range(REUSE_LAG + 6)]
    for h in tmp:
        be.marginalize(h)
    clones, planes, lms = [], [], []

    def clone(k):
        v = np.concatenate([_unit_quat(rng, small_q4=k < 4), rng.standard_normal(3)])
        h = be.add_clone_raw(100.0 + 0.05 * k, v, v + 1e-3 * rng.standard_normal(7))
        kinds[h], sig[h] = POSE, SIGMA[POSE]
        clones.append(h)

    def landmark(i):
        p = 3.0 * rng.standard_normal(3)
        h = be.add_slam_raw(5000000 + i, p, p + 1e-3 * rng.standard_normal(3))
        kinds[h], sig[h] = LANDMARK, SIGMA["lm"]
        lms.append(h)

    for k in range(12):
        clone(k)
    for pid in (1, 2, 3):
        cp = rng.standard_normal(3) + 3.0
        h = be.add_plane_raw(pid, cp, cp + 1e-3 * rng.standard_normal(3))
        kinds[h], sig[h] = VEC, SIGMA["plane"]
        planes.append(h)
    for i in range(6):
        landmark(i)
    for h in (clones[2], clones[5], lms[1], lms[4]):
        be.marginalize(h)
        del kinds[h], sig[h]
    clones = [h for h in clones if h in kinds]
    lms = [h for h in lms if h in kinds]
    for k in range(12, 14):
        clone(k)
    for i in range(6, 6 + extra_landmarks):
        landmark(i)
    assert be.cov_rows() == 123 + 3 * extra_landmarks
    return kinds, sig, dict(clones=clones, planes=planes, lms=lms)


def state_arrays(be, kinds, sig):
    """ids {handle: state id}, values {handle: value}, fejs {handle: fej} and the state's row standard deviations d (id order)."""
    ids = {h: be.var_id(h) for h in kinds}
    vals, fejs = {}, {}
    for h in kinds:
        vals[h], fejs[h] = be.var_get(h)
    d = np.zeros(be.cov_rows())
    for h in kinds:
        d[ids[h]:ids[h] + len(sig[h])] = sig[h]
    assert np.all(d > 0)
    return ids, vals, fejs, d


def update_handles(be, hs):
    """A non-contiguous subset of the variables, not in state order: a clone, the IMU, a plane, the intrinsics, the newest landmark and
    the extrinsics (41 columns)."""
    return [hs["clones"][2], be.handle_imu(), hs["planes"][1], be.handle_intrinsics(), hs["lms"][-1], be.handle_calib()]


def columns(be, handles):
    return [i for h in handles for i in range(be.var_id(h), be.var_id(h) + be.var_size(h))]


def measurement(rng, P, cols, rows, d, Rv):
    """H (rows x len(cols)) with columns scaled to the state's standard deviations (|H P H^T| ~ 1) and r = H dx_true + noise of R."""
    nc = len(cols)
    H = rng.standard_normal((rows, nc)) / (np.sqrt(nc) * d[cols])[None, :]
    dx = np.linalg.cholesky(P[np.ix_(cols, cols)]) @ rng.standard_normal(nc)
    r = H @ dx + np.sqrt(Rv) * rng.standard_normal(rows)
    return H, r


def update_case(be, extra_landmarks, rows, rdiag, seed):
    """State, covariance and measurement of one ovp_ekf_update case.  rdiag: None (unit R), "nonunit" (R_ii in [e^-1, e]) or "kappa"
    (R_ii ~ 1e-8 |H P H^T|_2, so kappa(S) ~ 1e8 when rows exceed the 41 columns).  Returns a dict."""
    kinds, sig, hs = build_state(be, extra_landmarks, seed)
    ids, vals, fejs, d = state_arrays(be, kinds, sig)
    P = correlated(d, seed)
    be.cov_upload(P)
    handles = update_handles(be, hs)
    cols = columns(be, handles)
    rng = np.random.default_rng(seed + 1000 * rows)
    if rdiag == "kappa":
        H, _ = measurement(rng, P, cols, rows, d, np.ones(rows))
        lam = np.linalg.eigvalsh(H @ P[np.ix_(cols, cols)] @ H.T)[-1]
        Rv = lam * 1e-8 * rng.uniform(1.0, 2.0, rows)
        H, r = measurement(np.random.default_rng(seed + 1000 * rows), P, cols, rows, d, Rv)
    else:
        Rv = np.ones(rows) if rdiag is None else np.exp(rng.uniform(-1.0, 1.0, rows))
        H, r = measurement(rng, P, cols, rows, d, Rv)
    return dict(kinds=kinds, hs=hs, ids=ids, vals=vals, fejs=fejs, d=d, P=P, handles=handles, cols=cols, H=H, r=r,
                Rdiag=None if rdiag is None else Rv)


def correlated(d, seed, cond=None):
    """P = D C D with D = diag(d) and C a correlation matrix with correlations of a few tenths between every pair of variables (a rank-4
    factor plus 0.3 I).  cond: the 6 smallest eigenvalues of C are lowered so that kappa_2(C) ~ cond."""
    rng = np.random.default_rng(seed)
    N = len(d)
    F = rng.standard_normal((N, 4))
    A = F @ F.T / 4.0 + 0.3 * np.eye(N)
    s = 1.0 / np.sqrt(np.diag(A))
    C = s[:, None] * A * s[None, :]
    if cond is not None:
        lam, V = np.linalg.eigh(C)
        lam[:6] = lam[-1] / cond
        C = (V * lam) @ V.T
        s = 1.0 / np.sqrt(np.diag(C))
        C = s[:, None] * C * s[None, :]
    P = np.asarray(d)[:, None] * C * np.asarray(d)[None, :]
    return 0.5 * (P + P.T)
