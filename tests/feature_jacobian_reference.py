"""Long-double reference of the measurement model of the feature kernels (mono radtan camera, JPL quaternions), written from the
mathematics: the whitened residual w (uv - h(x)) of every bearing measurement, its Jacobians H_f, H_clone, H_extrinsics and H_intrinsics,
the point-on-plane row, and d p_FinG / d (lambda, anchor, extrinsics) of the anchored landmark representations; with an entrywise
error bound for a double-precision evaluation of the same quantities (tests/test_cpu_feature_jacobian_reference.py,
tests/test_gpu_feature_jacobian_reference.py).

Forward model, generic over the dtype (np.longdouble or np.clongdouble, so r^2 is x^2 + y^2 and nothing takes abs or conj):
    R(q) = (2 w^2 - 1) I - 2 w [v]x + 2 v v^T          of the stored quaternion q = [v, w], not renormalised
    p_FinC = R_ItoC R_GtoI (p_FinG - p_IinG) + p_IinC,  (xn, yn) = (X / Z, Y / Z),  h = radtan(xn, yn),  r = w (uv - h)
with uv the float32 pixel the kernels receive.

Jacobians are complex steps, Im f(x + i s) / s with s = 1e-40: no cancellation, truncation error far below long-double rounding.
Rotations (clone, extrinsics, anchor) are perturbed as q <- dq(theta) (x) q with dq = [theta / 2, sqrt(1 - theta.theta / 4)];
positions, intrinsics, the global feature and the plane's closest point cp additively.  H = dh/dx (the residual is z - h).

First-estimate Jacobians compose the chain from factors evaluated where UpdaterHelper::get_feature_jacobian_full evaluates them:
dz/dzn and dz/dzeta at the value's (xn, yn); dzn/dp_FinC at the first-estimate camera point; dp_FinC/d{p_FinG, clone theta, clone p,
extrinsic theta, extrinsic p} at the clone's and the feature's first estimates with the extrinsics at their value (they are never
first-estimated); the plane row's Jacobians at (p_fej, cp_fej).  With do_fej = 0, or first estimates equal to the values, the product
equals the complex step of the whole chain (whole_chain).

Error bound, per entry: |computed - reference| <= C u mag with u = 2^-53 and mag the same factors evaluated in long double with every
operand replaced by its absolute value.  A coordinate of the camera point formed by cancellation (xn = 0 on an axis, a feature near the
image centre) is known only to an absolute error N_P u mag(X) / |Z|; its error reaches each factor through the magnitude of the
factor's derivative, which is added to the factor's magnitude (bearing_mags).  For the residual the magnitude holds |uv| and
|fx x1| + |cx|, so a residual near zero is held to absolute precision.  C is counted, not fitted: an expression of rounding depth d over
operands that carry errors of at most e u (relative to their magnitudes) is within (d + e) u of its value relative to its magnitude, to
first order.  The camera point coordinates have depth N_P = 11 (the rotation 3, the difference 1, two 3-term products 2 x 3, the offset
1, the division 1); each part adds its own depth, counted in C_PART."""
import numpy as np

LD, CLD = np.longdouble, np.clongdouble
U = 2.0 ** -53
STEP = LD("1e-40")
N_P = 11
C_PART = {
    # dz/dzn 12 (sqrt, r^2, r^4, the radial factor, the sums), dzn/dp_FinC 2, dp_FinC/dp_FinG = R_C R_i 6, the 2- and 3-term products
    # and the whitening 6
    "Hf": N_P + 12 + 2 + 6 + 6,
    # the rotation block's R_C [p_FinI]x: 9 instead of 6
    "clone": N_P + 12 + 2 + 9 + 6,
    # [p_FinC - p_IinC]x: the camera point's own depth plus one subtraction, already in N_P + 1
    "extrinsics": N_P + 12 + 2 + 1 + 6,
    # w dz/dzeta: fx x r^4 and x1, depth 14, the whitening 1
    "intrinsics": N_P + 14 + 1,
    # w (uv - (fx x1 + cx)): x1 14, then 3
    "res": N_P + 14 + 3,
    # |cp| 4, n 1, two 3-term products and the differences 6, 1 / d and the whitening 2; the inputs are the stored doubles
    "plane": 13,
}


def require_long_double():
    assert np.finfo(np.longdouble).eps < 1e-18, "the reference needs an extended-precision long double"


# ---------------------------------------------------------------------------------------------------------------------------------
# forward model (generic dtype)
# ---------------------------------------------------------------------------------------------------------------------------------
def rot(q):
    """JPL rotation of the stored quaternion [x y z w] (..., 4) -> (..., 3, 3)"""
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    s = 2 * w * w - 1
    R = np.stack([s + 2 * x * x, 2 * w * z + 2 * x * y, -2 * w * y + 2 * x * z,
                  -2 * w * z + 2 * y * x, s + 2 * y * y, 2 * w * x + 2 * y * z,
                  2 * w * y + 2 * z * x, -2 * w * x + 2 * z * y, s + 2 * z * z], axis=-1)
    return R.reshape(q.shape[:-1] + (3, 3))


def mv(R, v):
    return (R * v[..., None, :]).sum(axis=-1)


def cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def left_update(theta, q):
    """dq(theta) (x) q in the JPL product, dq = [theta / 2, sqrt(1 - theta.theta / 4)]"""
    dv = theta / 2
    dw = np.sqrt(1 - (theta * theta).sum(axis=-1) / 4)
    qv, qw = q[..., :3], q[..., 3]
    v = dw[..., None] * qv + qw[..., None] * dv - cross(dv, qv)
    return np.concatenate([v, (dw * qw - (dv * qv).sum(axis=-1))[..., None]], axis=-1)


def camera_point(q_cl, p_cl, q_C, p_C, pf):
    return mv(rot(q_C), mv(rot(q_cl), pf - p_cl)) + p_C


def distort(cam, x, y):
    """radtan, cam = [fx fy cx cy k1 k2 p1 p2] -> (..., 2)"""
    r2 = x * x + y * y
    r4 = r2 * r2
    k1, k2, p1, p2 = cam[..., 4], cam[..., 5], cam[..., 6], cam[..., 7]
    rad = 1 + k1 * r2 + k2 * r4
    x1 = x * rad + 2 * p1 * x * y + p2 * (r2 + 2 * x * x)
    y1 = y * rad + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
    return np.stack([cam[..., 0] * x1 + cam[..., 2], cam[..., 1] * y1 + cam[..., 3]], axis=-1)


def project(pc):
    return pc[..., :2] / pc[..., 2:3]


def plane_h(p, cp):
    """n^T p - d with d = |cp|, n = cp / d"""
    d = np.sqrt((cp * cp).sum(axis=-1))
    return (cp * p).sum(axis=-1) / d - d


def cstep(fun, x0, n, rotation=False):
    """d fun / d x at x0 (..., n) by complex step: (..., out, n).  rotation: x0 is a quaternion perturbed by dq(theta) (x) q."""
    cols = []
    for k in range(n):
        if rotation:
            th = np.zeros(x0.shape[:-1] + (3,), dtype=CLD)
            th[..., k] = 1j * STEP
            x = left_update(th, x0.astype(CLD))
        else:
            x = x0.astype(CLD).copy()
            x[..., k] += 1j * STEP
        cols.append(np.asarray(fun(x)).imag / STEP)
    return np.stack(cols, axis=-1)


# ---------------------------------------------------------------------------------------------------------------------------------
# the bearing rows
# ---------------------------------------------------------------------------------------------------------------------------------
def ld(a):
    return np.asarray(a, dtype=np.float64).astype(LD)


class Inputs(object):
    """One feature's measurements: clone values / first estimates (m x 7), extrinsics (7), intrinsics (8), the feature's value and first
    estimate, the float32 pixels (m x 2), whitening 1 / sigma_pix, do_fej."""

    def __init__(self, clone_val, clone_fej, calib, intr, pf, pf_fej, uv, sigma_pix, do_fej):
        self.cv, self.cf = ld(clone_val).reshape(-1, 7), ld(clone_fej).reshape(-1, 7)
        self.cal, self.cam = ld(calib), ld(intr)
        self.pf, self.pff = ld(pf), ld(pf_fej)
        self.uv = np.asarray(uv, dtype=np.float32).astype(np.float64).astype(LD).reshape(-1, 2)
        self.w = LD(1) / LD(float(sigma_pix))
        self.do_fej = bool(do_fej)
        self.m = self.cv.shape[0]

    def jac_point(self):
        """clone and feature where the Jacobians are evaluated"""
        return (self.cf, self.pff) if self.do_fej else (self.cv, self.pf)


def bearing_factors(I, mutate=None):
    """The factors of the FEJ composition, each at its own point (see the module docstring).  mutate: the name of one plausible
    wrong model (MUTATIONS), for the discrimination checks."""
    mutate = mutate or ""
    m = I.m
    qC, pC = I.cal[:4], I.cal[4:7]
    pfv = np.broadcast_to(I.pf, (m, 3))
    pc_val = camera_point(I.cv[:, :4], I.cv[:, 4:], qC, pC, pfv)
    zn = project(pc_val)
    cj, pfj = I.jac_point()
    if mutate == "clone rotation at its value" and I.do_fej:
        cj = np.concatenate([I.cv[:, :4], cj[:, 4:]], axis=1)
    pfj = np.broadcast_to(pfj, (m, 3))
    pc_j = camera_point(cj[:, :4], cj[:, 4:], qC, pC, pfj)
    zn_j = project(pc_j) if mutate == "uv_norm at the first estimate" else zn
    F = {}
    F["h"] = distort(I.cam, zn[:, 0], zn[:, 1])
    F["dz_dzn"] = cstep(lambda z: distort(I.cam, z[:, 0], z[:, 1]), zn_j, 2)
    if mutate == "2 p2 x tangential term":  # d x1 / dx = ... + 6 p2 x written as 2 p2 x
        F["dz_dzn"][:, 0, 0] -= I.cam[0] * 4 * I.cam[7] * zn_j[:, 0]
    F["dz_dzeta"] = cstep(lambda c: distort(c, zn_j[:, 0].astype(CLD), zn_j[:, 1].astype(CLD)), np.broadcast_to(I.cam, (m, 8)), 8)
    F["dzn_dpfc"] = cstep(project, pc_j, 3)
    cam_pt = lambda qc, pcl, qx, px, p: camera_point(qc, pcl, qx, px, p)
    F["dpfc_dpf"] = cstep(lambda p: cam_pt(cj[:, :4], cj[:, 4:], qC, pC, p), pfj, 3)
    if mutate == "skew(p_FinI) at the value" and I.do_fej:
        # the rotation block R_C [R_i^fej (p_f^fej - p_i^fej)]x with the clone-frame point taken at the value instead
        pI_val = mv(rot(I.cv[:, :4]), pfv - I.cv[:, 4:])
        F["dpfc_dth"] = np.einsum("ij,mjk->mik", rot(qC), _skew(pI_val))
    else:
        F["dpfc_dth"] = cstep(lambda q: cam_pt(q, cj[:, 4:], qC, pC, pfj), cj[:, :4], 3, rotation=True)
    F["dpfc_dp"] = cstep(lambda p: cam_pt(cj[:, :4], p, qC, pC, pfj), cj[:, 4:], 3)
    F["dpfc_dthC"] = cstep(lambda q: cam_pt(cj[:, :4], cj[:, 4:], q, pC, pfj), np.broadcast_to(qC, (m, 4)), 3, rotation=True)
    if mutate == "R_ItoC transposed in the extrinsic rotation block":
        # [R_C p_I]x -> [R_C^T p_I]x
        pI = mv(rot(cj[:, :4]), pfj - cj[:, 4:])
        F["dpfc_dthC"] = _skew(mv(np.swapaxes(rot(qC), -1, -2), pI))
    F["dpfc_dpC"] = cstep(lambda p: cam_pt(cj[:, :4], cj[:, 4:], qC, p, pfj), np.broadcast_to(pC, (m, 3)), 3)
    return F


def _skew(v):
    z = np.zeros_like(v[..., 0])
    return np.stack([z, -v[..., 2], v[..., 1], v[..., 2], z, -v[..., 0], -v[..., 1], v[..., 0], z], axis=-1).reshape(v.shape[:-1] + (3, 3))


def bearing_rows(I, mutate=None):
    """{res (m, 2), Hf (m, 2, 3), clone (m, 2, 6), extrinsics (m, 2, 6), intrinsics (m, 2, 8)} in long double"""
    F = bearing_factors(I, mutate)
    A = I.w * (F["dz_dzn"] @ F["dzn_dpfc"])
    return {"res": I.w * (I.uv - F["h"]), "Hf": A @ F["dpfc_dpf"],
            "clone": np.concatenate([A @ F["dpfc_dth"], A @ F["dpfc_dp"]], axis=-1),
            "extrinsics": np.concatenate([A @ F["dpfc_dthC"], A @ F["dpfc_dpC"]], axis=-1), "intrinsics": I.w * F["dz_dzeta"]}


def whole_chain(I):
    """The complex step of the whole measurement function at the values: the reference of bearing_rows when no first estimate differs"""
    m = I.m
    qC, pC, cam = I.cal[:4], I.cal[4:7], I.cam
    pfv = np.broadcast_to(I.pf, (m, 3))
    qv, pv = I.cv[:, :4], I.cv[:, 4:]

    def h(qc, pcl, qx, px, p, c):
        z = project(camera_point(qc, pcl, qx, px, p))
        return distort(c, z[:, 0], z[:, 1])

    def w(x):
        return I.w * x
    camm = np.broadcast_to(cam, (m, 8))
    return {"res": I.w * (I.uv - h(qv, pv, qC, pC, pfv, cam)),
            "Hf": w(cstep(lambda p: h(qv, pv, qC, pC, p, cam), pfv, 3)),
            "clone": w(np.concatenate([cstep(lambda q: h(q, pv, qC, pC, pfv, cam), qv, 3, rotation=True),
                                       cstep(lambda p: h(qv, p, qC, pC, pfv, cam), pv, 3)], axis=-1)),
            "extrinsics": w(np.concatenate([cstep(lambda q: h(qv, pv, q, pC, pfv, cam), np.broadcast_to(qC, (m, 4)), 3, rotation=True),
                                            cstep(lambda p: h(qv, pv, qC, p, pfv, cam), np.broadcast_to(pC, (m, 3)), 3)], axis=-1)),
            "intrinsics": w(cstep(lambda c: h(qv, pv, qC, pC, pfv, c), camm, 8))}


# ---------------------------------------------------------------------------------------------------------------------------------
# magnitudes (the same factors with every operand replaced by its absolute value)
# ---------------------------------------------------------------------------------------------------------------------------------
def rot_mag(q):
    x, y, z, w = (abs(q[..., i]) for i in range(4))
    s = 2 * w * w + 1
    R = np.stack([s + 2 * x * x, 2 * w * z + 2 * x * y, 2 * w * y + 2 * x * z,
                  2 * w * z + 2 * y * x, s + 2 * y * y, 2 * w * x + 2 * y * z,
                  2 * w * y + 2 * z * x, 2 * w * x + 2 * z * y, s + 2 * z * z], axis=-1)
    return R.reshape(q.shape[:-1] + (3, 3))


def _camera_point_mag(q_cl, p_cl, q_C, p_C, pf):
    """magnitudes of p_FinI and p_FinC; the difference of the two stored positions is rounded relative to itself"""
    pI = mv(rot_mag(q_cl), abs(pf - p_cl))
    return pI, mv(rot_mag(q_C), pI) + abs(p_C)


def _distort_mags(cam, x, y):
    """[dz/dzn (4), dz/dzeta (16), x1, y1] evaluated with the absolute values of every operand, at x, y >= 0 (..., 22); a polynomial
    with positive coefficients, so its complex step is the magnitude of its derivative"""
    fx, fy = abs(cam[0]), abs(cam[1])
    k1, k2, p1, p2 = (abs(cam[i]) for i in range(4, 8))
    r2 = x * x + y * y
    r4 = r2 * r2
    rad = 1 + k1 * r2 + k2 * r4
    x1 = x * rad + 2 * p1 * x * y + p2 * (r2 + 2 * x * x)
    y1 = y * rad + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
    dxx = rad + 2 * k1 * x * x + 4 * k2 * x * x * r2 + 2 * p1 * y + 6 * p2 * x
    dxy = 2 * k1 * x * y + 4 * k2 * x * y * r2 + 2 * p1 * x + 2 * p2 * y
    dyy = rad + 2 * k1 * y * y + 4 * k2 * y * y * r2 + 2 * p2 * x + 6 * p1 * y
    z = 0 * x
    one = z + 1
    return np.stack([fx * dxx, fx * dxy, fy * dxy, fy * dyy,
                     x1, z, one, z, fx * x * r2, fx * x * r4, 2 * fx * x * y, fx * (r2 + 2 * x * x),
                     z, y1, z, one, fy * y * r2, fy * y * r4, fy * (r2 + 2 * y * y), 2 * fy * x * y, x1, y1], axis=-1)


def _coords_err(pc, pcm):
    """magnitudes of the absolute rounding errors of x = X / Z, y = Y / Z (in units of N_P u): mag(X) / |Z| + |x| mag(Z) / |Z|"""
    aZ = abs(pc[..., 2])
    return (pcm[..., 0] + abs(pc[..., 0] / pc[..., 2]) * pcm[..., 2]) / aZ, (pcm[..., 1] + abs(pc[..., 1] / pc[..., 2]) * pcm[..., 2]) / aZ


def bearing_mags(I):
    """entrywise magnitudes of bearing_rows' parts: the abs-evaluation at |xn|, |yn| plus the magnitude of its derivative times the
    error magnitude of the coordinates (so a coordinate formed by cancellation, e.g. xn = 0, is held to its absolute precision)"""
    m = I.m
    qC, pC = I.cal[:4], I.cal[4:7]
    pfv = np.broadcast_to(I.pf, (m, 3))
    pc_val = camera_point(I.cv[:, :4], I.cv[:, 4:], qC, pC, pfv)
    _, pcm_val = _camera_point_mag(I.cv[:, :4], I.cv[:, 4:], qC, pC, pfv)
    x, y = abs(pc_val[:, 0] / pc_val[:, 2]), abs(pc_val[:, 1] / pc_val[:, 2])
    ex, ey = _coords_err(pc_val, pcm_val)
    xy = np.stack([x, y], axis=-1)
    D = _distort_mags(I.cam, x, y) + (cstep(lambda v: _distort_mags(I.cam.astype(CLD), v[:, 0], v[:, 1]), xy, 2) *
                                      np.stack([ex, ey], axis=-1)[:, None, :]).sum(axis=-1)
    dzn, dzeta, x1, y1 = D[:, :4].reshape(m, 2, 2), D[:, 4:20].reshape(m, 2, 8), D[:, 20], D[:, 21]
    cj, pfj = I.jac_point()
    pfj = np.broadcast_to(pfj, (m, 3))
    pc_j = camera_point(cj[:, :4], cj[:, 4:], qC, pC, pfj)
    pIm, pcm_j = _camera_point_mag(cj[:, :4], cj[:, 4:], qC, pC, pfj)
    X, Y, Z = abs(pc_j[:, 0]), abs(pc_j[:, 1]), abs(pc_j[:, 2])
    mX, mY, mZ = pcm_j[:, 0], pcm_j[:, 1], pcm_j[:, 2]
    zero = 0 * Z
    inv = 1 / Z + mZ / (Z * Z)  # 1 / Z and its first-order error through Z
    dp = np.stack([inv, zero, (X + mX) / (Z * Z) + 2 * X * mZ / (Z * Z * Z),
                   zero, inv, (Y + mY) / (Z * Z) + 2 * Y * mZ / (Z * Z * Z)], axis=-1).reshape(m, 2, 3)
    A = I.w * (dzn @ dp)
    RC = rot_mag(qC)
    B = RC @ rot_mag(cj[:, :4])
    sk = lambda v: abs(_skew(v))
    cam = I.cam
    res = I.w * (abs(I.uv) + np.stack([abs(cam[0]) * x1 + abs(cam[2]), abs(cam[1]) * y1 + abs(cam[3])], axis=-1))
    return {"res": res, "Hf": A @ B, "clone": np.concatenate([A @ (RC @ sk(pIm)), A @ B], axis=-1),
            "extrinsics": np.concatenate([A @ sk(pcm_j + abs(pC)), A], axis=-1), "intrinsics": I.w * dzeta}


# ---------------------------------------------------------------------------------------------------------------------------------
# the point-on-plane row
# ---------------------------------------------------------------------------------------------------------------------------------
def plane_row(pf, pf_fej, cp, cp_fej, sigma_c, do_fej, mutate=None):
    """(res, H_f (3), H_cp (3)) and their magnitudes: the residual at (p, cp), the Jacobians at (p_fej, cp_fej) with do_fej"""
    w = LD(1) / LD(float(sigma_c))
    pf, pff, cp, cpf = ld(pf), ld(pf_fej), ld(cp), ld(cp_fej)
    pj, cj = (pff, cpf) if do_fej else (pf, cp)
    if mutate == "plane row at cp instead of cp_fej":
        cj = cp
    res = -w * plane_h(pf, cp)
    Hf = w * cstep(lambda p: plane_h(p, cj), pj, 3)
    Hcp = w * cstep(lambda c: plane_h(pj, c), cj, 3)
    # magnitudes: d = |cp| (a sum of squares, no cancellation), n = |cp| / d
    d, dj = np.sqrt((cp * cp).sum()), np.sqrt((cj * cj).sum())
    n, nj = abs(cp) / d, abs(cj) / dj
    mag = {"res": w * ((n * abs(pf)).sum() + d), "Hf": w * nj,
           "Hcp": (w / dj) * (abs(pj) + (nj * abs(pj)).sum() * nj + dj * nj)}
    return res, Hf.reshape(3), Hcp.reshape(3), mag


# ---------------------------------------------------------------------------------------------------------------------------------
# anchored representations
# ---------------------------------------------------------------------------------------------------------------------------------
def get_xyz(rep, v):
    """ov_type::Landmark::get_xyz: the position a representation's 3-vector stands for (generic dtype)"""
    if rep in (0, 2):
        return v
    if rep in (1, 3):
        return np.stack([(1 / v[..., 2]) * np.cos(v[..., 0]) * np.sin(v[..., 1]), (1 / v[..., 2]) * np.sin(v[..., 0]) * np.sin(v[..., 1]),
                         (1 / v[..., 2]) * np.cos(v[..., 1])], axis=-1)
    if rep == 4:
        return np.stack([v[..., 0] / v[..., 2], v[..., 1] / v[..., 2], 1 / v[..., 2]], axis=-1)
    raise ValueError(rep)


def to_lambda(rep, p):
    """the representation's 3-vector of the position p (long double); rep 5: its single inverse depth"""
    if rep in (0, 2):
        return p.copy()
    if rep in (1, 3):
        rho = 1 / np.sqrt((p * p).sum())
        return np.array([np.arctan2(p[1], p[0]), np.arccos(rho * p[2]), rho], dtype=LD)
    if rep == 4:
        return np.array([p[0] / p[2], p[1] / p[2], 1 / p[2]], dtype=LD)
    return np.array([1 / p[2]], dtype=LD)


def anchor_to_global(anchor7, calib7, pA):
    """p_FinG = R_GtoA^T R_ItoC^T (p_FinA - p_IinC) + p_AinG (generic dtype)"""
    RA, RC = rot(anchor7[..., :4]), rot(calib7[..., :4])
    return mv(np.swapaxes(RA, -1, -2), mv(np.swapaxes(RC, -1, -2), pA - calib7[..., 4:7])) + anchor7[..., 4:7]


def global_to_anchor(anchor7, calib7, pG):
    return mv(rot(calib7[..., :4]), mv(rot(anchor7[..., :4]), pG - anchor7[..., 4:7])) + calib7[..., 4:7]


def representation_jacobians(rep, do_fej, pF, pF_fej, anchor_val=None, anchor_fej=None, calib=None):
    """(p_FinG, p_FinG_fej, d p_FinG / d lambda (3 x k), d p_FinG / d anchor (3 x 6) or None, d p_FinG / d extrinsics (3 x 6) or None),
    evaluated where ovp_feature_jacobian_full_rep / UpdaterHelper::get_feature_jacobian_representation evaluate them: the global
    representations at p_F (p_F_fej with do_fej); the anchored ones at the value of the anchor and the extrinsics, or with do_fej at
    the anchor's first estimate and the best global point seen from it.  pF: the global position (rep 0, 1) or the position in the
    anchor camera (rep 2..5)."""
    pF, pFf = ld(pF), ld(pF_fej)
    if rep < 2:
        p = pFf if do_fej else pF
        L = np.eye(3, dtype=LD) if rep == 0 else cstep(lambda v: get_xyz(1, v), to_lambda(1, p), 3)
        return pF, pFf, L, None, None
    av, af, cal = ld(anchor_val), ld(anchor_fej), ld(calib)
    pG = anchor_to_global(av, cal, pF)
    anc, pA = av, pF
    if do_fej:
        anc = af
        pA = global_to_anchor(af, cal, pG)
    if rep == 5:  # p_FinA = bearing / rho with the bearing fixed
        bearing = pA / pA[2]
        L = cstep(lambda r: anchor_to_global(anc.astype(CLD), cal.astype(CLD), bearing.astype(CLD) / r[..., 0:1]), to_lambda(5, pA), 1)
    else:
        L = cstep(lambda v: anchor_to_global(anc.astype(CLD), cal.astype(CLD), get_xyz(rep, v)), to_lambda(rep, pA), 3)
    pA_c = pA.astype(CLD)
    Ha = np.concatenate([cstep(lambda q: anchor_to_global(np.concatenate([q, anc[4:].astype(CLD)]), cal.astype(CLD), pA_c), anc[:4], 3,
                               rotation=True),
                         cstep(lambda p: anchor_to_global(np.concatenate([anc[:4].astype(CLD), p]), cal.astype(CLD), pA_c), anc[4:], 3)], axis=-1)
    Hc = np.concatenate([cstep(lambda q: anchor_to_global(anc.astype(CLD), np.concatenate([q, cal[4:].astype(CLD)]), pA_c), cal[:4], 3,
                               rotation=True),
                         cstep(lambda p: anchor_to_global(anc.astype(CLD), np.concatenate([cal[:4].astype(CLD), p]), pA_c), cal[4:7], 3)], axis=-1)
    return pG, pG.copy(), L, Ha, Hc


# ---------------------------------------------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------------------------------------------
def ratio(got, ref, mag, part):
    """entrywise |got - ref| / (C u mag) (0 where both sides are 0, inf where the bound is 0 and they differ)"""
    err = abs(np.asarray(got, dtype=np.float64).astype(LD) - ref)
    bound = LD(C_PART[part]) * LD(U) * mag
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, LD(0), err / bound)
    return np.where(np.isnan(r), LD(np.inf), r)


def worst(got, ref, mag, part):
    r = ratio(got, ref, mag, part)
    return float(r.max()) if r.size else 0.0


MUTATIONS = ("2 p2 x tangential term", "uv_norm at the first estimate", "clone rotation at its value", "skew(p_FinI) at the value",
             "R_ItoC transposed in the extrinsic rotation block", "plane row at cp instead of cp_fej")


def ulp_diff(a, b):
    """largest distance in units in the last place between two float64 arrays of the same shape"""
    a, b = np.asarray(a, dtype=np.float64).ravel(), np.asarray(b, dtype=np.float64).ravel()
    ia, ib = a.view(np.int64), b.view(np.int64)
    ia = np.where(ia < 0, np.int64(-0x8000000000000000) - ia, ia)
    ib = np.where(ib < 0, np.int64(-0x8000000000000000) - ib, ib)
    return int(np.abs(ia - ib).max()) if a.size else 0
