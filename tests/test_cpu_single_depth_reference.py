"""The single-depth landmark form checked without a GPU: the library's context-free host helpers (ovp_landmark_set_from_xyz /
ovp_landmark_get_xyz, ovp_anchor_change_jacobian: the functions ovp_slam_perform_anchor_change and the value tables use) against the
long-double restatement of tests/single_depth_reference.py, and that restatement against what it restates:
- Landmark::set_from_xyz / get_xyz of the library for every representation against long double, and the round trip;
- the library's anchor-change Phi, new value and first estimate against the long-double restatement (both anchors, with and without the
  extrinsics and FEJ);
- the anchor-change Jacobian Phi of UpdaterSLAM::perform_anchor_change (:802-838) against a numerical derivative of what it linearises: the
  inverse depth along the new bearing that puts the point where the old anchor's inverse depth puts it, in the least-squares sense;
- the representation Jacobian of the form (the library's context-free ovp_feature_jacobian_representation and the oracle's) equal to the
  third column of ANCHORED_MSCKF_INVERSE_DEPTH's at the same p_FinA, and to the long-double one of feature_jacobian_reference."""
import numpy as np
import pytest

import feature_jacobian_reference as fjr
import single_depth_reference as sd
from test_cpu_abi import _rep_call

LD = np.longdouble


def _pose(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    if q[3] < 0:
        q = -q
    return np.concatenate([q, rng.normal(size=3)])


def _near(rng, pose, s=0.05):
    """a clone near pose: rotated by ~s rad and moved by ~s"""
    from ov_plane_b200 import jpl
    out = pose.copy()
    out[:4] = jpl.quat_left_update(pose[:4], s * rng.normal(size=3))
    out[4:] += s * rng.normal(size=3)
    return out


def _lib():
    import ctypes as C
    from ov_plane_b200 import api
    return C.CDLL(api.LIB_PATH)


def _ptr(a):
    import ctypes as C
    return a.ctypes.data_as(C.c_void_p)


def test_library_set_from_xyz_and_get_xyz_against_long_double():
    lib = _lib()
    rng = np.random.default_rng(9)
    for _ in range(20):
        p = np.array([0.5, -0.4, 4.0]) + rng.normal(size=3) * [1.0, 1.0, 1.5]
        for rep in range(6):
            n = 4 if rep == 5 else 3
            v, back = np.zeros(n), np.zeros(3)
            assert lib.ovp_landmark_set_from_xyz(rep, _ptr(p), _ptr(v)) == 0
            want = sd.set_from_xyz(fjr.ld(p)) if rep == 5 else fjr.to_lambda(rep, fjr.ld(p))
            # a few ulps (the angles of 1 / 3 go through atan2 / acos)
            assert np.abs(np.asarray(fjr.ld(v) - want, dtype=np.float64)).max() <= 2e-15 * max(1.0, float(np.abs(np.asarray(want, dtype=np.float64)).max()))
            assert lib.ovp_landmark_get_xyz(rep, _ptr(v), _ptr(back)) == 0
            got_ld = sd.get_xyz(fjr.ld(v)) if rep == 5 else fjr.get_xyz(rep, fjr.ld(v))
            assert np.abs(np.asarray(fjr.ld(back) - got_ld, dtype=np.float64)).max() <= 4e-15 * float(np.abs(p).max())
            assert np.abs(back - p).max() <= 1e-14 * np.abs(p).max()
    assert lib.ovp_landmark_get_xyz(6, _ptr(p), _ptr(np.zeros(3))) != 0


@pytest.mark.parametrize("do_fej", [0, 1])
@pytest.mark.parametrize("calib_pose", [0, 1])
@pytest.mark.parametrize("same_anchor", [0, 1])
def test_library_anchor_change_against_long_double(do_fej, calib_pose, same_anchor):
    import ctypes as C
    fjr.require_long_double()
    lib = _lib()
    rng = np.random.default_rng(31 + 4 * do_fej + 2 * calib_pose + same_anchor)
    for _ in range(6):
        old, cal = _pose(rng), _pose(rng)
        oldf = _near(rng, old, 0.01)
        new, newf = (old.copy(), oldf.copy()) if same_anchor else (_near(rng, old), None)
        if newf is None:
            newf = _near(rng, new, 0.01)
        pA = np.array([0.3, -0.2, 3.5]) + 0.2 * rng.normal(size=3)
        v = np.asarray(sd.set_from_xyz(fjr.ld(pA)), dtype=np.float64)
        vf = np.asarray(sd.set_from_xyz(fjr.ld(pA * 1.01)), dtype=np.float64)
        Phi, vn, fn = np.zeros(63), np.zeros(4), np.zeros(4)
        rows, cols = C.c_int(0), C.c_int(0)
        st = lib.ovp_anchor_change_jacobian(5, do_fej, calib_pose, same_anchor, _ptr(v), _ptr(vf), _ptr(old), _ptr(oldf), _ptr(new), _ptr(newf),
                                            _ptr(cal), _ptr(Phi), C.byref(rows), C.byref(cols), _ptr(vn), _ptr(fn))
        assert st == 0 and rows.value == 1
        ref = sd.anchor_change(v, vf, old, oldf, new, newf, cal, do_fej, bool(calib_pose))
        P_ref = np.asarray(ref["Phi"], dtype=np.float64)
        assert cols.value == P_ref.shape[1]
        got = Phi[:cols.value]
        assert np.abs(got - P_ref[0]).max() <= 1e-13 * np.abs(P_ref).max(), (got, P_ref)
        assert np.allclose(vn, np.asarray(ref["value"], dtype=np.float64), rtol=1e-14, atol=1e-15)
        assert np.allclose(fn, np.asarray(ref["fej"], dtype=np.float64), rtol=1e-14, atol=1e-15)
    # a global form is not anchored
    assert lib.ovp_anchor_change_jacobian(1, 0, 0, 0, _ptr(v), _ptr(vf), _ptr(old), _ptr(oldf), _ptr(new), _ptr(newf), _ptr(cal), _ptr(Phi),
                                          C.byref(rows), C.byref(cols), _ptr(vn), _ptr(fn)) != 0


def test_set_from_xyz_and_get_xyz_round_trip():
    fjr.require_long_double()
    rng = np.random.default_rng(5)
    for _ in range(50):
        p = fjr.ld(np.array([0.5, -0.4, 4.0]) + rng.normal(size=3) * [1.0, 1.0, 1.5])
        v = sd.set_from_xyz(p)
        assert abs(v[3] - 1) <= float(np.finfo(LD).eps) and v[0] == 1 / p[2]
        back = sd.get_xyz(v)
        assert float(np.abs(back - p).max() / np.abs(p).max()) < 8 * float(np.finfo(LD).eps)
        vf = sd.set_from_xyz(p * LD(1.01))  # the first estimate: its own bearing and depth
        assert np.abs(sd.get_xyz(vf) - p * LD(1.01)).max() < 8 * float(np.finfo(LD).eps) * float(np.abs(p).max())
        assert np.abs(v[1:] - vf[1:]).max() < 8 * float(np.finfo(LD).eps)  # a scaled point keeps its bearing


@pytest.mark.parametrize("calib_pose", [False, True])
@pytest.mark.parametrize("same_anchor", [False, True])
def test_anchor_change_phi_against_a_numerical_derivative(calib_pose, same_anchor):
    """Phi = H_f_new^+ (H_f_old d rho_old + H_x_old dx_old - H_x_new dx_new) is the derivative of rho_new(x) = argmin_rho |g_new(rho) - g_old|^2,
    g_new(rho) = p_FinG of the new bearing at inverse depth rho from the new anchor, g_old = p_FinG from the old anchor; at the linearisation
    point the residual is zero, so the least-squares solution's derivative is exactly the pseudo-inverse times the residual's."""
    rng = np.random.default_rng(7 + 2 * calib_pose + same_anchor)
    old, cal = _pose(rng), _pose(rng)
    new = old.copy() if same_anchor else _near(rng, old)
    pA = np.array([0.3, -0.2, 3.5])
    v = sd.set_from_xyz(fjr.ld(pA))
    ref = sd.anchor_change(v, v, old, old, new, new, cal, 0, calib_pose)
    b_new = np.asarray(ref["value"][1:], dtype=np.float64)

    from ov_plane_b200 import jpl

    def pert(pose, d):
        out = pose.copy()
        out[:4] = jpl.quat_left_update(pose[:4], d[:3])
        out[4:] += d[3:]
        return out

    def rho_new(x):
        o, c, n, r = x["old"], x["cal"], x["new"], x["rho"]
        g_old = fjr.anchor_to_global(o, c, np.asarray(v[1:], dtype=np.float64) / r)
        # p_FinG(rho) = A / rho + t along the fixed new bearing: the least-squares 1/rho is u^T (g_old - t) / u^T u
        t = fjr.anchor_to_global(n, c, np.zeros(3))
        u = fjr.anchor_to_global(n, c, b_new) - t
        return 1.0 / (u @ (g_old - t) / (u @ u))

    x0 = dict(old=old, cal=cal, new=new, rho=float(v[0]))
    assert abs(rho_new(x0) - float(ref["value"][0])) < 1e-12
    eps, num = 1e-6, []
    blocks = [("old", 6)] + ([("cal", 6)] if calib_pose else []) + ([] if same_anchor else [("new", 6)]) + [("rho", 1)]
    for name, n in blocks:
        for k in range(n):
            d = np.zeros(n)
            d[k] = eps
            xs = []
            for sgn in (1, -1):
                x = dict(x0)
                if name == "rho":
                    x["rho"] = x0["rho"] + sgn * eps
                elif same_anchor and name == "old":  # one clone: old and new anchor move together
                    x["old"] = x["new"] = pert(old, sgn * d)
                else:
                    x[name] = pert(x0[name], sgn * d)
                xs.append(rho_new(x))
            num.append((xs[0] - xs[1]) / (2 * eps))
    Phi = np.asarray(ref["Phi"], dtype=np.float64)[0]
    assert Phi.shape == (len(num),)
    assert np.allclose(Phi, num, rtol=1e-6, atol=1e-7), (Phi, num)


@pytest.mark.parametrize("do_fej", [0, 1])
def test_single_depth_jacobian_is_the_third_column_of_the_msckf_inverse_depth_one(do_fej):
    import ctypes as C
    import oracle_backend as ob
    from ov_plane_b200 import api
    lib, orc = C.CDLL(api.LIB_PATH), C.CDLL(ob._LIB)
    rng = np.random.default_rng(3 + do_fej)
    for _ in range(8):
        anc, cal = _pose(rng), _pose(rng)
        ancf = _near(rng, anc)
        pA = np.array([0.4, -0.3, 3.0]) + 0.2 * rng.normal(size=3)
        pG = fjr.anchor_to_global(anc, cal, pA)
        for who in (lib, orc):
            fn = "ovp_feature_jacobian_representation" if who is lib else "orc_feature_jacobian_representation"
            H4, Ha4, Hc4, _ = _rep_call(who, fn, 4, do_fej, pG, pG, pA, anc, ancf, cal)
            H5, Ha5, Hc5, has = _rep_call(who, fn, 5, do_fej, pG, pG, pA, anc, ancf, cal)
            assert has == 1 and H5.shape == (3, 1)
            assert np.allclose(H5[:, 0], H4[:, 2], rtol=1e-13, atol=1e-15)
            assert np.array_equal(Ha5, Ha4) and np.array_equal(Hc5, Hc4)
        _, _, L5, _, _ = fjr.representation_jacobians(5, do_fej, pA, pA, anc, ancf, cal)
        _, _, L4, _, _ = fjr.representation_jacobians(4, do_fej, pA, pA, anc, ancf, cal)
        assert np.abs(np.asarray(L5[:, 0] - L4[:, 2], dtype=np.float64)).max() < 1e-15 * float(np.abs(np.asarray(L4, dtype=np.float64)).max())
        assert np.allclose(H5[:, 0], np.asarray(L5[:, 0], dtype=np.float64), rtol=1e-12, atol=1e-14)
