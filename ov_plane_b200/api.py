"""ctypes binding of the C ABI in include/ovp.h (libovp.so).  Plumbing only: every method is one C call.

There is NO CPU fallback: importing this module fails loudly when the CUDA library has not been built
(`python -c "import __graft_entry__ as g; g.build()"`), and creating a Context fails loudly without a CUDA device.
Method names mirror the reference's call surface (StateHelper::EKFUpdate -> Context.ekf_update, ...).
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("OVP_LIB", os.path.join(_HERE, "lib", "libovp.so"))  # OVP_LIB: A/B builds while tuning

OVP_KIND_VEC, OVP_KIND_POSE, OVP_KIND_IMU, OVP_KIND_LANDMARK = 0, 1, 2, 3


class OvpError(RuntimeError):
    def __init__(self, status, msg):
        RuntimeError.__init__(self, "ovp status %d: %s" % (status, msg))
        self.status = status


class StateOptions(C.Structure):
    _fields_ = [("do_fej", C.c_int), ("imu_avg", C.c_int), ("use_rk4_integration", C.c_int), ("do_calib_camera_pose", C.c_int),
                ("do_calib_camera_intrinsics", C.c_int), ("do_calib_camera_timeoffset", C.c_int), ("max_clone_size", C.c_int),
                ("max_aruco_features", C.c_int), ("sigma_constraint", C.c_double), ("const_init_multi", C.c_double),
                ("const_init_chi2", C.c_double), ("sigma_plane_merge", C.c_double), ("plane_merge_chi2", C.c_double),
                ("plane_merge_deg_max", C.c_double)]


class FeatureBatch(C.Structure):
    _fields_ = [("F", C.c_int), ("meas_offset", C.c_void_p), ("meas_clone", C.c_void_p), ("uv", C.c_void_p), ("p_FinG", C.c_void_p),
                ("p_FinG_original", C.c_void_p), ("featid", C.c_void_p), ("planeid", C.c_void_p), ("nplanes", C.c_int),
                ("plane_ids", C.c_void_p), ("plane_cp", C.c_void_p)]


class PlaneLandmarks(C.Structure):
    _fields_ = [("n", C.c_int), ("featid", C.c_void_p), ("planeid", C.c_void_p)]


class UpdaterOptions(C.Structure):
    _fields_ = [("sigma_pix", C.c_double), ("chi2_multipler", C.c_double)]


class PlaneFitOptions(C.Structure):
    _fields_ = [("min_inlier_num", C.c_int), ("max_cond_number", C.c_double), ("shuffle_kind", C.c_int)]


class PlaneRefineOptions(C.Structure):
    _fields_ = [("sigma_px_norm", C.c_double), ("sigma_c", C.c_double), ("max_num_iterations", C.c_int)]


class FeatureTracks(C.Structure):
    _fields_ = [("F", C.c_int), ("meas_offset", C.c_void_p), ("meas_clone", C.c_void_p), ("uv", C.c_void_p), ("uv_norm", C.c_void_p),
                ("featid", C.c_void_p), ("planeid", C.c_void_p)]


class PlaneInitOptions(C.Structure):
    _fields_ = [("sigma_pix", C.c_double), ("max_msckf_plane", C.c_int), ("plane_init_min_feat", C.c_int), ("plane_init_max_cond", C.c_double),
                ("shuffle_kind", C.c_int), ("tri", C.c_void_p)]


DEBUG_LIB_PATH = os.path.join(_HERE, "lib", "libovp_debug.so")  # product sources + include/ovp_debug.h hooks (tools/, kernel unit tests)


def load_library(path=None):
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise ImportError("ov_plane_b200: %s is missing. Build the CUDA library first: "
                          "python -c 'import __graft_entry__ as g; g.build()'  (no CPU fallback exists)" % path)
    lib = C.CDLL(path)
    lib.ovp_last_error.restype = C.c_char_p
    lib.ovp_status_string.restype = C.c_char_p
    lib.ovp_get_timestamp.restype = C.c_double
    lib.ovp_launch_count.restype = C.c_int64
    lib.ovp_stream.restype = C.c_void_p
    lib.ovp_slam_plane_of.restype = C.c_int64
    return lib


_lib = None


_debug_lib = None


def lib(debug=False):
    global _lib, _debug_lib
    if debug:
        if _debug_lib is None:
            _debug_lib = load_library(DEBUG_LIB_PATH)
        return _debug_lib
    if _lib is None:
        _lib = load_library()
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _colmajor(a):
    return np.asfortranarray(a, dtype=np.float64)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


class Context(object):
    """One device-resident filter state (the reference's `State` + `StateHelper` + `Propagator` seam)."""

    def __init__(self, options, device=0, max_state=640, max_meas_rows=40000, debug=False):
        self.lib = lib(debug)  # debug=True: libovp_debug.so (exports the include/ovp_debug.h hooks as well)
        self.opt = StateOptions(**{k: options[k] for k, _ in StateOptions._fields_})
        self.h = C.c_void_p()
        st = self.lib.ovp_create(C.byref(self.opt), int(device), int(max_state), int(max_meas_rows), C.byref(self.h))
        if st != 0:
            msg = self.lib.ovp_last_error(self.h).decode() if self.h else self.lib.ovp_status_string(st).decode()
            raise OvpError(st, "ovp_create failed (a CUDA device is required, there is no CPU fallback): " + msg)

    def close(self):
        if self.h:
            self.lib.ovp_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, st):
        if st != 0:
            raise OvpError(st, self.lib.ovp_last_error(self.h).decode())

    # ---- State ----
    def set_chi2_table(self, q):
        q = _f64(q)
        self._ck(self.lib.ovp_set_chi2_table(self.h, _p(q), len(q)))

    def cov_rows(self):
        return self.lib.ovp_cov_rows(self.h)

    def cov(self):
        n = self.cov_rows()
        out = np.zeros((n, n), order="F")
        self._ck(self.lib.ovp_cov_download(self.h, _p(out), n))
        return out

    def cov_upload(self, P):
        P = _colmajor(P)
        self._ck(self.lib.ovp_cov_upload(self.h, _p(P), P.shape[0], P.shape[0]))

    def handle_imu(self):
        return self.lib.ovp_handle_imu(self.h)

    def handle_dt(self):
        return self.lib.ovp_handle_dt(self.h)

    def handle_calib(self):
        return self.lib.ovp_handle_calib(self.h)

    def handle_intrinsics(self):
        return self.lib.ovp_handle_intrinsics(self.h)

    def var_id(self, h):
        return self.lib.ovp_var_id(self.h, h)

    def var_size(self, h):
        return self.lib.ovp_var_size(self.h, h)

    def var_set(self, h, value, fej=None):
        v = _f64(value)
        f = _f64(fej) if fej is not None else None
        self._ck(self.lib.ovp_var_set(self.h, h, _p(v), _p(f)))

    def var_get(self, h):
        n = self.lib.ovp_var_value_size(self.h, h)
        v, f = np.zeros(n), np.zeros(n)
        self._ck(self.lib.ovp_var_get(self.h, h, _p(v), _p(f)))
        return v, f

    def variable_order(self):
        n = self.lib.ovp_num_variables(self.h)
        o = np.zeros(n, dtype=np.int32)
        self._ck(self.lib.ovp_variable_order(self.h, _p(o)))
        return o.tolist()

    def set_timestamp(self, t):
        self.lib.ovp_set_timestamp(self.h, C.c_double(t))

    def get_timestamp(self):
        return self.lib.ovp_get_timestamp(self.h)

    def add_clone_raw(self, t, value7, fej7):
        v, f, h = _f64(value7), _f64(fej7), C.c_int(-1)
        self._ck(self.lib.ovp_add_clone_raw(self.h, C.c_double(t), _p(v), _p(f), C.byref(h)))
        return h.value

    def add_plane_raw(self, planeid, cp, cp_fej):
        v, f, h = _f64(cp), _f64(cp_fej), C.c_int(-1)
        self._ck(self.lib.ovp_add_plane_raw(self.h, C.c_int64(int(planeid)), _p(v), _p(f), C.byref(h)))
        return h.value

    def add_slam_raw(self, featid, p, p_fej):
        v, f, h = _f64(p), _f64(p_fej), C.c_int(-1)
        self._ck(self.lib.ovp_add_slam_raw(self.h, C.c_int64(int(featid)), _p(v), _p(f), C.byref(h)))
        return h.value

    def plane_handle(self, planeid):
        return self.lib.ovp_plane_handle(self.h, C.c_int64(int(planeid)))

    def clone_handle(self, t):
        return self.lib.ovp_clone_handle(self.h, C.c_double(t))

    # ---- StateHelper ----
    def set_initial_covariance(self, cov, handles):
        cov, hs = _colmajor(cov), _i32(handles)
        self._ck(self.lib.ovp_set_initial_covariance(self.h, _p(cov), cov.shape[0], _p(hs), len(hs)))

    def get_marginal_covariance(self, handles):
        hs = _i32(handles)
        n = sum(self.var_size(int(h)) for h in hs)
        out = np.zeros((n, n), order="F")
        self._ck(self.lib.ovp_get_marginal_covariance(self.h, _p(hs), len(hs), _p(out)))
        return out

    def ekf_propagation(self, new_handles, old_handles, Phi, Q):
        nh, oh, Phi, Q = _i32(new_handles), _i32(old_handles), _colmajor(Phi), _colmajor(Q)
        self._ck(self.lib.ovp_ekf_propagation(self.h, _p(nh), len(nh), _p(oh), len(oh), _p(Phi), Phi.shape[0], Phi.shape[1], _p(Q)))

    def ekf_update(self, handles, H, res, Rdiag=None):
        hs, H, res = _i32(handles), _colmajor(H), _f64(res)
        R = _f64(Rdiag) if Rdiag is not None else None
        self._ck(self.lib.ovp_ekf_update(self.h, _p(hs), len(hs), _p(H), H.shape[0], _p(res), _p(R)))

    def marginalize(self, h):
        self._ck(self.lib.ovp_marginalize(self.h, h))

    def clone(self, h):
        nh = C.c_int(-1)
        self._ck(self.lib.ovp_clone(self.h, h, C.byref(nh)))
        return nh.value

    def augment_clone(self, t, last_w):
        w, nh = _f64(last_w), C.c_int(-1)
        self._ck(self.lib.ovp_augment_clone(self.h, C.c_double(t), _p(w), C.byref(nh)))
        return nh.value

    def marginalize_old_clone(self):
        self._ck(self.lib.ovp_marginalize_old_clone(self.h))

    def marginalize_slam(self):
        self._ck(self.lib.ovp_marginalize_slam(self.h))

    def initialize(self, kind, value, fej, tag, handles, H_R, H_L, res, sigma2, chi2_mult, do_update=True):
        v, f, hs = _f64(value), _f64(fej), _i32(handles)
        H_R, H_L, res = _colmajor(H_R), _colmajor(H_L), _f64(res)
        acc, nh = C.c_int(0), C.c_int(-1)
        self._ck(self.lib.ovp_initialize(self.h, kind, len(v), _p(v), _p(f), C.c_int64(int(tag)), _p(hs), len(hs), _p(H_R), _p(H_L),
                                         _p(res), H_R.shape[0], C.c_double(sigma2), C.c_double(chi2_mult), int(do_update), C.byref(acc),
                                         C.byref(nh)))
        return bool(acc.value), nh.value

    def initialize_invertible(self, kind, value, fej, tag, handles, H_R, H_L, res, sigma2):
        v, f, hs = _f64(value), _f64(fej), _i32(handles)
        H_R, H_L, res = _colmajor(H_R), _colmajor(H_L), _f64(res)
        nh = C.c_int(-1)
        self._ck(self.lib.ovp_initialize_invertible(self.h, kind, len(v), _p(v), _p(f), C.c_int64(int(tag)), _p(hs), len(hs), _p(H_R),
                                                    _p(H_L), _p(res), C.c_double(sigma2), C.byref(nh)))
        return nh.value

    def merge_planes_and_marginalize(self, feat2plane, plane2oldplane):
        ff = np.array(list(feat2plane.keys()), dtype=np.int64)
        fp = np.array(list(feat2plane.values()), dtype=np.int64)
        mn, mo = [], []
        for k, olds in plane2oldplane.items():
            for o in olds:
                mn.append(k)
                mo.append(o)
        mn, mo = np.array(mn, dtype=np.int64), np.array(mo, dtype=np.int64)
        self._ck(self.lib.ovp_merge_planes_and_marginalize(self.h, _p(ff), _p(fp), len(ff), _p(mn), _p(mo), len(mn)))

    # ---- UpdaterHelper / UpdaterPlane statics ----
    def feature_jacobian_full(self, clone_handles, uv, p_FinG, p_FinG_fej, planeid, cp, cp_fej, sigma_px, sigma_c):
        ch, uv = _i32(clone_handles), np.ascontiguousarray(uv, dtype=np.float32)
        m = len(ch)
        rows_cap, cols_cap = 3 * m + 1, 14 + 6 * m + 3
        Hf, Hx, res = np.zeros(rows_cap * 6), np.zeros(rows_cap * cols_cap), np.zeros(rows_cap)
        xo = np.zeros(m + 3, dtype=np.int32)
        hfc, hxc, rows, xon = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        pf, pff = _f64(p_FinG), _f64(p_FinG_fej)
        cpv = _f64(cp) if cp is not None else np.zeros(3)
        cpf = _f64(cp_fej) if cp_fej is not None else np.zeros(3)
        self._ck(self.lib.ovp_feature_jacobian_full(self.h, m, _p(ch), _p(uv), _p(pf), _p(pff), C.c_int64(int(planeid)), _p(cpv), _p(cpf),
                                                    C.c_double(sigma_px), C.c_double(sigma_c), _p(Hf), C.byref(hfc), _p(Hx), C.byref(hxc),
                                                    _p(res), C.byref(rows), _p(xo), C.byref(xon)))
        r = rows.value
        return (Hf[:r * hfc.value].reshape((r, hfc.value), order="F").copy(), Hx[:r * hxc.value].reshape((r, hxc.value), order="F").copy(),
                res[:r].copy(), xo[:xon.value].tolist())

    def feature_jacobian_full_rep(self, clone_handles, uv, representation, anchor_clone_handle, p_F, p_F_fej, sigma_px):
        ch, uv = _i32(clone_handles), np.ascontiguousarray(uv, dtype=np.float32)
        m = len(ch)
        rows_cap, cols_cap = 2 * m, 14 + 6 * (m + 1)
        Hf, Hx, res = np.zeros(rows_cap * 3), np.zeros(rows_cap * cols_cap), np.zeros(rows_cap)
        xo = np.zeros(m + 4, dtype=np.int32)
        hfc, hxc, rows, xon = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        pf, pff = _f64(p_F), _f64(p_F_fej)
        self._ck(self.lib.ovp_feature_jacobian_full_rep(self.h, m, _p(ch), _p(uv), int(representation), int(anchor_clone_handle), _p(pf), _p(pff),
                                                        C.c_double(sigma_px), _p(Hf), C.byref(hfc), _p(Hx), C.byref(hxc), _p(res), C.byref(rows),
                                                        _p(xo), C.byref(xon)))
        r = rows.value
        return (Hf[:r * hfc.value].reshape((r, hfc.value), order="F").copy(), Hx[:r * hxc.value].reshape((r, hxc.value), order="F").copy(),
                res[:r].copy(), xo[:xon.value].tolist())

    def slam_set_representation(self, featid, representation, anchor_clone_handle=-1):
        self._ck(self.lib.ovp_slam_set_representation(self.h, C.c_int64(int(featid)), int(representation), int(anchor_clone_handle)))

    def slam_get_representation(self, featid):
        rep, anc = C.c_int(-1), C.c_int(-1)
        self._ck(self.lib.ovp_slam_get_representation(self.h, C.c_int64(int(featid)), C.byref(rep), C.byref(anc)))
        return rep.value, anc.value

    def slam_perform_anchor_change(self, featid, new_anchor_clone_handle):
        self._ck(self.lib.ovp_slam_perform_anchor_change(self.h, C.c_int64(int(featid)), int(new_anchor_clone_handle)))

    def slam_change_anchors(self):
        n = C.c_int(0)
        self._ck(self.lib.ovp_slam_change_anchors(self.h, C.byref(n)))
        return n.value

    def nullspace_project_inplace(self, H_f, H_x, res, H_cp=None):
        H_f, H_x, res = _colmajor(H_f).copy(order="F"), _colmajor(H_x).copy(order="F"), _f64(res).copy()
        rows, ro = H_f.shape[0], C.c_int()
        if H_cp is None:
            self._ck(self.lib.ovp_nullspace_project_inplace(self.h, _p(H_f), H_f.shape[1], _p(H_x), H_x.shape[1], _p(res), rows, C.byref(ro)))
            r = ro.value
            return H_x.ravel(order="F")[:r * H_x.shape[1]].reshape((r, H_x.shape[1]), order="F").copy(), res[:r].copy()
        H_cp = _colmajor(H_cp).copy(order="F")
        self._ck(self.lib.ovp_plane_nullspace_project_inplace(self.h, _p(H_f), H_f.shape[1], _p(H_x), H_x.shape[1], _p(H_cp), _p(res), rows,
                                                              C.byref(ro)))
        r = ro.value
        return (H_x.ravel(order="F")[:r * H_x.shape[1]].reshape((r, H_x.shape[1]), order="F").copy(),
                H_cp.ravel(order="F")[:r * 3].reshape((r, 3), order="F").copy(), res[:r].copy())

    def measurement_compress_inplace(self, H_x, res, H_cp=None):
        H_x, res = _colmajor(H_x).copy(order="F"), _f64(res).copy()
        rows, cols, ro = H_x.shape[0], H_x.shape[1], C.c_int()
        if H_cp is None:
            self._ck(self.lib.ovp_measurement_compress_inplace(self.h, _p(H_x), cols, _p(res), rows, C.byref(ro)))
            r = ro.value
            return H_x.ravel(order="F")[:r * cols].reshape((r, cols), order="F").copy(), res[:r].copy()
        H_cp = _colmajor(H_cp).copy(order="F")
        self._ck(self.lib.ovp_plane_measurement_compress_inplace(self.h, _p(H_x), cols, _p(H_cp), _p(res), rows, C.byref(ro)))
        r = ro.value
        return (H_x.ravel(order="F")[:r * cols].reshape((r, cols), order="F").copy(), H_cp.ravel(order="F")[:r * 3].reshape((r, 3), order="F").copy(),
                res[:r].copy())

    # ---- UpdaterMSCKF ----
    @staticmethod
    def _batch_struct(b):
        fb = FeatureBatch()
        fb.F = int(b["F"])
        keep = []
        for k in ("meas_offset", "meas_clone", "uv", "p_FinG", "p_FinG_original", "featid", "planeid", "plane_ids", "plane_cp"):
            a = np.ascontiguousarray(b[k])
            keep.append(a)
            setattr(fb, k, a.ctypes.data)
        fb.nplanes = len(b["plane_ids"])
        return fb, keep

    def msckf_update(self, batch, sigma_pix=1.0, chi2_mult=1.0):
        fb, keep = self._batch_struct(batch)
        uo = UpdaterOptions(sigma_pix, chi2_mult)
        F, npl = fb.F, max(1, fb.nplanes)
        fs, fc = np.zeros(F, dtype=np.int32), np.zeros(F)
        ps, pc = np.zeros(npl, dtype=np.int32), np.zeros(npl)
        hx, hxn = np.zeros(4096, dtype=np.int32), C.c_int(0)
        self._ck(self.lib.ovp_msckf_update(self.h, C.byref(fb), C.byref(uo), _p(fs), _p(fc), _p(ps), _p(pc), _p(hx), C.byref(hxn)))
        return dict(feat_status=fs, feat_chi2=fc, plane_status=ps[:fb.nplanes], plane_chi2=pc[:fb.nplanes], hx_order=hx[:hxn.value].tolist())

    @staticmethod
    def _landmarks_struct(featid, planeid):
        fid = np.ascontiguousarray(featid, dtype=np.int64).ravel()
        pid = np.ascontiguousarray(planeid, dtype=np.int64).ravel()
        if fid.shape != pid.shape:
            raise ValueError("featid and planeid need one entry per landmark")
        return PlaneLandmarks(len(fid), fid.ctypes.data, pid.ctypes.data), (fid, pid)

    def msckf_update_landmarks(self, batch, lm_featid, lm_planeid, sigma_pix=1.0, chi2_mult=1.0):
        """msckf_update with use_plane_constraint_slamu: (lm_featid[i], lm_planeid[i]) are the feat2plane entries of the caller's SLAM
        landmarks; the ones on planes of the batch that are not in the state join those planes' updates."""
        fb, keep = self._batch_struct(batch)
        lm, keep_lm = self._landmarks_struct(lm_featid, lm_planeid)
        uo = UpdaterOptions(sigma_pix, chi2_mult)
        F, npl = fb.F, max(1, fb.nplanes)
        fs, fc = np.zeros(F, dtype=np.int32), np.zeros(F)
        ps, pc = np.zeros(npl, dtype=np.int32), np.zeros(npl)
        hx, hxn = np.zeros(4096, dtype=np.int32), C.c_int(0)
        self._ck(self.lib.ovp_msckf_update_landmarks(self.h, C.byref(fb), C.byref(lm), C.byref(uo), _p(fs), _p(fc), _p(ps), _p(pc), _p(hx),
                                                     C.byref(hxn)))
        return dict(feat_status=fs, feat_chi2=fc, plane_status=ps[:fb.nplanes], plane_chi2=pc[:fb.nplanes], hx_order=hx[:hxn.value].tolist())

    def plane_init(self, batch, sigma_pix=1.0, chi2_mult=1.0):
        fb, keep = self._batch_struct(batch)
        uo = UpdaterOptions(sigma_pix, chi2_mult)
        npl = max(1, fb.nplanes)
        ps, nh = np.zeros(npl, dtype=np.int32), np.zeros(npl, dtype=np.int32)
        self._ck(self.lib.ovp_plane_init(self.h, C.byref(fb), C.byref(uo), _p(ps), _p(nh)))
        return dict(plane_status=ps[:fb.nplanes], new_handles=nh[:fb.nplanes])

    def plane_init_tracks(self, tracks, sigma_pix=1.0, max_msckf_plane=20, plane_init_min_feat=8, plane_init_max_cond=200.0, shuffle_kind=0):
        """UpdaterPlane::init_vio_plane end to end on raw tracks (dict: meas_offset, meas_clone, uv, uv_norm, featid, planeid; see
        include/ovp.h ovp_plane_init_tracks).  Returns feat_status, p_FinG, plane_ids, plane_status, new_handles, cp."""
        mo, mc = _i32(tracks["meas_offset"]), _i32(tracks["meas_clone"])
        uv = np.ascontiguousarray(tracks["uv"], dtype=np.float32)
        uvn = np.ascontiguousarray(tracks["uv_norm"], dtype=np.float32)
        fid = np.ascontiguousarray(tracks["featid"], dtype=np.int64)
        pid = np.ascontiguousarray(tracks["planeid"], dtype=np.int64)
        F = len(mo) - 1
        t = FeatureTracks(F, mo.ctypes.data, mc.ctypes.data, uv.ctypes.data, uvn.ctypes.data, fid.ctypes.data, pid.ctypes.data)
        o = PlaneInitOptions(float(sigma_pix), int(max_msckf_plane), int(plane_init_min_feat), float(plane_init_max_cond), int(shuffle_kind), None)
        n = max(1, F)
        fs, pf, npl = np.zeros(n, dtype=np.int32), np.zeros((n, 3)), C.c_int(0)
        pids, ps, nh, cp = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32), np.zeros((n, 3))
        self._ck(self.lib.ovp_plane_init_tracks(self.h, C.byref(t), C.byref(o), _p(fs), _p(pf), C.byref(npl), _p(pids), _p(ps), _p(nh), _p(cp)))
        k = npl.value
        return dict(feat_status=fs[:F], p_FinG=pf[:F], plane_ids=pids[:k], plane_status=ps[:k], new_handles=nh[:k], cp=cp[:k])

    # ---- UpdaterSLAM ----
    def slam_update(self, b, sigma_pix=1.0, chi2_mult=1.0, use_plane_constraint=True):
        F = int(b["F"])
        uo = UpdaterOptions(sigma_pix, chi2_mult)
        fs, fc = np.zeros(max(1, F), dtype=np.int32), np.zeros(max(1, F))
        mo, mc = _i32(b["meas_offset"]), _i32(b["meas_clone"])
        uv = np.ascontiguousarray(b["uv"], dtype=np.float32)
        fid = np.ascontiguousarray(b["featid"], dtype=np.int64)
        pid = np.ascontiguousarray(b["planeid"], dtype=np.int64)
        self._ck(self.lib.ovp_slam_update(self.h, F, _p(mo), _p(mc), _p(uv), _p(fid), _p(pid), C.byref(uo), int(bool(use_plane_constraint)),
                                          _p(fs), _p(fc)))
        return dict(feat_status=fs[:F], feat_chi2=fc[:F])

    def slam_delayed_init(self, b, sigma_pix=1.0, chi2_mult=1.0, use_plane_constraint=True):
        F = int(b["F"])
        uo = UpdaterOptions(sigma_pix, chi2_mult)
        fs, nh = np.zeros(max(1, F), dtype=np.int32), np.zeros(max(1, F), dtype=np.int32)
        mo, mc = _i32(b["meas_offset"]), _i32(b["meas_clone"])
        uv = np.ascontiguousarray(b["uv"], dtype=np.float32)
        pf, pfo = _f64(b["p_FinG"]), _f64(b["p_FinG_original"])
        fid = np.ascontiguousarray(b["featid"], dtype=np.int64)
        pid = np.ascontiguousarray(b["planeid"], dtype=np.int64)
        self._ck(self.lib.ovp_slam_delayed_init(self.h, F, _p(mo), _p(mc), _p(uv), _p(pf), _p(pfo), _p(fid), _p(pid), C.byref(uo),
                                                int(bool(use_plane_constraint)), _p(fs), _p(nh)))
        return dict(feat_status=fs[:F], new_handles=nh[:F])

    def slam_handle(self, featid):
        return self.lib.ovp_slam_handle(self.h, C.c_int64(int(featid)))

    def slam_should_marg(self, featid):
        return self.lib.ovp_slam_should_marg(self.h, C.c_int64(int(featid)))

    def slam_plane_of(self, featid):
        return int(self.lib.ovp_slam_plane_of(self.h, C.c_int64(int(featid))))

    # ---- multi-GPU shard halves ----
    def msckf_shard_columns(self, all_clone_handles):
        ch, n = _i32(all_clone_handles), C.c_int()
        self._ck(self.lib.ovp_msckf_shard_columns(self.h, _p(ch), len(ch), C.byref(n)))
        return n.value

    def msckf_shard_compress(self, batch, all_clone_handles, d_out_ptr, sigma_pix=1.0, chi2_mult=1.0):
        fb, keep = self._batch_struct(batch)
        uo = UpdaterOptions(sigma_pix, chi2_mult)
        ch = _i32(all_clone_handles)
        fs, fc = np.zeros(max(1, fb.F), dtype=np.int32), np.zeros(max(1, fb.F))
        self._ck(self.lib.ovp_msckf_shard_compress(self.h, C.byref(fb), C.byref(uo), _p(ch), len(ch), C.c_void_p(d_out_ptr), _p(fs), _p(fc)))
        return dict(feat_status=fs[:fb.F], feat_chi2=fc[:fb.F])

    # ---- collective inside the library (ovp_nccl_*): the ctx owns the communicator ----
    def nccl_unique_id(self):
        buf = C.create_string_buffer(128)
        self._ck(self.lib.ovp_nccl_unique_id(self.h, buf))
        return buf.raw

    def nccl_init(self, id128, nranks, rank):
        self._ck(self.lib.ovp_nccl_init(self.h, C.c_char_p(bytes(id128)), int(nranks), int(rank)))

    def nccl_finalize(self):
        self._ck(self.lib.ovp_nccl_finalize(self.h))

    def msckf_update_sharded(self, batch, all_clone_handles, sigma_pix=1.0, chi2_mult=1.0):
        """This rank's features of ONE large point update; collective over the ctx's communicator (see include/ovp.h)."""
        hs = _i32(all_clone_handles)
        uo = UpdaterOptions(sigma_pix, chi2_mult)
        F = int(batch["F"])
        fs, fc = np.zeros(max(1, F), dtype=np.int32), np.zeros(max(1, F))
        fb, keep = self._batch_struct(batch)
        self._ck(self.lib.ovp_msckf_update_sharded(self.h, C.byref(fb), C.byref(uo), _p(hs), len(hs), _p(fs), _p(fc)))
        return dict(feat_status=fs[:F], feat_chi2=fc[:F])

    def msckf_update_gathered(self, d_blocks_ptr, G, all_clone_handles):
        ch = _i32(all_clone_handles)
        self._ck(self.lib.ovp_msckf_update_gathered(self.h, C.c_void_p(d_blocks_ptr), int(G), _p(ch), len(ch)))

    # ---- Propagator ----
    def propagator_set_noise(self, sigma_w, sigma_wb, sigma_a, sigma_ab, gravity_mag=9.81):
        self._ck(self.lib.ovp_propagator_set_noise(self.h, C.c_double(sigma_w), C.c_double(sigma_wb), C.c_double(sigma_a), C.c_double(sigma_ab),
                                                   C.c_double(gravity_mag)))

    def feed_imu(self, t, wm, am):
        w, a = _f64(wm), _f64(am)
        self._ck(self.lib.ovp_propagator_feed_imu(self.h, C.c_double(t), _p(w), _p(a)))

    # ---- FeatureInitializer (triangulation, the step before the update path) ----
    def triangulate_features(self, meas_offset, meas_clone, uv_norm):
        mo, mc = _i32(meas_offset), _i32(meas_clone)
        uvn = np.ascontiguousarray(uv_norm, dtype=np.float32)
        F = len(mo) - 1
        pf, st = np.zeros((max(1, F), 3)), np.zeros(max(1, F), dtype=np.int32)
        self._ck(self.lib.ovp_triangulate_features(self.h, F, _p(mo), _p(mc), _p(uvn), None, _p(pf), _p(st)))
        return pf[:F], st[:F]

    # ---- PlaneFitting (plane hypothesis + refinement, the step before the plane Jacobians) ----
    def plane_fitting(self, feat_offset, p_FinG, min_inlier_num, max_cond, shuffle_kind=0):
        fo, pf = _i32(feat_offset), _f64(p_FinG).reshape(-1, 3)
        nP, Ft = len(fo) - 1, int(fo[-1])
        opt = PlaneFitOptions(int(min_inlier_num), float(max_cond), int(shuffle_kind))
        st, ab, inl = np.zeros(max(1, nP), dtype=np.int32), np.zeros((max(1, nP), 4)), np.zeros(max(1, Ft), dtype=np.int32)
        self._ck(self.lib.ovp_plane_fitting(self.h, nP, _p(fo), _p(pf), C.byref(opt), _p(st), _p(ab), _p(inl)))
        return st[:nP], ab[:nP], inl[:Ft]

    def optimize_plane(self, feat_offset, meas_offset, meas_clone, uv_norm, p_FinG, cp_inG, fix_plane, sigma_px_norm, sigma_c, max_num_iterations=0):
        fo, mo, mc = _i32(feat_offset), _i32(meas_offset), _i32(meas_clone)
        uvn = np.ascontiguousarray(uv_norm, dtype=np.float32)
        pf, cp, fx = _f64(p_FinG).reshape(-1, 3), _f64(cp_inG).reshape(-1, 3), _i32(fix_plane)
        nP, Ft = len(fo) - 1, int(fo[-1])
        opt = PlaneRefineOptions(float(sigma_px_norm), float(sigma_c), int(max_num_iterations))
        po, co = np.zeros((max(1, Ft), 3)), np.zeros((max(1, nP), 3))
        inl, st, info = np.zeros(max(1, Ft), dtype=np.int32), np.zeros(max(1, nP), dtype=np.int32), np.zeros((max(1, nP), 5))
        self._ck(self.lib.ovp_optimize_plane(self.h, nP, _p(fo), _p(mo), _p(mc), _p(uvn), _p(pf), _p(cp), _p(fx), C.byref(opt), _p(po), _p(co),
                                             _p(inl), _p(st), _p(info)))
        return st[:nP], po[:Ft], co[:nP], inl[:Ft], info[:nP]

    # ---- UpdaterZeroVelocity ----
    def zupt_feed_imu(self, t, wm, am):
        w, a = _f64(wm), _f64(am)
        self._ck(self.lib.ovp_zupt_feed_imu(self.h, C.c_double(t), _p(w), _p(a)))

    def zupt_try_update(self, t, average_disparity, num_features, gravity_mag=9.81, max_velocity=1.0, noise_multiplier=1.0, max_disparity=1.0,
                        chi2_mult=1.0):
        zo = (C.c_double * 5)(gravity_mag, max_velocity, noise_multiplier, max_disparity, chi2_mult)
        acc, chi = C.c_int(0), C.c_double(0.0)
        self._ck(self.lib.ovp_zupt_try_update(self.h, zo, C.c_double(t), C.c_double(average_disparity), int(num_features), C.byref(acc), C.byref(chi)))
        return bool(acc.value), chi.value

    def fast_state_propagate(self, t):
        sp, cv, ok = np.zeros(13), np.zeros((12, 12), order="F"), C.c_int(0)
        self._ck(self.lib.ovp_fast_state_propagate(self.h, C.c_double(t), _p(sp), _p(cv), C.byref(ok)))
        return (sp, cv) if ok.value else None

    def propagate_and_clone(self, t):
        Phi, Q, nh = np.zeros((15, 15), order="F"), np.zeros((15, 15), order="F"), C.c_int(-1)
        self._ck(self.lib.ovp_propagate_and_clone(self.h, C.c_double(t), _p(Phi), _p(Q), C.byref(nh)))
        return nh.value, Phi, Q

    # ---- instrumentation ----
    def launch_count(self):
        return int(self.lib.ovp_launch_count(self.h))

    def stream(self):
        return self.lib.ovp_stream(self.h)

    def synchronize(self):
        self._ck(self.lib.ovp_synchronize(self.h))

    def last_timing(self):
        ms = np.zeros(4)
        self.lib.ovp_last_timing(self.h, _p(ms))
        return ms

    def selftest_dgemm_tflops(self, n=2048, iters=10):
        t = C.c_double()
        self._ck(self.lib.ovp_selftest_dgemm_tflops(self.h, n, iters, C.byref(t)))
        return t.value

    # ---- prepared batch / snapshots / profiling (measurement support) ----
    def msckf_prepare(self, batch, sigma_pix=1.0, chi2_mult=1.0):
        fb, keep = self._batch_struct(batch)
        self._prep_F, self._prep_np = fb.F, fb.nplanes
        uo = UpdaterOptions(sigma_pix, chi2_mult)
        self._ck(self.lib.ovp_msckf_prepare(self.h, C.byref(fb), C.byref(uo)))

    def msckf_prepare_landmarks(self, batch, lm_featid, lm_planeid, sigma_pix=1.0, chi2_mult=1.0):
        fb, keep = self._batch_struct(batch)
        lm, keep_lm = self._landmarks_struct(lm_featid, lm_planeid)
        self._prep_F, self._prep_np = fb.F, fb.nplanes
        uo = UpdaterOptions(sigma_pix, chi2_mult)
        self._ck(self.lib.ovp_msckf_prepare_landmarks(self.h, C.byref(fb), C.byref(lm), C.byref(uo)))

    def msckf_launch(self):
        self._ck(self.lib.ovp_msckf_launch(self.h))

    def msckf_finish(self):
        F, npl = self._prep_F, max(1, self._prep_np)
        fs, fc = np.zeros(F, dtype=np.int32), np.zeros(F)
        ps, pc = np.zeros(npl, dtype=np.int32), np.zeros(npl)
        hx, hxn = np.zeros(4096, dtype=np.int32), C.c_int(0)
        self._ck(self.lib.ovp_msckf_finish(self.h, _p(fs), _p(fc), _p(ps), _p(pc), _p(hx), C.byref(hxn)))
        return dict(feat_status=fs, feat_chi2=fc, plane_status=ps[:self._prep_np], plane_chi2=pc[:self._prep_np],
                    hx_order=hx[:hxn.value].tolist())

    def snapshot(self):
        self._ck(self.lib.ovp_snapshot(self.h))

    def restore(self):
        self._ck(self.lib.ovp_restore(self.h))

    def set_rank_tolerance(self, tol):
        self._ck(self.lib.ovp_set_rank_tolerance(self.h, C.c_double(tol)))

    def set_use_graphs(self, on):
        self._ck(self.lib.ovp_set_use_graphs(self.h, int(on)))

    def set_profiling(self, on):
        self._ck(self.lib.ovp_set_profiling(self.h, int(on)))

    def profile_report(self):
        ms, cnt, work = np.zeros(5), np.zeros(5, dtype=np.int64), np.zeros(5)
        self._ck(self.lib.ovp_profile_report(self.h, _p(ms), _p(cnt), _p(work)))
        names = ["gemm_f64_kernel", "gram_kernel", "chol_fused_kernel", "feature_kernel", "other"]
        return {n: dict(ms=float(ms[i]), launches=int(cnt[i]), work=float(work[i])) for i, n in enumerate(names)}

    def transfer_bytes(self):
        a, b = C.c_int64(0), C.c_int64(0)
        self._ck(self.lib.ovp_transfer_bytes(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value
