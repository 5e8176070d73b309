"""TEST INFRASTRUCTURE: ctypes binding of tests/oracle_slam_init.cpp (UpdaterSLAM::delayed_init composed on the CPU oracle's own stages, built
by __graft_entry__.build() into oracle/liboracle_slam_init.so).  Runs on the context of an oracle_backend.OracleContext."""
import ctypes as C
import os

import numpy as np

import oracle_backend

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_lib = None


def lib():
    global _lib
    if _lib is None:
        oracle_backend.lib()  # liboracle.so first: the composition runs on the same library instance
        _lib = C.CDLL(os.path.join(_ROOT, "oracle", "liboracle_slam_init.so"))
        _lib.orc_slam_plane_of.restype = C.c_longlong
    return _lib


def slam_plane_of(orc, featid):
    """State::_features_SLAM_to_PLANE[featid] of the oracle context, -1 = no entry"""
    return int(lib().orc_slam_plane_of(orc.h, C.c_longlong(int(featid))))


def set_slam_plane_of(orc, featid, planeid):
    lib().orc_slam_set_plane_of(orc.h, C.c_longlong(int(featid)), C.c_longlong(int(planeid)))


def slam_delayed_init_tracks(orc, tracks, sigma_constraint, sigma_pix=1.0, chi2_mult=1.0, use_plane_constraint=True, use_refine_plane_feat=True,
                             tri=None):
    """the outputs of api.Context.slam_delayed_init_tracks.  tri = optional (p_FinG, status) of the tracks with >= 2 measurements, in input
    order, used instead of the oracle's triangulation."""
    mo = np.ascontiguousarray(tracks["meas_offset"], dtype=np.int32)
    mc = np.ascontiguousarray(tracks["meas_clone"], dtype=np.int32)
    uv = np.ascontiguousarray(tracks["uv"], dtype=np.float32)
    uvn = np.ascontiguousarray(tracks["uv_norm"], dtype=np.float32)
    fid = np.ascontiguousarray(tracks["featid"], dtype=np.int64)
    pid = np.ascontiguousarray(tracks["planeid"], dtype=np.int64)
    F = len(mo) - 1
    n = max(1, F)
    tp = np.ascontiguousarray(tri[0], dtype=np.float64) if tri is not None else None
    ts = np.ascontiguousarray(tri[1], dtype=np.int32) if tri is not None else None
    fs, ps, po, nh = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32), np.zeros((n, 3)), np.zeros(n, dtype=np.int32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None  # noqa: E731
    st = lib().orcsi_slam_delayed_init_tracks(orc.h, F, ptr(mo), ptr(mc), ptr(uv), ptr(uvn), ptr(fid), ptr(pid), C.c_double(sigma_pix),
                                              C.c_double(chi2_mult), C.c_double(sigma_constraint), int(bool(use_plane_constraint)),
                                              int(bool(use_refine_plane_feat)), ptr(tp), ptr(ts), ptr(fs), ptr(ps), ptr(po), ptr(nh))
    if st != 0:
        raise oracle_backend.OracleError("orcsi_slam_delayed_init_tracks failed (%d)" % st)
    return dict(feat_status=fs[:F], plane_status=ps[:F], p_FinG=po[:F], new_handles=nh[:F])
