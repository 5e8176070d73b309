"""TEST INFRASTRUCTURE: ctypes binding of tests/oracle_plane_init.cpp (init_vio_plane composed on the CPU oracle's own stages, built by
__graft_entry__.build() into oracle/liboracle_plane_init.so).  Runs on the context of an oracle_backend.OracleContext."""
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
        _lib = C.CDLL(os.path.join(_ROOT, "oracle", "liboracle_plane_init.so"))
    return _lib


def plane_init_tracks(orc, tracks, sigma_constraint, sigma_pix=1.0, max_msckf_plane=20, plane_init_min_feat=8, plane_init_max_cond=200.0,
                      shuffle_kind=0, tri=None):
    """the outputs of api.Context.plane_init_tracks, plus `stage` per feature (1 grouped, 2 RANSAC inlier, 3 refinement inlier).  tri = optional
    (p_FinG, status) of the candidates with >= 2 measurements, in input order, used instead of the oracle's triangulation."""
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
    fs, po, stg, npl = np.zeros(n, dtype=np.int32), np.zeros((n, 3)), np.zeros(n, dtype=np.int32), C.c_int(0)
    pids, ps, nh, cp = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32), np.zeros((n, 3))
    ptr = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None  # noqa: E731
    st = lib().orcpi_plane_init_tracks(orc.h, F, ptr(mo), ptr(mc), ptr(uv), ptr(uvn), ptr(fid), ptr(pid), C.c_double(sigma_pix),
                                       C.c_double(sigma_constraint), int(max_msckf_plane), int(plane_init_min_feat), C.c_double(plane_init_max_cond),
                                       int(shuffle_kind), ptr(tp), ptr(ts), ptr(fs), ptr(po), ptr(stg), C.byref(npl), ptr(pids), ptr(ps), ptr(nh), ptr(cp))
    if st != 0:
        raise oracle_backend.OracleError("orcpi_plane_init_tracks failed (%d)" % st)
    k = npl.value
    return dict(feat_status=fs[:F], p_FinG=po[:F], stage=stg[:F], plane_ids=pids[:k], plane_status=ps[:k], new_handles=nh[:k], cp=cp[:k])


def stages_of(r, plane_ids_of_feature):
    """per plane id: the feature sets after grouping, RANSAC and refinement (the `stages` of plane_init_chain.chain, as sets)"""
    out = {}
    for p in r["plane_ids"]:
        on = plane_ids_of_feature == p
        out[int(p)] = dict(grouped=set(np.nonzero(on & (r["stage"] >= 1))[0]), ransac=set(np.nonzero(on & (r["stage"] >= 2))[0]),
                           refined=set(np.nonzero(on & (r["stage"] >= 3))[0]))
    return out
