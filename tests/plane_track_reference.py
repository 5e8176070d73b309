"""Host restatement of TrackPlane::perform_plane_detection_monocular (track_plane/TrackPlane.cpp:580-1121), the reference the device tracker
(ovp_plane_track_*) is tested against.  Double where the reference computes in double; float where it does (pixels, the mesh's inputs,
the spatial filter's k-NN distances); long double for the bearing-system solves.  The Delaunay mesh comes from the reference's own CDT,
built into oracle/_ref/libref_cdt.so by build()."""
import ctypes as C
import math
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_CDT = os.path.join(ROOT, "oracle", "_ref", "libref_cdt.so")
_cdt = None


def ref_cdt():
    global _cdt
    if _cdt is None:
        if not os.path.exists(REF_CDT):
            raise FileNotFoundError("%s is missing: build() compiles it from the reference checkout's thirdparty/cdt" % REF_CDT)
        _cdt = C.CDLL(REF_CDT)
    return _cdt


def cdt_triangulate(xy):
    """CDT's triangles (T, 3) of float pixels xy (n, 2), inserted as given, super-triangle erased"""
    xy = np.ascontiguousarray(xy, dtype=np.float32).reshape(-1, 2)
    n = len(xy)
    cap = 2 * n + 8
    tri = np.zeros((cap, 3), dtype=np.int32)
    nt = ref_cdt().ref_cdt_triangulate(n, xy.ctypes.data_as(C.c_void_p), cap, tri.ctypes.data_as(C.c_void_p))
    if nt < 0:
        raise RuntimeError("CDT threw")
    return tri[:nt].copy()


def quat_2_rot(q):
    q = np.asarray(q, dtype=np.float64)
    v, w = q[:3], q[3]
    sk = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])
    return (2 * w * w - 1) * np.eye(3) - 2 * w * sk + 2 * np.outer(v, v)


def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def norm3(v):
    return math.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])


def px_dist(a, b):
    """cv::norm of a Point2f difference: float subtraction, then double"""
    d = np.float32(a[0]) - np.float32(b[0]), np.float32(a[1]) - np.float32(b[1])
    return math.sqrt(float(d[0]) * float(d[0]) + float(d[1]) * float(d[1]))


def solve_ld(A, b):
    """A x = b in long double, Gaussian elimination with partial pivoting"""
    M = np.zeros((3, 4), dtype=np.longdouble)
    M[:, :3], M[:, 3] = A, b
    for k in range(3):
        p = k + int(np.argmax(np.abs(M[k:, k])))
        M[[k, p]] = M[[p, k]]
        for i in range(k + 1, 3):
            M[i] -= M[i, k] / M[k, k] * M[k]
    x = np.zeros(3, dtype=np.longdouble)
    for k in range(2, -1, -1):
        x[k] = (M[k, 3] - M[k, k + 1:3] @ x[k + 1:]) / M[k, k]
    return x


def avg_norm(norms, o, trace=None):
    """TrackPlane::avg_norm (:1123-1171), with the NaN behaviour of its comparisons; trace: a dict the compared values are appended to"""
    if len(norms) == 0:
        return np.zeros(3)
    count, s = 0, np.zeros(3)
    for nk in norms:
        if norm3(nk) <= 0:
            continue
        s = s + nk
        count += 1
    with np.errstate(invalid="ignore", divide="ignore"):
        s = s / norm3(s)
    if count < 2:
        return np.zeros(3)
    max_deg, var_deg = 0.0, 0.0
    for nk in norms:
        if norm3(nk) <= 0:
            continue
        dt = (nk[0] * s[0] + nk[1] * s[1]) + nk[2] * s[2]
        d = (180.0 / math.pi) * (math.acos(dt) if -1.0 <= dt <= 1.0 else float("nan"))
        var_deg += d * d
        max_deg = d if max_deg < d else max_deg  # std::max(max_deg, d)
    var_deg /= (count - 1)
    if trace is not None:
        trace.setdefault("max_norm_avg_var", []).append(math.sqrt(var_deg))
        trace.setdefault("max_norm_avg_max", []).append(max_deg)
    if math.sqrt(var_deg) > o["max_norm_avg_var"] or max_deg > o["max_norm_avg_max"]:  # NaN compares false
        return np.zeros(3)
    return s


def knn_mean(pts, i, k):
    """mean of the k smallest squared float distances from pts[i] to the other points, ikd-tree's calc_dist unfused, summed ascending in
    double"""
    p = pts[i]
    d = []
    for j in range(len(pts)):
        if j == i:
            continue
        dx, dy, dz = p[0] - pts[j][0], p[1] - pts[j][1], p[2] - pts[j][2]  # float32 arithmetic
        d.append(np.float32(np.float32(np.float32(dx * dx) + np.float32(dy * dy)) + np.float32(dz * dz)))
    d.sort()
    acc = 0.0
    for v in d[:k]:
        acc += float(v)
    return acc / k


class PlaneTrackRef(object):
    """The tracker's hist_* members and one method per reference step."""

    def __init__(self, options):
        self.o = dict(options)
        self.A, self.b, self.cnt, self.inG, self.norms = {}, {}, {}, {}, {}
        self.f2p, self.p2o = {}, {}
        self.currplaneid = 0
        self.tri, self.tri_norms, self.events = np.zeros((0, 3), dtype=np.int32), np.zeros((0, 3)), {}
        self.trace = {}  # per rule, every value the last frame compared with its threshold

    def _tr(self, rule, v):
        self.trace.setdefault(rule, []).append(float(v))

    def remove_feats(self, ids):
        keep = set(ids)
        for d in (self.A, self.b, self.cnt, self.inG, self.norms):
            for k in [k for k in d if k not in keep]:
                del d[k]

    def update_plane_ids(self, min_planeid, oldplaneid):
        if min_planeid == oldplaneid:
            return
        for f in list(self.f2p):
            if self.f2p[f] == oldplaneid:
                self.f2p[f] = min_planeid
        self.p2o.setdefault(min_planeid, set()).add(oldplaneid)
        if oldplaneid in self.p2o:
            self.p2o[min_planeid] |= self.p2o.pop(oldplaneid)

    def frame(self, pose7, calib7, featid, uv, uv_norm, tri=None):
        """one perform_plane_detection_monocular; tri: the mesh to use (default: CDT's)"""
        o = self.o
        self.trace = {}
        ev = self.events = {"new_plane": 0, "merge": 0, "merge_nonneighbour": 0, "z_removed": 0, "pruned": 0, "removed_feats": 0}
        featid = [int(f) for f in featid]
        uv = np.asarray(uv, dtype=np.float32).reshape(-1, 2)
        uvn = np.asarray(uv_norm, dtype=np.float32).reshape(-1, 2)
        if len(featid) == 0:
            return
        before = set(self.A)
        self.remove_feats(featid)
        ev["removed_feats"] = len(before - set(self.A))
        R_GtoI, p_IinG = quat_2_rot(pose7[:4]), np.asarray(pose7[4:7], dtype=np.float64)
        R_ItoC, p_IinC = quat_2_rot(calib7[:4]), np.asarray(calib7[4:7], dtype=np.float64)
        R = R_ItoC @ R_GtoI
        pc = p_IinG - R.T @ p_IinC
        for i, f in enumerate(featid):
            bi = R.T @ np.array([float(uvn[i, 0]), float(uvn[i, 1]), 1.0])
            bi = bi / np.linalg.norm(bi)
            B = skew(bi)
            Ai = B.T @ B
            self.A[f] = Ai + self.A.get(f, np.zeros((3, 3)))
            self.b[f] = Ai @ pc + self.b.get(f, np.zeros(3))
            self.cnt[f] = 1 + self.cnt.get(f, 0)
            if self.cnt[f] >= o["feat_init_min_obs"]:
                A, b = self.A[f], self.b[f]
                p = solve_ld(A.astype(np.longdouble), b.astype(np.longdouble))
                pz = (R.astype(np.longdouble) @ (p - pc.astype(np.longdouble)))
                sv = np.linalg.svd(A, compute_uv=False)
                with np.errstate(divide="ignore", invalid="ignore"):
                    cond = sv[0] / sv[-1]
                self._tr("max_cond_number", cond)
                self._tr("min_dist", pz[2])
                self._tr("max_dist", pz[2])
                if abs(cond) <= o["max_cond_number"] and o["min_dist"] <= float(pz[2]) <= o["max_dist"] and not np.isnan(float(np.linalg.norm(pz.astype(np.float64)))):
                    self.inG[f] = p.astype(np.float64)
        keep = [i for i, f in enumerate(featid) if f in self.inG]
        ids = [featid[i] for i in keep]
        pts = uv[keep]
        if tri is None:
            tri = cdt_triangulate(pts) if len(ids) else np.zeros((0, 3), dtype=np.int32)
        close, tri_norms = {}, []
        for t in tri:
            i1, i2, i3 = (ids[t[0]], ids[t[1]], ids[t[2]])
            for a, b in ((i1, i2), (i1, i3), (i2, i1), (i2, i3), (i3, i1), (i3, i2)):
                close.setdefault(a, set()).add(b)
            side = float(o["max_tri_side_px"])
            self._tr("max_tri_side_px", max(px_dist(pts[t[0]], pts[t[1]]), px_dist(pts[t[1]], pts[t[2]]), px_dist(pts[t[2]], pts[t[0]])))
            if px_dist(pts[t[0]], pts[t[1]]) > side or px_dist(pts[t[1]], pts[t[2]]) > side or px_dist(pts[t[2]], pts[t[0]]) > side:
                tri_norms.append(np.zeros(3))
                continue
            d1 = self.inG[i2] - self.inG[i1]
            d1 = d1 / norm3(d1)
            d2 = self.inG[i3] - self.inG[i1]
            d2 = d2 / norm3(d2)
            nrm = np.array([d1[1] * d2[2] - d1[2] * d2[1], d1[2] * d2[0] - d1[0] * d2[2], d1[0] * d2[1] - d1[1] * d2[0]])
            nrm = nrm / norm3(nrm)
            if (R @ nrm) @ (R @ (self.inG[i1] - pc)) < 0:
                nrm = -nrm
            tri_norms.append(nrm)
            for f in (i1, i2, i3):
                w = self.norms.setdefault(f, [])
                w.append(nrm)
                if len(w) > o["max_norm_count"]:
                    del w[:len(w) - o["max_norm_count"]]
        avg = {f: avg_norm(w, o, self.trace) for f, w in self.norms.items()}
        pix = {f: pts[k] for k, f in enumerate(ids)}
        if len(tri):
            self.merge_loop(close, pix, avg)
        self.filter_and_prune(ids)
        self.tri, self.tri_norms = np.asarray(tri, dtype=np.int32).reshape(-1, 3), np.asarray(tri_norms).reshape(-1, 3)
        self.survivors = ids

    def merge_loop(self, close, pix, avg):
        """the matching and merging loop (:816-979) over the features with a normal window, ascending id: close = the mesh neighbours of
        each feature, pix = its pixel, avg = its average normal"""
        o, ev = self.o, self.events
        done = set()
        for f in sorted(self.norms):
            norms, nv = self.norms[f], avg[f]
            if len(norms) < o["min_norms"] or not (norm3(nv) > 0):
                continue
            d = float(self.inG[f] @ nv)
            if not o["check_old_feats"] and f in self.f2p:
                continue
            if f not in close:
                continue
            matches = []
            for g in sorted(close[f]):
                if g not in self.norms or len(self.norms[g]) < o["min_norms"] or not (norm3(avg[g]) > 0) or g in done:
                    continue
                self._tr("max_pairwise_px", px_dist(pix[f], pix[g]))
                if px_dist(pix[f], pix[g]) > o["max_pairwise_px"]:
                    continue
                plane_dist = float(self.inG[g] @ nv) - d
                dt = float(nv @ avg[g])
                angle = (180.0 / math.pi) * (math.acos(dt) if -1.0 <= dt <= 1.0 else float("nan"))
                if abs(dt - 1.0) < 1e-12:  # acos is NaN or not by the last bits of the two normals: the match is decided by rounding
                    self._tr("unit_dot", dt)
                if not math.isnan(angle):
                    self._tr("max_norm_deg", angle)
                self._tr("max_dist_between_z", abs(plane_dist))
                if not math.isnan(angle) and angle < o["max_norm_deg"] and abs(plane_dist) < o["max_dist_between_z"]:
                    matches.append(g)
            if not matches:
                continue
            mp = self.f2p.get(f, -1)
            for g in matches:
                if g in self.f2p:
                    mp = self.f2p[g] if mp == -1 else min(mp, self.f2p[g])
            if mp != -1:
                neigh = set(matches) | {f}
                for g in matches + [f]:
                    if g in self.f2p and self.f2p[g] != mp:
                        old = self.f2p[g]
                        ev["merge"] += 1
                        ev["merge_nonneighbour"] += any(v == old and k not in neigh for k, v in self.f2p.items())
                        self.update_plane_ids(mp, old)
                for g in matches:
                    self.f2p[g] = mp
                self.f2p[f] = mp
                done.add(f)
            else:
                self.currplaneid += 1
                ev["new_plane"] += 1
                for g in matches:
                    self.f2p[g] = self.currplaneid
                self.f2p[f] = self.currplaneid

    def filter_and_prune(self, ids):
        """the spatial filter (:989-1058) and the pruning to the frame's planes with more than 3 features (:1064-1095)"""
        o, ev = self.o, self.events
        assert o["filter_num_feat"] > 1
        active = set(ids)
        plane_to_feat = {}
        for f in sorted(self.f2p):
            if f in active:
                plane_to_feat.setdefault(self.f2p[f], []).append(f)
        for pid in sorted(plane_to_feat):
            fs = plane_to_feat[pid]
            self._tr("filter_num_feat", len(fs))
            if len(fs) <= o["filter_num_feat"]:
                continue
            P = [self.inG[f].astype(np.float32) for f in fs]
            dist = np.array([knn_mean(P, i, o["filter_num_feat"]) for i in range(len(fs))])
            mean = 0.0
            for v in dist:
                mean += v
            mean /= len(dist)
            ss = 0.0
            for v in dist:
                ss += (v - mean) * (v - mean)
            std = math.sqrt(ss / (len(dist) - 1))
            for f, v in zip(fs, dist):
                with np.errstate(divide="ignore", invalid="ignore"):
                    sigma = np.float64(abs(v - mean)) / np.float64(std)
                self._tr("filter_z_thresh", sigma)
                if sigma > o["filter_z_thresh"]:
                    del self.f2p[f]
                    ev["z_removed"] += 1
        tmp = {f: self.f2p[f] for f in ids if f in self.f2p}
        ct = {}
        for p in tmp.values():
            ct[p] = ct.get(p, 0) + 1
        for c in ct.values():
            self._tr("prune", c)
        kept = {f: p for f, p in tmp.items() if ct[p] > 3}
        ev["pruned"] = len(tmp) - len(kept)
        self.f2p = kept
        self.p2o = {p: set(self.p2o[p]) for p in set(kept.values()) if p in self.p2o}
