"""UpdaterPlane::init_vio_plane (UpdaterPlane.cpp:61-481) restated as a chain of the C ABI's stage calls, plus synthetic track scenes for it.

`chain(be, tracks, ...)` runs triangulate_features -> plane_fitting -> optimize_plane -> plane_init on any object with the C ABI's method
names: on an `api.Context` it is the hand-chained counterpart of `Context.plane_init_tracks` (same kernels, host round trips between the
stages); on the test oracle it is the reference's orchestration over the oracle's own stages.  The host-side decisions are the reference's:
candidates, the track-length `std::sort` (restated below as libstdc++'s introsort, since its order of equal keys decides RANSAC's draws), the
off-by-one cap, the init thresholds, the refinement with the plane free.

`tracks_scene(...)` builds the raw tracks of a synthetic room (ov_plane_b200.synth) with pixels re-projected through the poses the state
holds, and optional hazards: planes over the cap, a plane RANSAC must reject, planes whose refinement or initialisation fails, one-measurement
tracks, a feature too far to triangulate, an in-state plane and off-plane features.  Pure numpy.
"""
import numpy as np

from . import jpl, synth, vio_sim

_S_THRESHOLD = 16  # libstdc++ _S_threshold


def libstdcxx_sort(seq, less):
    """std::sort(seq.begin(), seq.end(), less) as libstdc++ implements it (introsort, median-of-three pivot, final insertion sort); returns a
    new list.  The order of elements that compare equal is the one libstdc++ leaves, which is what RANSAC's point order depends on."""
    a = list(seq)
    n = len(a)
    if n < 2:
        return a

    def move_median_to_first(result, x, y, z):
        if less(a[x], a[y]):
            if less(a[y], a[z]):
                a[result], a[y] = a[y], a[result]
            elif less(a[x], a[z]):
                a[result], a[z] = a[z], a[result]
            else:
                a[result], a[x] = a[x], a[result]
        elif less(a[x], a[z]):
            a[result], a[x] = a[x], a[result]
        elif less(a[y], a[z]):
            a[result], a[z] = a[z], a[result]
        else:
            a[result], a[y] = a[y], a[result]

    def unguarded_partition(first, last, pivot):
        while True:
            while less(a[first], a[pivot]):
                first += 1
            last -= 1
            while less(a[pivot], a[last]):
                last -= 1
            if not first < last:
                return first
            a[first], a[last] = a[last], a[first]
            first += 1

    def adjust_heap(first, hole, length, value):
        top = hole
        child = hole
        while child < (length - 1) // 2:
            child = 2 * (child + 1)
            if less(a[first + child], a[first + child - 1]):
                child -= 1
            a[first + hole] = a[first + child]
            hole = child
        if (length & 1) == 0 and child == (length - 2) // 2:
            child = 2 * (child + 1)
            a[first + hole] = a[first + child - 1]
            hole = child - 1
        parent = (hole - 1) // 2
        while hole > top and less(a[first + parent], value):
            a[first + hole] = a[first + parent]
            hole = parent
            parent = (hole - 1) // 2
        a[first + hole] = value

    def heap_sort(first, last):  # std::__partial_sort(first, last, last): make_heap + sort_heap
        length = last - first
        if length >= 2:
            parent = (length - 2) // 2
            while True:
                adjust_heap(first, parent, length, a[first + parent])
                if parent == 0:
                    break
                parent -= 1
        while last - first > 1:
            last -= 1
            value = a[last]
            a[last] = a[first]
            adjust_heap(first, 0, last - first, value)

    def introsort_loop(first, last, depth):
        while last - first > _S_THRESHOLD:
            if depth == 0:
                heap_sort(first, last)
                return
            depth -= 1
            mid = first + (last - first) // 2
            move_median_to_first(first, first + 1, mid, last - 1)
            cut = unguarded_partition(first + 1, last, first)
            introsort_loop(cut, last, depth)
            last = cut

    def insertion_sort(first, last):
        for i in range(first + 1, last):
            val = a[i]
            if less(val, a[first]):
                a[first + 1:i + 1] = a[first:i]
                a[first] = val
            else:
                unguarded_linear_insert(i)

    def unguarded_linear_insert(last):
        val = a[last]
        nxt = last - 1
        while less(val, a[nxt]):
            a[last] = a[nxt]
            last = nxt
            nxt -= 1
        a[last] = val

    introsort_loop(0, n, 2 * (n.bit_length() - 1))
    if n > _S_THRESHOLD:
        insertion_sort(0, _S_THRESHOLD)
        for i in range(_S_THRESHOLD, n):
            unguarded_linear_insert(i)
    else:
        insertion_sort(0, n)
    return a


def chain(be, tracks, sigma_constraint, sigma_pix=1.0, max_msckf_plane=20, plane_init_min_feat=8, plane_init_max_cond=200.0, shuffle_kind=0, tri=None):
    """init_vio_plane from the stage calls of `be` (sigma_constraint: StateOptions of the state in `be`).  tri = optional (p_FinG, status) of the candidates with >= 2 measurements, in input order,
    used instead of be.triangulate_features (feeds one backend's triangulation to another).  Returns the outputs of
    Context.plane_init_tracks plus `stages`: per plane id, the feature indices after grouping, RANSAC and refinement."""
    mo, mc = np.asarray(tracks["meas_offset"]), np.asarray(tracks["meas_clone"])
    uv, uvn = np.asarray(tracks["uv"], dtype=np.float32).reshape(-1, 2), np.asarray(tracks["uv_norm"], dtype=np.float32).reshape(-1, 2)
    fid, pid = np.asarray(tracks["featid"]), np.asarray(tracks["planeid"])
    F = len(mo) - 1
    fs, pout = np.zeros(F, dtype=np.int32), np.zeros((F, 3))
    empty = dict(feat_status=fs, p_FinG=pout, plane_ids=np.zeros(0, dtype=np.int64), plane_status=np.zeros(0, dtype=np.int32),
                 new_handles=np.zeros(0, dtype=np.int32), cp=np.zeros((0, 3)), stages={})
    count = np.diff(mo)
    cand = []
    for f in range(F):
        if pid[f] == 0 or be.plane_handle(int(pid[f])) >= 0:
            continue
        if count[f] < 2:
            fs[f] = -1
            continue
        cand.append(f)
    if not cand:
        return empty

    def sub(idx):
        offs = np.concatenate([[0], np.cumsum(count[idx])]).astype(np.int32)
        sel = np.concatenate([np.arange(mo[f], mo[f + 1]) for f in idx]).astype(np.int64)
        return offs, np.ascontiguousarray(mc[sel], dtype=np.int32), np.ascontiguousarray(uvn[sel]), np.ascontiguousarray(uv[sel])

    offs, cl, un, _ = sub(cand)
    if tri is None:
        p_tri, st_tri = be.triangulate_features(offs, cl, un)
    else:
        p_tri, st_tri = np.asarray(tri[0]).reshape(-1, 3), np.asarray(tri[1])
    for k, f in enumerate(cand):
        pout[f] = p_tri[k]
    valid = [f for k, f in enumerate(cand) if st_tri[k]]
    for k, f in enumerate(cand):
        if not st_tri[k]:
            fs[f] = -2
    valid = libstdcxx_sort(valid, lambda a, b: count[a] < count[b])
    groups = {}
    for f in valid:
        fs[f] = 2
        g = groups.setdefault(int(pid[f]), [])
        if len(g) > max_msckf_plane:
            continue
        g.append(f)
    plane_ids = sorted(groups)
    P = len(plane_ids)
    if P == 0:
        return empty
    stages = {p: dict(grouped=list(groups[p])) for p in plane_ids}
    plane_status, new_handles, cp_out = np.full(P, -2, dtype=np.int32), np.full(P, -1, dtype=np.int32), np.zeros((P, 3))
    fo = np.concatenate([[0], np.cumsum([len(groups[p]) for p in plane_ids])]).astype(np.int32)
    pts = np.vstack([pout[groups[p]] for p in plane_ids])
    r_st, r_ab, r_il = be.plane_fitting(fo, pts, plane_init_min_feat, plane_init_max_cond, shuffle_kind=shuffle_kind)
    ref = []  # (plane index, inlier features, cp0)
    for i, p in enumerate(plane_ids):
        if not r_st[i]:
            continue
        keep = [f for k, f in enumerate(groups[p]) if r_il[fo[i] + k]]
        stages[p]["ransac"] = keep
        stages[p]["abcd"] = np.array(r_ab[i])
        ref.append((i, keep, -r_ab[i][:3] * r_ab[i][3]))
    if not ref:
        return dict(feat_status=fs, p_FinG=pout, plane_ids=np.array(plane_ids, dtype=np.int64), plane_status=plane_status, new_handles=new_handles,
                    cp=cp_out, stages=stages)
    ofo = np.concatenate([[0], np.cumsum([len(k) for _, k, _ in ref])]).astype(np.int32)
    oidx = [f for _, k, _ in ref for f in k]
    omo, omc, ouv, _ = sub(oidx)
    fx = float(be.var_get(be.handle_intrinsics())[0][0])
    o_st, o_p, o_cp, o_il, _ = be.optimize_plane(ofo, omo, omc, ouv, pout[oidx], np.array([c for _, _, c in ref]), np.zeros(len(ref), dtype=np.int32),
                                                 sigma_pix / fx, sigma_constraint)
    for k, f in enumerate(oidx):
        pout[f] = o_p[k]
    fin = []
    for q, (i, keep, _) in enumerate(ref):
        cp_out[i] = o_cp[q]
        if not o_st[q]:
            plane_status[i] = -3
            continue
        kept = [f for k, f in enumerate(keep) if o_il[ofo[q] + k]]
        stages[plane_ids[i]]["refined"] = kept
        plane_status[i] = -1
        fin.append((i, kept))
    if fin:
        idx = [f for _, k in fin for f in k]
        bmo, bmc, _, buv = sub(idx)
        b = dict(F=len(idx), meas_offset=bmo, meas_clone=bmc, uv=buv, p_FinG=np.ascontiguousarray(pout[idx]),
                 p_FinG_original=np.ascontiguousarray(pout[idx]), featid=np.ascontiguousarray(fid[idx], dtype=np.int64),
                 planeid=np.array([plane_ids[i] for i, k in fin for _ in k], dtype=np.int64),
                 plane_ids=np.array([plane_ids[i] for i, _ in fin], dtype=np.int64), plane_cp=np.ascontiguousarray(cp_out[[i for i, _ in fin]]))
        r = be.plane_init(b, sigma_pix=sigma_pix)
        for j, (i, kept) in enumerate(fin):
            plane_status[i] = r["plane_status"][j]
            new_handles[i] = r["new_handles"][j]
            if plane_status[i] == 1:
                fs[kept] = 1
    return dict(feat_status=fs, p_FinG=pout, plane_ids=np.array(plane_ids, dtype=np.int64), plane_status=plane_status, new_handles=new_handles,
                cp=cp_out, stages=stages)


def true_plane_cp(pid):
    """CP = n * d of the synthetic room's plane `pid` (synth._PLANES; ids start at 1)"""
    n, d = synth._PLANES[(pid - 1) % len(synth._PLANES)]
    n = np.asarray(n) / np.linalg.norm(n)
    return n * (d + 0.15 * ((pid - 1) // len(synth._PLANES)))


def tracks_scene(name="small_planes", seed=0, px_noise=0.5, keep_in_state=(), off_plane=(), inconsistent=(), noisy=(), ransac_fail_plane=0, n_single=0,
                 n_far=0, **override):
    """Scenario + raw tracks for plane initialisation.  Planes not in keep_in_state are taken out of the state.  off_plane = ((plane id, metres), ...):
    those planes' points are displaced along their normal by +-metres (RANSAC still fits them; the refinement or the initialisation's chi2
    rejects them, depending on the distance).  noisy = ((plane id, pixels), ...):
    those planes' pixel noise instead of px_noise (a plane whose noise is well above the updater's sigma_pix fails the initialisation's chi2
    while RANSAC and the refinement still accept it).  inconsistent:
    planes whose pixels are the scenario's own (taken through the TRUE poses while the state holds perturbed ones).  ransac_fail_plane != 0:
    six off-plane features are assigned to that (new) plane id.  n_single one-measurement candidate tracks, n_far candidates placed 100 m out
    (the triangulation's depth check rejects them).  Returns (S, make_tracks) where make_tracks(clone_handles) gives the track dict."""
    S = synth.make_scenario(name, seed=seed, **override)
    rng = np.random.RandomState(4242 + seed)
    drop = [pl for pl in S.planes if pl[0] not in keep_in_state]
    rows = set()
    for p, _, _ in drop:
        b = S.ids["plane%d" % p]
        rows.update(range(b, b + 3))
    keep = [i for i in range(S.N) if i not in rows]
    S.P0, S.N = np.ascontiguousarray(S.P0[np.ix_(keep, keep)]), len(keep)
    S.planes = [pl for pl in S.planes if pl[0] in keep_in_state]
    pf = S.pf_true.copy()
    planeid = S.planeid.copy()
    for p, dist in off_plane:
        n = true_plane_cp(p) / np.linalg.norm(true_plane_cp(p))
        idx = np.nonzero(planeid == p)[0]
        pf[idx] += (dist * rng.choice([-1.0, 1.0], size=len(idx)))[:, None] * n
    if ransac_fail_plane:
        planeid[np.nonzero(planeid == 0)[0][:6]] = ransac_fail_plane
    cand = [f for f in range(S.F) if planeid[f] and planeid[f] not in keep_in_state and planeid[f] not in inconsistent]
    far = cand[:n_far]
    single = cand[n_far:n_far + n_single]
    Rc, pic = jpl.quat_2_Rot(S.calib_value[:4]), S.calib_value[4:7]
    for f in far:  # 100 m out along the ray from the first camera of its track
        v = S.clones[S.meas_clone_idx[S.meas_offset[f]]][1]
        c0 = v[4:7] - jpl.quat_2_Rot(v[:4]).T @ (Rc.T @ pic)
        pf[f] = c0 + 100.0 * (pf[f] - c0) / np.linalg.norm(pf[f] - c0)
    noisy_px = dict(noisy)
    cam = S.intr_value
    uv = np.zeros((len(S.meas_clone_idx), 2))
    for f in range(S.F):
        for q in range(S.meas_offset[f], S.meas_offset[f + 1]):
            if planeid[f] in inconsistent:
                uv[q] = S.uv[q]
                continue
            v = S.clones[S.meas_clone_idx[q]][1]
            pc = Rc @ (jpl.quat_2_Rot(v[:4]) @ (pf[f] - v[4:7])) + pic
            uv[q] = jpl.radtan_distort(cam, pc[0] / pc[2], pc[1] / pc[2])
            uv[q] += noisy_px.get(int(planeid[f]), px_noise) * rng.randn(2)
    uv = uv.astype(np.float32)
    uvn = np.array([vio_sim.undistort(cam, u.astype(np.float64)) for u in uv], dtype=np.float32).reshape(-1, 2)
    keep_m = [np.arange(S.meas_offset[f], S.meas_offset[f + 1] if f not in single else S.meas_offset[f] + 1) for f in range(S.F)]
    sel = np.concatenate(keep_m)
    mo = np.concatenate([[0], np.cumsum([len(k) for k in keep_m])]).astype(np.int32)
    S.scene_pf, S.scene_planeid = pf, planeid

    def make_tracks(clone_handles):
        ch = np.asarray(clone_handles, dtype=np.int32)
        return dict(meas_offset=mo, meas_clone=np.ascontiguousarray(ch[S.meas_clone_idx[sel]], dtype=np.int32),
                    uv=np.ascontiguousarray(uv[sel]), uv_norm=np.ascontiguousarray(uvn[sel]), featid=S.featid.copy(),
                    planeid=np.ascontiguousarray(planeid, dtype=np.int64))
    return S, make_tracks
