"""The covariance operations between updates (ovp_ekf_propagation, ovp_clone / ovp_augment_clone, ovp_marginalize*,
ovp_get_marginal_covariance, ovp_set_initial_covariance) against the references of tests/state_reference.py, through the public C ABI,
on a state that holds every variable kind, has holes in its handle table and recycled slots (update_reference.build_state), and on three
covariances: correlated, correlated with kappa(C) ~ 1e10, and asymmetric (the reference's propagation leaves P asymmetric every frame,
and the copies that follow are defined on that P).  Copies are checked bit for bit, arithmetic element by element within a-priori
bounds; each test prints its worst error / bound."""
import numpy as np
import pytest

import state_reference as sr
import update_reference as ur
from ov_plane_b200 import api

pytestmark = pytest.mark.gpu

OVP_ERR_BAD_ARGS, OVP_ERR_NEGATIVE_DIAGONAL, OVP_ERR_NON_CONTIGUOUS, OVP_ERR_CAPACITY = 1, 2, 3, 7
COVS = ("corr", "cond", "asym")
SIGMA_IMU_POSE = ur.SIGMA[ur.IMU][:6]


def extra_for(residue, delta=0, minimum=0):
    """The number of extra landmarks of build_state that makes N + delta = 123 + 3 e + delta congruent to `residue` mod 64 and at least
    `minimum` (3 is invertible mod 64, so one of 64 consecutive e does)."""
    e = 0
    while (123 + 3 * e + delta) % 64 != residue % 64 or 123 + 3 * e + delta < minimum:
        e += 1
    return e


class State(object):
    """build_state on a fresh context, with the bookkeeping the tests extend as they clone and marginalise.  make(options): the backend
    (default: a GPU context)."""

    def __init__(self, extra, seed=0, max_state=640, options=ur.STATE_OPTIONS, make=None):
        self.ctx = make(options) if make else api.Context(options, device=0, max_state=max_state, max_meas_rows=4096)
        self.kinds, self.sig, self.hs = ur.build_state(self.ctx, extra, seed)

    def clone(self, src):
        nh = self.ctx.clone(src)
        imu = src == self.ctx.handle_imu()
        self.kinds[nh] = ur.POSE if imu else self.kinds[src]
        self.sig[nh] = SIGMA_IMU_POSE if imu else self.sig[src]
        return nh

    def marginalize(self, h):
        self.ctx.marginalize(h)
        del self.kinds[h], self.sig[h]

    def upload(self, cov, seed):
        ids, _, _, d = ur.state_arrays(self.ctx, self.kinds, self.sig)
        P = sr.covariance(cov, d, seed)
        self.ctx.cov_upload(P)
        self.d = d
        return P

    def ids(self, handles):
        return [i for h in handles for i in range(self.ctx.var_id(h), self.ctx.var_id(h) + self.ctx.var_size(h))]

    def snapshot(self):
        c = self.ctx
        return c.cov().copy(), c.variable_order(), {h: c.var_get(h) for h in self.kinds}, {h: c.var_id(h) for h in self.kinds}

    def assert_unchanged(self, snap):
        P, order, vals, ids = snap
        sr.bits(self.ctx.cov(), P, "P")
        assert self.ctx.variable_order() == order
        for h, (v, f) in vals.items():
            g, gf = self.ctx.var_get(h)
            assert np.array_equal(g, v) and np.array_equal(gf, f), "handle %d: value or FEJ changed" % h
            assert self.ctx.var_id(h) == ids[h]


# ---- ovp_ekf_propagation ------------------------------------------------------------------------------------------------------------
TAILS = {"rows17": ("intr", "clone", "plane"), "rows64": ("intr",) * 8, "rows65": ("intr",) * 8 + ("dt",)}
TAIL_SIZE = {k: sum({"intr": 8, "clone": 6, "plane": 3, "dt": 1}[t] for t in v) for k, v in TAILS.items()}


def prop_shape(st, name):
    """(new, old) handle lists of a propagation shape; the rows* shapes first append their NEW variables (clones) to the state."""
    c, hs = st.ctx, st.hs
    imu, dt, cal, intr = c.handle_imu(), c.handle_dt(), c.handle_calib(), c.handle_intrinsics()
    cl, pl, lm = hs["clones"], hs["planes"], hs["lms"]
    if name == "imu":
        return [imu], [imu]
    if name == "anchor":  # perform_anchor_change: old anchor, extrinsics, new anchor, the landmark (3 x 21)
        return [lm[1]], [cl[0], cal, cl[5], lm[1]]
    if name == "anchor_nocal":
        return [lm[1]], [cl[0], cl[5], lm[1]]
    if name == "calib_incl":  # old permuted, non-contiguous, holding the new variables
        return [cal, intr], [intr, cl[3], cal, lm[0], imu]
    if name == "calib_excl":
        return [cal, intr], [cl[6], imu, pl[1]]
    if name == "rows1":
        return [dt], [pl[2], dt, cl[1]]
    if name == "rows16":
        return [imu, dt], [cal, imu, lm[0], dt]
    src = {"intr": intr, "clone": cl[0], "plane": pl[0], "dt": dt}
    tail = [st.clone(src[t]) for t in TAILS[name]]
    old = tail[::-1] + [imu] if name == "rows64" else ([tail[2], imu, tail[0], cl[4], tail[1]] if name == "rows17" else tail[1::2] + [cal] + tail[::2])
    return tail, old


def phi_q(st, new, old, seed):
    """Phi (rows x cols) scaled by the standard deviations of its rows and columns (|Phi P_old Phi^T| ~ P_new) and Q = 0.1 diag(d) W diag(d)
    with W a random positive definite matrix; Qg is Q with random garbage of 1e3 |Q| in its strictly lower triangle."""
    rng = np.random.default_rng(seed)
    ni, oi = st.ids(new), st.ids(old)
    dn, do = st.d[ni], st.d[oi]
    Phi = rng.standard_normal((len(ni), len(oi))) * dn[:, None] / (do[None, :] * np.sqrt(len(oi)))
    A = rng.standard_normal((len(ni), len(ni)))
    Q = 0.1 * dn[:, None] * (A @ A.T / len(ni) + 0.1 * np.eye(len(ni))) * dn[None, :]
    Qg = np.triu(Q) + np.tril(1e3 * np.abs(Q).max() * rng.standard_normal(Q.shape), -1)
    return Phi, Q, Qg, ni, oi


PROP_SHAPES = ("imu", "anchor", "anchor_nocal", "calib_incl", "calib_excl", "rows1", "rows16", "rows17", "rows64", "rows65")
PROP_CASES = [(s, m, cov) for s in PROP_SHAPES for m in (0, 1, 63) for cov in COVS]
PROP_CASES += [(s, "large", cov) for s in ("imu", "rows65") for cov in COVS]


@pytest.mark.parametrize("shape,nmod,cov", PROP_CASES)
def test_ekf_propagation_against_long_double(shape, nmod, cov):
    """nmod: N % 64, or "large": N a multiple of 64 of at least 1000 (1152 and 1088 rows), the capacity of the context."""
    ur.require_long_double()
    delta = TAIL_SIZE.get(shape, 0)
    if nmod == "large":
        extra = extra_for(0, delta, 1000)
        max_state = 123 + 3 * extra + delta
    else:
        extra, max_state = extra_for(nmod, delta), 640
    st = State(extra, seed=7, max_state=max_state)
    new, old = prop_shape(st, shape)
    N = st.ctx.cov_rows()
    assert N % 64 == (0 if nmod == "large" else nmod), N
    P = st.upload(cov, seed=N)
    Phi, Q, Qg, ni, oi = phi_q(st, new, old, seed=N + len(old))
    assert ni == list(range(ni[0], ni[0] + len(ni)))
    st.ctx.ekf_propagation(new, old, Phi, Qg)  # Q's lower triangle is garbage: the reference reads the upper one only
    got = st.ctx.cov()
    ref, B = sr.propagate(P, ni, oi, Phi, Q)
    q = sr.within(got, ref, B, "P+")  # zero bound outside the new rows and columns: those entries are bit-identical
    other = np.setdiff1d(np.arange(N), ni)
    sr.bits(got[np.ix_(other, ni)], got[np.ix_(ni, other)].T, "P[other, new] against P[new, other]^T")
    st.ctx.cov_upload(P)
    st.ctx.ekf_propagation(new, old, Phi, sr.upper_sym(Q))
    sr.bits(st.ctx.cov(), got, "P+ with Q's lower triangle garbage against P+ with Q symmetric")
    print("%s N %d %s: Phi %d x %d, worst error / bound %.3e" % (shape, N, cov, len(ni), len(oi), q))
    st.ctx.close()


def test_ekf_propagation_negative_diagonal_and_refusals():
    """A Q with a negative diagonal entry (Phi = 0) gives OVP_ERR_NEGATIVE_DIAGONAL (the reference exits there) and the next call succeeds;
    a non-contiguous NEW set and a Phi of the wrong shape are refused with the state bit-identical."""
    ur.require_long_double()
    st = State(extra_for(1))
    c, hs = st.ctx, st.hs
    P = st.upload("asym", seed=5)
    imu, cal, intr = c.handle_imu(), c.handle_calib(), c.handle_intrinsics()
    Phi, Q, _, ni, oi = phi_q(st, [imu], [imu, cal], seed=5)
    Qn = Q.copy()
    Qn[4, 4] = -1.0
    with pytest.raises(api.OvpError) as e:
        c.ekf_propagation([imu], [imu, cal], np.zeros_like(Phi), Qn)
    assert e.value.status == OVP_ERR_NEGATIVE_DIAGONAL
    c.cov_upload(P)
    c.ekf_propagation([imu], [imu, cal], Phi, Q)
    ref, B = sr.propagate(P, ni, oi, Phi, Q)
    q = sr.within(c.cov(), ref, B, "P+ after the negative-diagonal call")
    snap = st.snapshot()
    with pytest.raises(api.OvpError) as e:  # calib and intrinsics are contiguous, calib and a clone are not
        c.ekf_propagation([cal, hs["clones"][0]], [imu], np.zeros((12, 15)), np.eye(12))
    assert e.value.status == OVP_ERR_NON_CONTIGUOUS
    st.assert_unchanged(snap)
    for shp in ((14, 13), (13, 14), (15, 15)):  # [calib, intrinsics] is 14 x 14
        with pytest.raises(api.OvpError) as e:
            c.ekf_propagation([cal, intr], [cal, intr], np.zeros(shp), np.eye(shp[0]))
        assert e.value.status == OVP_ERR_BAD_ARGS
        st.assert_unchanged(snap)
    print("propagation after the negative diagonal: worst error / bound %.3e" % q)
    c.close()


# ---- ovp_clone / ovp_augment_clone --------------------------------------------------------------------------------------------------
CLONE_SIZE = {"imu": 6, "clone": 6, "plane": 3, "intr": 8, "dt": 1}


def clone_source(st, target):
    c = st.ctx
    return {"imu": c.handle_imu(), "clone": st.hs["clones"][3], "plane": st.hs["planes"][1], "intr": c.handle_intrinsics(),
            "dt": c.handle_dt()}[target]


@pytest.mark.parametrize("cov", COVS)
@pytest.mark.parametrize("where", ["straddle", "nmax"])
@pytest.mark.parametrize("target", list(CLONE_SIZE))
def test_clone_is_the_reference_copy(target, where, cov):
    """N = 255 before the clone (it straddles or ends at 256), or a clone that ends exactly at Nmax followed by one that would pass it."""
    s = CLONE_SIZE[target]
    if where == "straddle":
        extra, max_state = extra_for(63), 640
    else:  # build_state needs 240 rows on the way: Nmax >= 256
        extra = extra_for(0, s, 256)
        max_state = 123 + 3 * extra + s
    outs = []
    for run in range(2 if cov == "asym" else 1):
        st = State(extra, seed=7, max_state=max_state)
        c = st.ctx
        src = clone_source(st, target)
        N, old = c.cov_rows(), c.var_id(src)
        P = st.upload(cov, seed=N)
        order = c.variable_order()
        v0, f0 = c.var_get(src)
        nh = c.clone(src)
        got = c.cov()
        sr.bits(got, sr.clone(P, old, s), "P after the clone")
        assert c.var_id(nh) == N and c.var_size(nh) == s and c.cov_rows() == N + s
        assert c.variable_order() == order + [nh]
        v, f = c.var_get(nh)
        n = 7 if target == "imu" else len(v0)  # the IMU's pose sub-variable: q and p
        assert len(v) == n and np.array_equal(v, v0[:n]) and np.array_equal(f, f0[:n]), "the clone's value / FEJ is not the source's"
        if where == "nmax":
            assert c.cov_rows() == (max_state + 63) // 64 * 64
            st.kinds[nh], st.sig[nh] = ur.VEC, [1.0] * s
            snap = st.snapshot()
            with pytest.raises(api.OvpError) as e:
                c.clone(src)
            assert e.value.status == OVP_ERR_CAPACITY
            st.assert_unchanged(snap)
        outs.append(got)
        c.close()
    if len(outs) == 2:
        sr.bits(outs[1], outs[0], "P after the clone, second run")
    print("clone of %s (%d) at N %d -> %d, %s: bit-exact" % (target, s, N, N + s, cov))


def dt_d(c, last_w):
    return np.concatenate([last_w, c.var_get(c.handle_imu())[0][7:10]])


@pytest.mark.parametrize("cov", COVS)
@pytest.mark.parametrize("nmod", [63, 0])
def test_augment_clone_with_time_offset(nmod, cov):
    """StateHelper::augment_clone with the time offset calibrated: the clone of the IMU pose, then the two passes of d = [w; v]."""
    ur.require_long_double()
    st = State(extra_for(nmod), seed=3)
    c = st.ctx
    N = c.cov_rows()
    P = st.upload(cov, seed=N)
    w = np.array([0.31, -0.12, 0.07])
    d = dt_d(c, w)
    v0, f0 = c.var_get(c.handle_imu())
    nh = c.augment_clone(200.0, w)
    assert c.var_id(nh) == N and c.clone_handle(200.0) == nh and c.get_timestamp() == 200.0
    v, f = c.var_get(nh)
    assert np.array_equal(v, v0[:7]) and np.array_equal(f, f0[:7])
    ref, B = sr.augment_dt(sr.clone(P, 0, 6), N, c.var_id(c.handle_dt()), d)
    q = sr.within(c.cov(), ref, B, "P after augment_clone")  # zero bound outside the new rows and columns: bit-exact copies
    print("augment_clone N %d -> %d, %s: worst error / bound %.3e" % (N, N + 6, cov, q))
    c.close()


def small_state(timeoffset, make=None):
    """A state of its own for the time-offset-off case (build_state puts dt in the state): IMU, extrinsics, intrinsics, 5 clones, 2 planes
    and 3 landmarks, one clone marginalised in the middle.  make(options): the backend (default: a GPU context)."""
    opt = dict(ur.STATE_OPTIONS, do_calib_camera_timeoffset=timeoffset)
    c = make(opt) if make else api.Context(opt, device=0, max_state=128, max_meas_rows=1024)
    rng = np.random.default_rng(2)
    clones = []
    imu = np.concatenate([[0.1, -0.2, 0.3, 0.927], rng.standard_normal(12)])
    imu[:4] /= np.linalg.norm(imu[:4])
    c.var_set(c.handle_imu(), imu, imu)
    kinds = {c.handle_imu(): ur.IMU, c.handle_calib(): ur.POSE, c.handle_intrinsics(): ur.VEC}
    sig = {c.handle_imu(): ur.SIGMA[ur.IMU], c.handle_calib(): ur.SIGMA[ur.POSE], c.handle_intrinsics(): ur.SIGMA["intr"]}
    for k in range(5):
        q = rng.standard_normal(4)
        h = c.add_clone_raw(10.0 + k, np.concatenate([q / np.linalg.norm(q), rng.standard_normal(3)]), np.zeros(7))
        kinds[h], sig[h] = ur.POSE, ur.SIGMA[ur.POSE]
        clones.append(h)
    for p in (1, 2):
        h = c.add_plane_raw(p, rng.standard_normal(3) + 3.0, np.zeros(3))
        kinds[h], sig[h] = ur.VEC, ur.SIGMA["plane"]
    for i in range(3):
        h = c.add_slam_raw(5000 + i, rng.standard_normal(3), np.zeros(3))
        kinds[h], sig[h] = ur.LANDMARK, ur.SIGMA["lm"]
    h = clones[2]
    c.marginalize(h)
    del kinds[h], sig[h]
    return c, kinds, sig


@pytest.mark.parametrize("cov", COVS)
def test_augment_clone_without_time_offset_is_a_pure_clone(cov):
    c, kinds, sig = small_state(0)
    _, _, _, d = ur.state_arrays(c, kinds, sig)
    P = sr.covariance(cov, d, 9)
    c.cov_upload(P)
    N = c.cov_rows()
    nh = c.augment_clone(20.0, [0.5, 0.5, 0.5])
    sr.bits(c.cov(), sr.clone(P, 0, 6), "P after augment_clone without the time offset")
    assert c.var_id(nh) == N
    print("augment_clone without the time offset, N %d, %s: bit-exact" % (N, cov))
    c.close()


def feed_constant_imu(c, t0, t1, wm):
    """IMU readings every 2.5 ms over [t0, t1] with one angular rate (so the last one before the clone time is wm whatever the
    interpolation picks) and a slowly varying specific force."""
    c.propagator_set_noise(1.6968e-04, 1.9393e-05, 2.0e-3, 3.0e-3, 9.81)
    for k, t in enumerate(np.arange(t0, t1, 0.0025)):
        c.feed_imu(t, wm, np.array([0.2, 9.7, 0.4]) + 0.05 * np.sin(0.3 * k))


def compose_prop_dt(B1, N, dt, d):
    """The bound of propagation errors B1 carried through the clone of the IMU pose and the two dt passes (first order)."""
    Bc = sr.clone(B1, 0, 6)
    ad = np.abs(d)
    Bc[:, N:N + 6] += np.outer(Bc[:, dt], ad)
    Bc[N:N + 6, :] += np.outer(ad, Bc[dt, :])
    return Bc


@pytest.mark.parametrize("cov", ["corr", "asym"])
def test_propagate_and_clone_composite(cov):
    """ovp_propagate_and_clone on a correlated P: propagate with the Phi and Q the call returns, clone, augment_dt."""
    ur.require_long_double()
    st = State(extra_for(1), seed=4)
    c = st.ctx
    N = c.cov_rows()
    P = st.upload(cov, seed=N)
    c.set_timestamp(101.0)
    wm = np.array([0.12, -0.05, 0.2])
    feed_constant_imu(c, 100.99, 101.2, wm)
    nh, Phi, Q = c.propagate_and_clone(101.1)
    assert c.var_id(nh) == N
    d = np.concatenate([wm - c.var_get(c.handle_imu())[0][10:13], c.var_get(c.handle_imu())[0][7:10]])
    P1, B1 = sr.propagate(P, list(range(15)), list(range(15)), Phi, Q)
    dt = c.var_id(c.handle_dt())
    ref, B3 = sr.augment_dt(sr.clone(P1, 0, 6), N, dt, d)
    B = B3 + compose_prop_dt(B1, N, dt, d)
    q = sr.within(c.cov(), ref, B, "P after propagate_and_clone")
    print("propagate_and_clone N %d, %s: worst error / bound %.3e" % (N, cov, q))
    c.close()


# ---- marginalisation -------------------------------------------------------------------------------------------------------------
MARG = [(15, "first"), (1, "first"), (1, "middle"), (1, "last"), (3, "first"), (3, "middle"), (3, "last"), (6, "first"), (6, "middle"),
        (6, "last"), (8, "first"), (8, "middle"), (8, "last")]


def marg_target(st, size, where):
    """Prepare the state so that a variable of `size` sits at `where` and return it: first = every variable before it marginalised,
    last = a clone of it appended."""
    c, hs = st.ctx, st.hs
    src = {15: c.handle_imu(), 1: c.handle_dt(), 3: hs["planes"][0] if where == "first" else hs["planes"][1],
           6: c.handle_calib() if where == "first" else hs["clones"][4], 8: c.handle_intrinsics()}[size]
    if where == "last":
        return st.clone(src)
    if where == "first":
        for h in sorted(st.kinds, key=c.var_id):
            if c.var_id(h) < c.var_id(src):
                st.marginalize(h)
    return src


def marg_delta(size, where):
    """N after marg_target minus build_state's N (the ids of build_state do not depend on its extra landmarks)."""
    if where == "last":
        return size
    if where == "middle":
        return 0
    st = State(0)
    t = {15: st.ctx.handle_imu(), 1: st.ctx.handle_dt(), 3: st.hs["planes"][0], 6: st.ctx.handle_calib(), 8: st.ctx.handle_intrinsics()}[size]
    i = st.ctx.var_id(t)
    st.ctx.close()
    return -i


def check_marginalize(st, h, P, what):
    c = st.ctx
    mid, ms = c.var_id(h), c.var_size(h)
    order = c.variable_order()
    ids = {o: c.var_id(o) for o in st.kinds if o != h}
    st.marginalize(h)
    sr.bits(c.cov(), sr.marginalize(P, mid, ms), what)
    assert c.variable_order() == [o for o in order if o != h]
    for o, i in ids.items():
        assert c.var_id(o) == (i - ms if i > mid else i), "handle %d: id %d -> %d" % (o, i, c.var_id(o))
    assert c.var_id(h) == -1
    return mid, ms


@pytest.mark.parametrize("cov", COVS)
@pytest.mark.parametrize("cross", [False, True])
@pytest.mark.parametrize("size,where", MARG)
def test_marginalize_is_the_reference_copy(size, where, cross, cov):
    """cross: N - size and N on either side of a multiple of 64 (N % 64 < size); otherwise N % 64 = size + 5."""
    delta = marg_delta(size, where)
    extra = extra_for(size - 1 if cross else size + 5, delta)
    st = State(extra, seed=size)
    h = marg_target(st, size, where)
    N = st.ctx.cov_rows()
    assert (N % 64 < size) == cross, N
    P = st.upload(cov, seed=N)
    mid, ms = check_marginalize(st, h, P, "P after marginalize")
    assert (where == "first") == (mid == 0) and (where != "last" or mid + ms == N)
    print("marginalize %d at %d (%s) N %d -> %d, %s: bit-exact" % (ms, mid, where, N, N - ms, cov))
    st.ctx.close()


@pytest.mark.parametrize("cov", COVS)
def test_marginalize_old_clone_takes_the_oldest_timestamp(cov):
    """With max_clone_size = 11 and 13 clones: a clone added last with the oldest timestamp (the highest id, a recycled handle) goes
    first, then the clone at 100.0 (the lowest id); with 11 left nothing happens."""
    st = State(extra_for(5), seed=8, options=dict(ur.STATE_OPTIONS, max_clone_size=11))
    c = st.ctx
    q = np.array([0.0, 0.0, 0.0, 1.0])
    h_old = c.add_clone_raw(99.0, np.concatenate([q, [1.0, 2.0, 3.0]]), np.concatenate([q, [1.0, 2.0, 3.0]]))
    st.kinds[h_old], st.sig[h_old] = ur.POSE, ur.SIGMA[ur.POSE]
    assert c.var_id(h_old) + 6 == c.cov_rows()  # the newest id, the oldest timestamp
    for expect, ts in ((h_old, 99.0), (c.clone_handle(100.0), 100.0)):
        P = st.upload(cov, seed=c.cov_rows())
        assert c.clone_handle(ts) == expect
        order = c.variable_order()
        mid, ms = c.var_id(expect), 6
        c.marginalize_old_clone()
        del st.kinds[expect], st.sig[expect]
        sr.bits(c.cov(), sr.marginalize(P, mid, ms), "P after marginalize_old_clone")
        assert c.variable_order() == [o for o in order if o != expect] and c.clone_handle(ts) == -1
    snap = st.snapshot()
    c.marginalize_old_clone()
    st.assert_unchanged(snap)
    print("marginalize_old_clone, %s: bit-exact" % cov)
    c.close()


@pytest.mark.parametrize("cov", ["corr", "asym"])
def test_vio_sequence_propagate_clone_marginalize(cov):
    """One VioManager frame on a correlated P: EKFPropagation of the IMU, augment_clone, marginalize_old_clone.  The propagation within
    its bound against the long-double reference; each copy step against the restatement applied to the library's own P of the step
    before (bit-exact, the dt terms within their bound)."""
    ur.require_long_double()
    st = State(extra_for(2), seed=6, options=dict(ur.STATE_OPTIONS, max_clone_size=12))
    c = st.ctx
    imu = c.handle_imu()
    P = st.upload(cov, seed=31)
    Phi, Q, _, ni, _ = phi_q(st, [imu], [imu], seed=31)
    c.ekf_propagation([imu], [imu], Phi, Q)
    P1 = c.cov()
    ref, B = sr.propagate(P, ni, ni, Phi, Q)
    q1 = sr.within(P1, ref, B, "P after the propagation")
    N = c.cov_rows()
    w = np.array([0.02, 0.3, -0.1])
    d = dt_d(c, w)
    c.augment_clone(300.0, w)
    P2 = c.cov()
    ref2, B2 = sr.augment_dt(sr.clone(P1, 0, 6), N, c.var_id(c.handle_dt()), d)
    q2 = sr.within(P2, ref2, B2, "P after augment_clone")
    h0 = c.clone_handle(100.0)
    mid = c.var_id(h0)
    c.marginalize_old_clone()
    assert c.clone_handle(100.0) == -1
    sr.bits(c.cov(), sr.marginalize(P2, mid, 6), "P after marginalize_old_clone")
    print("VioManager frame N %d, %s: worst error / bound: propagation %.3e, augment_clone %.3e; marginalisation bit-exact" % (N, cov, q1, q2))
    c.close()


# ---- get_marginal_covariance / set_initial_covariance ----------------------------------------------------------------------------
@pytest.mark.parametrize("cov", COVS)
def test_marginal_and_initial_covariance(cov):
    st = State(extra_for(63), seed=9)
    c = st.ctx
    P = st.upload(cov, seed=9)
    handles = ur.update_handles(c, st.hs)  # out of id order, non-contiguous
    ids = st.ids(handles)
    sr.bits(c.get_marginal_covariance(handles), sr.marginal(P, ids), "get_marginal_covariance")
    rng = np.random.default_rng(9)
    n = len(ids)
    A = rng.standard_normal((n, n))
    cov_in = A @ A.T / n + rng.standard_normal((n, n)) * 1e-3  # not symmetric: only its upper part survives where it lands above
    c.set_initial_covariance(cov_in, handles)
    sr.bits(c.cov(), sr.set_initial(P, cov_in, ids), "set_initial_covariance")
    print("marginal / initial covariance on %d columns, %s: bit-exact" % (n, cov))
    c.close()
