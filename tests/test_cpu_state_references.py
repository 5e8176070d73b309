"""The references of tests/state_reference.py against the oracle (StateHelper in double) and numpy on the inputs the GPU tests use, and
against planted mistakes: each arithmetic mistake moves some entry by more than twice its bound, each copy mistake changes at least one
bit, so a kernel that made it could not pass tests/test_gpu_state_ops.py."""
import numpy as np
import pytest

import oracle_backend
import state_reference as sr
import update_reference as ur
from test_gpu_state_ops import COVS, State, extra_for, phi_q, prop_shape, small_state


def ostate(extra, seed=0, options=ur.STATE_OPTIONS):
    return State(extra, seed=seed, options=options, make=oracle_backend.OracleContext)


# ---- propagation ---------------------------------------------------------------------------------------------------------------------
ORACLE_SHAPES = ("imu", "anchor", "anchor_nocal", "calib_incl", "calib_excl", "rows1", "rows16")  # the rows* tails need ovp_clone


@pytest.mark.parametrize("cov", COVS)
@pytest.mark.parametrize("shape", ORACLE_SHAPES)
def test_propagation_reference_against_oracle_and_numpy(shape, cov):
    """StateHelper::EKFPropagation of the oracle and the same products in float64 numpy stay within the bound; the oracle's entries
    outside the new rows and columns are bit-identical and its Q's lower triangle is ignored."""
    ur.require_long_double()
    st = ostate(extra_for(1), seed=7)
    new, old = prop_shape(st, shape)
    P = st.upload(cov, seed=3)
    Phi, Q, Qg, ni, oi = phi_q(st, new, old, seed=3)
    st.ctx.ekf_propagation(new, old, Phi, Qg)
    ref, B = sr.propagate(P, ni, oi, Phi, Q)
    qo = sr.within(st.ctx.cov(), ref, B, "oracle P+")
    C = P[:, oi] @ Phi.T
    Pn = P.copy()
    Pn[ni, :], Pn[:, ni] = C.T, C
    Pn[np.ix_(ni, ni)] = sr.upper_sym(Q) + Phi @ C[oi, :]
    qn = sr.within(Pn, ref, B, "numpy P+")
    print("%s %s: worst error / bound: oracle %.3e, numpy %.3e" % (shape, cov, qo, qn))
    st.ctx.close()


# ---- exact copies --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cov", COVS)
def test_copy_restatements_against_oracle(cov):
    """marginalize (first, middle and last variable, sizes 1 to 15), get_marginal_covariance and set_initial_covariance with handles out
    of id order, augment_clone with and without the time offset: the oracle equals the restatements bit for bit (the dt terms within
    their bound)."""
    ur.require_long_double()
    st = ostate(extra_for(0), seed=2)
    c = st.ctx
    for h in (c.handle_dt(), st.hs["planes"][2], c.handle_imu(), st.hs["lms"][-1], c.handle_intrinsics(), st.hs["clones"][1]):
        P = st.upload(cov, seed=c.cov_rows())
        mid, ms = c.var_id(h), c.var_size(h)
        st.marginalize(h)
        sr.bits(c.cov(), sr.marginalize(P, mid, ms), "oracle marginalize of %d at %d" % (ms, mid))
    P = st.upload(cov, seed=1)
    handles = [st.hs["clones"][3], c.handle_calib(), st.hs["planes"][1], st.hs["lms"][0]]
    ids = st.ids(handles)
    sr.bits(c.get_marginal_covariance(handles), sr.marginal(P, ids), "oracle get_marginal_covariance")
    A = np.random.default_rng(4).standard_normal((len(ids), len(ids)))
    c.set_initial_covariance(A, handles)
    sr.bits(c.cov(), sr.set_initial(P, A, ids), "oracle set_initial_covariance")
    st.ctx.close()
    st = ostate(extra_for(0), seed=2)
    c = st.ctx
    P = st.upload(cov, seed=5)
    N, w = c.cov_rows(), np.array([0.3, -0.2, 0.1])
    d = np.concatenate([w, c.var_get(c.handle_imu())[0][7:10]])
    c.set_timestamp(300.0)
    c.augment_clone(300.0, w)
    ref, B = sr.augment_dt(sr.clone(P, 0, 6), N, c.var_id(c.handle_dt()), d)
    q = sr.within(c.cov(), ref, B, "oracle augment_clone")
    c.close()
    c, kinds, sig = small_state(0, make=oracle_backend.OracleContext)
    _, _, _, dd = ur.state_arrays(c, kinds, sig)
    P = sr.covariance(cov, dd, 9)
    c.cov_upload(P)
    c.set_timestamp(20.0)
    c.augment_clone(20.0, [0.5, 0.5, 0.5])
    sr.bits(c.cov(), sr.clone(P, 0, 6), "oracle augment_clone without the time offset")
    c.close()
    print("%s: copies bit-exact, augment_clone worst error / bound %.3e" % (cov, q))


def test_long_sequence_on_an_asymmetric_covariance():
    """Every operation in turn on the oracle, starting from the asymmetric P, each against its reference applied to the oracle's own P of
    the step before: propagations of the IMU and of an anchor change, augment_clone, marginalisations, set_initial_covariance."""
    ur.require_long_double()
    st = ostate(extra_for(9), seed=11, options=dict(ur.STATE_OPTIONS, max_clone_size=11))
    c, hs = st.ctx, st.hs
    imu = c.handle_imu()
    P = st.upload("asym", seed=11)
    dt = c.handle_dt()
    worst = 0.0
    for k in range(4):
        Phi, Q, Qg, ni, oi = phi_q(st, [imu], [imu], seed=20 + k)
        c.ekf_propagation([imu], [imu], Phi, Qg)
        ref, B = sr.propagate(P, ni, oi, Phi, Q)
        worst = max(worst, sr.within(c.cov(), ref, B, "step %d propagation" % k))
        P = c.cov()
        assert not np.array_equal(P, P.T)
        N, w = P.shape[0], np.array([0.1 * k, 0.2, -0.3])
        d = np.concatenate([w, c.var_get(imu)[0][7:10]])
        t = 400.0 + k
        c.set_timestamp(t)
        nh = c.augment_clone(t, w)
        st.kinds[nh], st.sig[nh] = ur.POSE, ur.SIGMA[ur.POSE]
        ref, B = sr.augment_dt(sr.clone(P, 0, 6), N, c.var_id(dt), d)
        worst = max(worst, sr.within(c.cov(), ref, B, "step %d augment_clone" % k))
        P = c.cov()
        before = {h: c.var_id(h) for h in st.kinds}
        c.marginalize_old_clone()
        gone = [h for h in before if c.var_id(h) == -1]
        assert len(gone) == 1 and c.var_size(gone[0]) == 6
        del st.kinds[gone[0]], st.sig[gone[0]]
        sr.bits(c.cov(), sr.marginalize(P, before[gone[0]], 6), "step %d marginalize_old_clone" % k)
        P = c.cov()
        lm, a0, a1 = hs["lms"][k % 2], hs["clones"][5 + k], hs["clones"][-1]
        Phi, Q, Qg, ni, oi = phi_q(st, [lm], [a0, c.handle_calib(), a1, lm], seed=30 + k)
        c.ekf_propagation([lm], [a0, c.handle_calib(), a1, lm], Phi, Qg)
        ref, B = sr.propagate(P, ni, oi, Phi, Q)
        worst = max(worst, sr.within(c.cov(), ref, B, "step %d anchor change" % k))
        P = c.cov()
        h = hs["planes"][k] if k < 3 else hs["lms"][-1]
        mid, ms = c.var_id(h), c.var_size(h)
        st.marginalize(h)
        sr.bits(c.cov(), sr.marginalize(P, mid, ms), "step %d marginalize" % k)
        P = c.cov()
    handles = [hs["clones"][-1], imu, c.handle_intrinsics()]
    ids = st.ids(handles)
    A = np.random.default_rng(1).standard_normal((len(ids), len(ids)))
    c.set_initial_covariance(A, handles)
    sr.bits(c.cov(), sr.set_initial(P, A, ids), "set_initial_covariance")
    print("sequence of 21 operations: copies bit-exact, worst error / bound %.3e" % worst)
    c.close()


# ---- planted mistakes ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cov", COVS)
def test_planted_arithmetic_mistakes_exceed_the_bounds(cov):
    """Phi transposed, Q's lower triangle used, D written transposed (asymmetric P: D is not symmetric), the second dt pass reading the dt
    row from before the first: each moves some entry by more than twice its bound."""
    ur.require_long_double()
    st = ostate(extra_for(63), seed=7)
    c = st.ctx
    imu = c.handle_imu()
    P = st.upload(cov, seed=3)
    ratios = {}
    Phi, Q, Qg, ni, oi = phi_q(st, [imu], [imu], seed=3)
    ref, B = sr.propagate(P, ni, oi, Phi, Q)
    ratios["Phi transposed"] = sr.exceed(sr.propagate(P, ni, oi, Phi.T, Q)[0], ref, B)
    ratios["Q lower triangle"] = sr.exceed(sr.propagate(P, ni, oi, Phi, Qg, lower=True)[0], ref, B)
    new, old = prop_shape(st, "calib_incl")
    Phi, Q, Qg, ni, oi = phi_q(st, new, old, seed=4)
    ref, B = sr.propagate(P, ni, oi, Phi, Q)
    bad = ref.copy()
    bad[np.ix_(ni, ni)] = ref[np.ix_(ni, ni)].T
    if cov == "asym":
        ratios["D transposed"] = sr.exceed(bad, ref, B)
    N, d = P.shape[0], np.concatenate([[0.3, -0.2, 0.1], c.var_get(imu)[0][7:10]])
    Pc = sr.clone(P, 0, 6)
    ref, B = sr.augment_dt(Pc, N, c.var_id(c.handle_dt()), d)
    ratios["dt row read before the first pass"] = sr.exceed(sr.augment_dt(Pc, N, c.var_id(c.handle_dt()), d, stale_row=True)[0], ref, B)
    print("%s: %s" % (cov, ", ".join("%s %.1e" % kv for kv in ratios.items())))
    for name, q in ratios.items():
        assert q > 2.0, "%s moves no entry beyond twice its bound (%.3e)" % (name, q)
    c.close()


def _mismatches(a, b):
    return int(np.sum(np.asarray(a).view(np.uint64) != np.asarray(b).view(np.uint64)))


@pytest.mark.parametrize("cov", COVS)
def test_planted_copy_mistakes_change_bits(cov):
    """The clone's row block taken from columns and x2x1 copied instead of mirrored change bits exactly when P is asymmetric (which is
    why the parity tests on synth's symmetric P0 could not see them); x2 read one row late changes bits on every P."""
    st = ostate(extra_for(1), seed=5)
    c = st.ctx
    P = st.upload(cov, seed=6)
    n = {}
    for name, h in (("IMU pose", c.handle_imu()), ("clone", st.hs["clones"][2]), ("intrinsics", c.handle_intrinsics())):
        o, s = c.var_id(h), 6 if h == c.handle_imu() else c.var_size(h)
        n["clone of %s: rows from columns" % name] = _mismatches(sr.clone(P, o, s, rows_from_cols=True), sr.clone(P, o, s))
    for name, h in (("dt", c.handle_dt()), ("plane", st.hs["planes"][1]), ("clone", st.hs["clones"][4])):
        mid, ms = c.var_id(h), c.var_size(h)
        ref = sr.marginalize(P, mid, ms)
        n["marginalize %s: x2x1 copied" % name] = _mismatches(sr.marginalize(P, mid, ms, copy_x2x1=True), ref)
        n["marginalize %s: shifted by one" % name] = _mismatches(sr.marginalize(P, mid, ms, shift=1), ref)
    print("%s: %s" % (cov, ", ".join("%s %d" % kv for kv in n.items())))
    for name, k in n.items():
        if cov == "asym" or "shifted" in name:
            assert k > 0, "%s changes no bit" % name
        else:
            assert k == 0, "%s: P is symmetric, so the mistake is invisible on it (%d bits)" % (name, k)
    c.close()
