"""The oracle's per-feature chi2 (UpdaterMSCKF's point gate and UpdaterSLAM's gate, its plane -> no-plane retry included) against the
long-double references of tests/gate_reference.py on a correlated covariance.  Every feature status of the GPU tests is compared with
this oracle, and the references are the ones tests/test_gpu_feature_gate.py holds the CUDA kernels to."""
import numpy as np
import pytest

import gate_reference as gr
import oracle_backend
from ov_plane_b200 import synth


def _oracle(S, chi2_table):
    orc = oracle_backend.OracleContext(S.options)
    orc.set_chi2_table(chi2_table)
    return orc, synth.load_scenario_into(orc, S)


def _check(tag, got, ref, bound, status, thr, accept_status):
    """chi2 within the bound; the status is the reference's decision where the reference lies outside the bound of the threshold."""
    err = abs(float(got) - float(ref))
    assert err <= bound, "%s: chi2 %.17g, reference %.17g: error %.3e above the bound %.3e" % (tag, got, float(ref), err, bound)
    if abs(float(ref) - thr) > bound:
        assert (status == accept_status) == (float(ref) <= thr), "%s: status %d, reference chi2 %.6g against %.6g" % (tag, status, float(ref), thr)
    return err / bound if bound > 0 else 0.0


@pytest.mark.parametrize("ncal,cond", [(0, None), (14, None), (6, 1e10), (8, None)])
def test_oracle_point_gate_against_long_double_reference(ncal, cond, chi2_table):
    gr.require_long_double()
    from test_gpu_compression import _scenario
    S = _scenario(("points", ncal))
    orc, ch = _oracle(S, chi2_table)
    orc.cov_upload(gr.correlated_cov(S, S.N, seed=5 + ncal, cond=cond))
    P = orc.cov()
    b = synth.feature_batch(S, ch)
    cal = gr.calib_ids(orc, S.options)
    refs = []  # at the linearisation point of the gate: before the update moves the clones
    for f in range(S.F):
        a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
        pf = b["p_FinG_original"][f]
        Hf, Hx, r, xo = orc.feature_jacobian_full(b["meas_clone"][a:e], b["uv"][a:e], pf, pf, 0, None, None, 1.0, S.options["sigma_constraint"])
        ids = gr.block_ids(orc, xo)
        assert ids[:len(cal)] == cal
        refs.append(gr.point_gate(Hf, Hx, r, P[np.ix_(ids, ids)]))
        assert refs[-1][2] == 2 * (e - a) - 3
    o = orc.msckf_update(b, 1.0, 1.0)
    worst, n = 0.0, {0: 0, 1: 0}
    for f in range(S.F):
        ref, bound, dof = refs[f]
        st = int(o["feat_status"][f])
        assert st in (0, 1)
        n[st] += 1
        worst = max(worst, _check("feature %d" % f, o["feat_chi2"][f], ref, bound, st, chi2_table[dof], 1))
    print("oracle point gate ncal=%d cond=%s: accepted %d rejected %d, worst error / bound %.3e" % (ncal, cond, n[1], n[0], worst))
    assert n[0] >= 2 and n[1] >= 20


def slam_gate_reference(be, S, b, f, status, has_plane, P):
    """Reference chi2, bound and dof of the gate whose result the status reports: with the plane row when the feature had one and was
    accepted with it, otherwise on the bearing rows alone."""
    a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
    lm = be.slam_handle(int(b["featid"][f]))
    val, fej = be.var_get(lm)
    with_plane = has_plane and status == 1
    pid = int(b["planeid"][f]) if with_plane else 0
    cp = cpf = None
    if with_plane:
        cp, cpf = be.var_get(be.plane_handle(pid))
    Hf, Hx, r, xo = be.feature_jacobian_full(b["meas_clone"][a:e], b["uv"][a:e], val, fej, pid, cp, cpf, 1.0, S.options["sigma_constraint"])
    ids = gr.block_ids(be, [lm]) + gr.block_ids(be, xo)
    return gr.slam_gate(np.hstack([Hf, Hx]), r, P[np.ix_(ids, ids)])


@pytest.mark.parametrize("ncal,cond", [(0, None), (14, None), (14, 1e10)])
def test_oracle_slam_gate_against_long_double_reference(ncal, cond, chi2_table):
    gr.require_long_double()
    S = gr.slam_scenario(ncal)
    orc, ch = _oracle(S, chi2_table)
    g = orc.slam_delayed_init(synth.feature_batch(S, ch), 1.0, 1.0)
    keep = np.nonzero(g["feat_status"] > 0)[0]
    attached = {int(S.featid[f]) for f in keep if g["feat_status"][f] == 1 and S.planeid[f] != 0}
    assert len(keep) >= 16 and len(attached) >= 6, (len(keep), len(attached))
    orc.cov_upload(gr.correlated_cov(S, orc.cov_rows(), seed=7 + ncal, cond=cond))
    P = orc.cov()
    b = gr.slam_update_batch(S, ch, keep, seed=ncal, wrong_plane=3)
    # both gates of every landmark at the linearisation point of the update, before it moves the state
    refs = [{st: slam_gate_reference(orc, S, b, f, st, int(b["featid"][f]) in attached, P) for st in (0, 1)} for f in range(b["F"])]
    o = orc.slam_update(b, 1.0, 1.0)
    worst, count = 0.0, np.zeros(4, dtype=int)
    for f in range(b["F"]):
        st = int(o["feat_status"][f])
        has_plane = int(b["featid"][f]) in attached
        assert st in (0, 1, 3) and (st != 3 or has_plane)
        ref, bound, dof = refs[f][1 if st == 1 else 0]
        count[st] += 1
        worst = max(worst, _check("landmark %d" % f, o["feat_chi2"][f], ref, bound, st, chi2_table[dof], 3 if has_plane and st != 1 else 1))
    print("oracle SLAM gate ncal=%d cond=%s: statuses %s, worst error / bound %.3e" % (ncal, cond, count.tolist(), worst))
    assert count[1] >= 8 and count[3] >= 1
