"""Programmatic dependent launches of the update chain (chain_launch, ovp_internal.h): the feature kernels, the Gram SYRK, its D part and
reduction, and the update's tail start while the launch before them runs, each waiting for it before touching memory.  Nothing of the
arithmetic moves, so with the launches programmatic (the default) and with ovp_debug_programmatic_launches(0) every output carries the same
bits: P+, every value and first estimate, the statuses, the chi2 values and the Hx order of the benchmarked step (replayed from its graph
and launched eagerly), of a prepared batch replayed three times, of the SLAM update, of ovp_ekf_update, and of a step whose gates all
reject (the update tail's early exits, which must leave the state untouched)."""
import threading

import numpy as np
import pytest

from ov_plane_b200 import api, synth

pytestmark = pytest.mark.gpu

CFG3 = "cfg3_n512_f600_p8"


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _state(ctx):
    vals = [ctx.var_get(int(h)) for h in ctx.variable_order()]
    return ctx.cov(), np.concatenate([np.concatenate([v, f]) for v, f in vals])


def _same(a, b, tag):
    """a, b: (gates dict, (P, values)) of two runs"""
    (ga, sa), (gb, sb) = a, b
    assert ga.keys() == gb.keys(), tag
    for k in ga:
        assert _bits_equal(np.asarray(ga[k]), np.asarray(gb[k])), "%s: %s differs" % (tag, k)
    assert _bits_equal(sa[0], sb[0]), "%s: P differs" % tag
    assert _bits_equal(sa[1], sb[1]), "%s: values / FEJs differ" % tag


def _cfg3_ctx(chi2_table, programmatic, extra_state=0):
    S = synth.make_scenario(CFG3, seed=0)
    ctx = api.Context(S.options, device=0, max_state=S.N + extra_state + 64, max_meas_rows=60000, debug=True)
    ctx.set_chi2_table(chi2_table)
    ch = synth.load_scenario_into(ctx, S)
    ctx._ck(ctx.lib.ovp_debug_programmatic_launches(ctx.h, 1 if programmatic else 0))
    return S, ch, ctx


@pytest.mark.parametrize("graphs", [True, False])
def test_cfg3_step_programmatic_and_serial(chi2_table, graphs):
    """The benchmarked step (8 plane updates + the point update), replayed from its CUDA graph or launched eagerly: the same bits either
    way, with as many launches."""
    runs = {}
    for prog in (0, 1):
        S, ch, ctx = _cfg3_ctx(chi2_table, prog)
        ctx.set_use_graphs(graphs)
        batch = synth.feature_batch(S, ch)
        ctx.snapshot()
        ctx.msckf_update(batch, 1.0, 1.0)  # the first launch of a plan runs eagerly, the next one is captured
        ctx.restore()
        l0 = ctx.launch_count()
        g = ctx.msckf_update(batch, 1.0, 1.0)
        runs[prog] = ((g, _state(ctx)), ctx.launch_count() - l0)
        ctx.close()
    assert (runs[1][0][0]["feat_status"] == 1).any() and (runs[1][0][0]["plane_status"] == 1).any()
    _same(runs[0][0], runs[1][0], "cfg3 step, graphs=%s" % graphs)
    assert runs[0][1] == runs[1][1]


def test_prepared_batch_replayed_three_times(chi2_table):
    """One prepared batch launched three times in a row on the evolving state (no restore in between), then switched to serial launches
    in the same context: the switch drops the captured graph, and the serial replays reproduce the programmatic ones."""
    S, ch, ctx = _cfg3_ctx(chi2_table, 1)
    try:
        batch = synth.feature_batch(S, ch)
        ctx.snapshot()
        ctx.msckf_prepare(batch, 1.0, 1.0)
        runs = {}
        for prog in (1, 0):
            ctx._ck(ctx.lib.ovp_debug_programmatic_launches(ctx.h, prog))
            ctx.restore()
            seq = []
            for _ in range(3):
                ctx.msckf_launch()
                seq.append((ctx.msckf_finish(), _state(ctx)))
            runs[prog] = seq
        for k in range(3):
            _same(runs[0][k], runs[1][k], "replay %d" % k)
        assert not _bits_equal(runs[1][0][1][0], runs[1][2][1][0])  # the replays did update the state
    finally:
        ctx.close()


def test_slam_update_programmatic_and_serial(chi2_table):
    """UpdaterSLAM's delayed initialisation and update of 20 landmarks on the benchmark's state."""
    out = {}
    for prog in (0, 1):
        S, ch, ctx = _cfg3_ctx(chi2_table, prog, extra_state=3 * 20)
        g = ctx.slam_delayed_init(synth.feature_batch(S, ch, np.arange(20)), 1.0, 1.0)
        keep = np.nonzero(g["feat_status"] > 0)[0]
        ub = synth.feature_batch(S, ch, keep)
        ub["uv"] = ub["uv"] + np.random.default_rng(7).normal(0.0, 0.5, ub["uv"].shape).astype(np.float32)
        g2 = ctx.slam_update(ub, 1.0, 1.0)
        out[prog] = (g, g2, _state(ctx))
        ctx.close()
    assert (out[1][1]["feat_status"] == 1).any()
    _same((out[0][0], out[0][2]), (out[1][0], out[1][2]), "SLAM delayed init + update")
    _same((out[0][1], out[0][2]), (out[1][1], out[1][2]), "SLAM update")


def test_ekf_update_programmatic_and_serial(chi2_table):
    """ovp_ekf_update (StateHelper::EKFUpdate) with a dense H over the IMU and three clones."""
    out = {}
    for prog in (0, 1):
        S, ch, ctx = _cfg3_ctx(chi2_table, prog)
        order = [int(h) for h in ctx.variable_order()]
        hs = [ctx.handle_imu()] + [h for h in order if h != ctx.handle_imu()][:3]
        ncol = sum(ctx.var_size(h) for h in hs)
        rng = np.random.default_rng(3)
        H = rng.standard_normal((40, ncol))
        res = 0.01 * rng.standard_normal(40)
        ctx.ekf_update(hs, H, res, np.full(40, 0.5))
        out[prog] = ({}, _state(ctx))
        ctx.close()
    _same(out[0], out[1], "ovp_ekf_update")


def test_all_gates_rejected_leave_the_state_untouched(chi2_table):
    """A chi2 multiplier so small that every plane update and every point feature is rejected: the plane updates and the point update
    take the early exits of the update tail (the gate flag, and no accepted feature), and the state keeps its bits."""
    out = {}
    for prog in (0, 1):
        S, ch, ctx = _cfg3_ctx(chi2_table, prog)
        before = _state(ctx)
        batch = synth.feature_batch(S, ch)
        ctx.snapshot()
        ctx.msckf_update(batch, 1.0, 1e-12)
        ctx.restore()
        g = ctx.msckf_update(batch, 1.0, 1e-12)  # replayed from the captured graph
        after = _state(ctx)
        assert not (g["plane_status"] == 1).any() and not (g["feat_status"] == 1).any()
        assert _bits_equal(before[0], after[0]) and _bits_equal(before[1], after[1])
        out[prog] = (g, after)
        ctx.close()
    _same(out[0], out[1], "all gates rejected")


def test_two_contexts_at_once_match_their_serial_runs(chi2_table):
    """Two contexts run the benchmarked step at the same time on their own streams, each from its own thread: each one's result is its
    serial (non-programmatic, one context at a time) result."""
    ctxs, refs = [], []
    for seed in (0, 1):
        S = synth.make_scenario(CFG3, seed=seed)
        c = api.Context(S.options, device=0, max_state=S.N + 64, max_meas_rows=60000, debug=True)
        c.set_chi2_table(chi2_table)
        ch = synth.load_scenario_into(c, S)
        b = synth.feature_batch(S, ch)
        c.snapshot()
        c._ck(c.lib.ovp_debug_programmatic_launches(c.h, 0))
        refs.append((c.msckf_update(b, 1.0, 1.0), _state(c)))
        c.restore()
        c._ck(c.lib.ovp_debug_programmatic_launches(c.h, 1))
        c.msckf_update(b, 1.0, 1.0)  # captures the plan's graph; the runs below replay it
        c.msckf_prepare(b, 1.0, 1.0)
        ctxs.append(c)
    try:
        for rnd in range(3):
            for c in ctxs:
                c.restore()
            start = threading.Barrier(2)

            def run(c):
                start.wait()
                c.msckf_launch()

            th = [threading.Thread(target=run, args=(c,)) for c in ctxs]
            for t in th:
                t.start()
            for t in th:
                t.join()
            for i, c in enumerate(ctxs):
                _same(refs[i], (c.msckf_finish(), _state(c)), "context %d, round %d" % (i, rnd))
    finally:
        for c in ctxs:
            c.close()
