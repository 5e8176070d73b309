"""Reuse of a prepared MSCKF batch: an update whose batch layout and state layout equal the last one's replays the last plan (and its
CUDA graph) and uploads only the measurement values.  What the plan read must then be what a fresh plan would read: the state handle of
each plane of the batch, and whether the batch carries plane_cp."""
import ctypes as C

import numpy as np
import pytest

from ov_plane_b200 import api, synth

pytestmark = pytest.mark.gpu

OVP_ERR_BAD_ARGS = 1
TOL = 1e-11  # the context's default rank tolerance; setting it again drops the prepared batch (ovp_set_rank_tolerance)
PLANE_B = 9001  # a plane id that is not in the scenario


def _context(S, chi2):
    ctx = api.Context(S.options, device=0, max_state=256, max_meas_rows=4096)
    ctx.set_chi2_table(chi2)
    ctx.set_rank_tolerance(TOL)
    return ctx


def _recycled_handle_sequence(chi2, drop_plan_before_second_update):
    """Plane A is in the state at handle h for a first update; A is marginalised, and a new plane B takes handle h and A's covariance
    columns.  The second update of the same batch sees the same batch layout, the same variable ids and as many planes in the state,
    but A is now a plane that is not in the state (the batch carries its plane_cp)."""
    S = synth.make_scenario("tiny_planes", seed=1)
    ctx = _context(S, chi2)
    batch = synth.feature_batch(S, synth.load_scenario_into(ctx, S))
    for fid, _, _ in S.slam:  # A, the scenario's last plane, becomes the last variable of the state
        ctx.marginalize(ctx.slam_handle(fid))
    pid_a, cp_a, _ = S.planes[-1]
    h = ctx.plane_handle(pid_a)
    assert ctx.var_id(h) + 3 == ctx.cov_rows()
    # 64 freed handles queue up behind the landmark's: from here on every new variable takes the oldest freed handle, so the handle
    # table keeps its size
    for k in range(64):
        ctx.marginalize(ctx.add_slam_raw(10**6 + k, np.ones(3), np.ones(3)))
    out = [ctx.msckf_update(batch)]
    ctx.marginalize(h)
    for _ in range(100):  # B goes in and out of the state until the free list hands it h
        hb = ctx.add_plane_raw(PLANE_B, cp_a, cp_a)
        if hb == h:
            break
        ctx.marginalize(hb)
    assert ctx.plane_handle(PLANE_B) == h and ctx.plane_handle(pid_a) == -1
    if drop_plan_before_second_update:
        ctx.set_rank_tolerance(TOL)
    out.append(ctx.msckf_update(batch))
    handles = ctx.variable_order()
    state = [ctx.cov()] + [a for hv in handles for a in ctx.var_get(hv)]
    ctx.close()
    return out, handles, state


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def test_recycled_plane_handle_is_planned_again(chi2_table):
    """A plan reused across the recycled handle would update A's features against B as an in-state plane."""
    got, got_handles, got_state = _recycled_handle_sequence(chi2_table, False)
    ref, ref_handles, ref_state = _recycled_handle_sequence(chi2_table, True)
    assert got_handles == ref_handles
    for i, (g, r) in enumerate(zip(got, ref)):
        for k in ("feat_status", "feat_chi2", "plane_status", "plane_chi2"):
            assert _same_bits(g[k], r[k]), "update %d: %s" % (i + 1, k)
        assert g["hx_order"] == r["hx_order"]
    assert len(got_state) == len(ref_state) and all(_same_bits(g, r) for g, r in zip(got_state, ref_state))


def _update_without_plane_cp(ctx, batch):
    fb, keep = ctx._batch_struct(batch)
    fb.plane_cp = None
    return ctx.lib.ovp_msckf_update(ctx.h, C.byref(fb), C.byref(api.UpdaterOptions(1.0, 1.0)), None, None, None, None, None, None)


def test_null_plane_cp_is_refused_on_a_reused_layout(chi2_table):
    """A plane that is not in the state needs the batch's plane_cp: a layout prepared with it does not run without it."""
    S = synth.make_scenario("tiny_planes", seed=0)
    planes = synth.drop_planes_from_state(S)
    fresh, ctx = _context(S, chi2_table), _context(S, chi2_table)
    batches = []
    for c in (fresh, ctx):
        b = synth.feature_batch(S, synth.load_scenario_into(c, S))
        b["plane_ids"] = np.array([p[0] for p in planes], dtype=np.int64)
        b["plane_cp"] = np.ascontiguousarray([p[1] for p in planes], dtype=np.float64)
        batches.append(b)
    assert _update_without_plane_cp(fresh, batches[0]) == OVP_ERR_BAD_ARGS
    ctx.msckf_update(batches[1])
    assert _update_without_plane_cp(ctx, batches[1]) == OVP_ERR_BAD_ARGS
    assert "plane_cp" in ctx.lib.ovp_last_error(ctx.h).decode()
    fresh.close()
    ctx.close()
