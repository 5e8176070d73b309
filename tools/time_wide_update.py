"""Time updates wider than one co-resident launch of the fused Cholesky (DESIGN.md 4.1, 9), with the width declared up to the context's
column capacity (ovp_set_max_update_width):
  - ovp_ekf_update with n = rows in {960, 1024, 1536, 2048} innovation rows over about as many landmark columns of a state of
    N ~ 2048 (960 runs the one fused launch, the others run panels);
  - ovp_slam_update of about 330 GLOBAL_3D landmarks with two measurements each (compressed width past 960);
  - ovp_debug_chol_panels forced at a 960-column panel against ovp_debug_chol_solve_gated on the same 960-wide system with a 2048-row
    right-hand side: the cost of running one system as a panel rather than as the fused launch.  Both hook calls include the same host
    copies of the system; their difference is the panel path's own cost.
Before every timed call the covariance and values are restored outside the timed window.  Time is host wall time around the call and a
synchronise of the library's stream (so it covers the device work); each line prints the median and spread over --iters calls, the
kernel launches per call, and the card name and power limit read in the same run.

  python tools/time_wide_update.py [--iters 20]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from ov_plane_b200 import api, synth  # noqa: E402

STATE_OPTIONS = dict(do_fej=1, imu_avg=0, use_rk4_integration=1, do_calib_camera_pose=1, do_calib_camera_intrinsics=1,
                     do_calib_camera_timeoffset=1, max_clone_size=11, max_aruco_features=1024, sigma_constraint=0.01, const_init_multi=1.0,
                     const_init_chi2=1.0, sigma_plane_merge=0.01, plane_merge_chi2=0.75, plane_merge_deg_max=1.0)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:  # the timing is still reported; the card is then unknown
        return "unknown (%s)" % e


def timed(ctx, call, iters, restore=True):
    """median / min / max ms and launches of call() over iters runs, after two warm-up runs"""
    ts, launches = [], 0
    for it in range(iters + 2):
        if restore:
            ctx.restore()
        ctx.synchronize()
        l0 = ctx.launch_count()
        t0 = time.perf_counter()
        call()
        ctx.synchronize()
        t1 = time.perf_counter()
        if it >= 2:
            ts.append(1e3 * (t1 - t0))
            launches = ctx.launch_count() - l0
    return dict(ms_median=float(np.median(ts)), ms_min=float(np.min(ts)), ms_max=float(np.max(ts)), launches=int(launches))


def ekf_cases(iters, gpu):
    ctx = api.Context(STATE_OPTIONS, device=0, max_state=2048, max_meas_rows=4096)
    rng = np.random.default_rng(0)
    lms = []
    for i in range((2048 - ctx.cov_rows()) // 3):
        p = 3.0 * rng.standard_normal(3)
        lms.append(ctx.add_slam_raw(5000000 + i, p, p))
    N = ctx.cov_rows()
    F = rng.standard_normal((N, 4))
    d = np.exp(rng.uniform(-2.0, 0.0, N))
    A = F @ F.T / 4.0 + 0.3 * np.eye(N)
    s = d / np.sqrt(np.diag(A))
    ctx.cov_upload(s[:, None] * A * s[None, :])
    ctx.set_max_update_width((2048 + 63) // 64 * 64 + 64)
    ctx.snapshot()
    for rows in (960, 1024, 1536, 2048):
        hs = lms[:min(len(lms), (rows + 2) // 3)]
        H = rng.standard_normal((rows, 3 * len(hs))) / np.sqrt(3 * len(hs))
        r = rng.standard_normal(rows)
        res = timed(ctx, lambda: ctx.ekf_update(hs, H, r), iters)
        print(json.dumps(dict(case="ekf_update", N=N, rows=rows, cols=3 * len(hs), card=gpu, **res)), flush=True)
    ctx.close()


def slam_case(iters, gpu):
    import gate_reference as gr
    S = gr.slam_scenario(0, seed=0, F=330)
    ctx = api.Context(S.options, device=0, max_state=S.N + 3 * S.F + 64, max_meas_rows=60000)
    ctx.set_chi2_table(synth.chi2_table())
    chg = synth.load_scenario_into(ctx, S)
    g = ctx.slam_delayed_init(synth.feature_batch(S, chg), 1.0, 1.0)
    keep = np.nonzero(g["feat_status"] > 0)[0]
    b = gr.slam_update_batch(S, chg, keep, seed=0, wrong_plane=3)
    offs, mc, uv = [0], [], []
    for f in range(b["F"]):  # every landmark with its newest two measurements: a wide, short batch
        a, e = int(b["meas_offset"][f]), int(b["meas_offset"][f + 1])
        n = min(2, e - a)
        mc.append(b["meas_clone"][e - n:e])
        uv.append(b["uv"][e - n:e])
        offs.append(offs[-1] + n)
    b.update(meas_offset=np.array(offs, dtype=np.int32), meas_clone=np.concatenate(mc).astype(np.int32),
             uv=np.concatenate(uv).astype(np.float32))
    ctx.set_max_update_width((S.N + 3 * S.F + 64 + 63) // 64 * 64 + 64)
    ctx.snapshot()
    res = timed(ctx, lambda: ctx.slam_update(b, 1.0, 1.0, True), iters)
    print(json.dumps(dict(case="slam_update", landmarks=int(b["F"]), N=ctx.cov_rows(), card=gpu, **res)), flush=True)
    ctx.close()


def panel_cost(iters, gpu):
    S = synth.make_scenario("tiny_points")
    ctx = api.Context(S.options, device=0, max_state=2048, max_meas_rows=4096, debug=True)
    rng = np.random.default_rng(1)
    n, mrows = 960, 2048
    B = rng.standard_normal((n + 16, n))
    A = np.asfortranarray(np.tril(B.T @ B + 0.5 * np.eye(n)))
    M = np.asfortranarray(rng.standard_normal((mrows, n)))
    z = rng.standard_normal(n)
    L, Y, w = np.zeros((n, n), order="F"), np.zeros((mrows, n), order="F"), np.zeros(n)
    p = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
    args = (p(A), n, n, C.c_double(0.0), p(M), mrows, p(z), 1, C.c_double(-1.0), p(L), p(Y), p(w), None, None)
    for name, call in (("fused", lambda: ctx._ck(ctx.lib.ovp_debug_chol_solve_gated(ctx.h, *args))),
                       ("panel_960", lambda: ctx._ck(ctx.lib.ovp_debug_chol_panels(ctx.h, 960, *args)))):
        res = timed(ctx, call, iters, restore=False)
        print(json.dumps(dict(case="chol_960_rhs_2048", path=name, card=gpu, **res)), flush=True)
    ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    gpu = card()
    ekf_cases(a.iters, gpu)
    slam_case(a.iters, gpu)
    panel_cost(a.iters, gpu)


if __name__ == "__main__":
    main()
