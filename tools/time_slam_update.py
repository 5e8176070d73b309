"""Time ovp_slam_update with 25 landmarks (the sim config's max_slam_in_update) held as GLOBAL_3D against the same landmarks held as
ANCHORED_MSCKF_INVERSE_DEPTH and as ANCHORED_INVERSE_DEPTH_SINGLE (both then run feature_kernel<true, true>), over an 11-clone and a 30-clone
window.  Both paths start
from the same scene and raw tracks, and the landmarks are created by ovp_slam_delayed_init_tracks under ovp_set_landmark_representations(rep, rep):
each path's covariance is then the library's own for its representation (anchored in the clone of the newest measurement), so both gate
alike and accept the same landmarks.  Each landmark is then updated with its whole track; before every timed call the covariance and every
value are restored (outside the timed window), so every call does the same work.  Prints one JSON line per size and path with the median /
spread of device time (CUDA events on the library's stream) and of host wall time (with a synchronise), the kernel launches and accepted
landmarks per call, and the card name and power limit read in the same run.

  python tools/time_slam_update.py [--iters 30]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ov_plane_b200 import api, synth  # noqa: E402
from ov_plane_b200 import plane_init_chain as pic  # noqa: E402

N_SLAM = 25
SIZES = {
    "sim_11_clones": dict(n_clones=11, n_planes=4, F=200, m_min=3, m_max=11, plane_frac=0.5, n_slam=0, dtheta=0.05),
    "sim_30_clones": dict(n_clones=30, n_planes=4, F=400, m_min=6, m_max=20, plane_frac=0.5, n_slam=0, dtheta=0.03),
}
REPS = {"GLOBAL_3D": 0, "ANCHORED_MSCKF_INVERSE_DEPTH": 4, "ANCHORED_INVERSE_DEPTH_SINGLE": 5}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:  # the timing is still reported; the card is then unknown
        return "unknown (%s)" % e


def _pick(t, sel):
    mo = t["meas_offset"]
    idx = np.concatenate([np.arange(mo[f], mo[f + 1]) for f in sel])
    return dict(F=len(sel), meas_offset=np.concatenate([[0], np.cumsum(np.diff(mo)[sel])]).astype(np.int32),
                meas_clone=np.ascontiguousarray(t["meas_clone"][idx]), uv=np.ascontiguousarray(t["uv"][idx]),
                uv_norm=np.ascontiguousarray(t["uv_norm"][idx]), featid=np.ascontiguousarray(t["featid"][sel]),
                planeid=np.zeros(len(sel), dtype=np.int64))


def setup(size, rep):
    """a context with N_SLAM landmarks in representation rep, created from the scene's first N_SLAM tracks of 2 .. 29 measurements"""
    S, mk = pic.tracks_scene(name="small_planes", seed=0, px_noise=0.3, **SIZES[size])
    ctx = api.Context(S.options, device=0, max_state=S.N + 3 * N_SLAM + 64, max_meas_rows=60000)
    ctx.set_chi2_table(synth.chi2_table())
    full = mk(synth.load_scenario_into(ctx, S))
    n = np.diff(full["meas_offset"])
    t = _pick(full, [f for f in range(len(n)) if 2 <= n[f] <= 29][:N_SLAM])
    ctx.set_landmark_representations(rep, rep)
    r = ctx.slam_delayed_init_tracks(t, use_plane_constraint=False)
    b = _pick(t, [f for f in range(t["F"]) if r["new_handles"][f] >= 0])
    return ctx, b


def run(size, path, iters):
    import torch
    ctx, b = setup(size, REPS[path])
    stream = torch.cuda.ExternalStream(ctx.stream())
    P0, order = ctx.cov().copy(), ctx.variable_order()
    vals = [ctx.var_get(h) for h in order]
    dev, wall, launches, acc = [], [], [], []
    for it in range(iters + 2):
        ctx.cov_upload(P0)  # every call updates the same prior
        for h, (v, f) in zip(order, vals):
            ctx.var_set(h, v, f)
        l0 = ctx.launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ctx.synchronize()
        w0 = time.perf_counter()
        e0.record(stream)
        r = ctx.slam_update(b, 1.0, 1.0, False)
        e1.record(stream)
        ctx.synchronize()
        w1 = time.perf_counter()
        if it >= 2:  # warm-up: module loading and the first allocations of the process
            dev.append(e0.elapsed_time(e1))
            wall.append(1e3 * (w1 - w0))
            launches.append(ctx.launch_count() - l0)
            acc.append(int((r["feat_status"] > 0).sum()))
    rows = int(2 * b["meas_offset"][-1])
    ctx.close()

    def stat(x):
        x = np.asarray(x)
        return dict(median=float(np.median(x)), p10=float(np.percentile(x, 10)), p90=float(np.percentile(x, 90)))

    return dict(size=size, path=path, landmarks=int(b["F"]), rows=rows, accepted=int(np.median(acc)), device_ms=stat(dev), wall_ms=stat(wall),
                launches=int(np.median(launches)), iters=iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    a = ap.parse_args()
    gpu = card()
    for size in SIZES:
        for path in REPS:
            out = run(size, path, a.iters)
            out["card"] = gpu
            print(json.dumps(out))


if __name__ == "__main__":
    main()
