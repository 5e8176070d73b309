"""Time SLAM delayed initialisation from raw tracks: one ovp_slam_delayed_init_tracks call against the same work as the three existing entry
points chained from Python (triangulate_features, optimize_plane, slam_delayed_init; ov_plane_b200.slam_init_chain).  The sim config's sizes:
25 new features (max_slam 50), about half of them on the four in-state planes, over an 11-clone and a 30-clone window.  Every call runs on a
fresh context loaded with the same state (outside the timed window): the call leaves _features_SLAM_to_PLANE entries that no call erases, and
they would shrink the work of the next one.  Prints one JSON line per size and path with the median / spread of device time (CUDA events on
the library's stream) and of host wall time (with a synchronise), the host<->device bytes and kernel launches per call, and the card name and
power limit read in the same run.

  python tools/time_slam_init.py [--iters 30]
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
from ov_plane_b200 import slam_init_chain as sic  # noqa: E402

SIZES = {
    "sim_11_clones": dict(n_clones=11, n_planes=4, F=200, m_min=3, m_max=11, plane_frac=0.5, n_slam=0, dtheta=0.05),
    "sim_30_clones": dict(n_clones=30, n_planes=4, F=400, m_min=6, m_max=20, plane_frac=0.5, n_slam=0, dtheta=0.03),
}
N_NEW = 25


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:  # the timing is still reported; the card is then unknown
        return "unknown (%s)" % e


def tracks(S, mk, ch):
    """N_NEW features of the scene: the first half on the in-state planes, the rest without a plane"""
    full = mk(ch)
    on = np.nonzero(full["planeid"] != 0)[0]
    pick = np.sort(np.concatenate([on[:N_NEW // 2], np.nonzero(full["planeid"] == 0)[0][:N_NEW - N_NEW // 2]]))
    mo = full["meas_offset"]
    sel = np.concatenate([np.arange(mo[f], mo[f + 1]) for f in pick])
    return dict(meas_offset=np.concatenate([[0], np.cumsum(np.diff(mo)[pick])]).astype(np.int32), meas_clone=np.ascontiguousarray(full["meas_clone"][sel]),
                uv=np.ascontiguousarray(full["uv"][sel]), uv_norm=np.ascontiguousarray(full["uv_norm"][sel]), featid=full["featid"][pick],
                planeid=full["planeid"][pick])


def run(size, path, iters):
    import torch
    S, mk = pic.tracks_scene(name="small_planes", seed=0, px_noise=0.3, keep_in_state=(1, 2, 3, 4), **SIZES[size])
    chi2 = synth.chi2_table()
    dev, wall, h2d, d2h, launches, n_init, n_ref = [], [], [], [], [], [], []
    for it in range(iters + 2):
        # a fresh context per call: the call writes _features_SLAM_to_PLANE for features that get no landmark, and no call erases those entries
        ctx = api.Context(S.options, device=0, max_state=S.N + 3 * N_NEW + 64, max_meas_rows=60000)
        ctx.set_chi2_table(chi2)
        t = tracks(S, mk, synth.load_scenario_into(ctx, S))
        cnt = np.diff(t["meas_offset"])
        trk = [f for f in range(len(cnt)) if cnt[f] >= 2]
        sel = np.concatenate([np.arange(t["meas_offset"][f], t["meas_offset"][f + 1]) for f in trk])
        ctx.triangulate_features(np.concatenate([[0], np.cumsum(cnt[trk])]).astype(np.int32), t["meas_clone"][sel], t["uv_norm"][sel])  # staging buffer
        stream = torch.cuda.ExternalStream(ctx.stream())
        b0, l0 = ctx.transfer_bytes(), ctx.launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ctx.synchronize()
        w0 = time.perf_counter()
        e0.record(stream)
        if path == "composed":
            r = ctx.slam_delayed_init_tracks(t)
        else:
            r = sic.chain(ctx, t, S.options["sigma_constraint"])
        e1.record(stream)
        ctx.synchronize()
        w1 = time.perf_counter()
        b1, l1 = ctx.transfer_bytes(), ctx.launch_count()
        if it >= 2:  # warm-up: module loading and the first allocations of the process
            dev.append(e0.elapsed_time(e1))
            wall.append(1e3 * (w1 - w0))
            h2d.append(b1[0] - b0[0])
            d2h.append(b1[1] - b0[1])
            launches.append(l1 - l0)
            n_init.append(int((r["new_handles"] >= 0).sum()))
            n_ref.append(int((r["plane_status"] == 1).sum()))
        ctx.close()

    def stat(x):
        x = np.asarray(x)
        return dict(median=float(np.median(x)), p10=float(np.percentile(x, 10)), p90=float(np.percentile(x, 90)))
    return dict(size=size, path=path, iters=iters, device_ms=stat(dev), wall_ms=stat(wall), h2d_bytes=int(np.median(h2d)),
                d2h_bytes=int(np.median(d2h)), launches=int(np.median(launches)), landmarks_initialised=int(np.median(n_init)), features=len(t["featid"]),
                refined=int(np.median(n_ref)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    a = ap.parse_args()
    gpu = card()
    for size in SIZES:
        for path in ("composed", "hand_chain"):
            r = run(size, path, a.iters)
            r["gpu"] = gpu
            print(json.dumps(r))


if __name__ == "__main__":
    main()
