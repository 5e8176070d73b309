"""Median device time of one ovp_plane_track_frame at 200 and 2048 features (CUDA events on the context's stream around the call, which
ends in a stream synchronise), and beside it the reference CDT's host time for the mesh alone (oracle/_ref/libref_cdt.so).  Prints one
JSON line with the card's name and power limit.  Run on the GPU: python tools/time_plane_track.py"""
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
import torch  # noqa: E402
import plane_track_reference as ref  # noqa: E402
from ov_plane_b200 import api, vio_sim  # noqa: E402


def frames(n, k, seed):
    """k frames of n features that all triangulate from the second frame on: points at 3-6 m seen from a sideways-moving camera"""
    rng = np.random.RandomState(seed)
    P = np.c_[rng.uniform(-3, 3, n), rng.uniform(-2, 2, n), rng.uniform(3, 6, n)]
    out = []
    for j in range(k):
        px = 0.05 * j
        uvn = ((P[:, :2] - [px, 0.0]) / P[:, 2:3]).astype(np.float32)
        uv = (uvn * 458.0 + [376.0, 240.0]).astype(np.float32)
        out.append((np.r_[0, 0, 0, 1, px, 0, 0], np.arange(1, n + 1), uv, uvn))
    return out


def time_frames(n, iters=30):
    ctx = api.Context(vio_sim.state_options(), device=0, max_state=64, max_meas_rows=256)
    ctx.plane_track_set_options(dict(api.PLANE_TRACK_DEFAULTS, feat_init_min_obs=2))
    fr = frames(n, iters + 5, n)
    calib = np.r_[0, 0, 0, 1, 0, 0, 0.0]
    stream = torch.cuda.ExternalStream(ctx.lib.ovp_stream(ctx.h))
    ms = []
    for j, (pose, fid, uv, uvn) in enumerate(fr):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        ctx.plane_track_frame(pose, calib, fid, uv, uvn)
        e1.record(stream)
        e1.synchronize()
        if j >= 5:  # warm-up, and the first frames before every feature has triangulated
            ms.append(e0.elapsed_time(e1))
    tri, _ = ctx.plane_track_mesh()
    ctx.close()
    uv = fr[-1][2]
    t_cdt = []
    for _ in range(iters):
        t0 = time.perf_counter()
        ref.cdt_triangulate(uv)
        t_cdt.append((time.perf_counter() - t0) * 1e3)
    return dict(n=n, triangles=int(len(tri)), device_ms_median=float(np.median(ms)), device_ms_min=float(np.min(ms)),
                ref_cdt_host_ms_median=float(np.median(t_cdt)))


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=q, results=[time_frames(200), time_frames(2048)])))


if __name__ == "__main__":
    main()
