"""Time ovp_triangulate_features in each triangulation mode (ovp_set_triangulation_mode: the 3-D or 1-D linear stage, with or without
Gauss-Newton) on 600 and 4000 tracks of 20 measurements over a 110-clone window, 1 px of noise, points 1.5 .. 25 m out.  Prints one JSON
line per size and mode with the median / spread of device time (CUDA events on the library's stream around the call, its copies
included), the features triangulated, the launches per call and the card name and power limit read in the same run.

  python tools/time_triangulation.py [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ov_plane_b200 import api, jpl, synth  # noqa: E402

MODES = {"3d_refine": (0, 1), "3d_linear": (0, 0), "1d_refine": (1, 1), "1d_linear": (1, 0)}
SIZES = (600, 4000)
TRACK = 20


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:  # the timing is still reported; the card is then unknown
        return "unknown (%s)" % e


def tracks(ctx, handles, F, seed=0):
    """F tracks of TRACK consecutive clones ending at a random clone; the point along the track's mean optical axis"""
    cal = np.asarray(ctx.var_get(ctx.handle_calib())[0], dtype=np.float64)
    RC = jpl.quat_2_Rot(cal[:4])
    poses = []
    for h in handles:
        v = np.asarray(ctx.var_get(int(h))[0], dtype=np.float64)
        R = RC @ jpl.quat_2_Rot(v[:4])
        poses.append((R, v[4:7] - R.T @ cal[4:7]))
    rng = np.random.RandomState(seed)
    mc, uvn = [], []
    for _ in range(F):
        a = rng.randint(TRACK - 1, len(handles))
        idx = range(a - TRACK + 1, a + 1)
        d = np.mean([poses[i][0][2] for i in idx], axis=0)
        d = d / np.linalg.norm(d) + 0.1 * rng.randn(3) * np.array([1, 1, 0.2])
        p = np.mean([poses[i][1] for i in idx], axis=0) + d / np.linalg.norm(d) * rng.uniform(1.5, 25.0)
        for i in idx:
            c = poses[i][0] @ (p - poses[i][1])
            uvn.append(c[:2] / c[2] + rng.randn(2) / 458.0)
            mc.append(int(handles[i]))
    mo = np.arange(0, TRACK * F + 1, TRACK, dtype=np.int32)
    return mo, np.array(mc, dtype=np.int32), np.array(uvn, dtype=np.float32)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    gpu = card()
    S = synth.make_scenario("cfg2_n256_f200", seed=5, n_clones=110, F=40)
    ctx = api.Context(S.options, device=0, max_state=S.N + 64, max_meas_rows=4096)
    handles = synth.load_scenario_into(ctx, S)
    stream = torch.cuda.ExternalStream(ctx.stream())
    for F in SIZES:
        mo, mc, uvn = tracks(ctx, handles, F)
        for mode, m in MODES.items():
            ctx.set_triangulation_mode(*m)
            dev, launches = [], []
            for it in range(a.iters + 3):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ctx.synchronize()
                l0 = ctx.launch_count()
                e0.record(stream)
                _, st = ctx.triangulate_features(mo, mc, uvn)
                e1.record(stream)
                ctx.synchronize()
                if it >= 3:  # warm-up: module loading and the staging buffer's first allocation
                    dev.append(e0.elapsed_time(e1))
                    launches.append(ctx.launch_count() - l0)
            x = np.asarray(dev)
            print(json.dumps(dict(tracks=F, track_length=TRACK, mode=mode, iters=a.iters, device_ms=dict(
                median=float(np.median(x)), p10=float(np.percentile(x, 10)), p90=float(np.percentile(x, 90))), triangulated=int(st.sum()),
                launches=int(np.median(launches)), gpu=gpu)))
    ctx.set_triangulation_mode(None)
    ctx.close()


if __name__ == "__main__":
    main()
