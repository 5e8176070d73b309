"""Time plane initialisation from raw tracks: one ovp_plane_init_tracks call against the same work as the four existing entry points chained
from Python (triangulate_features, plane_fitting, optimize_plane, plane_init; ov_plane_b200.plane_init_chain).  Two sizes: the shipped window
(11 clones, 4 new planes of ~25 candidates) and a cfg4-like 30-clone window.  The state is restored outside the timed window after every call
(initialisation adds variables, so the new planes are marginalised and the covariance and values written back).  Prints one JSON line per
size and path with the median / spread of device time (CUDA events on the library's stream) and of host wall time (with a synchronise), the
host<->device bytes and kernel launches per call, and the card name and power limit read in the same run.

  python tools/time_plane_init.py [--iters 30]
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

SIZES = {
    "shipped_11_clones": dict(n_clones=11, n_planes=4, F=200, m_min=3, m_max=11, plane_frac=0.5, n_slam=0, dtheta=0.05),
    "cfg4_30_clones": dict(n_clones=30, n_planes=4, F=400, m_min=6, m_max=20, plane_frac=0.5, n_slam=0, dtheta=0.03),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:  # the timing is still reported; the card is then unknown
        return "unknown (%s)" % e


def run(size, path, iters):
    import torch
    S, mk = pic.tracks_scene(name="small_planes", seed=0, px_noise=0.3, **SIZES[size])
    ctx = api.Context(S.options, device=0, max_state=S.N + 64, max_meas_rows=60000)
    ctx.set_chi2_table(synth.chi2_table())
    ch = synth.load_scenario_into(ctx, S)
    t = mk(ch)
    order0 = ctx.variable_order()
    P0 = ctx.cov()
    vals0 = [ctx.var_get(h) for h in order0]
    stream = torch.cuda.ExternalStream(ctx.stream())
    dev, wall, h2d, d2h, launches, n_init = [], [], [], [], [], []
    for it in range(iters + 2):
        b0, l0 = ctx.transfer_bytes(), ctx.launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ctx.synchronize()
        w0 = time.perf_counter()
        e0.record(stream)
        if path == "composed":
            r = ctx.plane_init_tracks(t, max_msckf_plane=40)
        else:
            r = pic.chain(ctx, t, S.options["sigma_constraint"], max_msckf_plane=40)
        e1.record(stream)
        ctx.synchronize()
        w1 = time.perf_counter()
        b1, l1 = ctx.transfer_bytes(), ctx.launch_count()
        if it >= 2:  # warm-up: allocation of the staging buffers
            dev.append(e0.elapsed_time(e1))
            wall.append(1e3 * (w1 - w0))
            h2d.append(b1[0] - b0[0])
            d2h.append(b1[1] - b0[1])
            launches.append(l1 - l0)
            n_init.append(int((r["plane_status"] == 1).sum()))
        for h in r["new_handles"][r["new_handles"] >= 0]:  # restore, outside the timed window
            ctx.marginalize(int(h))
        ctx.cov_upload(P0)
        for h, (v, f) in zip(order0, vals0):
            ctx.var_set(h, v, f)
    ctx.close()

    def stat(x):
        x = np.asarray(x)
        return dict(median=float(np.median(x)), p10=float(np.percentile(x, 10)), p90=float(np.percentile(x, 90)))
    return dict(size=size, path=path, iters=iters, device_ms=stat(dev), wall_ms=stat(wall), h2d_bytes=int(np.median(h2d)),
                d2h_bytes=int(np.median(d2h)), launches=int(np.median(launches)), planes_initialised=int(np.median(n_init)), features=len(t["featid"]))


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
