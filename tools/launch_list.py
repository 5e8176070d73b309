"""Per-launch list of the kernels of one MSCKF + plane update step, from torch.profiler (CUDA activities): every launch in stream
order with its duration, grid and the update it belongs to, then a per-kernel summary.  The step runs eagerly (profiling mode,
no CUDA graph) after a warm-up, so every launch is listed under its own name.  Prints the card name and power limit with the
numbers; `--out DIR` also writes the list as DIR/launch_list.json."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402
from ov_plane_b200 import api, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="cfg3_n512_f600_p8")
ap.add_argument("--steps", type=int, default=3, help="profiled steps; the list shows the last one, the summary averages all")
ap.add_argument("--out", default=None)
a = ap.parse_args()

card = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
S = synth.make_scenario(a.workload, seed=0)
ctx = api.Context(S.options, device=0, max_state=576, max_meas_rows=40000)
ctx.set_chi2_table(synth.chi2_table())
ch = synth.load_scenario_into(ctx, S)
batch = synth.feature_batch(S, ch)
ctx.snapshot()
for _ in range(3):
    ctx.restore()
    ctx.msckf_update(batch, 1.0, 1.0)
ctx.msckf_prepare(batch, 1.0, 1.0)
ctx.set_profiling(1)  # eager launches: no graph, one named kernel per launch
ctx.restore()
ctx.msckf_launch()
ctx.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(a.steps):
        ctx.restore()
        ctx.msckf_launch()
    ctx.synchronize()
ctx.set_profiling(0)
ctx.msckf_finish()

evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
       and "memset" not in e.name.lower()]
evs.sort(key=lambda e: e.time_range.start)
names = [e.name.split("(")[0].replace("void ", "") for e in evs]
# one step = the launches between consecutive restores; the restore is the first kernel of each step
per_step = len(evs) // a.steps
last = list(zip(names, evs))[-per_step:]
rows, upd = [], 0
for n, e in last:
    if n.startswith("init_flags_kernel"):
        upd = 0
    if "feature" in n:
        upd += 1
    rows.append({"kernel": n, "us": e.time_range.elapsed_us(), "update": upd})
print("card, power limit: %s   workload %s, %d launches per step" % (card, a.workload, per_step))
print("%-4s %-34s %10s" % ("upd", "kernel", "us"))
for r in rows:
    print("%-4d %-34s %10.1f" % (r["update"], r["kernel"], r["us"]))
summ = {}
for n, e in zip(names, evs):
    s = summ.setdefault(n, [0, 0.0])
    s[0] += 1
    s[1] += e.time_range.elapsed_us()
print("\nper kernel, per step (%d steps):" % a.steps)
for n, (cnt, us) in sorted(summ.items(), key=lambda kv: -kv[1][1]):
    print("  %-34s launches %5.1f  %9.1f us" % (n, cnt / a.steps, us / a.steps))
print("  %-34s %25.1f us" % ("sum of kernel time", sum(s[1] for s in summ.values()) / a.steps))
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "launch_list.json"), "w") as fh:
        json.dump({"card": card, "workload": a.workload, "last_step": rows,
                   "per_step_us": {n: s[1] / a.steps for n, s in summ.items()}}, fh, indent=1)
ctx.close()
