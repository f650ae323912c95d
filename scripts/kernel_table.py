"""Per-kernel time of the captured bench update: torch.profiler (CUDA activities) over N graph replays of the learner
bench.py times.  Prints one row per kernel -- launches per update, mean us per launch, us per update and share of the
summed kernel time -- and writes the Chrome trace to --out.
Usage: python scripts/kernel_table.py [--workload dqn] [--replay async|sync] [--replays 50] [--out DIR]"""
import argparse
import collections
import os
import re
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import deeprl_b200 as rl  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="dqn")
ap.add_argument("--replay", default="async")
ap.add_argument("--replays", type=int, default=50)
ap.add_argument("--capacity", type=int, default=bench.CAP)
ap.add_argument("--out", default=None, help="directory for the Chrome trace")
a = ap.parse_args()
rl.select_device(0)
rl.Config.COMPUTE_DTYPE = torch.bfloat16
bench.CAP = a.capacity
dev = torch.device("cuda", 0)
learner = bench.build_learner(rl, a.workload, dev, 0, 1, prefetch=(a.replay == "async"))
learner.capture(warmup=3, with_h2d=False)
for _ in range(20):
    learner.update()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(a.replays):
        learner.update()
    torch.cuda.synchronize()
if a.out:
    os.makedirs(a.out, exist_ok=True)
    prof.export_chrome_trace(os.path.join(a.out, "kernels_%s_%s.json" % (a.workload, a.replay)))


def short(name):
    """Kernel name without namespace, return type and argument list; template arguments stay (they name the instance)."""
    name = re.sub(r"^void ", "", name)
    depth, out = 0, []
    for ch in name:                                        # drop the parenthesised argument list at template depth 0
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            break
        out.append(ch)
    return "".join(out).replace("b2rl::", "")


tot = collections.defaultdict(float)
cnt = collections.Counter()
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset")):
        k = short(e.name)
        tot[k] += e.time_range.elapsed_us()
        cnt[k] += 1
if not tot:
    sys.exit("the profiler recorded no kernels of the graph replays")
step_us = sum(tot.values()) / a.replays
print("# %s, replay %s: %d replays, summed kernel time per update %.1f us (kernels overlap on side streams: the "
      "shares are of this sum, not of the wall-clock step)" % (a.workload, a.replay, a.replays, step_us))
print("%-72s %8s %9s %9s %6s" % ("kernel", "per upd", "us/launch", "us/upd", "share"))
for k in sorted(tot, key=lambda k: -tot[k]):
    per = tot[k] / a.replays
    print("%-72s %8.2f %9.2f %9.2f %5.1f%%" % (k[:72], cnt[k] / a.replays, tot[k] / cnt[k], per, 100 * per / step_us))
