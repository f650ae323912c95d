"""Run a few EAGER gradient updates of the bench workload (same kernels as the captured graph) for ncu."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import deeprl_b200 as rl  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--updates", type=int, default=3)
ap.add_argument("--workload", default="dqn")
ap.add_argument("--capacity", type=int, default=200_000)
ap.add_argument("--replay", default="async")
a = ap.parse_args()
rl.select_device(0)
rl.Config.COMPUTE_DTYPE = torch.bfloat16
bench.CAP = a.capacity
learner = bench.build_learner(rl, a.workload, torch.device("cuda", 0), 0, 1, prefetch=(a.replay == "async"))
learner.refresh_packed()                             # as capture() does: the target operands are otherwise packed at sync only
for _ in range(2):                                     # warm-up (cuDNN plan selection)
    learner._main(), learner._opt()
torch.cuda.synchronize()
torch.cuda.nvtx.range_push("timed_updates")
for _ in range(a.updates):
    learner._main(), learner._opt()
torch.cuda.synchronize()
torch.cuda.nvtx.range_pop()
# the raw uint8 gather variant too
rp = learner.replay
bufs = rp._buffers(bench.B, torch.uint8, "nchw", tag=9)
rp.select(bench.B, bufs["idx"])
rp.gather(bufs["idx"], bench.B, bufs)
torch.cuda.synchronize()
print("done")
