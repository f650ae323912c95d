"""Where the DQN update's backward pass loses time to the weight gradients beside it, and the side-branch CTA budget
(``nature_tc.SIDE_CTAS``, ``b2rl_set_cta_budget``) that keeps them off the dgrad chain's SMs.

1. Alone: each backward kernel at the bench's batch, timed in a CUDA graph of back-to-back launches
   (bench.time_kernel_graph, best of 5 replays), with its full grid and with each budget of the sweep; CTAs from
   b2rl_last_grid_ctas; work in SM-us = alone time x CTAs.
2. In the update: the captured DQN update (async replay) with timing events in the graph (learner.StepTrace), mean of the
   replays: the intervals of the dgrad chain (head_bwd -> d_fc4 -> d_conv3 -> d_conv2), where each weight gradient on
   the side branch ends (w_fc4 / w_conv3 / w_conv2 / w_conv1 marks), kernel A (w_conv1 -> reduce) -- once per side budget
   of the sweep (0: full grids, the schedule without a budget) and once with B2RL_SINGLE_STREAM=1 (no side branch).
3. The back-to-back replay period of the same update graphs WITHOUT event nodes, the sweep alternated --rounds times.

Prints the card's name, power limit and clocks first.
Usage: python scripts/bwd_sm_budget.py [--sweep 0,16,24,32,40,48] [--replays 40] [--rounds 2]"""
import argparse
import ctypes
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import deeprl_b200 as rl  # noqa: E402
from deeprl_b200 import _lib  # noqa: E402
from deeprl_b200.learner import StepTrace  # noqa: E402
from deeprl_b200.network import nature_tc  # noqa: E402
from deeprl_b200.network.nature_tc import RingFrames  # noqa: E402
from deeprl_b200.ops import gemm_bf16  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=512)
ap.add_argument("--sweep", default="0,16,24,32,40,48", help="side-branch CTA budgets (0: full grids)")
ap.add_argument("--replays", type=int, default=40)
ap.add_argument("--rounds", type=int, default=2)
ap.add_argument("--iters", type=int, default=50)
ap.add_argument("--capacity", type=int, default=200_000)
a = ap.parse_args()
sweep = [int(x) for x in a.sweep.split(",")]
bench.CAP = a.capacity
rl.select_device(0)
rl.Config.COMPUTE_DTYPE = torch.bfloat16
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True)
print("# card: %s (%s)" % (torch.cuda.get_device_name(0), q.stdout.strip() or "nvidia-smi: " + q.stderr.strip()))
dev = torch.device("cuda", 0)
SMS = torch.cuda.get_device_properties(dev).multi_processor_count
B = a.batch


# ---------------------------------------------------------------------------------------------- 1. alone
def alone_table():
    gen = torch.Generator(device=dev).manual_seed(0)
    r = lambda *s: (torch.randn(s, generator=gen, device=dev) * 0.1).to(torch.bfloat16)
    g4, y3c, w4p = r(B, 512), r(B, 3136).relu_(), r(512, 3136)
    y2, x1, g3, g2 = r(B * 100, 64).relu_(), r(B * 100, 128).relu_(), r(B * 100, 64), r(B * 100, 64)
    w3d, w2d = r(64, 576), r(128, 256)
    g3o, g2o, g1o = (torch.zeros(s, dtype=torch.bfloat16, device=dev) for s in ((B * 100, 64), (B * 100, 64), (B * 441, 32)))
    db = torch.zeros(160, device=dev)
    e3, e2, e1 = (_lib.bwd_epilogue(y3c, db[96:], 64, 64), _lib.bwd_epilogue(y2, db[32:96], 64, 0),
                  _lib.bwd_epilogue(x1, db[:32], 32, 32))
    ring = torch.randint(0, 256, (20_000, 84 * 84), dtype=torch.uint8, device=dev, generator=gen)
    rf = RingFrames(ring, torch.randint(3, 20_000 - 1, (B,), device=dev, generator=gen), -3, 84 * 84, 84, 4)
    g1 = r(B * 441, 32)
    kernels = [
        ("fc4 dgrad", "main", lambda: _lib.call("b2rl_gemm_bwd_bf16", _lib.ptr(g4), 512, _lib.ptr(w4p), 1, 3136, _lib.ptr(g3o),
                                                64, B, 3136, 512, 4, 10, 7, ctypes.byref(e3), 128, _lib.stream())),
        ("fc4 wgrad", "side", lambda: gemm_bf16(g4, y3c, a_major="mn", b_major="mn", out_dtype=torch.float32, block_n=128)),
        ("conv3 dgrad", "main", lambda: _lib.call("b2rl_conv_gemm_bwd_bf16", _lib.ptr(g3), B * 100, 64, _lib.ptr(w3d), 64, 9,
                                                  3, 10, _lib.ptr(g2o), 64, 0, 0, 0, ctypes.byref(e2), 64, _lib.stream())),
        ("conv3 wgrad", "side", lambda: nature_tc.wgrad_partials(y2, g3, 64, 9, 3, 10)),
        ("conv2 dgrad", "main", lambda: _lib.call("b2rl_conv_gemm_bwd_bf16", _lib.ptr(g2), B * 100, 64, _lib.ptr(w2d), 128,
                                                  4, 2, 10, _lib.ptr(g1o), 32, 3, 21, 20, ctypes.byref(e1), 128,
                                                  _lib.stream())),
        ("conv2 wgrad", "side", lambda: nature_tc.wgrad_partials(x1, g2, 64, 4, 2, 10)),
        ("conv1 wgrad (ring, never budgeted)", None, lambda: nature_tc.wgrad_partials_ring(rf, g1, 32)),
    ]
    n = ctypes.c_int32(0)
    print("\n## 1. alone: us per launch (CTAs), %d back-to-back launches in a graph, best of 5; SM-us = us x CTAs" % a.iters)
    cols = [0] + [w for w in sweep if w]
    print("%-36s %s" % ("kernel", "  ".join("%20s" % ("full grid" if w == 0 else "side W=%d" % w) for w in cols)))
    side_work = {w: 0.0 for w in cols}
    for name, role, fn in kernels:
        cells = []
        for w in cols if role else [0]:
            budget = 0 if w == 0 else (SMS - w if role == "main" else w)
            with nature_tc._cta_budget(budget):
                t = bench.time_kernel_graph(fn, iters=a.iters) * 1e3
                out = fn()
            _lib.call("b2rl_last_grid_ctas", ctypes.byref(n))
            ctas = out[1] if role is None else n.value            # conv1's launcher reports its CTAs as the partial count
            cells.append("%8.2f (%3d) %6.0f" % (t, ctas, t * ctas))
            if role == "side":
                side_work[w] += t * ctas
        print("%-36s %s" % (name, "  ".join("%20s" % c for c in cells)))
    print("%-36s %s" % ("side branch work, SM-us", "  ".join("%20.0f" % side_work[w] for w in cols)))


# ---------------------------------------------------------------------------------------------- 2./3. in the update
def learner():
    lr = bench.build_learner(rl, "dqn", dev, 0, 1, prefetch=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            lr._main(), lr._opt()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    return lr


def capture(lr, side, traced):
    nature_tc.SIDE_CTAS = side
    tr = nature_tc.TRACE = StepTrace() if traced else None
    g = torch.cuda.CUDAGraph()
    try:
        with torch.cuda.graph(g):
            lr._main(0 if lr.prefetch else None)
            lr._opt()
    finally:
        nature_tc.TRACE = None
    return g, tr


def timeline(g, tr):
    acc = None
    for i in range(a.replays + 5):
        g.replay()
        torch.cuda.synchronize()
        t = np.array([x for _, x in tr.timeline()])
        if i >= 5:
            acc = t if acc is None else acc + t
    return {n: v for (n, _), v in zip(tr.marks, acc / a.replays)}


def period(g, n=200):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g.replay()
    e0.record()
    for _ in range(n):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n


alone_table()
torch.cuda.synchronize()
default_side = nature_tc.SIDE_CTAS
lr = learner()
rows = []
for w in sweep:
    rows.append(("side W=%d" % w if w else "full grids (no budget)", timeline(*capture(lr, w, True))))
os.environ["B2RL_SINGLE_STREAM"] = "1"
lr1 = learner()
del os.environ["B2RL_SINGLE_STREAM"]
assert lr1.plan.single_stream
rows.append(("B2RL_SINGLE_STREAM=1", timeline(*capture(lr1, 0, True))))

print("\n## 2. in the update (event nodes in the graph), mean of %d replays, us" % a.replays)
hdr = ["head_bwd", "->d_fc4", "->d_conv3", "->d_conv2", "d_conv2", "w_fc4", "w_conv3", "w_conv2", "w_conv1", "A", "reduce", "opt"]
print("%-24s %s" % ("schedule", " ".join("%9s" % h for h in hdr)))
for name, m in rows:
    h = m["head_bwd"]
    side = lambda k: "%9.1f" % (m[k] - h) if k in m else "%9s" % "-"
    cells = ["%9.1f" % h, "%9.1f" % (m["d_fc4"] - h), "%9.1f" % (m["d_conv3"] - m["d_fc4"]),
             "%9.1f" % (m["d_conv2"] - m["d_conv3"]), "%9.1f" % (m["d_conv2"] - h), side("w_fc4"), side("w_conv3"),
             side("w_conv2"), side("w_conv1"), "%9.1f" % (m["reduce"] - max(m["w_conv1"], m["d_conv2"])),
             "%9.1f" % (m["reduce"] - h), "%9.1f" % m["opt"]]
    print("%-24s %s" % (name, " ".join(cells)))
print("# head_bwd: us after 'start'; ->x: interval from the previous dgrad mark; d_conv2 / w_* / reduce: us after head_bwd;\n"
      "# A: kernel A (split-K reduce) after the later of w_conv1 and d_conv2; opt: us after 'start'")

print("\n## 3. replay period of the update graph without event nodes, us (200 back-to-back replays per entry)")
graphs = {w: capture(lr, w, False)[0] for w in sweep}
per = {w: [] for w in sweep}
for _ in range(a.rounds):
    for w in sweep:
        per[w].append(period(graphs[w]))
for w in sweep:
    print("%-24s %s" % ("side W=%d" % w if w else "full grids (no budget)", "  ".join("%7.1f" % x for x in per[w])))
nature_tc.SIDE_CTAS = default_side
print("# SMs %d, default side budget %d" % (SMS, default_side))
