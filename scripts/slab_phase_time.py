"""Every convolution slab launch of the DQN update (conv_slab_body in csrc/gemm.cu) at the bench's batch, each timed alone in
a CUDA graph of back-to-back calls (bench.time_kernel_graph, best of 5 replays), as the update issues it: the paired conv1
forward, the single K1 conv1 forward (BN 32), the dual conv2 and conv3 forwards of the online and target networks, and the
conv3 and conv2 dgrads with their fused epilogues on the dgrad chain's CTA budget (100 CTAs).  Prints the card's name and
power limit first.  --phases: the clock64 probe (b2rl_conv1_set_phase_clocks) of each launch -- cycles per tile of each
role: producer, converters (K1), the MMA warpgroup and the two epilogue warpgroups (per 64-row half).
Usage: python scripts/slab_phase_time.py [--batch 512] [--iters 50] [--budget 100] [--phases]"""
import argparse
import ctypes
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import deeprl_b200 as rl  # noqa: E402
from deeprl_b200 import _lib  # noqa: E402
from deeprl_b200.network import nature_tc as tc  # noqa: E402
from deeprl_b200.network.nature_tc import RingFrames  # noqa: E402

# K1_CLK_* slots of csrc/gemm.cu: (label, divisor: 1 per tile, 2 for the epilogue slots, which sum both warpgroups)
CLK = [("CTA run", 0), ("producer: wait for a free stage", 1), ("converters: wait for a free slab", 1),
       ("converters: wait for pixels", 1), ("converters: convert", 1), ("MMA: wait for the slab", 1),
       ("MMA: chain issue -> retire", 1), ("MMA: wait for a free staging half", 1), ("MMA: accumulator staging", 1),
       ("epilogue: wait for a staged half (per half)", 2), ("epilogue: work (per half)", 2), ("tiles", 0)]

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=512)
ap.add_argument("--iters", type=int, default=50)
ap.add_argument("--capacity", type=int, default=20_000)
ap.add_argument("--budget", type=int, default=100, help="CTA budget of the dgrad launches (0: every SM)")
ap.add_argument("--phases", action="store_true", help="also print the per-role cycles of the clock64 probe")
a = ap.parse_args()
rl.select_device(0)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True)
print("# card: %s (%s)" % (torch.cuda.get_device_name(0), q.stdout.strip() or "nvidia-smi: " + q.stderr.strip()))
B, dev = a.batch, torch.device("cuda", 0)
gen = torch.Generator(device=dev).manual_seed(0)
rnd = lambda *s, scale=0.05: (torch.randn(s, generator=gen, device=dev) * scale).to(torch.bfloat16)
ring = torch.randint(0, 256, (a.capacity, 84 * 84), dtype=torch.uint8, device=dev, generator=gen)
idx = torch.randint(3, a.capacity - 1, (B,), device=dev, generator=gen)
s, s2 = RingFrames(ring, idx, -3, 84 * 84, 84, 4), RingFrames(ring, idx, -2, 84 * 84, 84, 4)
w1f, v1f = rnd(32, 256, scale=0.01), rnd(32, 256, scale=0.01)
b1, c1 = (torch.randn(32, generator=gen, device=dev) for _ in range(2))
x1, z1 = (torch.empty((B * 100, 128), dtype=torch.bfloat16, device=dev) for _ in range(2))
w2f, v2f, w3f, v3f = rnd(64, 512), rnd(64, 512), rnd(64, 576), rnd(64, 576)
b2, c2, b3, c3 = (torch.randn(64, generator=gen, device=dev) for _ in range(4))
y2, z2 = (torch.empty((B * 100, 64), dtype=torch.bfloat16, device=dev) for _ in range(2))
y3, z3 = (torch.empty((B * 49, 64), dtype=torch.bfloat16, device=dev) for _ in range(2))
# dgrad operands: output gradients, dgrad weights, the saved activations as ReLU masks (half of them <= 0)
g3, w3d, w2d = rnd(B * 100, 64), rnd(64, 576), rnd(128, 256)
m2, m1 = rnd(B * 100, 64, scale=1.0), rnd(B * 100, 128, scale=1.0)
g2 = torch.empty((B * 100, 64), dtype=torch.bfloat16, device=dev)
g1 = torch.zeros((B * 441, 32), dtype=torch.bfloat16, device=dev)
db2, db1 = torch.zeros(64, device=dev), torch.zeros(32, device=dev)
e2, e1 = _lib.bwd_epilogue(m2, db2, 64, 0), _lib.bwd_epilogue(m1, db1, 32, 32)


def k1_single():
    _lib.call("b2rl_conv1_u8_fwd", *s.args(), _lib.ptr(w1f), 32, _lib.ptr(x1), x1.stride(0), _lib.ptr(b1), 1, 1, 20, _lib.stream())


def k1_pair():
    _lib.call("b2rl_conv1_u8_fwd_pair", *s.args(), _lib.ptr(w1f), _lib.ptr(v1f), _lib.ptr(x1), _lib.ptr(z1), x1.stride(0),
              _lib.ptr(b1), _lib.ptr(c1), 1, 1, 20, _lib.stream())


def conv2_fwd():
    tc.conv_gemm_dual(x1, z1, w2f, v2f, 64, 4, 2, 10, y2, z2, b2, c2, block_n=64)


def conv3_fwd():
    tc.conv_gemm_dual(y2, z2, w3f, v3f, 64, 9, 3, 10, y3, z3, b3, c3, out_map=2, G=10, V=7, block_n=64)


def budgeted(fn):
    def run():
        _lib.call("b2rl_set_cta_budget", a.budget)
        try:
            fn()
        finally:
            _lib.call("b2rl_set_cta_budget", 0)
    return run


@budgeted
def conv3_dgrad():
    _lib.call("b2rl_conv_gemm_bwd_bf16", _lib.ptr(g3), B * 100, 64, _lib.ptr(w3d), 64, 9, 3, 10, _lib.ptr(g2), 64, 0, 0, 0,
              ctypes.byref(e2), 64, _lib.stream())


@budgeted
def conv2_dgrad():
    _lib.call("b2rl_conv_gemm_bwd_bf16", _lib.ptr(g2), B * 100, 64, _lib.ptr(w2d), 128, 4, 2, 10, _lib.ptr(g1), 32, 3, 21, 20,
              ctypes.byref(e1), 128, _lib.stream())


LAUNCHES = [("conv1 pair forward (K1, BN 64)", k1_pair), ("conv1 single forward (K1, BN 32)", k1_single),
            ("conv2 forward, dual <64,F,F,2,2,2>", conv2_fwd), ("conv3 forward, dual <64,F,F,3,3,1>", conv3_fwd),
            ("conv3 dgrad <64,T,F,3,3,1>", conv3_dgrad), ("conv2 dgrad <128,T,F,2,2,1>", conv2_dgrad)]


def grid_ctas():
    n = ctypes.c_int32(0)
    _lib.call("b2rl_last_grid_ctas", ctypes.byref(n))
    return n.value


print("# batch %d, %d back-to-back calls per graph, best of 5 replays; dgrads on %s CTAs" % (
    B, a.iters, a.budget or "all"))
for name, fn in LAUNCHES:
    fn()
    torch.cuda.synchronize()
    print("%-40s %9.2f us   (%d CTAs)" % (name, bench.time_kernel_graph(fn, iters=a.iters) * 1e3, grid_ctas()))

if a.phases:
    clocks = torch.zeros(len(CLK), dtype=torch.int64, device=dev)
    n = 20
    for name, fn in LAUNCHES:
        fn()
        torch.cuda.synchronize()
        ctas = grid_ctas()
        clocks.zero_()
        _lib.call("b2rl_conv1_set_phase_clocks", _lib.ptr(clocks))
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
        _lib.call("b2rl_conv1_set_phase_clocks", None)
        c = clocks.cpu().tolist()
        tiles = max(c[-1], 1)
        print("# %s: %d launches, %.2f tiles per CTA, %.0f cycles per CTA run, %.0f cycles per tile of the CTA run" % (
            name, n, tiles / (n * ctas), c[0] / (n * ctas), c[0] / tiles))
        for (label, div), v in zip(CLK, c):
            if div and v:
                print("    %-46s %8.0f cycles / tile" % (label, v / tiles / div))
