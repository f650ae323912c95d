"""The paired conv1 forward (b2rl_conv1_u8_fwd_pair: online conv1 on s and target conv1 on s' from one five-frame ring
window) against the two b2rl_conv1_u8_fwd launches it replaces, at the bench's batch: each form timed alone in a CUDA
graph of back-to-back calls (bench.time_kernel_graph, best of 5 replays), beside its HBM and MMA floors.  Prints the card's
name and power limit first.  --phases: the K1 kernels' clock64 probe (b2rl_conv1_set_phase_clocks) -- cycles per tile of
each role (producer, converters, MMA warpgroup, epilogue warpgroups) -- for the single launch and the pair.
Usage: python scripts/conv1_pair_time.py [--batch 512] [--iters 50] [--phases]"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import deeprl_b200 as rl  # noqa: E402
from deeprl_b200 import _lib  # noqa: E402
from deeprl_b200.network.nature_tc import RingFrames  # noqa: E402

PEAK, HBM = 989e12, 3.35e12          # H100 SXM data sheet: dense bf16 FLOP/s, HBM3 bytes/s
CLK = ["CTA run", "producer: wait for a free uint8 stage", "converters: wait for a free slab", "converters: wait for pixels",
       "converters: convert", "MMA: wait for the slab", "MMA: chain issue -> retire", "MMA: wait for a free staging half",
       "MMA: accumulator staging", "epilogue: wait for a staged half (2 warpgroups)",
       "epilogue: work (2 warpgroups)", "tiles"]

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=512)
ap.add_argument("--iters", type=int, default=50)
ap.add_argument("--capacity", type=int, default=20_000)
ap.add_argument("--phases", action="store_true", help="also print the per-role cycles of the clock64 probe")
a = ap.parse_args()
rl.select_device(0)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True)
print("# card: %s (%s)" % (torch.cuda.get_device_name(0), q.stdout.strip() or "nvidia-smi: " + q.stderr.strip()))
B, dev = a.batch, torch.device("cuda", 0)
gen = torch.Generator(device=dev).manual_seed(0)
ring = torch.randint(0, 256, (a.capacity, 84 * 84), dtype=torch.uint8, device=dev, generator=gen)
idx = torch.randint(3, a.capacity - 1, (B,), device=dev, generator=gen)
s, s2 = RingFrames(ring, idx, -3, 84 * 84, 84, 4), RingFrames(ring, idx, -2, 84 * 84, 84, 4)
w1f, v1f = ((torch.randn((32, 256), generator=gen, device=dev) * 0.01).to(torch.bfloat16) for _ in range(2))
b1, c1 = torch.randn(32, generator=gen, device=dev), torch.randn(32, generator=gen, device=dev)
x1, z1 = (torch.empty((B * 100, 128), dtype=torch.bfloat16, device=dev) for _ in range(2))


def single(rf, w, b, out):
    _lib.call("b2rl_conv1_u8_fwd", *rf.args(), _lib.ptr(w), 32, _lib.ptr(out), out.stride(0), _lib.ptr(b), 1, 1, 20, _lib.stream())


def two():
    single(s, w1f, b1, x1)
    single(s2, v1f, c1, z1)


def pair():
    _lib.call("b2rl_conv1_u8_fwd_pair", *s.args(), _lib.ptr(w1f), _lib.ptr(v1f), _lib.ptr(x1), _lib.ptr(z1), x1.stride(0),
              _lib.ptr(b1), _lib.ptr(c1), 1, 1, 20, _lib.stream())


# floors of the pair: the MMAs of the stacked N = 64 chain (5 k16 steps per tap) and the HBM bytes of 5 frames per sample
# read once plus the two bf16 outputs
flops = 2 * B * 441 * 64 * 4 * 80
hbm = 5 * 84 * 84 * B + 2 * B * 400 * 32 * 2
print("# batch %d, %d back-to-back calls per graph, best of 5 replays; pair floors: MMA %.1f us, HBM %.1f us" % (
    B, a.iters, flops / PEAK * 1e6, hbm / HBM * 1e6))
t_two = bench.time_kernel_graph(two, iters=a.iters) * 1e3
t_pair = bench.time_kernel_graph(pair, iters=a.iters) * 1e3
print("%-52s %9.2f us" % ("two b2rl_conv1_u8_fwd launches (s, s')", t_two))
print("%-52s %9.2f us   (%.2fx the two launches)" % ("one b2rl_conv1_u8_fwd_pair launch", t_pair, t_pair / t_two))

if a.phases:
    clocks = torch.zeros(len(CLK), dtype=torch.int64, device=dev)
    for name, fn, launches in (("single b2rl_conv1_u8_fwd (s)", lambda: single(s, w1f, b1, x1), 1), ("pair", pair, 1)):
        fn()
        torch.cuda.synchronize()
        clocks.zero_()
        _lib.call("b2rl_conv1_set_phase_clocks", _lib.ptr(clocks))
        n = 20
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
        _lib.call("b2rl_conv1_set_phase_clocks", None)
        c = clocks.cpu().tolist()
        tiles = c[-1]
        ctas = min(torch.cuda.get_device_properties(0).multi_processor_count, -(-B * 441 // 128))
        print("# %s: %d launches, %.1f tiles per CTA, %.0f cycles per CTA run" % (name, n, tiles / (n * ctas), c[0] / (n * ctas)))
        for i in range(1, len(CLK) - 1):
            print("    %-44s %8.0f cycles / tile" % (CLK[i], c[i] / tiles))
