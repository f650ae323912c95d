"""conv1's weight gradient at the bench's batch, each form timed alone in a CUDA graph of back-to-back calls
(bench.time_kernel_graph, best of 5 replays), beside its MMA and byte floors:
  * b2rl_conv1_u8_wgrad_partials  -- conv1_taps_conv_wgrad_wgmma_kernel<true>, activations built from the uint8 ring (K1)
  * b2rl_conv1_wgrad_partials     -- conv1_taps_conv_wgrad_wgmma_kernel<false>, activations from the bf16 stacks
Prints the card's name and power limit first.  --phases: the clock64 probe (b2rl_conv1_set_phase_clocks) of the two taps
kernels -- cycles per k-block of each role.
Usage: python scripts/conv1_wgrad_time.py [--batch 512] [--iters 50] [--phases]"""
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
from deeprl_b200.network.nature_tc import RingFrames  # noqa: E402

PEAK, HBM = 989e12, 3.35e12          # H100 SXM data sheet: dense bf16 FLOP/s, HBM3 bytes/s
CLK = ["CTA run", "producer: wait for free stages", "converters: wait for a free stage", "converters: wait for pixels",
       "converters: convert", "MMA: wait for a full stage", "MMA: issue + retire-one wait", "", "", "", "", "k-blocks"]

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
rows = B * 441
gen = torch.Generator(device=dev).manual_seed(0)
ring = torch.randint(0, 256, (a.capacity, 84 * 84), dtype=torch.uint8, device=dev, generator=gen)
idx = torch.randint(3, a.capacity - 1, (B,), device=dev, generator=gen)
s = RingFrames(ring, idx, -3, 84 * 84, 84, 4)
x0m = s.materialize().permute(0, 2, 3, 1).reshape(rows, 64).contiguous()
g1 = torch.randn((rows, 32), generator=gen, device=dev).to(torch.bfloat16)
sms = torch.cuda.get_device_properties(0).multi_processor_count
bufs = {name: torch.empty((sms, 32, 256), device=dev) for name in ("ring", "bf16")}
n = ctypes.c_int32(0)


def ring_form():
    _lib.call("b2rl_conv1_u8_wgrad_partials", *s.args(), _lib.ptr(g1), 32, _lib.ptr(bufs["ring"]), ctypes.byref(n), _lib.stream())


def bf16_form():
    _lib.call("b2rl_conv1_wgrad_partials", _lib.ptr(x0m), rows, 21, _lib.ptr(g1), 32, _lib.ptr(bufs["bf16"]), ctypes.byref(n),
              _lib.stream())


# floors: the useful MMAs (2 rows x 32 x 256 per grid row) and the bytes of four frames per sample (ring) or the bf16
# stacks, plus the output gradient read once
flops = 2 * rows * 32 * 256
bytes_ring = 4 * 84 * 84 * B + rows * 32 * 2
bytes_bf16 = rows * 64 * 2 + rows * 32 * 2
print("# batch %d, %d back-to-back calls per graph, best of 5 replays; floors: MMA %.1f us, bytes %.1f us (ring) / %.1f us "
      "(bf16)" % (B, a.iters, flops / PEAK * 1e6, bytes_ring / HBM * 1e6, bytes_bf16 / HBM * 1e6))
times = {}
for name, fn in (("b2rl_conv1_wgrad_partials (taps kernel, bf16)", bf16_form),
                 ("b2rl_conv1_u8_wgrad_partials (taps kernel, ring)", ring_form)):
    times[name] = bench.time_kernel_graph(fn, iters=a.iters) * 1e3
    print("%-52s %9.2f us" % (name, times[name]))
ring_form()
bf16_form()
torch.cuda.synchronize()
print("# ring and bf16 taps partials bit-identical: %s (%d partials)" % (torch.equal(bufs["ring"][:n.value], bufs["bf16"][:n.value]),
                                                                        n.value))

if a.phases:
    clocks = torch.zeros(len(CLK), dtype=torch.int64, device=dev)
    for name, fn in (("taps kernel, ring", ring_form), ("taps kernel, bf16", bf16_form)):
        fn()
        torch.cuda.synchronize()
        clocks.zero_()
        _lib.call("b2rl_conv1_set_phase_clocks", _lib.ptr(clocks))
        reps = 20
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        _lib.call("b2rl_conv1_set_phase_clocks", None)
        c = clocks.cpu().tolist()
        blocks = c[-1]
        print("# %s: %d launches, %d partials, %.1f k-blocks per CTA, %.0f cycles per CTA run" % (
            name, reps, n.value, blocks / (reps * n.value), c[0] / (reps * n.value)))
        for i in range(1, 7):
            if name.endswith("bf16") and 2 <= i <= 4:
                continue
            # the MMA slots sum both warpgroups
            print("    %-44s %8.0f cycles / k-block" % (CLK[i], c[i] / blocks / (2 if i >= 5 else 1)))
