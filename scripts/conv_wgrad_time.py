"""conv2's and conv3's weight gradients at the bench's batch, each entry timed alone in a CUDA graph of back-to-back calls
(bench.time_kernel_graph, best of 5 replays), with the full grid and with the side branch's CTA budget:
  * b2rl_conv_wgrad_partials       -- conv_wgrad_wgmma_kernel: 64-row k-tiles, one CTA per 128-column group of taps
  * b2rl_conv_taps_wgrad_partials  -- conv_taps_wgrad_wgmma_kernel: 128-row k-blocks, every tap in one CTA
beside the MMA floor on the SMs the launch may use (dense bf16 data-sheet rate x SMs / all SMs) and the share of it reached.
Prints the card's name, power limit and clocks first.  --phases: the clock64 probe (b2rl_conv1_set_phase_clocks) of the
taps kernel -- cycles per k-block of each role.
Usage: python scripts/conv_wgrad_time.py [--batch 512] [--iters 50] [--budgets 0,32] [--phases]"""
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
from deeprl_b200.network import nature_tc  # noqa: E402

PEAK = 989e12                        # H100 SXM data sheet: dense bf16 FLOP/s
CLK = ["CTA run", "producer: wait for a free stage", "", "", "", "MMA: wait for a full stage", "MMA: issue + retire-one wait",
       "", "", "", "", "k-blocks"]
LAYERS = {"conv3": (64, 64, 9, 3, 10), "conv2": (128, 64, 4, 2, 10)}     # C, n_out, taps, taps_x, grid_w

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=512)
ap.add_argument("--iters", type=int, default=50)
ap.add_argument("--budgets", default="0,32", help="CTA budgets (0: full grid)")
ap.add_argument("--phases", action="store_true", help="also print the per-role cycles of the clock64 probe")
a = ap.parse_args()
rl.select_device(0)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True)
print("# card: %s (%s)" % (torch.cuda.get_device_name(0), q.stdout.strip() or "nvidia-smi: " + q.stderr.strip()))
dev = torch.device("cuda", 0)
SMS = torch.cuda.get_device_properties(dev).multi_processor_count
gen = torch.Generator(device=dev).manual_seed(0)
n = ctypes.c_int32(0)


def entry(name, X, G, geo, buf):
    C, n_out, taps, tx, gw = geo
    return lambda: _lib.call(name, _lib.ptr(X), X.shape[0], C, _lib.ptr(G), n_out, taps, tx, gw, _lib.ptr(buf), ctypes.byref(n),
                             _lib.stream())


print("# batch %d, %d back-to-back calls per graph, best of 5 replays; floor = MMA FLOP / (%.0f TFLOP/s x SMs usable / %d)"
      % (a.batch, a.iters, PEAK / 1e12, SMS))
print("%-6s %-32s %8s %10s %10s %8s %8s" % ("layer", "entry", "budget", "us", "floor us", "share", "CTAs"))
news = {}
for layer, geo in LAYERS.items():
    C, n_out, taps, tx, gw = geo
    rows = a.batch * gw * gw
    X = (torch.randn((rows, C), generator=gen, device=dev) * 0.1).relu_().to(torch.bfloat16)
    G = (torch.randn((rows, n_out), generator=gen, device=dev) * 0.1).to(torch.bfloat16)
    flops = 2 * rows * n_out * taps * C
    bufs, cnt = {}, {}
    for budget in [int(x) for x in a.budgets.split(",")]:
        usable = budget if 0 < budget < SMS else SMS
        floor = flops / (PEAK * usable / SMS) * 1e6
        for name in ("b2rl_conv_wgrad_partials", "b2rl_conv_taps_wgrad_partials"):
            buf = bufs.setdefault(name, torch.empty((SMS, n_out, taps * C), device=dev))
            fn = entry(name, X, G, geo, buf)
            with nature_tc._cta_budget(budget):
                t = bench.time_kernel_graph(fn, iters=a.iters) * 1e3
                fn()
            ctas = ctypes.c_int32(0)
            _lib.call("b2rl_last_grid_ctas", ctypes.byref(ctas))
            torch.cuda.synchronize()
            cnt[name] = n.value
            print("%-6s %-32s %8s %10.2f %10.2f %7.0f%% %8d" % (layer, name, budget or "full", t, floor, 100 * floor / t,
                                                                ctas.value))
            if name.startswith("b2rl_conv_taps"):
                news[(layer, budget)] = (fn, n.value)
        old, new = (bufs[k][:cnt[k]].double().sum(0) for k in ("b2rl_conv_wgrad_partials", "b2rl_conv_taps_wgrad_partials"))
        print("# %s, budget %s: the two entries' summed partials differ by %.1e normwise" % (
            layer, budget or "full", float((new - old).norm() / old.norm())))

if a.phases:
    clocks = torch.zeros(len(CLK), dtype=torch.int64, device=dev)
    for (layer, budget), (fn, parts) in news.items():
        reps = 20
        with nature_tc._cta_budget(budget):
            fn()
            torch.cuda.synchronize()
            clocks.zero_()
            _lib.call("b2rl_conv1_set_phase_clocks", _lib.ptr(clocks))
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
            _lib.call("b2rl_conv1_set_phase_clocks", None)
        c = clocks.cpu().tolist()
        blocks = c[-1]
        wgs = 3 if layer == "conv3" else 2                               # the MMA slots sum every MMA warpgroup
        print("# %s taps kernel, budget %s: %d launches, %d partials, %.1f k-blocks per CTA, %.0f cycles per CTA run" % (
            layer, budget or "full", reps, parts, blocks / (reps * parts), c[0] / (reps * parts)))
        for i in (1, 5, 6):
            print("    %-44s %8.0f cycles / k-block" % (CLK[i], c[i] / blocks / (wgs if i >= 5 else 1)))
