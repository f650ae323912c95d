"""Isolated time of every plain-GEMM shape the bench update issues (fc4 of NatureConvBody and the distributional heads), each
launch timed alone in a CUDA graph of back-to-back launches (bench.time_kernel_graph), against its MMA floor at the
989 TFLOP/s dense-bf16 data-sheet peak of the H100 SXM.  Prints the card's name and power limit first.
Usage: python scripts/fc4_gemm_time.py [--batch 512] [--iters 50]"""
import argparse
import ctypes
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import deeprl_b200 as rl  # noqa: E402
from deeprl_b200 import _lib, ops  # noqa: E402

PEAK = 989e12

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=512)
ap.add_argument("--iters", type=int, default=50)
ap.add_argument("--sweep", action="store_true", help="also time the fc4 forward at every cluster size and BN")
a = ap.parse_args()
rl.select_device(0)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True)
print("# card: %s (%s)" % (torch.cuda.get_device_name(0), q.stdout.strip() or "nvidia-smi: " + q.stderr.strip()))
B, dev = a.batch, torch.device("cuda", 0)
gen = torch.Generator(device=dev).manual_seed(0)
bf = lambda *s: (torch.randn(s, generator=gen, device=dev) * 0.1).to(torch.bfloat16)
f32 = torch.float32

y3c, w4p, b4 = bf(B, 3136), bf(512, 3136), torch.randn(512, generator=gen, device=dev)
g4 = bf(B, 512)
g3 = torch.zeros((B * 100, 64), dtype=torch.bfloat16, device=dev)
db3 = torch.zeros(64, device=dev)
e3 = _lib.bwd_epilogue(y3c, db3, 64, 64)
acc = torch.empty((B, 512), dtype=f32, device=dev)
y4 = torch.empty((B, 512), dtype=torch.bfloat16, device=dev)
gw4 = torch.empty((512, 3136), dtype=f32, device=dev)


def fc4_three():
    ops.gemm_bf16(y3c, w4p, out_dtype=f32, splits=4, block_n=64, out=acc)
    _lib.call("b2rl_bias_act_f32_to_bf16", _lib.ptr(acc), _lib.ptr(b4), _lib.ptr(y4), B, 512, 1, _lib.stream())


def fc4_dgrad():
    _lib.call("b2rl_gemm_bwd_bf16", _lib.ptr(g4), g4.stride(0), _lib.ptr(w4p), 1, w4p.stride(0), _lib.ptr(g3), 64, B, 3136, 512,
              4, 10, 7, ctypes.byref(e3), 128, _lib.stream())


rows = [  # (name, launches per call, flops, fn)
    ("fc4 forward: zero fill + split-K 4 atomics + bias/ReLU pass", 3, 2 * B * 512 * 3136, fc4_three),
    ("fc4 forward: b2rl_gemm_splitk_bf16, splits 4, BN 64", 1, 2 * B * 512 * 3136,
     lambda: ops.gemm_splitk_bf16(y3c, w4p, bias=b4, relu=True, splits=4, block_n=64, out=y4)),
    ("fc4 forward: b2rl_gemm_splitk_bf16, splits 0 (launcher's), BN 64", 1, 2 * B * 512 * 3136,
     lambda: ops.gemm_splitk_bf16(y3c, w4p, bias=b4, relu=True, splits=0, block_n=64, out=y4)),
    ("fc4 forward: gemm_bf16, BN 32", 1, 2 * B * 512 * 3136,
     lambda: ops.gemm_bf16(y3c, w4p, bias=b4, relu=True, block_n=32, out=y4)),
    ("fc4 dgrad + mask / db3 / map 4, BN 128", 1, 2 * B * 512 * 3136, fc4_dgrad),
    ("fc4 weight gradient, MN x MN, fp32, BN 128", 1, 2 * B * 512 * 3136,
     lambda: ops.gemm_bf16(g4, y3c, a_major="mn", b_major="mn", out_dtype=f32, block_n=128, out=gw4)),
]
for kind, AN in (("C51", 4 * 51), ("QR", 4 * 200)):
    phi, w16, bias = bf(B, 512), bf(AN, 512), torch.randn(AN, generator=gen, device=dev)
    ld = (AN + 7) // 8 * 8
    gv = bf(B, ld)[:, :AN]
    logits = torch.empty((B, AN), dtype=f32, device=dev)
    gw = torch.zeros((AN, 512), dtype=f32, device=dev)
    gphi = torch.empty_like(phi)
    colsum = torch.zeros(512, device=dev)
    e = _lib.bwd_epilogue(phi, colsum, 0, 0)

    def head_dgrad(gv=gv, w16=w16, gphi=gphi, e=e, AN=AN):
        _lib.call("b2rl_gemm_bwd_bf16", _lib.ptr(gv), gv.stride(0), _lib.ptr(w16), 1, w16.stride(0), _lib.ptr(gphi), gphi.stride(0),
                  B, 512, AN, 0, 0, 0, ctypes.byref(e), 128, _lib.stream())

    fl = 2 * B * AN * 512
    rows += [
        ("%s head logits, N %d, fp32 + bias, BN 64" % (kind, AN), 1, fl,
         lambda phi=phi, w16=w16, bias=bias, logits=logits: ops.gemm_bf16(phi, w16, bias=bias, out_dtype=f32, block_n=64, out=logits)),
        ("%s head weight gradient, accumulate, BN 128" % kind, 1, fl,
         lambda gv=gv, phi=phi, gw=gw: ops.gemm_bf16(gv, phi, a_major="mn", b_major="mn", out_dtype=f32, block_n=128, out=gw,
                                                      accumulate=True)),
        ("%s head feature gradient + mask / db4, BN 128" % kind, 1, fl, head_dgrad),
    ]

if a.sweep:
    for bn in (32, 64, 128):
        for S in (1, 2, 4, 8):
            rows.append(("fc4 forward: b2rl_gemm_splitk_bf16, splits %d, BN %d" % (S, bn), 1, 2 * B * 512 * 3136,
                         lambda S=S, bn=bn: ops.gemm_splitk_bf16(y3c, w4p, bias=b4, relu=True, splits=S, block_n=bn, out=y4)))

print("# batch %d, %d back-to-back calls per graph, best of 5 replays" % (B, a.iters))
print("%-62s %8s %9s %9s %7s" % ("GEMM", "launches", "us/call", "floor us", "share"))
for name, n, fl, fn in rows:
    try:
        us = bench.time_kernel_graph(fn, iters=a.iters) * 1e3
    except _lib.B2RLError as e:                # a form this build does not have
        print("%-62s %8d %9s  (%s)" % (name, n, "n/a", str(e)[:60]))
        continue
    floor = fl / PEAK * 1e6
    print("%-62s %8d %9.2f %9.2f %6.1f%%" % (name, n, us, floor, 100 * floor / us))
