"""conv2's and conv3's weight gradients with every tap of a k-block in one CTA (csrc/gemm.cu
``conv_taps_wgrad_wgmma_kernel``, entry ``b2rl_conv_taps_wgrad_partials``).

The kernel reads the gradient rows shifted by each tap (one 128-byte-swizzled TMA box of 128 + halo rows per k-block, one
descriptor start per tap) and the activations unshifted.  With integer operands every fp32 sum is exact in any order (see
test_gpu_conv_exact.py), so the summed partials must EQUAL the float64 reference; Gaussian operands at batch 512 bound the
rounding.  Batches 1 and 37 end in a partial k-block (100 and 3 700 rows are not multiples of 128), and at every batch
k-blocks and CTA ranges start and end inside images."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_conv_exact import (BATCHES, CONV2, CONV3, check_partials, draw, exact_ok, gen_for, k,  # noqa: E402,F401
                                 nan_partials, row_wgrad)
from test_epilogue import GEMM_CU  # noqa: E402

gpu = pytest.mark.gpu
BK = 128          # rows of one k-block
LAYERS = {"conv2": CONV2, "conv3": CONV3}


def partition(rows, ctas):
    """Partials the launcher writes: 128-row k-blocks in equal contiguous ranges over at most `ctas` CTAs."""
    blocks = -(-rows // BK)
    per = -(-blocks // min(blocks, ctas))
    return -(-blocks // per)


def operands(layer, B, kind, gen):
    C, n, taps, tx, gw = LAYERS[layer]
    rows = B * gw * gw
    return draw(gen, (rows, C), kind, 0, 7), draw(gen, (rows, n), kind, -1, 1)


def taps_call(k, layer, X, Gr):
    """(partials, count) of b2rl_conv_taps_wgrad_partials into a NaN-filled buffer."""
    C, n, taps, tx, gw = LAYERS[layer]
    buf, cnt = nan_partials(k, n, taps * C), ctypes.c_int32(0)
    k.lib.call("b2rl_conv_taps_wgrad_partials", k.lib.ptr(X), X.shape[0], C, k.lib.ptr(Gr), n, taps, tx, gw, k.lib.ptr(buf),
               ctypes.byref(cnt), k.lib.stream())
    torch.cuda.synchronize()
    return buf, int(cnt.value)


def last_ctas(k):
    n = ctypes.c_int32(0)
    k.lib.call("b2rl_last_grid_ctas", ctypes.byref(n))
    return int(n.value)


@gpu
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("layer", list(LAYERS))
def test_taps_wgrad_exact(k, layer, B):
    """Integer operands: the fp64 sum of the partials equals the reference; the partial count is the partition over one
    CTA per SM and equals the CTAs launched; a second call gives the same bits."""
    _, _, taps, tx, gw = LAYERS[layer]
    X, Gr = operands(layer, B, "int", gen_for("taps_wgrad", layer, B))
    exact_ok(row_wgrad(X.double().abs(), Gr.double().abs(), taps, tx, gw), layer + " wgrad")
    buf, n = taps_call(k, layer, X, Gr)
    assert n == partition(B * gw * gw, k.sms) == last_ctas(k), (n, last_ctas(k))
    check_partials(k, buf, n, row_wgrad(X.double(), Gr.double(), taps, tx, gw), "%s taps wgrad B=%d" % (layer, B))
    again, n2 = taps_call(k, layer, X, Gr)
    assert n2 == n and torch.equal(again[:n], buf[:n]), "two calls differ"


@gpu
@pytest.mark.parametrize("layer", list(LAYERS))
def test_taps_wgrad_gaussian(k, layer):
    """Batch 512, Gaussian operands: within 1e-5 normwise of float64, bit-identical across calls."""
    _, _, taps, tx, gw = LAYERS[layer]
    X, Gr = operands(layer, 512, "gauss", gen_for("taps_wgrad", layer, "gauss"))
    buf, n = taps_call(k, layer, X, Gr)
    check_partials(k, buf, n, row_wgrad(X.double(), Gr.double(), taps, tx, gw), "%s taps wgrad" % layer, kind="gauss")
    again, _ = taps_call(k, layer, X, Gr)
    assert torch.equal(again[:n], buf[:n])


@gpu
@pytest.mark.parametrize("budget", [8, 16, 32])
@pytest.mark.parametrize("layer", list(LAYERS))
def test_taps_wgrad_budget(k, layer, budget):
    """Under a CTA budget the grid stays within it and writes one partial per CTA; the sum is still exact."""
    _, _, taps, tx, gw = LAYERS[layer]
    X, Gr = operands(layer, 512, "int", gen_for("taps_wgrad", layer, "budget"))
    with k.tc._cta_budget(budget):
        buf, n = taps_call(k, layer, X, Gr)
        ctas = last_ctas(k)
    assert n == ctas == partition(512 * gw * gw, budget) and n <= budget, (n, ctas, budget)
    check_partials(k, buf, n, row_wgrad(X.double(), Gr.double(), taps, tx, gw), "%s budget %d" % (layer, budget))
    _, n_full = taps_call(k, layer, X, Gr)                            # the context cleared the budget
    assert n_full == partition(512 * gw * gw, k.sms) <= k.sms


@gpu
def test_wgrad_partials_routes_every_conv_layer_to_its_taps_kernel(k):
    """nature_tc.wgrad_partials sends conv1 to conv1's taps kernel and conv2 / conv3 to this one (the same bits as the
    entries called directly); the entry refuses other geometries."""
    for layer, (C, n, taps, tx, gw) in LAYERS.items():
        X, Gr = operands(layer, 37, "int", gen_for("taps_wgrad", layer, "routes"))
        want, nw = taps_call(k, layer, X, Gr)
        got, ng = k.tc.wgrad_partials(X, Gr, n, taps, tx, gw)
        assert ng == nw and torch.equal(got[:ng], want[:nw]), layer
    gen = gen_for("taps_wgrad", "conv1")
    x0m, g1 = draw(gen, (37 * 441, 64), "int", 0, 7), draw(gen, (37 * 441, 32), "int", -1, 1)
    buf, cnt = nan_partials(k, 32, 256), ctypes.c_int32(0)
    k.lib.call("b2rl_conv1_wgrad_partials", k.lib.ptr(x0m), x0m.shape[0], 21, k.lib.ptr(g1), 32, k.lib.ptr(buf),
               ctypes.byref(cnt), k.lib.stream())
    got, n1 = k.tc.wgrad_partials(x0m, g1, 32, 4, 2, 21)
    torch.cuda.synchronize()
    assert n1 == cnt.value and torch.equal(got[:n1], buf[:n1])
    X, Gr = operands("conv3", 37, "int", gen)
    with pytest.raises(k.lib.B2RLError, match="taps weight gradient"):
        k.lib.call("b2rl_conv_taps_wgrad_partials", k.lib.ptr(X), X.shape[0], 64, k.lib.ptr(Gr), 64, 4, 2, 10,
                   k.lib.ptr(buf), ctypes.byref(cnt), k.lib.stream())


def test_taps_wgrad_kernels_compile_without_spills(tmp_path):
    """Both instantiations of conv_taps_wgrad_wgmma_kernel: no spill stores, no stack frame."""
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not on PATH")
    cubin = str(tmp_path / "gemm.cubin")
    r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
                        "-o", cubin, GEMM_CU], capture_output=True, text=True, timeout=900, cwd=os.path.dirname(GEMM_CU))
    assert r.returncode == 0, r.stderr[-2000:]
    found = re.findall(r"Function properties for \S*conv_taps_wgrad_wgmma_kernelILi(\d+)E\S*\n"
                       r".*?(\d+) bytes stack frame, (\d+) bytes spill stores", r.stderr)
    assert sorted(f[0] for f in found) == ["128", "64"], found
    for c, stack, spills in found:
        assert (int(stack), int(spills)) == (0, 0), (c, stack, spills)
