"""conv1's weight gradient with the taps in the MMA rows (csrc/gemm.cu ``conv1_taps_conv_wgrad_wgmma_kernel``): the ring
form ``b2rl_conv1_u8_wgrad_partials`` and the bf16 form ``b2rl_conv1_wgrad_partials``.

The kernel reads the gradient rows shifted by each tap (one 64-byte-swizzled TMA box per 128-row k-block, four descriptor
starts into it) and the activations unshifted.  With integer operands (pixels 0..15, gradients -1..1) every fp32 sum is
exact in any order (see test_gpu_conv_exact.py), so the summed partials must EQUAL the float64 reference; Gaussian
operands at batch 512 bound the rounding.  The two forms share the partition, the k order and the MMA chain, so their
partials must be bit-identical on the same frames.  Batch 1 and 37 end in a partial k-block (441 and 16 317 rows are not
multiples of 128), and at every batch k-blocks and CTA ranges start and end inside images."""
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
from test_gpu_conv_exact import (BATCHES, check_partials, draw, exact_ok, gen_for, k, k1_case, nan_partials,  # noqa: E402,F401
                                 row_wgrad)
from test_epilogue import GEMM_CU  # noqa: E402

gpu = pytest.mark.gpu
BK = 128          # rows of one k-block


def partition(rows, sms):
    """Partials the launcher writes: 128-row k-blocks in equal contiguous ranges over at most one CTA per SM."""
    blocks = -(-rows // BK)
    per = -(-blocks // min(blocks, sms))
    return -(-blocks // per)


def both_forms(k, rf, x0, g1):
    """(partials, count) of the ring form and of the bf16 form on the stacks x0 (float64 grid matrix [rows][64])."""
    lib = k.lib
    rows = x0.shape[0]
    out = []
    for form in ("ring", "bf16"):
        buf = nan_partials(k, 32, 256)
        cnt = ctypes.c_int32(0)
        if form == "ring":
            lib.call("b2rl_conv1_u8_wgrad_partials", *rf.args(), lib.ptr(g1), 32, lib.ptr(buf), ctypes.byref(cnt), lib.stream())
        else:
            x0m = x0.to(torch.bfloat16).contiguous()
            lib.call("b2rl_conv1_wgrad_partials", lib.ptr(x0m), rows, 21, lib.ptr(g1), 32, lib.ptr(buf), ctypes.byref(cnt),
                     lib.stream())
        out.append((buf, int(cnt.value)))
    torch.cuda.synchronize()
    return out


@gpu
@pytest.mark.parametrize("which", [0, 1], ids=["state", "next_state"])
@pytest.mark.parametrize("n_step", [1, 3])
@pytest.mark.parametrize("B", BATCHES)
def test_conv1_wgrad_exact(k, B, n_step, which):
    """Both forms against float64 on the ring's own frames (duplicate indices, stacks at both ends of the ring), the
    partial contract (NaN sentinel intact past n, n <= SMs, n = the partition) and bit-identity between the forms."""
    gen = gen_for("conv1_wgrad", B, n_step, which)
    rf, x0 = k1_case(k, B, n_step, which, "int", gen)
    g1 = draw(gen, (B * 441, 32), "int", -1, 1)
    ref = row_wgrad(x0, g1.double(), 4, 2, 21)
    exact_ok(row_wgrad(x0, g1.double().abs(), 4, 2, 21), "conv1 wgrad")
    (pr, nr), (pb, nb) = both_forms(k, rf, x0, g1)
    assert nr == nb == partition(B * 441, k.sms), (nr, nb)
    check_partials(k, pr, nr, ref, "ring form B=%d n_step=%d" % (B, n_step))
    check_partials(k, pb, nb, ref, "bf16 form B=%d n_step=%d" % (B, n_step))
    assert torch.equal(pr[:nr], pb[:nb]), "the ring and bf16 forms differ"


@gpu
def test_conv1_wgrad_gaussian(k):
    """Batch 512, full-range pixels and Gaussian output gradients: within 1e-5 normwise of float64, both forms the same bits."""
    gen = gen_for("conv1_wgrad", "gauss")
    rf, x0 = k1_case(k, 512, 1, 0, "gauss", gen)
    g1 = draw(gen, (512 * 441, 32), "gauss", 0, 0)
    ref = row_wgrad(x0, g1.double(), 4, 2, 21)
    (pr, nr), (pb, nb) = both_forms(k, rf, x0, g1)
    check_partials(k, pr, nr, ref, "ring form", kind="gauss")
    check_partials(k, pb, nb, ref, "bf16 form", kind="gauss")
    assert torch.equal(pr[:nr], pb[:nb])


@gpu
def test_conv1_wgrad_routes(k):
    """nature_tc.wgrad_partials sends conv1's geometry to the taps kernel (the ring form's bits); both entries refuse an
    n_out other than 32."""
    gen = gen_for("conv1_wgrad", "routes")
    rf, x0 = k1_case(k, 37, 1, 0, "int", gen)
    g1 = draw(gen, (37 * 441, 32), "int", -1, 1)
    x0m = x0.to(torch.bfloat16).contiguous()
    pw, nw = k.tc.wgrad_partials(x0m, g1, 32, 4, 2, 21)
    pg, ng = k.tc.wgrad_partials_ring(rf, g1, 32)
    assert nw == ng and torch.equal(pw[:nw], pg[:ng])
    buf, cnt = nan_partials(k, 64, 256), ctypes.c_int32(0)
    g64 = draw(gen, (37 * 441, 64), "int", -1, 1)
    with pytest.raises(k.lib.B2RLError, match="n_out 32"):
        k.lib.call("b2rl_conv1_u8_wgrad_partials", *rf.args(), k.lib.ptr(g64), 64, k.lib.ptr(buf), ctypes.byref(cnt),
                   k.lib.stream())
    with pytest.raises(k.lib.B2RLError, match="n_out 32"):
        k.lib.call("b2rl_conv1_wgrad_partials", k.lib.ptr(x0m), x0m.shape[0], 21, k.lib.ptr(g64), 64, k.lib.ptr(buf),
                   ctypes.byref(cnt), k.lib.stream())


def test_conv1_wgrad_kernels_compile_without_spills(tmp_path):
    """Both instantiations of conv1_taps_conv_wgrad_wgmma_kernel: no spill stores, no stack frame."""
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not on PATH")
    cubin = str(tmp_path / "gemm.cubin")
    r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
                        "-o", cubin, GEMM_CU], capture_output=True, text=True, timeout=900, cwd=os.path.dirname(GEMM_CU))
    assert r.returncode == 0, r.stderr[-2000:]
    found = re.findall(r"Function properties for \S*conv1_taps_conv_wgrad_wgmma_kernelILb([01])E\S*\n"
                       r".*?(\d+) bytes stack frame, (\d+) bytes spill stores", r.stderr)
    assert sorted(f[0] for f in found) == ["0", "1"], found
    for u8, stack, spills in found:
        assert (int(stack), int(spills)) == (0, 0), (u8, stack, spills)
