"""What the compiler made of the convolution slab kernels' epilogue (slab_epilogue_half in csrc/gemm.cu), read from the
SASS of gemm.cu compiled for sm_90a.

* Loads first: every staged value of one pass (two 16-byte shared-memory loads per row, slab_epi_pass_rows rows) is
  requested before the epilogue's first global store, so that a pass waits for one shared-memory round trip instead of
  one per row.  In these kernels only the epilogue issues 16-byte shared-memory loads (LDS.128) and global stores (STG).
* One store form: the slab kernels store bf16 in whole 16-byte column groups, so every global store is an STG.E.128;
  no scalar bf16 (STG.E.U16) or fp32 (STG.E) store remains."""
import os
import re
import shutil
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_epilogue import GEMM_CU, _demangle  # noqa: E402

SLAB_KERNELS = ["conv_slab_wgmma_kernel<%d, %s, %s, %d, %d, %d>" % k for k in (
    (32, "false", "false", 2, 2, 1), (32, "true", "false", 2, 2, 1), (32, "false", "true", 2, 2, 1),
    (64, "false", "false", 2, 2, 2), (64, "true", "false", 2, 2, 2), (64, "false", "false", 3, 3, 1),
    (64, "true", "false", 3, 3, 1), (128, "false", "false", 2, 2, 1), (128, "true", "false", 2, 2, 1))] + [
    "conv1_pair_wgmma_kernel"]


def pass_rows(kernel):
    """slab_epi_pass_rows<BN, EXT>: BN/16 rows, BN/32 for BN 128 with the mask."""
    if kernel == "conv1_pair_wgmma_kernel":
        return 4
    bn, ext = re.search(r"<(\d+), (true|false),", kernel).groups()
    bn = int(bn)
    return bn // 32 if ext == "true" and bn == 128 else bn // 16


@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    """{kernel: [instruction, ...]} of the slab kernels, predicates stripped."""
    if shutil.which("nvcc") is None or shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("nvcc / cuobjdump / c++filt not on PATH")
    cubin = str(tmp_path_factory.mktemp("slab_sass") / "gemm.cubin")
    r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-o", cubin, GEMM_CU],
                       capture_output=True, text=True, timeout=900, cwd=os.path.dirname(GEMM_CU))
    assert r.returncode == 0, r.stderr[-2000:]
    out, name = {}, None
    for line in subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True, check=True).stdout.splitlines():
        if "Function :" in line:
            name = line.split("Function :")[1].strip()
            out[name] = []
        elif name is not None and line.count("*/") >= 2 and line.strip().startswith("/*"):
            out[name].append(re.sub(r"^@!?U?P\w+\s+", "", line.split("*/")[1].strip()))
    names = _demangle(sorted(out))
    return {names[n]: v for n, v in out.items() if names[n] in SLAB_KERNELS}


def test_every_slab_kernel_found(sass):
    assert set(sass) == set(SLAB_KERNELS), sorted(set(SLAB_KERNELS) ^ set(sass))


@pytest.mark.parametrize("kernel", SLAB_KERNELS)
def test_a_pass_of_loads_before_the_first_store(sass, kernel):
    ins = sass[kernel]
    stores = [i for i, x in enumerate(ins) if x.startswith("STG")]
    assert stores, "%s: no global store" % kernel
    loads = sum(1 for x in ins[:stores[0]] if x.startswith("LDS.128"))
    want = 2 * pass_rows(kernel)
    assert loads >= want, "%s: %d 16-byte shared-memory loads before the first global store, want >= %d" % (kernel, loads, want)


@pytest.mark.parametrize("kernel", SLAB_KERNELS)
def test_one_store_form(sass, kernel):
    forms = sorted({x.split()[0] for x in sass[kernel] if x.startswith("STG")})
    assert forms == ["STG.E.128"], "%s: global store forms %s" % (kernel, forms)
