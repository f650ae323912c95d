"""The GEMM epilogue of csrc/gemm.cu (epilogue_half): what the compiler made of it, and its bias-gradient sums at the largest
row count per CTA.

* CPU: gemm.cu compiled for sm_90a with ``-Xptxas -v``.  No convolution slab or plain-GEMM instantiation may spill more
  registers than before the row-contiguous epilogue, none may keep a stack frame (the per-chunk transpose-reduce of the
  old epilogue lived in one), and every one must store its epilogue results with 128-bit global stores.
* GPU: the bias gradient is summed per thread over its rows, then over warps and tiles in shared memory, in a different
  order from the float64 reference.  At B = 2048 a CTA of the slab kernel covers about 13 tiles; the check bounds the
  fp32 rounding of those sums by their summation depth, for dbias_mod 0 / 32 / 64."""
import os
import re
import shutil
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEMM_CU = os.path.join(ROOT, "deeprl_b200", "csrc", "gemm.cu")

# spill stores (bytes) per instantiation before the row-contiguous epilogue: the ceiling
PARENT_SPILLS = {
    "conv_slab_wgmma_kernel<128, false, false, 2, 2, 1>": 0,
    "conv_slab_wgmma_kernel<128, true, false, 2, 2, 1>": 0,
    "conv_slab_wgmma_kernel<64, false, false, 3, 3, 1>": 8,
    "conv_slab_wgmma_kernel<64, false, false, 2, 2, 2>": 8,
    "conv_slab_wgmma_kernel<64, true, false, 3, 3, 1>": 0,
    "conv_slab_wgmma_kernel<64, true, false, 2, 2, 2>": 0,
    "conv_slab_wgmma_kernel<32, false, false, 2, 2, 1>": 0,
    "conv_slab_wgmma_kernel<32, true, false, 2, 2, 1>": 0,
    "conv_slab_wgmma_kernel<32, false, true, 2, 2, 1>": 0,
    "gemm_wgmma_kernel<128, 4, false>": 0,
    "gemm_wgmma_kernel<128, 4, true>": 0,
    "gemm_wgmma_kernel<64, 6, false>": 36,
    "gemm_wgmma_kernel<64, 6, true>": 0,
    "gemm_wgmma_kernel<32, 6, false>": 0,
    "gemm_wgmma_kernel<32, 6, true>": 0,
}


def _demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
    return {m: d.split("(")[0].replace("void ", "").replace("b2rl::", "") for m, d in zip(names, out)}


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """(ptxas properties {kernel: (stack bytes, spill store bytes)}, SASS {kernel: text}) of the epilogue kernels."""
    if shutil.which("nvcc") is None or shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("nvcc / cuobjdump / c++filt not on PATH")
    cubin = str(tmp_path_factory.mktemp("epilogue") / "gemm.cubin")
    r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
                        "-o", cubin, GEMM_CU], capture_output=True, text=True, timeout=900, cwd=os.path.dirname(GEMM_CU))
    assert r.returncode == 0, r.stderr[-2000:]
    props, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores", line)
        if m and cur is not None:
            props[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    sass, name = {}, None
    for line in subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True, check=True).stdout.splitlines():
        if "Function :" in line:
            name = line.split("Function :")[1].strip()
            sass[name] = []
        elif name is not None:
            sass[name].append(line)
    names = _demangle(sorted(set(props) | set(sass)))
    keep = lambda n: n.startswith(("conv_slab_wgmma_kernel", "gemm_wgmma_kernel"))
    return ({names[k]: v for k, v in props.items() if keep(names[k])},
            {names[k]: "\n".join(v) for k, v in sass.items() if keep(names[k])})


def test_epilogue_kernels_do_not_spill_more(compiled):
    props, _ = compiled
    assert set(props) == set(PARENT_SPILLS), sorted(set(props) ^ set(PARENT_SPILLS))
    for k, (stack, spill) in props.items():
        assert spill <= PARENT_SPILLS[k], "%s spills %d bytes (before: %d)" % (k, spill, PARENT_SPILLS[k])
        assert stack == 0, "%s keeps a %d-byte stack frame (local memory)" % (k, stack)


def _bn(kernel):
    return int(re.search(r"<(\d+),", kernel).group(1))


def bf16_128_stores(text):
    """STG.E.128 instructions whose data was packed by F2FP.BF16.F32.PACK_AB within the 8 instructions before: the bf16
    epilogue's 16-byte stores."""
    ins = [l.split("*/")[1].strip() for l in text.splitlines() if l.count("*/") >= 2 and l.strip().startswith("/*")]
    return sum(1 for i, x in enumerate(ins)
               if re.search(r"\bSTG\.E\.128\s", x) and any("F2FP.BF16.F32.PACK_AB" in y for y in ins[max(0, i - 8):i]))


def test_epilogue_stores_are_128_bit(compiled):
    """The bf16 epilogue stores the 8 columns of each of a thread's BN/16 rows with one STG.E.128 of packed bf16 pairs: at
    least BN/16 such store sites per instantiation (the pass loop is unrolled).  The narrower stores left are the
    element-wise path of partial column groups (STG.E.U16 for bf16, STG.E for fp32), never 64-bit pairs, and no kernel
    touches local memory."""
    _, sass = compiled
    assert set(sass) == set(PARENT_SPILLS), sorted(set(sass) ^ set(PARENT_SPILLS))
    for k, text in sass.items():
        n = bf16_128_stores(text)
        assert n >= _bn(k) // 16, "%s: %d 128-bit bf16 store sites, want >= %d" % (k, n, _bn(k) // 16)
        assert not re.search(r"\bSTG\.E\.64\s", text), "%s: 64-bit global stores" % k
        assert not re.search(r"\b(LDL|STL)\b", text), "%s: local-memory traffic" % k


# ================================================================================================= GPU
@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import deeprl_b200 as rl
    from deeprl_b200 import _lib
    rl.select_device(0)
    return _lib


@pytest.mark.gpu
@pytest.mark.parametrize("layer,mod", [("conv3", 0), ("conv3", 64), ("conv2", 32), ("fc4", 64)])
def test_bias_gradient_sums_at_batch_2048(lib, layer, mod):
    """B = 2048 with operands whose GEMM values are exact in fp32 but whose bias-gradient sums are not: gradient rows are
    integers 0..3 times 2^-e (e = 0..8 per row), weights integers 0..3, so every dot product is a multiple of 2^-8 below
    2^13 (exact), while the column sums over ~2e5 rows need more than 24 bits.  All values are >= 0, so the float64 sum is
    also the sum of |terms|.  Each value passes through at most D fp32 additions: BN/16 in its thread, the warp fold,
    the shared-memory atomics on its s_dbias slot in its CTA (2 halves x 4 warps per tile, times the columns the fold
    maps onto one slot) and one global atomic per CTA.  So |dbias - ref| <= ((1 + 2^-24)^D - 1) ref.  The test also
    checks that this bound rejects a result scaled by 1 + 1e-3 and one that misses the first 128 rows' contribution."""
    import ctypes
    import math
    B = 2048
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    gen = torch.Generator(device="cuda").manual_seed(2048 + mod + len(layer))
    ints = lambda *s: torch.randint(0, 4, s, generator=gen, device="cuda").double()
    pow2 = torch.tensor([2.0 ** -e for e in range(9)], dtype=torch.float64, device="cuda")         # exact scales
    scaled = lambda r, c: ints(r, c) * pow2[torch.randint(0, 9, (r, 1), generator=gen, device="cuda")]
    if layer == "conv3":
        g, w, mask = scaled(B * 100, 64), ints(64, 576), torch.randn((B * 100, 64), generator=gen, device="cuda")
        out, N, BN, K = torch.empty((B * 100, 64), dtype=torch.bfloat16, device="cuda"), 64, 64, 576
        taps, tx, sub_c = 9, 3, 0
    elif layer == "conv2":
        g, w, mask = scaled(B * 100, 64), ints(128, 256), torch.randn((B * 100, 128), generator=gen, device="cuda")
        out, N, BN, K = torch.zeros((B * 441, 32), dtype=torch.bfloat16, device="cuda"), 128, 128, 256
        taps, tx, sub_c = 4, 2, 32
    else:
        g, w, mask = scaled(B, 512), ints(512, 3136), torch.randn((B, 3136), generator=gen, device="cuda")
        out, N, BN, K = torch.zeros((B * 100, 64), dtype=torch.bfloat16, device="cuda"), 3136, 128, 512
        taps, tx, sub_c = 0, 0, 64
    g16, w16, m16 = g.to(torch.bfloat16), w.to(torch.bfloat16), mask.to(torch.bfloat16)
    assert torch.equal(g16.double(), g) and torch.equal(w16.double(), w)
    # float64 GEMM values (dgrad: row r gathers rows r - offset(tap), as row_conv in test_gpu_conv_exact.py)
    if layer == "fc4":
        v = g @ w
    else:
        v = torch.zeros((g.shape[0], w.shape[0]), dtype=torch.float64, device="cuda")
        for t in range(taps):
            s = (t // tx) * 10 + t % tx
            v[s:] += g[:g.shape[0] - s] @ w[:, t * 64:(t + 1) * 64].t()
    assert float(v.max()) < 2.0 ** 13 and torch.equal(v * 256, (v * 256).round())    # exact in fp32
    vm = torch.where(m16.double() > 0, v, torch.zeros_like(v))
    n_idx = N if mod == 0 else mod
    fold = lambda x: x.sum(0).view(-1, n_idx).sum(0)
    ref = fold(vm)
    # the summation depth D of one bias index
    if layer == "fc4":
        tiles = -(-B // 128) * -(-N // BN)
    else:
        tiles = -(-(B * 100) // 128)
    n_cta = min(sms, tiles)
    per_cta = -(-tiles // n_cta)
    D = BN // 16 + 5 + per_cta * 2 * 4 * max(1, BN // n_idx) + n_cta + 1
    tol = (math.expm1(D * math.log1p(2.0 ** -24))) * ref
    db = torch.zeros(128 if mod == 0 and N <= 128 else n_idx, device="cuda")
    e = lib.bwd_epilogue(m16, db, mod, sub_c)
    if layer == "fc4":
        lib.call("b2rl_gemm_bwd_bf16", lib.ptr(g16), g16.stride(0), lib.ptr(w16), 1, w16.stride(0), lib.ptr(out), 64, B, 3136,
                 512, 4, 10, 7, ctypes.byref(e), 128, lib.stream())
    else:
        lib.call("b2rl_conv_gemm_bwd_bf16", lib.ptr(g16), B * 100, 64, lib.ptr(w16), w.shape[0], taps, tx, 10, lib.ptr(out),
                 out.shape[1], 3 if layer == "conv2" else 0, 21 if layer == "conv2" else 0, 20 if layer == "conv2" else 0,
                 ctypes.byref(e), BN, lib.stream())
    torch.cuda.synchronize()
    got = db[:n_idx].double()
    err = (got - ref).abs()
    assert bool((err <= tol).all()), "%s dbias_mod %d: max excess %g (max rel err %g, D %d)" % (
        layer, mod, float((err - tol).max()), float((err / ref).max()), D)
    if mod == 0:
        assert bool((db[n_idx:] == 0).all()), "columns past N must not be touched"
    # the bound is tight enough to see a 1e-3 scale error or one 128-row tile left out
    assert bool(((got * (1 + 1e-3) - ref).abs() > tol).all())
    assert bool(((got - fold(vm[:128]) - ref).abs() > tol).any())
