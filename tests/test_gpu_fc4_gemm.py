"""The plain-GEMM kernel of csrc/gemm.cu (dense_gemm_kernel: fc4 of NatureConvBody and the distributional heads) compared
EXACTLY with a float64 reference, in both of its launch modes: persistent CTAs (optionally with an atomic split-K over
blockIdx.z) and cluster split-K, where the CTAs of a thread-block cluster each compute one tile over a slice of K and add
the partials through distributed shared memory.

Exactness by choice of data, as in test_gpu_conv_exact.py: small integers in bf16, so every product is exact in fp32 and,
while sum |a*b| < 2**24, every partial sum in any order is too.  fp32 outputs then equal the float64 reference and bf16
outputs equal ``ref64.float().to(bfloat16)``.  The launcher picks the cluster size from the shape, so the batches 1, 37,
512 and 2048 and the C51 / QR head widths run different cluster sizes of each instantiation; b2rl_gemm_splitk_bf16 sets
it explicitly (1, 2, 4, 8), including K ranges that leave trailing ranks of a cluster without a k-tile.

Gaussian operands check what exactness cannot: two launches, two default forward passes and a graph replay give the same
bits (the cluster sum has a fixed order; the split-K forward it replaces added its partials with fp32 atomics).
The CPU test reads ptxas's report of every instantiation: no spills, no stack frame, no serialized wgmma."""
import ctypes
import os
import re
import shutil
import subprocess
import zlib

import pytest
import torch

gpu = pytest.mark.gpu
F64, BF = torch.float64, torch.bfloat16
EXACT = 2.0 ** 24
SENT = -12345.0
BATCHES = [1, 37, 512, 2048]
HEADS = {"c51": 4 * 51, "qr": 4 * 200}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEMM_CU = os.path.join(ROOT, "deeprl_b200", "csrc", "gemm.cu")
# dense_gemm_kernel<BN, STAGES, TA, TB, EXT>: every instantiation the launcher can reach
DENSE = {"dense_gemm_kernel<%d, %d, %d, %d, %s>" % (bn, st, ta, tb, ext)
         for bn, st in ((32, 6), (64, 6), (128, 4))
         for ta, tb, ext in ((0, 0, "false"), (1, 0, "false"), (0, 0, "true"), (0, 1, "false"), (1, 1, "false"), (0, 1, "true"))
         if bn >= 64 or tb == 0}


# ================================================================================================= CPU: ptxas report
def test_dense_kernels_compile_clean(tmp_path):
    """Each instantiation: 0 bytes stack frame, 0 bytes spilled, and no ptxas note about wgmma serialization or injected
    warpgroup waits (the k-loop keeps one k-tile of MMAs in flight only if the chain is not serialized)."""
    if shutil.which("nvcc") is None or shutil.which("c++filt") is None:
        pytest.skip("nvcc / c++filt not on PATH")
    r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
                        "-o", str(tmp_path / "gemm.cubin"), GEMM_CU], capture_output=True, text=True, timeout=900,
                       cwd=os.path.dirname(GEMM_CU))
    assert r.returncode == 0, r.stderr[-2000:]
    mangled = sorted(set(re.findall(r"_ZN4b2rl17dense_gemm_kernel\w+", r.stderr)))
    out = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.split("\n")
    names = {m: d.split("(")[0].replace("void ", "").replace("b2rl::", "") for m, d in zip(mangled, out)}
    assert set(names.values()) == DENSE, sorted(set(names.values()) ^ DENSE)
    props, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur in names:
            props[names[cur]] = tuple(int(x) for x in m.groups())
            cur = None
    assert set(props) == DENSE
    for k, (stack, st, ld) in props.items():
        assert (stack, st, ld) == (0, 0, 0), "%s: stack %d, spill stores %d, spill loads %d" % (k, stack, st, ld)
    notes = [l for l in r.stderr.splitlines() if re.search(r"\(C75\d\d\)", l) and "dense_gemm_kernel" in l]
    assert not notes, notes[:3]


# ================================================================================================= GPU helpers
@pytest.fixture(scope="module")
def k():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import deeprl_b200 as rl
    from deeprl_b200 import _lib, ops
    from deeprl_b200.network import nature_tc
    rl.select_device(0)
    return rl, _lib, ops, nature_tc


def gen_for(*key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(key).encode()))


def ints(gen, shape, lo, hi):
    return torch.randint(lo, hi + 1, shape, generator=gen, device="cuda").to(BF)


def exact_ok(S, what):
    assert float(S.max()) < EXACT, "%s: test data leaves the exact range (%g)" % (what, float(S.max()))


def bf(x):
    return x.float().to(BF)


def eq(got, want, what):
    assert torch.equal(got, want), "%s: %d elements differ" % (what, int((got != want).sum()))


# ================================================================================================= fc4 forward
@gpu
@pytest.mark.parametrize("splits", [0, 1, 2, 4, 8])
@pytest.mark.parametrize("B", BATCHES)
def test_fc4_forward_exact(k, B, splits):
    """relu(y3 W4^T + b4) in bf16 through b2rl_gemm_splitk_bf16 (cluster size = splits, 0: the launcher's choice) at
    forward_only's BN 64 and at BN 32 up to batch 1024, and through gemm_bf16 (cluster size picked by the launcher)."""
    _, _, ops, _ = k
    gen = gen_for("fwd", B, splits)
    x, w, b = ints(gen, (B, 3136), 0, 3), ints(gen, (512, 3136), -2, 2), ints(gen, (512,), -40, 40).float()
    exact_ok(x.double().abs() @ w.double().abs().t() + b.double().abs(), "fc4")
    want = bf(torch.relu(x.double() @ w.double().t() + b.double()))
    for bn in sorted({64, 32 if B <= 1024 else 64}):
        out = torch.full((B, 512), SENT, dtype=BF, device="cuda")
        ops.gemm_splitk_bf16(x, w, bias=b, relu=True, splits=splits, block_n=bn, out=out)
        torch.cuda.synchronize()
        eq(out, want, "splitk %d, BN %d" % (splits, bn))
    if splits == 0:
        got = ops.gemm_bf16(x, w, bias=b, relu=True, block_n=32 if B <= 1024 else 64)
        torch.cuda.synchronize()
        eq(got, want, "gemm_bf16")


@gpu
@pytest.mark.parametrize("M,N,K,splits,block_n", [(37, 200, 1000, 4, 64), (130, 72, 200, 8, 32), (1, 8, 64, 2, 128),
                                                  (300, 520, 3136, 4, 128), (129, 33, 136, 8, 64)])
def test_cluster_ragged_exact(k, M, N, K, splits, block_n):
    """Ragged M and N, K not a multiple of splits x 64 (the last k-tile partial, trailing ranks of a cluster without a
    k-tile), with and without bias / ReLU, into a wider destination whose columns past N keep the sentinel."""
    _, _, ops, _ = k
    gen = gen_for("ragged", M, N, K, splits, block_n)
    a, b, bias = ints(gen, (M, K), -3, 3), ints(gen, (N, K), -2, 2), ints(gen, (N,), -9, 9).float()
    exact_ok(a.double().abs() @ b.double().abs().t() + 9, "ragged")
    v = a.double() @ b.double().t()
    buf = torch.full((M, N + 24), SENT, dtype=BF, device="cuda")
    ops.gemm_splitk_bf16(a, b, bias=bias, relu=True, splits=splits, block_n=block_n, out=buf[:, :N])
    plain = ops.gemm_splitk_bf16(a, b, splits=splits, block_n=block_n)
    torch.cuda.synchronize()
    eq(buf[:, :N], bf(torch.relu(v + bias.double())), "bias + relu")
    assert bool((buf[:, N:] == bf(torch.tensor(SENT))).all()), "columns past N were written"
    eq(plain, bf(v), "plain")


# ================================================================================================= fc4 backward
@gpu
@pytest.mark.parametrize("B", BATCHES)
def test_fc4_dgrad_and_wgrad_exact(k, B):
    """fc4 dgrad with the backward extras exactly as _backward_fused calls it (ReLU mask of relu(conv3), db3 summed mod 64,
    map 4 onto conv3's 10-grid), and fc4's weight gradient g4^T y3 (both operands MN-major, fp32)."""
    _, lib, ops, _ = k
    gen = gen_for("bwd", B)
    g, w, y3 = ints(gen, (B, 512), -1, 1), ints(gen, (512, 3136), -2, 2), ints(gen, (B, 3136), 0, 3)
    mask = (torch.randint(0, 2, (B, 3136), generator=gen, device="cuda") * 2 - 1).to(BF)
    exact_ok(g.double().abs() @ w.double().abs(), "fc4 dgrad")
    v = torch.where(mask.double() > 0, g.double() @ w.double(), torch.zeros((), dtype=F64, device="cuda"))
    grid = torch.full((B * 100, 64), SENT, dtype=BF, device="cuda")
    want = grid.clone()
    pos = torch.arange(49, device="cuda")
    rows = (torch.arange(B, device="cuda").view(-1, 1) * 100 + (pos // 7) * 10 + pos % 7).view(-1)
    want[rows] = bf(v.view(B * 49, 64))
    db0 = torch.randint(-100, 101, (64,), generator=gen, device="cuda").float()
    db = db0.clone()
    exact_ok(v.abs().sum(0).view(49, 64).sum(0) + 100, "db3")
    e = lib.bwd_epilogue(mask, db, 64, 64)
    lib.call("b2rl_gemm_bwd_bf16", lib.ptr(g), g.stride(0), lib.ptr(w), 1, w.stride(0), lib.ptr(grid), 64, B, 3136, 512, 4, 10,
             7, ctypes.byref(e), 128, lib.stream())
    exact_ok(g.double().abs().t() @ y3.double().abs(), "fc4 wgrad")
    gw = ops.gemm_bf16(g, y3, a_major="mn", b_major="mn", out_dtype=torch.float32, block_n=128)
    torch.cuda.synchronize()
    eq(grid, want, "dgrad")
    assert torch.equal(db.double(), db0.double() + v.sum(0).view(49, 64).sum(0)), "db3"
    assert torch.equal(gw.double(), g.double().t() @ y3.double()), "weight gradient"


# ================================================================================================= distributional heads
@gpu
@pytest.mark.parametrize("head", sorted(HEADS))
@pytest.mark.parametrize("B", BATCHES)
def test_head_gemms_exact(k, B, head):
    """The three GEMMs of _DistHead: logits phi W^T + b (fp32, BN 64), the weight gradient g^T phi accumulated into .grad
    (MN x MN, BN 128) and dphi = relu_mask(g W) with fc4's per-column bias gradient (K x MN, BN 128, dbias_mod 0)."""
    _, lib, ops, _ = k
    AN = HEADS[head]
    ld = (AN + 7) // 8 * 8
    gen = gen_for("head", B, head)
    phi, w, bias = ints(gen, (B, 512), 0, 3), ints(gen, (AN, 512), -2, 2), ints(gen, (AN,), -9, 9).float()
    g = ints(gen, (B, ld), -1, 1)[:, :AN]
    exact_ok(phi.double().abs() @ w.double().abs().t() + 9, head + " logits")
    logits = ops.gemm_bf16(phi, w, bias=bias, out_dtype=torch.float32, block_n=64)
    gw0 = torch.randint(-50, 51, (AN, 512), generator=gen, device="cuda").float()
    gw = gw0.clone()
    exact_ok(g.double().abs().t() @ phi.double().abs() + 50, head + " weight gradient")
    ops.gemm_bf16(g, phi, a_major="mn", b_major="mn", out_dtype=torch.float32, block_n=128, out=gw, accumulate=True)
    gphi = torch.full((B, 512), SENT, dtype=BF, device="cuda")
    colsum = torch.zeros(512, device="cuda")
    v = torch.where(phi.double() > 0, g.double() @ w.double(), torch.zeros((), dtype=F64, device="cuda"))
    exact_ok(g.double().abs() @ w.double().abs(), head + " feature gradient")
    exact_ok(v.abs().sum(0), head + " db4")
    e = lib.bwd_epilogue(phi, colsum, 0, 0)
    lib.call("b2rl_gemm_bwd_bf16", lib.ptr(g), g.stride(0), lib.ptr(w), 1, w.stride(0), lib.ptr(gphi), gphi.stride(0), B, 512,
             AN, 0, 0, 0, ctypes.byref(e), 128, lib.stream())
    torch.cuda.synchronize()
    assert torch.equal(logits.double(), phi.double() @ w.double().t() + bias.double()), "logits"
    assert torch.equal(gw.double(), gw0.double() + g.double().t() @ phi.double()), "weight gradient"
    eq(gphi, bf(v), "feature gradient")
    assert torch.equal(colsum.double(), v.sum(0)), "db4"


# ================================================================================================= same bits every time
@gpu
@pytest.mark.parametrize("B", [37, 512])
def test_launches_repeat_bit_for_bit(k, B):
    """Gaussian operands (sums rounded in fp32): the cluster split-K forward, the auto-sized dgrad and the head GEMMs give the
    same bits in two launches, and the default forward_only (FC4_SPLITS) gives the same features twice."""
    rl, lib, ops, tc = k
    gen = gen_for("repeat", B)
    rn = lambda *s: (torch.randn(s, generator=gen, device="cuda") * 0.3).to(BF)
    x, w, b = rn(B, 3136), rn(512, 3136), torch.randn(512, generator=gen, device="cuda")
    phi, wh = rn(B, 512), rn(800, 512)
    runs = []
    for _ in range(2):
        y = ops.gemm_splitk_bf16(x, w, bias=b, relu=True, splits=4, block_n=64)
        lg = ops.gemm_bf16(phi, wh, out_dtype=torch.float32, block_n=64)
        gw = ops.gemm_bf16(phi, x, a_major="mn", b_major="mn", out_dtype=torch.float32, block_n=128)
        runs.append((y, lg, gw))
    torch.cuda.synchronize()
    for name, p, q in zip(("splitk", "logits", "wgrad"), *runs):
        assert torch.equal(p, q), name
    assert tc.FC4_SPLITS == 0, "the default forward: cluster size picked by the launcher"
    ws = [torch.randn(s, generator=gen, device="cuda") * 0.05 for s in ((32, 4, 8, 8), (64, 32, 4, 4), (64, 64, 3, 3), (512, 3136))]
    packed = tc.pack_weights(*ws, 1.0)
    biases = [torch.randn(n, generator=gen, device="cuda") * 0.1 for n in (32, 64, 64, 512)]
    x0 = (torch.rand((B, 21, 21, 64), generator=gen, device="cuda")).to(BF).permute(0, 3, 1, 2)
    y4a = tc.forward_only(x0, packed, *biases)[0].clone()
    y4b = tc.forward_only(x0, packed, *biases)[0]
    torch.cuda.synchronize()
    assert int((y4a > 0).sum()) > y4a.numel() // 8
    assert torch.equal(y4a, y4b), "forward_only: %d features differ between two calls" % int((y4a != y4b).sum())


@gpu
def test_graph_replay_matches_eager(k):
    """The cluster launches captured in a CUDA graph (fc4 forward, the fc4 dgrad with extras, a head's logits) replay to
    the same bits as the eager calls; the bias gradient, summed with atomics, to within rounding."""
    _, lib, ops, _ = k
    B = 512
    gen = gen_for("graph")
    rn = lambda *s: (torch.randn(s, generator=gen, device="cuda") * 0.3).to(BF)
    x, w, b, g4 = rn(B, 3136), rn(512, 3136), torch.randn(512, generator=gen, device="cuda"), rn(B, 512)
    mask, phi, wh = rn(B, 3136), rn(B, 512), rn(204, 512)
    y, grid = torch.empty((B, 512), dtype=BF, device="cuda"), torch.zeros((B * 100, 64), dtype=BF, device="cuda")
    db = torch.zeros(64, device="cuda")
    lg = torch.empty((B, 204), device="cuda")

    def step():
        ops.gemm_splitk_bf16(x, w, bias=b, relu=True, splits=4, block_n=64, out=y)
        db.zero_()
        e = lib.bwd_epilogue(mask, db, 64, 64)
        lib.call("b2rl_gemm_bwd_bf16", lib.ptr(g4), g4.stride(0), lib.ptr(w), 1, w.stride(0), lib.ptr(grid), 64, B, 3136, 512, 4,
                 10, 7, ctypes.byref(e), 128, lib.stream())
        ops.gemm_bf16(phi, wh, out_dtype=torch.float32, block_n=64, out=lg)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    eager = [t.clone() for t in (y, grid, db, lg)]
    for t in (y, grid, lg):
        t.fill_(0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for name, got, want in zip(("fc4 forward", "dgrad", "logits"), (y, grid, lg), eager[:2] + eager[3:]):
            assert torch.equal(got, want), name
        # (the bias gradient is summed with shared-memory and global fp32 atomics: same value, order-dependent last bits)
        torch.testing.assert_close(db, eager[2], rtol=1e-5, atol=1e-4)
