"""The schedule of the convolution slab kernel (conv_slab_body in csrc/gemm.cu): one MMA warpgroup issues and stages every
tile of its CTA, two epilogue warpgroups finish the tile's 64-row halves side by side, and per half two named barriers hand
the fp32 staging tile over (written / read).

* CPU: gemm.cu compiled for sm_90a.  Every slab instantiation (and the paired conv1 forward) is built for its block size
  (.maxntid 512, or 640 with the K1 converters), splits the register file with one setmaxnreg per role within what the
  launch allocates, and neither spills nor keeps a stack frame.
* GPU: the hand-over at the grid shapes the update runs that test_gpu_conv_exact.py does not: the dgrads on the dgrad
  chain's 100-CTA budget, where a CTA takes 1, 2, 3-4 or 16 tiles, checked exactly against float64 with its helpers; and
  run-to-run determinism of every output the epilogue stores (forward, dual forward, paired conv1, dgrad), across two
  launches and against a CUDA-graph replay."""
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
from test_epilogue import GEMM_CU, PARENT_SPILLS, _demangle  # noqa: E402
from test_gpu_conv_exact import (SENT, assert_bf16_equal, dgrad_case, exact_ok, fwd_call, fwd_operands, gen_for,  # noqa: E402,F401
                                 k, k1_case, sentinel)
from test_gpu_k1_pair import pair_call  # noqa: E402

gpu = pytest.mark.gpu

SLAB_KERNELS = sorted(n for n in PARENT_SPILLS if n.startswith("conv_slab_wgmma_kernel")) + ["conv1_pair_wgmma_kernel"]


def _is_k1(name):
    return name == "conv1_pair_wgmma_kernel" or name.endswith(", true, 2, 2, 1>")


# ================================================================================================= CPU: what the compiler made
@pytest.fixture(scope="module")
def build(tmp_path_factory):
    """(ptxas {kernel: (registers, stack bytes, spill store bytes)}, PTX {kernel: entry text}) of the slab kernels."""
    if shutil.which("nvcc") is None or shutil.which("c++filt") is None:
        pytest.skip("nvcc / c++filt not on PATH")
    d = tmp_path_factory.mktemp("slab")
    r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
                        "-keep", "-keep-dir", str(d), "-o", str(d / "gemm.cubin"), GEMM_CU], capture_output=True, text=True,
                       timeout=900, cwd=os.path.dirname(GEMM_CU))
    assert r.returncode == 0, r.stderr[-2000:]
    props, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores", line)
        if m and cur is not None:
            props[cur] = [int(m.group(1)), int(m.group(2))]
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur in props:
            props[cur] = (int(m.group(1)), *props[cur])
            cur = None
    ptx_files = [f for f in os.listdir(d) if f.endswith(".ptx")]
    assert len(ptx_files) == 1, ptx_files
    ptx = open(d / ptx_files[0]).read()
    entries = {m.group(1): m.start() for m in re.finditer(r"\.entry\s+(\w+)\(", ptx)}
    starts = sorted(entries.values()) + [len(ptx)]
    text = {n: ptx[s:starts[starts.index(s) + 1]] for n, s in entries.items()}
    names = _demangle(sorted(set(props) | set(text)))
    keep = lambda n: names[n] in SLAB_KERNELS
    return ({names[n]: v for n, v in props.items() if keep(n)}, {names[n]: v for n, v in text.items() if keep(n)})


def test_slab_kernels_compiled(build):
    props, ptx = build
    assert set(props) == set(SLAB_KERNELS) and set(ptx) == set(SLAB_KERNELS), sorted(set(SLAB_KERNELS) ^ set(props) ^ set(ptx))


@pytest.mark.parametrize("kernel", SLAB_KERNELS)
def test_block_size_registers_and_spills(build, kernel):
    """512 threads (producer, MMA, two epilogue warpgroups) or 640 (K1: + the converters); the launch allocates
    65536 / threads registers per thread (rounded down to 8), the roles' setmaxnreg shares add up to no more than that over
    the warpgroups, each role sets its share once (the two epilogue warpgroups share one), and nothing spills."""
    props, ptx = build
    regs, stack, spill = props[kernel]
    threads = 640 if _is_k1(kernel) else 512
    m = re.search(r"\.maxntid\s+(\d+),\s*(\d+),\s*(\d+)", ptx[kernel])
    assert m and (int(m.group(1)), int(m.group(2)), int(m.group(3))) == (threads, 1, 1), (kernel, m and m.group(0))
    per_thread = 65536 // threads // 8 * 8
    assert regs == per_thread, "%s: %d registers at launch, setmaxnreg shares assume %d" % (kernel, regs, per_thread)
    assert (stack, spill) == (0, 0), "%s: %d bytes stack frame, %d bytes spill stores" % (kernel, stack, spill)
    sets = re.findall(r"setmaxnreg\.(inc|dec)\.sync\.aligned\.u32\s+(\d+);", ptx[kernel])
    roles = 4 if _is_k1(kernel) else 3
    assert len(sets) == roles, (kernel, sets)
    for kind, n in sets:
        n = int(n)
        assert n % 8 == 0 and 24 <= n <= 256 and (n > per_thread if kind == "inc" else n < per_thread), (kernel, kind, n)
    shares = sorted(int(n) for _, n in sets)
    # the epilogue share counts twice; it is the one .dec that is not the producer's (the smallest)
    dec = sorted(int(n) for kind, n in sets if kind == "dec")
    assert len(dec) == 2, (kernel, sets)
    total = sum(shares) + dec[1]
    assert total <= (threads // 128) * per_thread, "%s: shares %s + one more epilogue %d exceed %d" % (
        kernel, shares, dec[1], (threads // 128) * per_thread)


# ================================================================================================= GPU: budgeted dgrads
@pytest.fixture
def budget(k):
    def set_budget(n):
        k.lib.call("b2rl_set_cta_budget", int(n))
    yield set_budget
    set_budget(0)


@gpu
@pytest.mark.parametrize("B", [1, 37, 256, 300, 512, 2048])
@pytest.mark.parametrize("layer", ["conv3", "conv2"])
def test_dgrad_exact_on_the_chain_budget(k, budget, layer, B):
    """The dgrads as the update launches them beside the weight gradients: on at most 100 CTAs.  B = 1: one tile on one CTA
    (no staging-tile wait at all); 37: one tile per CTA, ragged last tile; 256: two per CTA; 300: two or three; 512: four;
    2048: sixteen, the bias gradient summed over all of them.  Output and bias gradient exact against float64."""
    budget(100)
    c = dgrad_case(k, layer, B, "int", gen_for("dgrad-budget", layer, B))
    n = ctypes.c_int32(0)
    k.lib.call("b2rl_last_grid_ctas", ctypes.byref(n))
    assert n.value == min(100, -(-(B * 100) // 128)), n.value
    exact_ok(c.S, layer)
    exact_ok(c.db_abs, layer + " bias gradient")
    assert_bf16_equal(c.out, c.ref, "%s dgrad B=%d on 100 CTAs" % (layer, B))
    assert torch.equal(c.db.double(), c.db_ref), "%s bias gradient B=%d: max |err| %g" % (
        layer, B, float((c.db.double() - c.db_ref).abs().max()))


# ================================================================================================= GPU: determinism
def _launches(k, B):
    """name -> (launch, output buffers) of every slab instantiation the update runs, on Gaussian data at batch B."""
    gen = gen_for("slab-determinism", B)
    lib, out = k.lib, {}
    for layer in ("conv1", "conv2", "conv3"):
        X, W, b = fwd_operands(layer, B, "gauss", gen)
        o = sentinel(((B * 100, 128) if layer == "conv1" else (B * (49 if layer == "conv3" else 100), 64)))
        out[layer + " forward"] = ((lambda X=X, W=W, b=b, o=o, layer=layer: fwd_call(k, layer, X, W, b, o)), [o])
    X, W, b = fwd_operands("conv3", B, "gauss", gen)
    X2, W2, b2 = fwd_operands("conv3", B, "gauss", gen)
    o, o2 = sentinel((B * 49, 64)), sentinel((B * 49, 64))
    out["conv3 dual forward"] = (lambda X=X, X2=X2, W=W, W2=W2, o=o, o2=o2, b=b, b2=b2: k.tc.conv_gemm_dual(
        X, X2, W, W2, 64, 9, 3, 10, o, o2, b, b2, out_map=2, G=10, V=7, block_n=64), [o, o2])
    rf, _ = k1_case(k, B, 1, 0, "gauss", gen)
    w1f, v1f = (torch.randn((32, 256), generator=gen, device="cuda") * 0.01).to(torch.bfloat16), \
        (torch.randn((32, 256), generator=gen, device="cuda") * 0.01).to(torch.bfloat16)
    b1, c1 = torch.randn(32, generator=gen, device="cuda"), torch.randn(32, generator=gen, device="cuda")
    x1, z1 = sentinel((B * 100, 128)), sentinel((B * 100, 128))
    out["conv1 pair"] = (lambda rf=rf, w1f=w1f, v1f=v1f, b1=b1, c1=c1, x1=x1, z1=z1: pair_call(k, rf, w1f, v1f, b1, c1, x1, z1),
                         [x1, z1])
    for layer, n, taps, tx, bn, cols, rows, omap, G, V, mod, sub_c, mask_c in (
            ("conv3", 64, 9, 3, 64, 64, B * 100, 0, 0, 0, 64, 0, 64), ("conv2", 128, 4, 2, 128, 32, B * 441, 3, 21, 20, 32, 32, 128)):
        g = torch.randn((B * 100, 64), generator=gen, device="cuda").to(torch.bfloat16)
        w = (torch.randn((n, taps * 64), generator=gen, device="cuda") * 0.1).to(torch.bfloat16)
        mask = torch.randn((B * 100, mask_c), generator=gen, device="cuda").to(torch.bfloat16)
        o = sentinel((rows, cols))
        db = torch.zeros(mod, device="cuda")
        e = lib.bwd_epilogue(mask, db, mod, sub_c)

        def call(g=g, w=w, n=n, taps=taps, tx=tx, o=o, cols=cols, omap=omap, G=G, V=V, e=e, bn=bn, keep=(mask, db)):
            # keep: the mask and bias-gradient tensors e points to stay alive as long as the launch
            lib.call("b2rl_conv_gemm_bwd_bf16", lib.ptr(g), B * 100, 64, lib.ptr(w), n, taps, tx, 10, lib.ptr(o), cols, omap, G,
                     V, ctypes.byref(e), bn, lib.stream())
        out[layer + " dgrad"] = (call, [o])
    return out


@gpu
@pytest.mark.parametrize("B", [37, 512])
def test_outputs_are_deterministic(k, B):
    """Each output the slab epilogue stores has the same bits in two eager launches and in a CUDA-graph replay of the same
    launch: no hand-over lets an epilogue warpgroup read a half that is not yet, or no longer, the tile it finishes."""
    for name, (launch, outs) in _launches(k, B).items():
        launch()
        torch.cuda.synchronize()
        first = [o.clone() for o in outs]
        for o in outs:
            o.fill_(SENT)
        launch()
        torch.cuda.synchronize()
        for i, (o, f) in enumerate(zip(outs, first)):
            assert torch.equal(o, f), "%s B=%d output %d: two launches differ in %d elements" % (name, B, i, int((o != f).sum()))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
            launch()
        torch.cuda.current_stream().wait_stream(s)
        for o in outs:
            o.fill_(SENT)
        torch.cuda.synchronize()
        graph.replay()
        torch.cuda.synchronize()
        for i, (o, f) in enumerate(zip(outs, first)):
            assert torch.equal(o, f), "%s B=%d output %d: graph replay differs in %d elements" % (name, B, i, int((o != f).sum()))
