"""The paired conv1 forward (``b2rl_conv1_u8_fwd_pair``, ``nature_tc.paired_conv1``): the online network's conv1 on the
states and the target network's conv1 on the next states in ONE launch that reads each sample's five-frame ring window
once (n_step 1: s = idx-3 .. idx, s' = idx-2 .. idx+1).

Its chain adds one k16 step of exact zeros per tap to the products of the single launch, in the same k16 groups and tap
order, so the pair is checked for EQUALITY: against the float64 reference built from the ring's own frames (integer
operands, see test_gpu_conv_exact.py), against two ``b2rl_conv1_u8_fwd`` launches on full-range frames with Gaussian
weights, and in one captured update of the graph learner with and without it."""
import dataclasses
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from deeprl_b200.learner import update_plan  # noqa: E402
from test_gpu_conv_exact import (BATCHES, FRAME_W, HIST, SENT, bf, draw, exact_ok, gen_for, k, k1_case, place,  # noqa: E402,F401
                                 ring_grid, row_conv, sentinel)
from test_epilogue import GEMM_CU, bf16_128_stores  # noqa: E402
from test_learner_plan import BEST, ROWS  # noqa: E402

gpu = pytest.mark.gpu


def pair_call(k, rf, w1f, v1f, b1, c1, x1, z1, history=HIST):
    k.lib.call("b2rl_conv1_u8_fwd_pair", k.lib.ptr(rf.frames), int(rf.frames.shape[0]), k.lib.ptr(rf.idx), rf.first,
               rf.row_bytes, rf.frame_w, rf.batch, history, k.lib.ptr(w1f), k.lib.ptr(v1f), k.lib.ptr(x1), k.lib.ptr(z1),
               x1.stride(0), k.lib.ptr(b1), k.lib.ptr(c1), 1, 1, 20, k.lib.stream())


def single_call(k, rf, w, b, out):
    k.lib.call("b2rl_conv1_u8_fwd", *rf.args(), k.lib.ptr(w), 32, k.lib.ptr(out), out.stride(0), k.lib.ptr(b), 1, 1, 20,
               k.lib.stream())


def next_of(k, rf, step=1):
    return k.tc.RingFrames(rf.frames, rf.idx, rf.first + step, rf.row_bytes, rf.frame_w, rf.history)


def assert_equal(got, want, what):
    assert torch.equal(got, want), "%s: %d of %d elements differ" % (what, int((got != want).sum()), got.numel())


# ================================================================================================= the kernel
@gpu
@pytest.mark.parametrize("B", BATCHES)
def test_pair_exact(k, B):
    """x1 and z1 equal the fp64 reference of conv1 on s and s' read from the ring: duplicate indices, the window's oldest
    frame at ring row 0 and its newest at the last row (k1_case with n_step 1), rows outside the V x V output untouched."""
    gen = gen_for("k1-pair", B)
    rf, x0 = k1_case(k, B, 1, 0, "int", gen)
    x0n = ring_grid(rf.frames, rf.idx, rf.first + 1)
    w1f, v1f = draw(gen, (32, 256), "int", -1, 1), draw(gen, (32, 256), "int", -1, 1)
    b1, c1 = draw(gen, (32,), "int", -20, 20).float(), draw(gen, (32,), "int", -20, 20).float()
    refs = []
    for x, w, b in ((x0, w1f, b1), (x0n, v1f, c1)):
        exact_ok(row_conv(x, w.double().abs(), 4, 2, 21) + b.double().abs(), "paired K1 forward")
        v = row_conv(x, w.double(), 4, 2, 21) + b.double()
        refs.append(bf(place(torch.relu(v), 1, (B * 100, 128), SENT, 21, 20)))
    x1, z1 = sentinel((B * 100, 128)), sentinel((B * 100, 128))
    pair_call(k, rf, w1f, v1f, b1, c1, x1, z1)
    torch.cuda.synchronize()
    assert_equal(x1, refs[0], "online conv1(s), B=%d" % B)
    assert_equal(z1, refs[1], "target conv1(s'), B=%d" % B)


@gpu
def test_pair_equals_two_single_launches(k):
    """Full-range frames (0..255) and Gaussian weights and biases at batch 512: the pair's bits are those of the two
    ``b2rl_conv1_u8_fwd`` launches it replaces."""
    B = 512
    gen = gen_for("k1-pair-gauss")
    rf, _ = k1_case(k, B, 1, 0, "gauss", gen)
    assert int(rf.frames.max()) == 255
    w1f, v1f = draw(gen, (32, 256), "gauss", 0, 0) * 0.01, draw(gen, (32, 256), "gauss", 0, 0) * 0.01
    b1, c1 = torch.randn(32, generator=gen, device="cuda"), torch.randn(32, generator=gen, device="cuda")
    x1, z1, y1, u1 = (sentinel((B * 100, 128)) for _ in range(4))
    pair_call(k, rf, w1f, v1f, b1, c1, x1, z1)
    single_call(k, rf, w1f, b1, y1)
    single_call(k, next_of(k, rf), v1f, c1, u1)
    torch.cuda.synchronize()
    assert bool((x1 > 0).any()) and bool((z1 > 0).any())
    assert_equal(x1, y1, "online conv1(s)")
    assert_equal(z1, u1, "target conv1(s')")


@gpu
def test_pair_refusals(k):
    """The pair serves a state and its next state one ring row later, of the same batch, with history 4 and 84 x 84
    frames: anything else is refused before a launch."""
    gen = gen_for("k1-pair-refuse")
    rf, _ = k1_case(k, 37, 1, 0, "int", gen)
    w = draw(gen, (32, 256), "int", -1, 1)
    b = torch.zeros(32, device="cuda")
    x1, z1 = sentinel((37 * 100, 128)), sentinel((37 * 100, 128))
    with pytest.raises(ValueError, match="one ring row"):
        k.tc.conv1_pair(rf, next_of(k, rf, 3), w, b, w, b)              # n_step 3: the windows are not adjacent
    with pytest.raises(ValueError, match="one ring row"):
        k.tc.conv1_pair(rf, rf, w, b, w, b)
    other = k.tc.RingFrames(rf.frames, rf.idx.clone(), rf.first + 1, rf.row_bytes, rf.frame_w, rf.history)
    with pytest.raises(ValueError, match="same batch"):
        k.tc.conv1_pair(rf, other, w, b, w, b)                           # another index buffer
    with pytest.raises(ValueError, match="RingFrames"):
        k.tc.conv1_pair(rf, rf.materialize(), w, b, w, b)
    with pytest.raises(k.lib.B2RLError, match="4 frames"):
        pair_call(k, rf, w, w, b, b, x1, z1, history=3)
    with pytest.raises(k.lib.B2RLError, match="null pointer"):
        pair_call(k, rf, w, None, b, b, x1, z1)
    with pytest.raises(k.lib.B2RLError, match="distinct"):
        pair_call(k, rf, w, w, b, b, x1, x1)
    with pytest.raises(k.lib.B2RLError, match="both or neither bias"):
        pair_call(k, rf, w, w, b, None, x1, z1)
    torch.cuda.synchronize()
    assert bool((x1.float() == bf(torch.tensor(SENT)).float()).all()) and bool((z1.float() == bf(torch.tensor(SENT)).float()).all())


# ================================================================================================= what the compiler made of it
def test_pair_kernel_has_no_spills_and_stores_128_bit(tmp_path):
    """conv1_pair_wgmma_kernel under the rules test_epilogue.py sets for the slab instantiations: no spills, no stack frame,
    its bf16 epilogue stores packed 16-byte rows (at least BN/16 = 4 STG.E.128 sites), no 64-bit stores, no local memory."""
    if shutil.which("nvcc") is None or shutil.which("cuobjdump") is None:
        pytest.skip("nvcc / cuobjdump not on PATH")
    cubin = str(tmp_path / "gemm.cubin")
    r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
                        "-o", cubin, GEMM_CU], capture_output=True, text=True, timeout=900, cwd=os.path.dirname(GEMM_CU))
    assert r.returncode == 0, r.stderr[-2000:]
    m = re.search(r"Function properties for \S*conv1_pair_wgmma_kernel\S*\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores",
                  r.stderr)
    assert m, "no ptxas report for conv1_pair_wgmma_kernel"
    assert (int(m.group(1)), int(m.group(2))) == (0, 0), m.group(0)
    sass = subprocess.run(["cuobjdump", "-sass", "-fun", "_ZN4b2rl23conv1_pair_wgmma_kernelE14CUtensorMap_stS0_S0_S0_NS_10SlabParamsE",
                           cubin], capture_output=True, text=True, check=True).stdout
    assert bf16_128_stores(sass) >= 64 // 16
    assert not re.search(r"\bSTG\.E\.64\s", sass)
    assert not re.search(r"\b(LDL|STL)\b", sass)


# ================================================================================================= the plan
@pytest.mark.parametrize("case,args,ring,head,forward,prefetch,join", ROWS, ids=[r[0] for r in ROWS])
def test_plan_conv1(case, args, ring, head, forward, prefetch, join):
    """The learner pairs conv1 exactly when conv1 reads the ring, the forward is not the dual launch and both bodies are
    wgmma bodies (every row of the plan table has n_step 1)."""
    p = update_plan(**{**BEST, **args})
    assert p.conv1 == ("pair" if ring and forward != "dual" else "separate")
    if p.conv1 == "pair":
        assert update_plan(**{**BEST, **args, "n_step": 3}).conv1 == "separate"
        assert update_plan(**{**BEST, **args, "dual_body": False}).conv1 == "separate"
        q = update_plan(**{**BEST, **args, "n_step": 3})
        assert (q.ring, q.head, q.forward, q.prefetch, q.join) == (p.ring, p.head, p.forward, p.prefetch, p.join)


# ================================================================================================= the update
@pytest.fixture
def small(monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import bench
    import deeprl_b200 as rl
    from deeprl_b200.network import nature_tc
    rl.select_device(0)
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    monkeypatch.setattr(bench, "CAP", 2048)
    monkeypatch.setattr(nature_tc, "FC4_SPLITS", 1)                    # one fc4 GEMM: a deterministic forward
    return bench, rl


@gpu
@pytest.mark.parametrize("prefetch", [True, False], ids=["async", "sync"])
def test_captured_update_with_and_without_pair(small, monkeypatch, prefetch):
    """One captured DQN update with the paired conv1 and one with the two single launches, from identical parameters,
    ring and batch: bit-identical online q, target q and loss."""
    from test_gpu_k1_async import bufs, copy_model
    from deeprl_b200 import learner as L
    from deeprl_b200.network import nature_tc
    bench, rl = small
    a = bench.build_learner(rl, "dqn", torch.device("cuda", 0), 0, 1, prefetch=prefetch)
    b = bench.build_learner(rl, "dqn", torch.device("cuda", 0), 0, 1, prefetch=prefetch)
    assert a.plan.conv1 == "pair"
    b._plan = dataclasses.replace(b.plan, conv1="separate")
    seen, pairs = [], []
    loss_fn, pair_fn = L.ops.dqn_loss_fused, nature_tc.conv1_pair

    def spy_loss(q, q_next, *args, **kw):
        seen.append((q, q_next))
        return loss_fn(q, q_next, *args, **kw)

    def spy_pair(*args):
        pairs.append(1)
        return pair_fn(*args)

    monkeypatch.setattr(L.ops, "dqn_loss_fused", spy_loss)
    monkeypatch.setattr(nature_tc, "conv1_pair", spy_pair)
    graphs = 2 if prefetch else 1                                       # async replay: one graph per buffer parity
    a.capture(warmup=3)
    qa = seen[-graphs:][a._parity if prefetch else 0]                  # the loss inputs of the graph a.update() replays
    n_pair = len(pairs)
    b.capture(warmup=3)
    qb = seen[-graphs:][b._parity if prefetch else 0]
    assert n_pair > 0 and len(pairs) == n_pair, "the pair runs in the paired learner only"
    copy_model(b, a)
    for name in ("frames", "action", "reward", "mask", "ring_state"):
        getattr(b.replay, name).copy_(getattr(a.replay, name))
    b.d_pack.copy_(a.d_pack)
    if prefetch:
        for p in (0, 1):
            for key, v in bufs(a, p).items():
                bufs(b, p)[key].copy_(v)
        b._parity = a._parity
        qb = seen[-graphs:][b._parity]
    torch.cuda.synchronize()
    a.update(), b.update()
    torch.cuda.synchronize()
    assert torch.equal(qa[0], qb[0]), "online q"
    assert torch.equal(qa[1], qb[1]), "target q"
    assert torch.equal(a.loss, b.loss), (float(a.loss), float(b.loss))
