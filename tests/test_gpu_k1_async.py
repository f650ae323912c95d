"""K1 under async replay: conv1 reads the sampled frame stacks from the uint8 ring while the next batch is prefetched.

The prefetch branch (this update's feeds, the next index draw, the next batch's action / reward / mask) forks after the
batch's last ring read, conv1's weight gradient.  Every batch then sees the ring exactly as the materialising form
(``B2RL_K1=0``: gather into a bf16 batch) sees it.  The tests use a ring of 2 048 transitions, so the 4 rows each update
feeds regularly belong to stacks of the batch that update trains on: a feed that ran before the last read would change
what conv1 reads.

Bit-exactness: fc4's forward runs as one GEMM here (``nature_tc.FC4_SPLITS = 1``) instead of the default split-K with fp32
atomics, so the forward pass, and with it the loss, is deterministic.  The backward pass keeps fp32 atomics (bias
gradients), so parameters are compared within their run-to-run noise and each update starts from copied parameters."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CAP = 2048


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import bench
    import deeprl_b200 as rl
    rl.select_device(0)
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    return bench, rl


@pytest.fixture
def small(env, monkeypatch):
    bench, rl = env
    from deeprl_b200.network import nature_tc
    monkeypatch.setattr(bench, "CAP", CAP)
    monkeypatch.setattr(nature_tc, "FC4_SPLITS", 1)
    return env


def make(env, workload, prefetch=True, k1=True, monkeypatch=None):
    bench, rl = env
    if not k1:
        monkeypatch.setenv("B2RL_K1", "0")
    try:
        return bench.build_learner(rl, workload, torch.device("cuda", 0), 0, 1, prefetch=prefetch)
    finally:
        if not k1:
            monkeypatch.delenv("B2RL_K1")


def copy_model(dst, src):
    """Parameters, optimizer state and target network of ``src`` into ``dst`` (the replay stays ``dst``'s own)."""
    for a, b in ((dst.opt.flat, src.opt.flat), (dst.opt.s1, src.opt.s1), (dst.opt.s2, src.opt.s2),
                 (dst.opt.step_dev, src.opt.step_dev), (dst.opt.scratch, src.opt.scratch), (dst.opt.grad, src.opt.grad)):
        a.copy_(b)
    dst.tgt.load_state_dict(src.tgt.state_dict())
    dst.refresh_packed()
    torch.cuda.synchronize()


def bufs(learner, parity):
    rp = learner.replay
    layout = rp.LAYOUTS["ring" if learner.ring else "s2d"]
    return rp._bufs[(rp.batch_size, torch.bfloat16, layout, parity)]


def stacks_touch(idx, rows, hl, n_step):
    """True if a frame stack (state or next state) of a sample in ``idx`` contains one of ``rows``."""
    lo, hi = idx - (hl - 1), idx + n_step
    return bool(any(((lo <= r) & (r <= hi)).any() for r in rows))


def test_ring_path_selection(small, monkeypatch):
    """Uniform async replay takes K1; prioritized async replay, ``B2RL_K1=0`` and the dual forward keep the gather."""
    from deeprl_b200.learner import GraphedDQNLearner
    assert make(small, "dqn").ring
    assert make(small, "c51").ring and make(small, "qr").ring
    assert make(small, "dqn", prefetch=False).ring
    assert make(small, "per", prefetch=False).ring
    assert not make(small, "per").ring
    assert not make(small, "dqn", k1=False, monkeypatch=monkeypatch).ring
    lr = make(small, "dqn")
    dual = GraphedDQNLearner(lr.net, lr.tgt, lr.opt, lr.replay, feeds_per_update=4, prefetch=True, dual=True,
                             target_sync_every=0)
    assert not dual.ring


@pytest.mark.parametrize("workload", ["dqn", "c51", "qr"])
def test_async_k1_equals_async_gather(small, monkeypatch, workload):
    """10 captured updates of async + K1 against async + gather from identical state: the same ring, cursor, Philox counter,
    indices and scalars after every update, the frames K1 read are the ones the gather materialised, and the loss is
    bit-identical."""
    k1 = make(small, workload)
    mat = make(small, workload, k1=False, monkeypatch=monkeypatch)
    assert k1.ring and not mat.ring and k1.prefetch and mat.prefetch
    k1.capture(warmup=3)
    mat.capture(warmup=3)
    rp_k, rp_m = k1.replay, mat.replay
    hl, n = rp_k.history_length, rp_k.n_step
    hazards = 0
    for step in range(10):
        copy_model(k1, mat)
        parity = k1._parity
        assert mat._parity == parity
        ring_before = rp_k.frames.clone()
        pos = int(rp_k.ring_state[0])
        k1.update(), mat.update()
        torch.cuda.synchronize()
        assert torch.equal(rp_k.frames, rp_m.frames)
        assert torch.equal(rp_k.ring_state, rp_m.ring_state)            # cursor, size and Philox counter
        bk, bm = bufs(k1, parity), bufs(mat, parity)                     # the batch this update trained on
        for key in ("idx", "action", "reward", "mask"):
            assert torch.equal(bk[key], bm[key]), key
            assert torch.equal(bufs(k1, 1 - parity)[key], bufs(mat, 1 - parity)[key]), key     # and the prefetched one
        t = k1._batch[parity]
        for which, ring_x, mat_x in ((0, t.state, mat._batch[parity].state), (1, t.next_state, mat._batch[parity].next_state)):
            read = type(ring_x)(ring_before, ring_x.idx, ring_x.first, ring_x.row_bytes, ring_x.frame_w, ring_x.history)
            assert torch.equal(read.materialize(), mat_x), "the ring before this update's feeds, at the trained indices"
        fed = [(pos + i) % CAP for i in range(k1.feeds)]
        hazards += stacks_touch(bk["idx"].cpu(), fed, hl, n)
        assert torch.equal(k1.loss, mat.loss), "update %d: %r vs %r" % (step, float(k1.loss), float(mat.loss))
        np.testing.assert_allclose(k1.opt.flat.cpu().numpy(), mat.opt.flat.cpu().numpy(), rtol=0, atol=2e-6)
    assert hazards >= 2, "the feeds never overwrote a row of the batch trained on (%d times)" % hazards


@pytest.mark.parametrize("workload", ["dqn", "c51", "qr"])
def test_async_k1_graph_equals_eager(small, workload):
    """Async + K1: the eager ``_main`` / ``_opt`` sequence and the graph replay from identical state give the same loss, the
    same ring and the same prefetched batch."""
    a, b = make(small, workload), make(small, workload)
    assert a.ring and b.ring
    for _ in range(3):
        a._main(), a._opt()
    b.capture(warmup=3)
    for _ in range(3):
        copy_model(a, b)
        for name in ("frames", "action", "reward", "mask", "ring_state"):
            getattr(a.replay, name).copy_(getattr(b.replay, name))
        for p in (0, 1):
            for k, v in bufs(b, p).items():
                bufs(a, p)[k].copy_(v)
        a._parity = b._parity
        torch.cuda.synchronize()
        parity = a._parity
        a._main(), a._opt()
        b.update()
        torch.cuda.synchronize()
        assert torch.equal(a.loss, b.loss)
        np.testing.assert_allclose(a.opt.flat.cpu().numpy(), b.opt.flat.cpu().numpy(), rtol=0, atol=2e-6)
        assert torch.equal(a.replay.frames, b.replay.frames) and torch.equal(a.replay.ring_state, b.replay.ring_state)
        for k in ("idx", "action", "reward", "mask"):
            assert torch.equal(bufs(a, 1 - parity)[k], bufs(b, 1 - parity)[k])
        assert a._parity == b._parity == 1 - parity


@pytest.mark.parametrize("n_step", [1, 3])
@pytest.mark.parametrize("B", [512, 37])
@pytest.mark.parametrize("stream", ["philox", "dry"])
def test_select_with_scalars_equals_select_then_gather(env, n_step, B, stream):
    """``b2rl_replay_select_uniform_scalars`` (the K1 sample: index draw + action / n-step reward / mask in one launch) writes
    exactly what ``b2rl_replay_select_uniform`` followed by the scalar-only gather writes, and advances the ring state the
    same way.  "dry": a candidate stream with too few valid indices, so the unfilled tail is cycled first."""
    bench, rl = env
    dev = torch.device("cuda", 0)
    rp = bench.synthetic_ring(rl, rl.UniformReplay, dev, seed=7, capacity=CAP)
    rp.n_step = n_step
    cand = None
    if stream == "dry":
        g = torch.Generator(device=dev).manual_seed(B)
        cand = torch.full((B + 16,), -1, dtype=torch.int64, device=dev)
        cand[::5] = torch.randint(8, CAP // 3 - 8, (len(cand[::5]),), device=dev, generator=g)
    st0 = rp.ring_state.clone()
    fused, split = rp._buffers(B, torch.bfloat16, "ring", tag=11), rp._buffers(B, torch.bfloat16, "ring", tag=12)
    for bufs in (fused, split):
        for k in ("idx", "action", "reward", "mask"):
            bufs[k].fill_(-7)
    rp.select(B, fused["idx"], cand, scalars=fused)
    torch.cuda.synchronize()
    st1, status1 = rp.ring_state.clone(), rp._status.clone()
    rp.ring_state.copy_(st0)
    rp.select(B, split["idx"], cand)
    rp.gather_scalars(split["idx"], B, split)
    torch.cuda.synchronize()
    assert torch.equal(rp.ring_state, st1) and torch.equal(rp._status, status1)
    if stream == "dry":
        assert 0 < int(status1[0]) < B
    else:
        assert int(status1[0]) == B and int(st1[4]) > int(st0[4])
    for k in ("idx", "action", "reward", "mask"):
        assert torch.equal(fused[k], split[k]), k
    assert bool((fused["idx"] >= 0).all())
