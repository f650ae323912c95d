"""GPU tests of the rows the round-1 review found untested: the asynchronous ``ReplayWrapper`` (replay.py:199-278) ordering,
the asynchronous actor (BaseAgent.py:108-182), and the replay checkpoint (HBM ring + sum tree, SURVEY 8f-4)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


@pytest.fixture(scope="module")
def rl():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import deeprl_b200 as rl
    rl.select_device(0)
    rl.Config.COMPUTE_DTYPE = torch.float32
    return rl


def _items(rng, n, value=None):
    frames = [np.full((84, 84), value, dtype=np.uint8) if value is not None else rng.randint(0, 200, (84, 84)).astype(np.uint8)
              for _ in range(n)]
    return dict(state=frames, action=[int(rng.randint(4)) for _ in range(n)], reward=[0.0] * n, mask=[1] * n)


def test_async_replay_wrapper_is_one_sample_stale(rl):
    """The reference's replay worker answers sample() with the batch it drew right after the PREVIOUS sample() and at once
    draws the next one (replay.py:236-249): a batch can only contain transitions fed before the previous sample() call.
    Frames fed later carry the marker value 255; the first sample() after them must not see them, the next one may."""
    rng = np.random.RandomState(0)
    w = rl.ReplayWrapper(rl.UniformReplay, dict(memory_size=512, batch_size=64, n_step=1, discount=0.99, history_length=4),
                         async_=True)
    for _ in range(60):
        w.feed(_items(rng, 4))                              # 240 unmarked transitions
    t1 = w.sample()                                         # drawn now; the NEXT batch is drawn now as well
    assert int((t1.state >= 250).sum()) == 0
    for _ in range(60):
        w.feed(_items(rng, 4, value=255))                   # 240 marked transitions (half of the ring afterwards)
    t2 = w.sample()                                         # the batch prefetched BEFORE the marked feeds
    assert int((t2.state >= 250).sum()) == 0, "async replay must hand out the batch drawn before the later feeds"
    seen = 0
    for _ in range(3):
        seen += int((w.sample().state >= 250).sum())        # batches drawn after the marked feeds see them
    assert seen > 0
    w.close()


def test_dqn_agent_with_async_actor_thread(rl):
    """config.async_actor = True: the actor plays in its own thread and hands sgd_update_frequency transitions per step through
    a queue (BaseAgent.py:108-182; a thread instead of a process -- a CUDA context does not survive fork)."""
    c = rl.Config()
    c.merge(dict(tag=None))
    c.task_fn = lambda: rl.Task("SyntheticAtari-v0", seed=4)
    c.eval_env = rl.Task("SyntheticAtari-v0", seed=4)
    c.optimizer_fn = lambda p: torch.optim.RMSprop(p, lr=0.00025, alpha=0.95, eps=0.01, centered=True)
    c.network_fn = lambda: rl.VanillaNet(c.action_dim, rl.NatureConvBody(in_channels=4))
    c.random_action_prob = rl.LinearSchedule(1.0, 0.01, 1e6)
    c.batch_size = 32
    c.replay_fn = lambda: rl.ReplayWrapper(rl.UniformReplay, dict(memory_size=1000, batch_size=32, n_step=1, discount=0.99,
                                                                  history_length=4), async_=True)
    c.state_normalizer, c.reward_normalizer = rl.ImageNormalizer(), rl.SignNormalizer()
    c.discount, c.history_length, c.double_q, c.n_step = 0.99, 4, False, 1
    c.target_network_update_freq, c.exploration_steps, c.sgd_update_frequency, c.gradient_clip = 20, 100, 4, 5
    c.async_actor = True
    ag = rl.DQNAgent(c)
    p0 = [p.detach().clone() for p in ag.network.parameters()]
    for _ in range(60):
        ag.step()
    torch.cuda.synchronize()
    assert ag.total_steps == 60 * 4
    assert ag.actor._thread is not None and ag.actor._thread.is_alive()
    assert ag.last_loss is not None and torch.isfinite(ag.last_loss).all()
    assert any(not torch.equal(a, b.detach()) for a, b in zip(p0, ag.network.parameters()))
    ag.close()
    assert not ag.actor._thread.is_alive()


@pytest.mark.parametrize("cls_name", ["UniformReplay", "PrioritizedReplay"])
def test_replay_checkpoint_round_trip(rl, cls_name, tmp_path):
    """state_dict / load_state_dict of the HBM ring (+ sum tree): a restored replay samples the SAME batches from the same
    candidate / uniform streams and continues feeding at the same cursor."""
    rng = np.random.RandomState(1)
    cls = getattr(rl, cls_name)
    a = cls(300, 32, n_step=1, discount=0.99, history_length=4)
    for _ in range(90):
        a.feed(_items(rng, 4))
    if cls_name == "PrioritizedReplay":
        t = a.sample(uniforms=rng.rand(32), fills=rng.randint(0, 1 << 30, 32))
        a.update_priorities((t.idx, torch.rand(32, device=t.idx.device) + 0.1))
    f = str(tmp_path / "replay.pt")
    torch.save(a.state_dict(), f)
    b = cls(300, 32, n_step=1, discount=0.99, history_length=4)
    b.load_state_dict(torch.load(f, weights_only=False))
    assert b.size() == a.size() and b.pos == a.pos
    if cls_name == "PrioritizedReplay":
        assert torch.equal(a.tree.tree, b.tree.tree)
        u, fl = rng.rand(32), rng.randint(0, 1 << 30, 32)
        ta, tb = a.sample(uniforms=u, fills=fl), b.sample(uniforms=u, fills=fl)
        assert torch.equal(ta.idx, tb.idx) and torch.equal(ta.sampling_prob, tb.sampling_prob)
    else:
        cand = rng.randint(0, a.size(), 400)
        ta, tb = a.sample(candidates=cand), b.sample(candidates=cand)
    assert torch.equal(ta.state, tb.state) and torch.equal(ta.next_state, tb.next_state) and torch.equal(ta.reward, tb.reward)
    item = _items(rng, 4, value=7)
    a.feed(item), b.feed(item)
    assert torch.equal(a.frames, b.frames) and torch.equal(a.ring_state, b.ring_state)


@pytest.mark.parametrize("workload", ["dqn", "per"])
def test_host_cursor_follows_feeds_captured_in_the_graph(rl, workload):
    """The learner feeds the ring inside its captured graph: ``size()`` / ``full()`` / ``valid_index()`` / ``state_dict()``
    then read the cursor from the device (replay.py:80-90 keeps it on the host; ours lives in ``ring_state``)."""
    import bench
    bench.CAP = 30_000
    rl.Config.COMPUTE_DTYPE = torch.bfloat16             # (the learner bench.py builds: bf16 wgmma body)
    try:
        lr = bench.build_learner(rl, workload, torch.device("cuda", 0), 0, 1, prefetch=False)
        rp = lr.replay
        lr.capture(warmup=2)
        rp.size()
        pos0 = rp.pos
        for _ in range(7):
            lr.update()
        torch.cuda.synchronize()
        assert rp.size() == rp.memory_size and rp.full()
        assert (rp.pos, rp._size) == tuple(int(x) for x in rp.ring_state[:2].tolist())
        assert rp.pos == (pos0 + 7 * lr.feeds) % rp.memory_size and lr.feeds == 4
        assert int(rp.state_dict()["ring_state"][0]) == rp.pos
        assert rp.valid_index(rp.pos - 1) is False and rp.valid_index(rp.pos - 2) is True   # next state of pos-1 is the write slot
    finally:
        rl.Config.COMPUTE_DTYPE = torch.float32
