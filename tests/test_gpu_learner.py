"""The CUDA-graph learner (deeprl_b200/learner.py, the path bench.py times) against the same update run eagerly, and the
async-replay prefetch branch (the graph form of ReplayWrapper(async_=True), reference replay.py:214-262).

Tolerance: the captured graph replays exactly the kernels of the eager update; the only run-to-run freedom is the order
of fp32 atomic adds (split-K fc4 accumulation, bias gradients, narrow-head weight gradients).  Whole trajectories are NOT
comparable (an argmax or a prioritized draw can flip on one ulp), so the comparison is one update from copied state."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import bench
    import deeprl_b200 as rl
    rl.select_device(0)
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    bench.CAP = 30_000
    return bench, rl


def make(env, workload, prefetch):
    bench, rl = env
    return bench.build_learner(rl, workload, torch.device("cuda", 0), 0, 1, prefetch=prefetch)


def copy_state(dst, src):
    """Make learner ``dst`` an exact twin of ``src``: parameters, optimizer state, target network, ring, sum tree,
    cursors and the batch buffers of the prefetch branch."""
    do, so = dst.opt, src.opt
    for a, b in ((do.flat, so.flat), (do.s1, so.s1), (do.s2, so.s2), (do.step_dev, so.step_dev), (do.scratch, so.scratch)):
        a.copy_(b)
    dst.tgt.load_state_dict(src.tgt.state_dict())
    dst.opt.grad.copy_(src.opt.grad)
    dst.refresh_packed()
    dr, sr = dst.replay, src.replay
    for name in ("frames", "action", "reward", "mask", "ring_state"):
        getattr(dr, name).copy_(getattr(sr, name))
    dr.pos, dr._size = sr.pos, sr._size
    if dst.per:
        dr.tree.tree.copy_(sr.tree.tree), dr.tree.pending.copy_(sr.tree.pending)
        dr.max_priority_dev.copy_(sr.max_priority_dev)
        dr.tree.n_entries = sr.tree.n_entries
    for key, bufs in sr._bufs.items():
        if key in dr._bufs:
            for k, v in bufs.items():
                dr._bufs[key][k].copy_(v)
    dst._parity = src._parity
    dst.d_pack.copy_(src.d_pack)
    torch.cuda.synchronize()


def params(learner):
    return learner.opt.flat.detach().clone()


@pytest.mark.parametrize("workload", ["dqn", "per", "c51", "qr"])
@pytest.mark.parametrize("prefetch", [False, True])
def test_graph_replay_equals_eager_update(env, workload, prefetch):
    """One update from IDENTICAL state, once as eager launches and once as a graph replay.  The loss depends on the
    forward pass only and must agree to fp32 rounding; the updated parameters differ by the order of fp32 atomic adds in
    the bias / head gradients (|dp| <= lr * O(1e-6 relative gradient noise))."""
    a, b = make(env, workload, prefetch), make(env, workload, prefetch)
    for _ in range(3):
        a._main(), a._opt()                                # creates a's buffers (overwritten below)
    b.capture(warmup=3)
    copy_state(a, b)
    a._main(), a._opt()
    b.update()
    torch.cuda.synchronize()
    la, lb = float(a.loss), float(b.loss)
    assert np.isfinite(la) and la > 0
    np.testing.assert_allclose(lb, la, rtol=1e-4)
    np.testing.assert_allclose(params(b).cpu().numpy(), params(a).cpu().numpy(), rtol=0, atol=2e-6)
    assert a.replay.ring_state.cpu().tolist()[:4] == b.replay.ring_state.cpu().tolist()[:4]
    if a.per:                                              # same leaves updated, priorities equal to forward-pass noise
        np.testing.assert_allclose(a.replay.tree.tree.cpu().numpy(), b.replay.tree.tree.cpu().numpy(), rtol=1e-2)
    # and a second update, now from (almost) identical state: same batch, loss within bf16-activation noise
    a._main(), a._opt()
    b.update()
    torch.cuda.synchronize()
    np.testing.assert_allclose(float(b.loss), float(a.loss), rtol=5e-2)


@pytest.mark.parametrize("workload", ["dqn", "per"])
def test_prefetch_trains_on_the_previous_sample(env, workload):
    """async replay: update k uses the batch sampled during update k-1; the very first update samples its own batch
    (nothing was prefetched), so it equals the synchronous learner's first update."""
    sync, pre = make(env, workload, False), make(env, workload, True)
    sync._main(), sync._opt()
    pre._main(), pre._opt()
    torch.cuda.synchronize()
    np.testing.assert_allclose(float(pre.loss), float(sync.loss), rtol=1e-5)
    # the prefetch learner has fed twice (its own batch + the prefetched one) and holds the next batch in the other set
    assert int(pre.replay.ring_state[0]) == int(sync.replay.ring_state[0]) + pre.feeds
    assert pre._batch[0].state.data_ptr() != pre._batch[1].state.data_ptr()
    ready = pre._batch[pre._parity].state.clone()          # sampled during update 1
    pre._main(), pre._opt()                                # trains on it and refills the OTHER buffer set
    torch.cuda.synchronize()
    assert torch.equal(pre._batch[1 - pre._parity].state, ready)


def test_update_from_host_feeds_the_ring(env):
    bench, rl = env
    lr = make(env, "dqn", True)
    lr.capture(warmup=2, with_h2d=True)
    pos0 = int(lr.replay.ring_state[0])
    rng = np.random.RandomState(0)
    frames = rng.randint(0, 256, (4, 84 * 84)).astype(np.uint8)
    loss = lr.update_from_host(frames, np.arange(4, dtype=np.int32), np.ones(4), np.ones(4, dtype=np.int32))
    assert np.isfinite(loss)
    cap = lr.replay.memory_size if hasattr(lr.replay, "memory_size") else bench.CAP
    rows = [(pos0 + i) % cap for i in range(4)]
    got = lr.replay.frames[rows].cpu().numpy().reshape(4, -1)
    assert np.array_equal(got, frames)
    assert lr.replay.action[rows].cpu().tolist() == [0, 1, 2, 3]


def test_dual_forward_matches_separate_forwards(env):
    """nature_tc.dual_forward: online(s) and target(s') evaluated with one launch per layer give the features, Q values and
    parameter gradients of two separate forwards (convolutions bit-identical; fc4 differs by its summation order: split-K
    with fp32 atomics vs one pass, i.e. bf16 rounding of the 512 features)."""
    bench, rl = env
    from deeprl_b200.network import nature_tc
    from deeprl_b200.network.fused import frame_scale
    dev = torch.device("cuda", 0)
    torch.manual_seed(3)
    net = rl.VanillaNet(4, rl.NatureConvBody(in_channels=4))
    tgt = rl.VanillaNet(4, rl.NatureConvBody(in_channels=4))          # different weights
    s = torch.randint(0, 256, (64, 64, 21, 21), device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    s2 = torch.randint(0, 256, (64, 64, 21, 21), device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    with frame_scale(1.0 / 255):
        q_ref = net(s)["q"]
        q_ref.sum().backward()
        g_ref = [p.grad.clone() for p in net.parameters()]
        net.zero_grad()
        with torch.no_grad():
            t_ref = tgt(s2)["q"]
        with nature_tc.dual_forward(net.body, tgt.body, s2) as d:
            q = net(s)["q"]
            assert len(d.features) == 1                                  # the target features were computed alongside
            with torch.no_grad():
                t = tgt(s2)["q"]
        q.sum().backward()
    torch.cuda.synchronize()
    np.testing.assert_allclose(q.detach().cpu().numpy(), q_ref.detach().cpu().numpy(), rtol=2e-2, atol=2e-3)
    np.testing.assert_allclose(t.cpu().numpy(), t_ref.cpu().numpy(), rtol=2e-2, atol=2e-3)
    for g, r in zip([p.grad for p in net.parameters()], g_ref):
        scale = float(r.abs().max()) + 1e-12
        assert float((g - r).abs().max()) <= 3e-2 * scale


@pytest.mark.parametrize("persistent", [False, True])
def test_graphed_ppo_minibatches_match_the_eager_loop(env, persistent):
    """GraphedPPOLearner (one graph replay per minibatch, KL gate decided on the device by b2rl_clip_adam_gated) and
    PersistentPPOLearner (the whole loop in one persistent kernel, csrc/ppo_persistent.cu) against
    PPOAgent._minibatch (the eager loop with the host-side `if approx_kl <= 1.5 * target_kl`, PPO_agent.py:94) on the same
    rollout rows and the same permutations.  fp32 throughout: parameters agree to 1e-5 after 16 updates, and both took
    the same number of (gated) actor steps."""
    bench, rl = env
    from collections import namedtuple
    from deeprl_b200.utils import random_sample
    dev = torch.device("cuda", 0)
    rl.Config.COMPUTE_DTYPE = torch.float32
    try:
        def agent(graph):
            torch.manual_seed(11)
            c = rl.Config()
            c.merge(dict(tag=None))
            c.num_workers = 2
            c.task_fn = lambda: rl.Task("SyntheticCheetah-v0", num_envs=2, seed=1)
            c.eval_env = rl.Task("SyntheticCheetah-v0", seed=1)
            c.network_fn = lambda: rl.GaussianActorCriticNet(c.state_dim, c.action_dim,
                                                             actor_body=rl.FCBody(c.state_dim, gate=torch.tanh),
                                                             critic_body=rl.FCBody(c.state_dim, gate=torch.tanh))
            c.actor_opt_fn = lambda p: torch.optim.Adam(p, 3e-4)
            c.critic_opt_fn = lambda p: torch.optim.Adam(p, 1e-3)
            c.discount, c.use_gae, c.gae_tau, c.gradient_clip = 0.99, True, 0.95, 0.5
            c.rollout_length, c.optimization_epochs, c.mini_batch_size, c.ppo_ratio_clip = 8, 4, 64, 0.2
            c.target_kl = 2e-4                                             # small: some actor steps are skipped
            c.graph_minibatch = graph
            c.persistent_minibatch = persistent
            return rl.PPOAgent(c)

        a, b = agent(False), agent(True)
        for pa, pb in zip(a.network.parameters(), b.network.parameters()):
            assert torch.equal(pa, pb)
        g = torch.Generator(device=dev).manual_seed(5)
        rows = 256
        state = torch.randn(rows, a.config.state_dim, device=dev, generator=g)
        with torch.no_grad():
            pred = a.network(state)
        Entry = namedtuple("Entry", ["state", "action", "log_pi_a", "ret", "advantage"])
        entries = Entry(state, pred["action"].contiguous(), pred["log_pi_a"].contiguous(),
                        torch.randn(rows, 1, device=dev, generator=g), torch.randn(rows, 1, device=dev, generator=g))
        np.random.seed(3)
        for _ in range(a.config.optimization_epochs):
            for idx in random_sample(np.arange(rows), 64):
                a._minibatch(entries, idx)
        np.random.seed(3)
        b._graphed_epochs(entries)
        torch.cuda.synchronize()
        assert type(b._graph).__name__ == ("PersistentPPOLearner" if persistent else "GraphedPPOLearner")
        for (n, pa), pb in zip(a.network.named_parameters(), b.network.parameters()):
            np.testing.assert_allclose(pb.detach().cpu().numpy(), pa.detach().cpu().numpy(), rtol=1e-4, atol=1e-5, err_msg=n)
        steps_a = int(next(iter(a.actor_opt.state.values()))["step"])
        steps_b = int(b._graph.actor_opt.step_dev)
        assert steps_a == steps_b and 0 < steps_b < 16                     # the gate closed at least once, identically
        assert int(b._graph.critic_opt.step_dev) == 16
        np.testing.assert_allclose(b.last_stats.cpu().numpy()[:3], a.last_stats.cpu().numpy()[:3], rtol=1e-3, atol=1e-6)
        a.close(), b.close()
    finally:
        rl.Config.COMPUTE_DTYPE = torch.bfloat16


def test_fused_backward_epilogues_match_the_separate_passes(env):
    """B2RL_FUSED_BWD: ReLU mask + bias gradient + grid scatter inside the dgrad GEMM epilogues against the three
    b2rl_act_bwd_bias_grad_bf16 passes.  The masked gradients are the same bf16 values (masking commutes with rounding);
    the bias gradients sum fp32 accumulators instead of bf16-rounded values."""
    bench, rl = env
    from deeprl_b200.network import nature_tc
    from deeprl_b200.network.fused import frame_scale
    dev = torch.device("cuda", 0)
    torch.manual_seed(5)
    net = rl.VanillaNet(4, rl.NatureConvBody(in_channels=4))
    s = torch.randint(0, 256, (96, 64, 21, 21), device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    grads = {}
    saved = nature_tc.FUSED_BWD          # restored for the tests that follow: their learners' plans read it
    for fused in (False, True):
        nature_tc.FUSED_BWD = fused
        try:
            net.zero_grad()
            with frame_scale(1.0 / 255):
                q = net(s)["q"]
                (q * torch.linspace(-1, 1, q.numel(), device=dev).view_as(q)).sum().backward()
            torch.cuda.synchronize()
            grads[fused] = {n: p.grad.detach().clone() for n, p in net.named_parameters()}
        finally:
            nature_tc.FUSED_BWD = saved
    for n, ref in grads[False].items():
        got = grads[True][n]
        scale = float(ref.abs().max()) + 1e-12
        assert float((got - ref).abs().max()) <= 2e-2 * scale, n


@pytest.mark.parametrize("replay_cls_name", ["UniformReplay", "PrioritizedReplay"])
def test_dqn_agent_with_cuda_graph_option(env, replay_cls_name):
    """config.cuda_graph: DQNAgent.step() drives GraphedDQNLearner (one graph replay per update) through the reference's
    own agent API: transitions are fed by the agent, the update runs as a graph, the target is synchronised on schedule."""
    bench, rl = env
    c = rl.Config()
    c.merge(dict(tag=None))
    c.task_fn = lambda: rl.Task("SyntheticAtari-v0", seed=2)
    c.eval_env = rl.Task("SyntheticAtari-v0", seed=2)
    c.optimizer_fn = lambda p: torch.optim.RMSprop(p, lr=0.00025, alpha=0.95, eps=0.01, centered=True)
    c.network_fn = lambda: rl.VanillaNet(c.action_dim, rl.NatureConvBody(in_channels=4))
    c.random_action_prob = rl.LinearSchedule(1.0, 0.01, 1e6)
    c.batch_size = 32
    replay_cls = getattr(rl, replay_cls_name)
    c.replay_fn = lambda: rl.ReplayWrapper(replay_cls, dict(memory_size=2000, batch_size=32, n_step=1, discount=0.99,
                                                            history_length=4), async_=False)
    c.replay_eps, c.replay_alpha, c.replay_beta = 0.01, 0.5, rl.LinearSchedule(0.4, 1.0, 1e5)
    c.state_normalizer, c.reward_normalizer = rl.ImageNormalizer(), rl.SignNormalizer()
    c.discount, c.history_length, c.double_q, c.n_step = 0.99, 4, False, 1
    c.target_network_update_freq, c.exploration_steps, c.sgd_update_frequency, c.gradient_clip = 20, 200, 4, 5
    c.async_actor = False
    c.cuda_graph = True
    ag = rl.DQNAgent(c)
    before = None
    for i in range(120):
        ag.step()
        if ag.total_steps == 204:
            before = ag._flat.flat.clone()
    torch.cuda.synchronize()
    assert getattr(ag, "_learner", None) is not None and ag._learner.updates > 50
    assert torch.isfinite(ag.last_loss).all()
    assert not torch.equal(before, ag._flat.flat)
    ag.close()
