"""``dqn_pixel``, ``categorical_dqn_pixel`` and ``quantile_regression_dqn_pixel`` as written (async replay) on the captured
sm_90a path (``config.cuda_graph``; DQNAgent ``_async_graph_update``): each step's transitions staged in the learner's pinned
buffer and fed inside ONE update replay (learner.GraphedDQNLearner with ``prefetch`` and ``wrapper_order``), the actor's
forward a GraphedQActor replay, on the actor thread with ``async_actor`` (component/actor.py ``ParameterOrder``).

CPU: the coverage predicate (``dqn_graph_unsupported``) names every refused condition.
GPU: the batches, ring, cursors and Philox counter against the eager ReplayWrapper(async_=True), uniform and prioritized;
the first captured step is exactly one update (float64 oracle, Adam step count), and every update's loss is the float64
oracle's on its batch as the ring held it before the step's feeds; consecutive updates with target
syncs; a step is graph replays only; the async actor through run_steps; the fp32 launcher keeps the eager path."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LAUNCHERS = ("dqn_pixel", "categorical_dqn_pixel", "quantile_regression_dqn_pixel")
AGENTS = ("DQNAgent", "CategoricalDQNAgent", "QuantileRegressionDQNAgent")


def _launch(name, **kw):
    """(agent class, config) of ``examples.<name>(cuda_graph=True, **kw)``: run_steps and the agent constructors are
    intercepted (the launchers hard-code a 1e6-frame ring).  Built in a temporary directory: the logger opens ./log."""
    import examples
    got = []
    mp = pytest.MonkeyPatch()
    for a in AGENTS:
        mp.setattr(examples, a, lambda config, _c=getattr(examples, a): got.append((_c, config)))
    mp.setattr(examples, "run_steps", lambda ag: None)
    mp.chdir(tempfile.mkdtemp(prefix="dqn_pixel_"))
    try:
        getattr(examples, name)(game=kw.pop("game", "SyntheticAtari-v0"), cuda_graph=True, **kw)
    finally:
        mp.undo()
    return got[0]


def _small_replay(name, config, memory_size):
    """The launcher's ``replay_fn`` again, with a small ring (examples._replay with the launcher's other arguments)."""
    import examples
    if name == "dqn_pixel":
        examples._replay(config, config.replay_cls, config.async_replay, memory_size=memory_size, n_step=config.n_step,
                         discount=config.discount, history_length=config.history_length)
    else:
        examples._replay(config, examples.UniformReplay, True, memory_size=memory_size, history_length=4)


# ------------------------------------------------------------------------------------------------ CPU
def _wrapper_stub(config):
    """What ``config.replay_fn()`` builds, without its replay (a replay needs a CUDA device): the wrapper's class and
    keyword arguments, which the predicate reads."""
    import examples
    from deeprl_b200.component.replay import ReplayWrapper

    def make(cls, kw, async_=True):
        w = ReplayWrapper.__new__(ReplayWrapper)
        w.replay_cls, w.replay_kwargs, w.async_, w._primed = cls, kw, bool(async_), False
        return w

    mp = pytest.MonkeyPatch()
    mp.setattr(examples, "ReplayWrapper", make)
    try:
        return config.replay_fn()
    finally:
        mp.undo()


def _stub_agent(cls, config, network=None, optimizer_fn=None):
    ag = cls.__new__(cls)
    ag.config = config
    ag.network = network if network is not None else config.network_fn()
    ag.optimizer = (optimizer_fn or config.optimizer_fn)(ag.network.parameters())
    ag.replay = _wrapper_stub(config)
    return ag


def _predicate(cls, config, **kw):
    from deeprl_b200.component.coverage import dqn_graph_unsupported
    return dqn_graph_unsupported(config, _stub_agent(cls, config, **kw))


@pytest.fixture
def host_bf16():
    import deeprl_b200 as rl
    rl.select_device(-1)
    old = rl.Config.COMPUTE_DTYPE
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    yield rl
    rl.Config.COMPUTE_DTYPE = old


@pytest.mark.parametrize("name", LAUNCHERS)
def test_launchers_are_refused_on_the_host_for_the_device_only(host_bf16, name):
    """As written, and with either async_actor setting, the launcher's configuration meets every condition but the CUDA
    device."""
    cls, cfg = _launch(name)
    assert cfg.replay_fn is not None
    for async_actor in (True, False):
        cfg.async_actor = async_actor
        assert _predicate(cls, cfg) == "the network is not on a CUDA device (select_device(0))", (name, async_actor)
    if name == "dqn_pixel":
        import examples
        for kw in (dict(replay_cls=examples.PrioritizedReplay), dict(n_step=3)):
            c2, cfg2 = _launch(name, **kw)
            assert _predicate(c2, cfg2) == "the network is not on a CUDA device (select_device(0))", kw


def test_every_refusal_names_its_condition(host_bf16):
    rl = host_bf16
    import examples
    cls, cfg = _launch("dqn_pixel")

    class Hooked(cls):
        def reduce_loss(self, loss):
            return loss.pow(2).mean()

    cases = [
        ("fp32", dict(dtype=torch.float32), {}, "compute dtype"),
        ("noisy", dict(noisy_linear=True), {}, "NoisyLinear"),
        ("rainbow_net", {}, dict(network=rl.RainbowNet(4, 51, rl.NatureConvBody(), noisy_linear=False)), "RainbowNet"),
        ("fc_body", {}, dict(network=rl.VanillaNet(4, rl.FCBody(4 * 84 * 84))), "implements NatureConvBody"),
        ("normalizer", dict(state_normalizer=rl.MeanStdNormalizer()), {}, "RescaleNormalizer"),
        ("sgd", {}, dict(optimizer_fn=lambda p: torch.optim.SGD(p, 1e-3)), "optimizer is SGD"),
        ("device_dqn", dict(device_dqn=True), {}, "device_dqn"),
        ("no_cuda_graph", dict(cuda_graph=False), {}, "cuda_graph is not set"),
        ("workers", dict(num_workers=2), {}, "envs per actor step"),
    ]
    for what, change, agent_kw, why in cases:
        saved = {k: getattr(cfg, k, None) for k in change if k != "dtype"}
        for k, v in change.items():
            if k == "dtype":
                rl.Config.COMPUTE_DTYPE = v
            else:
                setattr(cfg, k, v)
        try:
            got = _predicate(cls, cfg, **agent_kw)
        finally:
            rl.Config.COMPUTE_DTYPE = torch.bfloat16
            for k, v in saved.items():
                setattr(cfg, k, v)
        assert got is not None and why in got, (what, got)
    # float frames of the right shape, the frame history, the replay kind, the hooks and a wrapper that has handed out an
    # eager batch
    space = cfg.eval_env.observation_space
    cfg.eval_env.observation_space = type("Space", (), dict(shape=(4, 84, 84), dtype=np.float32))
    try:
        assert "float32 (4, 84, 84)" in _predicate(cls, cfg)
    finally:
        cfg.eval_env.observation_space = space
    examples._replay(cfg, examples.UniformReplay, True, memory_size=100, history_length=1)
    assert "history_length 1" in _predicate(cls, cfg)
    examples._replay(cfg, examples.UniformReplay, False, memory_size=100, history_length=4)
    assert "async_=True" in _predicate(cls, cfg)
    examples._replay(cfg, examples.UniformReplay, True, memory_size=100, history_length=4)
    assert "overrides compute_loss / reduce_loss" in _predicate(Hooked, cfg)
    ag = _stub_agent(cls, cfg)
    ag.replay._primed = True
    from deeprl_b200.component.coverage import dqn_graph_unsupported
    assert "already handed out an eager batch" in dqn_graph_unsupported(cfg, ag)
    qcls, qcfg = _launch("quantile_regression_dqn_pixel")
    examples._replay(qcfg, examples.PrioritizedReplay, True, memory_size=100, history_length=4)
    assert "QR-DQN with prioritized replay" in _predicate(qcls, qcfg)
    ccls, ccfg = _launch("categorical_dqn_pixel")
    assert "implements CategoricalNet" in _predicate(ccls, ccfg, network=rl.VanillaNet(4, rl.NatureConvBody()))


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def rl():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import deeprl_b200 as rl
    rl.select_device(0)
    old = rl.Config.COMPUTE_DTYPE
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    yield rl
    rl.Config.COMPUTE_DTYPE = old


def _agent(name, seed=0, memory_size=300, exploration=800, cuda_graph=True, async_actor=False, uniform_actions=False,
           **kw):
    """The launcher's agent with a small ring and a short exploration; nothing else changed."""
    import deeprl_b200 as rl
    cls, cfg = _launch(name, **kw)
    _small_replay(name, cfg, memory_size)
    cfg.exploration_steps = exploration
    cfg.cuda_graph, cfg.async_actor = cuda_graph, async_actor
    if uniform_actions:
        cfg.random_action_prob = rl.LinearSchedule(1.0, 1.0, 1)
    np.random.seed(seed), torch.manual_seed(seed)
    return cls(cfg)


def _until_updates(ag, k=0):
    """Step through exploration, then ``k`` more steps (updates)."""
    while ag.total_steps <= ag.config.exploration_steps - ag.config.sgd_update_frequency:
        ag.step()
    for _ in range(k):
        ag.step()
    torch.cuda.synchronize()


def _bufs(rp, tag, graph):
    keys = [k for k in rp._bufs if k[3] == tag and (k[1] != torch.uint8) == graph]
    assert len(keys) == 1, keys
    return rp._bufs[keys[0]]


def _trained_tag(ag):
    """The buffer set the next update trains on: the learner's parity, or the wrapper's current cache."""
    lr = ag._learner
    if ag.config.cuda_graph:
        return lr._parity if lr is not None else 0
    return ag.replay._cur if ag.replay._primed else 0


def _oracle(ag, sd, tgt):
    """oracle/agents.py DQNFamilyOracle in float64 from state dicts of the agent's networks."""
    from oracle import agents
    cfg = ag.config
    head = {"VanillaNet": "vanilla", "CategoricalNet": "categorical", "QuantileNet": "quantile"}[type(ag.network).__name__]
    atoms = torch.linspace(cfg.categorical_v_min, cfg.categorical_v_max, cfg.categorical_n_atoms, dtype=torch.float64) \
        if head == "categorical" else None
    orc = agents.DQNFamilyOracle(sd, head, "nature", cfg.action_dim, cfg.optimizer_fn, cfg.discount, cfg.n_step,
                                 double_q=bool(cfg.double_q), gradient_clip=cfg.gradient_clip, state_coef=1.0 / 255, atoms=atoms,
                                 v_min=cfg.categorical_v_min, v_max=cfg.categorical_v_max, num_quantiles=cfg.num_quantiles)
    for k, v in tgt.items():
        orc.target_sd[k].copy_(v)
    return orc


def _batch64(frames, idx, bufs, n_step=1):
    """The batch of ``idx`` from a host copy of the ring's frame rows, as float64 tensors (state / next state stacks of
    4 rows; action / reward / mask as the draw gathered them)."""
    f = frames.view(-1, 84, 84)
    rows = torch.from_numpy(np.asarray(idx)).view(-1, 1) + torch.arange(-3, 1).view(1, -1)

    class Tr:
        state = f[rows.reshape(-1)].view(-1, 4, 84, 84).double()
        next_state = f[(rows + n_step).reshape(-1)].view(-1, 4, 84, 84).double()
        action, reward, mask = (bufs[k].double().cpu() for k in ("action", "reward", "mask"))
    return Tr


def _sd64(net):
    return {k: v.detach().double().cpu().clone() for k, v in net.state_dict().items()}


def _trace(ag, updates, check_loss=False):
    """Per update: the trained batch's indices (and tree indices), the ring's bytes and scalar columns, ring_state and the
    host cursor.  ``check_loss``: the update's loss against the float64 oracle on the batch as the ring held it BEFORE
    the step (from the parameters before the step) -- what the eager wrapper materialised before this step's feeds."""
    _until_updates(ag)
    rp = ag.replay.replay
    per = hasattr(rp, "tree")
    out = []
    for _ in range(updates):
        tag = _trained_tag(ag)
        leaves0 = rp.tree.tree[rp.memory_size - 1:].clone() if per else None
        pos0 = int(rp.ring_state[0])
        if check_loss:
            pre = dict(frames=rp.frames.cpu().clone(), sd=_sd64(ag.network), tgt=_sd64(ag.target_network))
        ag.step()
        torch.cuda.synchronize()
        b = _bufs(rp, tag, ag.config.cuda_graph)
        if check_loss:
            with torch.no_grad():
                orc = _oracle(ag, pre["sd"], pre["tgt"])
                tr_pre = _batch64(pre["frames"], b["idx"].cpu().numpy(), b, rp.n_step)
                want = float(orc.reduce_loss(orc.compute_loss(tr_pre)))
            np.testing.assert_allclose(float(ag.last_loss), want, rtol=2e-2, err_msg="update %d" % len(out))
        rec = dict(idx=b["idx"].cpu().numpy().copy(), frames=rp.frames.cpu().clone(), action=rp.action.cpu().clone(),
                   reward=rp.reward.cpu().clone(), mask=rp.mask.cpu().clone(), state=rp.ring_state.cpu().clone(),
                   host=(rp.size(), rp.pos), steps=ag.total_steps)
        if per:
            leaves = rp.tree.tree[rp.memory_size - 1:]
            rec.update(tree_idx=b["tree_idx"].cpu().numpy().copy(), changed=torch.nonzero(leaves != leaves0).view(-1).cpu().numpy(),
                       fed=(pos0 + np.arange(ag.config.sgd_update_frequency)) % rp.memory_size,
                       total=float(rp.tree.tree[0]), leaf_sum=float(leaves.sum()))
        out.append(rec)
    ag.close()
    return out


def _compare_traces(graph, eager, exact_draws):
    for k, (g, e) in enumerate(zip(graph, eager)):
        for key in ("frames", "action", "reward", "mask"):
            assert torch.equal(g[key], e[key]), (k, key)
        assert g["host"] == e["host"] and g["steps"] == e["steps"], k
        assert int(g["state"][0]) == g["steps"] % 300, k            # every transition stored once, in order
        if k < exact_draws:
            assert np.array_equal(np.sort(g["idx"]), np.sort(e["idx"])), k
            assert torch.equal(g["state"], e["state"]), (k, g["state"], e["state"])


@pytest.mark.gpu
def test_same_batches_as_the_eager_async_wrapper(rl):
    """Uniform replay, a 300-frame ring that wraps: the captured agent trains on the batches the eager ReplayWrapper(async_=True)
    hands out, and leaves the ring, both cursors and the Philox counter as the eager agent does, after every step.  Each
    captured update's loss is the float64 oracle's on its batch read from the ring as it was before the step's feeds (conv1
    reads the stacks from the ring: feeds ordered before that read would change the frames of the stacks they overwrite)."""
    traces = [_trace(_agent("dqn_pixel", uniform_actions=True, cuda_graph=g), 40, check_loss=g) for g in (True, False)]
    _compare_traces(traces[0], traces[1], exact_draws=40)


@pytest.mark.gpu
def test_prioritized_replay_order(rl):
    """PER: the first two batches are the eager wrapper's, both drawn before any priority write; afterwards each update changes
    only the leaves of its own batch (and of its feeds), and the tree's total is the sum of its leaves."""
    traces = []
    for g in (True, False):
        traces.append(_trace(_agent("dqn_pixel", uniform_actions=True, cuda_graph=g, replay_cls=rl.PrioritizedReplay), 12))
    _compare_traces(traces[0], traces[1], exact_draws=2)
    for k, t in enumerate(traces[0]):
        mine = set((t["tree_idx"] - (300 - 1)).tolist()) | set(t["fed"].tolist())
        assert set(t["changed"].tolist()) <= mine, k
        np.testing.assert_allclose(t["total"], t["leaf_sum"], rtol=1e-12)


def _cosine(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


@pytest.mark.gpu
@pytest.mark.parametrize("game", ["SyntheticAtari-v0", "SyntheticAtari-A18-v0"])
@pytest.mark.parametrize("name", LAUNCHERS)
def test_first_captured_step_is_one_update(rl, name, game):
    """The first captured step leaves the agent exactly one update further on: one Adam step, and the loss, gradient and
    parameter delta of the float64 oracle's update on the batch it trained on (oracle/agents.py DQNFamilyOracle), within
    the tolerances of bf16 operands with fp32 accumulation."""
    ag = _agent(name, game=game, memory_size=2000, exploration=400)
    _until_updates(ag)
    o = ag._flat
    sd0, tgt0 = _sd64(ag.network), _sd64(ag.target_network)
    flat0 = o.flat.clone()
    assert ag._learner is None and float(o.s1.abs().max()) == 0.0
    ag.step()
    torch.cuda.synchronize()
    lr = ag._learner
    assert lr is not None and lr.updates == 1 and ag.graph_refusal is None
    if o.kind == "adam":
        assert int(o.step_dev) == 1
    rp = ag.replay.replay
    b = _bufs(rp, 0, True)
    # the first update feeds before it draws: its batch is read from the ring as the step left it
    orc = _oracle(ag, sd0, tgt0)
    Tr = _batch64(rp.frames.cpu(), b["idx"].cpu().numpy(), b, rp.n_step)
    before = {k: v.detach().clone() for k, v in orc.sd.items()}
    loss_orc = float(orc.update(Tr))
    np.testing.assert_allclose(float(ag.last_loss), loss_orc, rtol=2e-2)
    # the clipped gradient from the first optimizer step's state: Adam's exp_avg = (1 - beta1) g, centered RMSprop's
    # grad_avg = (1 - alpha) g
    g_flat = o.s1 / (1 - o.betas[0]) if o.kind == "adam" else o.s2 / (1 - o.alpha)
    base = o.flat.data_ptr()
    g_dev, g_orc, d_dev, d_orc = [], [], [], []
    for n, p in ag.network.named_parameters():
        off = (p.data_ptr() - base) // 4
        g_dev.append(g_flat[off:off + p.numel()].float().cpu())
        g_orc.append(orc.sd[n].grad.flatten())
        d_dev.append((o.flat[off:off + p.numel()] - flat0[off:off + p.numel()]).float().cpu())
        d_orc.append((orc.sd[n].detach() - before[n]).flatten())
    g_dev, g_orc, d_dev, d_orc = (torch.cat(x) for x in (g_dev, g_orc, d_dev, d_orc))
    assert _cosine(g_dev, g_orc) > 0.995, _cosine(g_dev, g_orc)
    assert _cosine(d_dev, d_orc) > 0.98, _cosine(d_dev, d_orc)
    np.testing.assert_allclose(float(g_dev.norm()), float(g_orc.norm()), rtol=5e-2)
    np.testing.assert_allclose(float(d_dev.norm()), float(d_orc.norm()), rtol=5e-2)
    ag.step()                                              # the next step is a replay: a second Adam step
    torch.cuda.synchronize()
    assert lr.updates == 2
    if o.kind == "adam":
        assert int(o.step_dev) == 2
    ag.close()


def _flat(net):
    return torch.cat([v.detach().double().cpu().flatten() for v in net.state_dict().values()])


@pytest.mark.gpu
@pytest.mark.parametrize("name", LAUNCHERS)
def test_consecutive_updates_with_target_syncs(rl, name):
    """Ten captured steps with the target synchronised every third agent step: after a sync the target is the online network
    bit for bit, otherwise unchanged; the actor's next forward is an eager bf16 forward of a copy of the updated network."""
    from deeprl_b200.network.fused import frame_scale
    ag = _agent(name, memory_size=1000, exploration=300)
    ag.config.target_network_update_freq = 3
    _until_updates(ag, 1)
    synced = []
    for k in range(10):
        target = _flat(ag.target_network)
        ag.step()
        torch.cuda.synchronize()
        sync = ag.total_steps / ag.config.sgd_update_frequency % 3 == 0
        synced.append(sync)
        assert torch.equal(_flat(ag.target_network), _flat(ag.network) if sync else target), k
        ga = ag.actor._graph_actor
        q = ga.q_values(ag.actor._state)
        fresh = ag.config.network_fn()
        fresh.load_state_dict(ag.network.state_dict())
        for m, f in zip(ag.network.children(), fresh.children()):
            if getattr(m, "_w16", None) is not None:       # C51 / QR: the head reads a bf16 copy of its weight
                f._w16 = f.weight.detach().to(torch.bfloat16)
        with torch.no_grad(), frame_scale(ag.config.state_normalizer.coef):
            q_ref = ag.actor._q_tensor(fresh(ga.x.permute(0, 3, 1, 2))).float().cpu()
        assert torch.equal(torch.from_numpy(q), q_ref), k
        assert np.isfinite(float(ag.last_loss)), k
    assert any(synced) and not all(synced)
    ag.close()


@pytest.mark.gpu
def test_a_step_is_graph_replays_only(rl, monkeypatch):
    """After capture, a step without a target sync makes no C-ABI launch: four actor replays and one update replay."""
    from deeprl_b200 import _lib
    ag = _agent("dqn_pixel", memory_size=1000, exploration=300)
    ag.config.target_network_update_freq = 10 ** 9
    _until_updates(ag, 2)                                  # captures the learner, then the actor's graph for its operands
    replays = []
    real = torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda g: (replays.append(g), real(g))[1])
    _lib.reset_launch_count()
    ag.step()
    torch.cuda.synchronize()
    assert _lib.launch_count() == 0
    lr = ag._learner
    assert len(replays) == 5 and replays[-1] in lr.g_main
    assert all(r is ag.actor._graph_actor.graphs[0] for r in replays[:4])
    ag.close()


@pytest.mark.gpu
def test_async_actor_through_run_steps(rl):
    """dqn_pixel with async_actor=True through run_steps, 400 steps past exploration: the captured path ran, the loss is finite,
    the ring holds exactly the transitions the actor handed over, in order, and after close() the actor thread is gone and
    its forward matches an eager forward of the final weights."""
    from deeprl_b200.network.fused import frame_scale
    from deeprl_b200.utils.misc import run_steps
    ag = _agent("dqn_pixel", memory_size=2000, exploration=400, async_actor=True)
    ag.config.max_steps = 800
    ag.config.eval_interval = 0
    ag.config.log_interval = 0
    got = []
    inner_step = ag.actor.step

    def step():
        out = inner_step()
        got.extend(out)
        return out

    ag.actor.step = step
    run_steps(ag)
    assert ag.graph_refusal is None and ag._learner is not None and ag._learner.updates > 0
    assert np.isfinite(float(ag.last_loss))
    assert not ag.actor._thread.is_alive()
    rp = ag.replay.replay
    n = ag.total_steps
    assert n == 800 and len(got) == n and rp.size() == n and rp.pos == n
    frames = rp.frames[:n].view(n, 84, 84).cpu().numpy()
    want = np.stack([np.asarray(t[0][0])[-1] for t in got])
    assert np.array_equal(frames, want)
    assert np.array_equal(rp.action[:n].cpu().numpy(), np.asarray([t[1][0] for t in got]))
    ga = ag.actor._graph_actor
    assert ga and ga.replays > 0
    q = ga.q_values(ag.actor._state)
    fresh = ag.config.network_fn()
    fresh.load_state_dict(ag.network.state_dict())
    with torch.no_grad(), frame_scale(ag.config.state_normalizer.coef):
        q_ref = fresh(ga.x.permute(0, 3, 1, 2))["q"].float().cpu()
    assert torch.equal(torch.from_numpy(q), q_ref)


@pytest.mark.gpu
def test_fp32_launcher_keeps_the_eager_path(rl):
    """The launchers' default fp32 compute is refused for its dtype and trains on today's eager path."""
    rl.Config.COMPUTE_DTYPE = torch.float32
    try:
        ag = _agent("dqn_pixel", memory_size=500, exploration=100)
        _until_updates(ag, 2)
        assert "compute dtype" in ag.graph_refusal and ag._learner is None
        assert np.isfinite(float(ag.last_loss))
        ag.close()
    finally:
        rl.Config.COMPUTE_DTYPE = torch.bfloat16
