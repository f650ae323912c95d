"""``n_step_dqn_pixel`` on the captured sm_90a path (``config.cuda_graph``; NStepDQNAgent ``_step_graph``): one GraphedQActor
replay per env step, its uploads landing in the rollout arena, and one GraphedNStepLearner replay per rollout, whose n-step
target and loss are ONE ``b2rl_nstep_q_loss`` launch (csrc/losses.cu).

CPU: the coverage predicate (``nstep_q_graph_unsupported``) and the eager path of refused configurations; the float64
restatement of the pixel n-step update against oracle/agents.py ``nstep_dqn_update``; the float64 reference of the loss
kernel's outputs against autograd; the kernel's registers and spills.
GPU: the kernel bit for bit against float64 on exact small-integer inputs; the recomputed batch-T*N q against the actor's q;
one update and consecutive updates (with target syncs) against the float64 oracle at the tolerances of
tests/test_gpu_step_vs_oracle.py (bf16 operands, fp32 accumulation); launch accounting; checkpoints; the launcher."""
import os
import re
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import agents, nets  # noqa: E402

T5, N16 = 5, 16                                      # the launcher's rollout length and workers (examples.py n_step_dqn_pixel)


# ------------------------------------------------------------------------------------------------ float64 references
def nstep_q_update(sd, target_sd, params, opt, states, actions, rewards, masks, discount, gradient_clip, body):
    """NStepDQN_agent.py:26-70 for one rollout whose env interaction is given -- the statements of oracle/agents.py
    ``nstep_dqn_update`` with the body a function ``phi = body(sd, x)`` (``pixel_body`` for the NatureConvBody).  ``states``
    (T+1, N, ...), ``actions`` (T, N), ``rewards`` / ``masks`` (T, N, 1).  Returns (ret (T, N, 1), loss)."""
    T = actions.shape[0]
    q = [nets.vanilla_q(sd, body(sd, states[t])) for t in range(T)]
    with torch.no_grad():
        ret = nets.vanilla_q(target_sd, body(target_sd, states[T])).max(dim=1, keepdim=True)[0]
    rets = [None] * T
    for i in reversed(range(T)):
        ret = rewards[i] + discount * masks[i] * ret
        rets[i] = ret
    qa = torch.cat(q, dim=0).gather(1, actions.reshape(-1, 1).long())
    loss = 0.5 * (qa - torch.cat(rets, dim=0)).pow(2).mean()
    opt.zero_grad()
    loss.backward()
    agents.clip_grad_norm(params, gradient_clip)
    opt.step()
    return torch.stack(rets), loss.detach()


def pixel_body(sd, x):
    """ImageNormalizer (x / 255) then the NatureConvBody (network_bodies.py:27-33) on uint8 stacks [N, 4, 84, 84]."""
    return nets.nature_body(sd, x.to(torch.float64) / 255.0)


def nstep_q_reference(q, q_boot, action, reward, mask, discount):
    """float64 outputs of ``b2rl_nstep_q_loss``: ret, delta = ret - q[a], loss = 0.5 mean(delta^2), gq = dloss/dq.  Shapes:
    q [T*N, A], q_boot [N, A], action / reward / mask [T, N]."""
    q, qb = np.asarray(q, np.float64), np.asarray(q_boot, np.float64)
    T, N = np.shape(action)
    r, m = np.asarray(reward, np.float64), np.asarray(mask, np.float64)
    ret = np.zeros((T, N))
    nxt = qb.max(axis=1)
    for t in reversed(range(T)):
        nxt = r[t] + discount * m[t] * nxt
        ret[t] = nxt
    rows = np.arange(T * N)
    a = np.asarray(action).reshape(-1)
    delta = ret.reshape(-1) - q[rows, a]
    gq = np.zeros_like(q)
    gq[rows, a] = -delta / (T * N)
    return ret.reshape(-1), delta, 0.5 * np.mean(delta ** 2), gq


def small_int_case(T, N, A, seed):
    """Integers everywhere, discount 0.5 and 0/1 masks, with r_t a multiple of 2^t and q_boot one of 2^T, so that every
    return ret_t (a multiple of 2^t) and every delta is an integer: each value and each partial sum of delta^2 (below 2^24)
    is exact in fp32, whatever the order of the sums."""
    g = np.random.RandomState(seed)
    q = g.randint(-8, 9, size=(T * N, A)).astype(np.float32)
    qb = (g.randint(-1, 2, size=(N, A)) * 2.0 ** T).astype(np.float32)
    action = g.randint(0, A, size=(T, N)).astype(np.int64)
    reward = (g.randint(-1, 2, size=(T, N)) * 2.0 ** np.arange(T).reshape(T, 1)).astype(np.float32)
    mask = (g.rand(T, N) > 0.3).astype(np.float32)
    return q, qb, action, reward, mask


# ------------------------------------------------------------------------------------------------ CPU
def test_pixel_oracle_reduces_to_the_fc_oracle():
    """With the FC body, the pixel restatement is oracle/agents.py nstep_dqn_update statement for statement: same returns,
    same loss and the same parameters after the step."""
    g = torch.Generator().manual_seed(3)
    T, N, D, A = 5, 4, 6, 3
    sd = {"body.layers.0.weight": torch.randn(16, D, generator=g, dtype=torch.float64) * 0.3,
          "body.layers.0.bias": torch.randn(16, generator=g, dtype=torch.float64) * 0.1,
          "body.layers.1.weight": torch.randn(16, 16, generator=g, dtype=torch.float64) * 0.3,
          "body.layers.1.bias": torch.randn(16, generator=g, dtype=torch.float64) * 0.1,
          "fc_head.weight": torch.randn(A, 16, generator=g, dtype=torch.float64) * 0.3,
          "fc_head.bias": torch.randn(A, generator=g, dtype=torch.float64) * 0.1}
    tgt = {k: v + 0.01 for k, v in sd.items()}
    states = torch.randn(T + 1, N, D, generator=g, dtype=torch.float64)
    actions = torch.randint(0, A, (T, N), generator=g)
    rewards = torch.randint(-1, 2, (T, N, 1), generator=g).double()
    masks = (torch.rand(T, N, 1, generator=g) > 0.2).double()
    out = []
    for fn in (agents.nstep_dqn_update, None):
        leaves = agents.leafify(sd)
        params = list(leaves.values())
        opt = torch.optim.RMSprop(params, lr=1e-3, alpha=0.99, eps=1e-5)
        if fn is None:
            ret, loss = nstep_q_update(leaves, tgt, params, opt, states, actions, rewards, masks, 0.99, 5.0,
                                       lambda s, x: nets.fc_body(s, x, "body.", F.relu))
        else:
            ret, loss = fn(leaves, tgt, params, opt, states, actions, rewards, masks, 0.99, 5.0)
        out.append((ret, loss, {k: v.detach().clone() for k, v in leaves.items()}))
    (r0, l0, p0), (r1, l1, p1) = out
    assert torch.equal(r0, r1) and torch.equal(l0, l1)
    assert all(torch.equal(p0[k], p1[k]) for k in p0)


@pytest.mark.parametrize("T,N,A", [(1, 1, 2), (5, 16, 4), (7, 37, 18)])
def test_loss_reference_matches_autograd(T, N, A):
    """The float64 reference of ret / delta / loss / gq against autograd on 0.5 * mean((q[a] - ret)^2)."""
    g = np.random.RandomState(T * 100 + N)
    q, qb = g.randn(T * N, A), g.randn(N, A)
    action, reward = g.randint(0, A, size=(T, N)), g.randn(T, N)
    mask = (g.rand(T, N) > 0.2).astype(np.float64)
    ret, delta, loss, gq = nstep_q_reference(q, qb, action, reward, mask, 0.99)
    qt = torch.tensor(q, requires_grad=True)
    boot = torch.tensor(qb).max(dim=1)[0]
    rets, nxt = [None] * T, boot
    for t in reversed(range(T)):
        nxt = torch.tensor(reward[t]) + 0.99 * torch.tensor(mask[t]) * nxt
        rets[t] = nxt
    r = torch.cat(rets)
    qa = qt.gather(1, torch.tensor(action).reshape(-1, 1)).view(-1)
    lt = 0.5 * (qa - r).pow(2).mean()
    lt.backward()
    np.testing.assert_allclose(ret, r.numpy(), rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(delta, (r - qa).detach().numpy(), rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(loss, float(lt.detach()), rtol=1e-13)
    np.testing.assert_allclose(gq, qt.grad.numpy(), rtol=1e-12, atol=1e-15)


def _pixel_config(rl, **kw):
    """The configuration ``examples.n_step_dqn_pixel`` builds (examples.py), on whatever device is selected.  Built in a
    temporary directory: the launcher's logger opens its file under ./log."""
    import tempfile

    import examples
    got = []
    mp = pytest.MonkeyPatch()
    mp.setattr(examples, "run_steps", got.append)
    mp.chdir(tempfile.mkdtemp(prefix="nstep_pixel_"))
    try:
        examples.n_step_dqn_pixel(game=kw.pop("game", "SyntheticAtari-v0"), cuda_graph=True, **kw)
    finally:
        mp.undo()
    return got[0]


def _refusals(rl):
    """(name, config change, network_fn, expected reason) for every refused configuration."""
    nature = lambda **k: (lambda: rl.VanillaNet(4, rl.NatureConvBody(**k)))
    return [
        ("fp32", dict(dtype=torch.float32), None, "compute dtype"),
        ("fc_body", {}, lambda: rl.VanillaNet(4, rl.FCBody(4 * 84 * 84)), "captured update implements NatureConvBody"),
        ("noisy", {}, nature(noisy_linear=True), "NoisyLinear"),
        ("normalizer", dict(state_normalizer=rl.MeanStdNormalizer()), None, "RescaleNormalizer"),
        ("dueling", {}, lambda: rl.DuelingNet(4, rl.NatureConvBody()), "implements VanillaNet"),
        ("device_nstep_dqn", dict(device_nstep_dqn=True), None, "device_nstep_dqn"),
        ("no_cuda_graph", dict(cuda_graph=False), None, "cuda_graph is not set"),
        ("sgd", dict(optimizer_fn=lambda p: torch.optim.SGD(p, 1e-3)), None, "optimizer is SGD"),
    ]


def _predicate(rl, cfg, net, opt_fn=None):
    from deeprl_b200.component.coverage import nstep_q_graph_unsupported
    opt = (opt_fn or cfg.optimizer_fn)(net.parameters())
    states = cfg.task_fn().reset()
    return nstep_q_graph_unsupported(cfg, net, opt, states)


def test_coverage_predicate_on_the_host():
    """Every refusal names its condition; the launcher's configuration is refused on the host for its device only, and
    async_actor (default True) plays no part."""
    import deeprl_b200 as rl
    rl.select_device(-1)
    old = rl.Config.COMPUTE_DTYPE
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    try:
        ag = _pixel_config(rl, max_steps=0)
        cfg = ag.config
        assert cfg.async_actor
        assert _predicate(rl, cfg, cfg.network_fn()) == "the network is not on a CUDA device (select_device(0))"
        for name, change, net_fn, why in _refusals(rl):
            saved = {k: getattr(cfg, k, None) for k in change if k != "dtype"}
            for k, v in change.items():
                if k == "dtype":
                    rl.Config.COMPUTE_DTYPE = v
                else:
                    setattr(cfg, k, v)
            try:
                got = _predicate(rl, cfg, (net_fn or cfg.network_fn)())
            finally:
                rl.Config.COMPUTE_DTYPE = torch.bfloat16
                for k, v in saved.items():
                    setattr(cfg, k, v)
            assert got is not None and why in got, (name, got)
    finally:
        rl.Config.COMPUTE_DTYPE = old


def test_refused_configuration_takes_the_eager_path():
    """The launcher at its default fp32 compute on the host: the agent notes the refusal and its step() is the eager path."""
    import deeprl_b200 as rl
    rl.select_device(-1)
    np.random.seed(0), torch.manual_seed(0)
    ag = _pixel_config(rl, max_steps=0, num_workers=2)
    ag.config.rollout_length = 2
    before = {k: v.clone() for k, v in ag.network.state_dict().items()}
    ag.step()
    assert ag._graph is False and "compute dtype" in ag.graph_refusal
    assert isinstance(ag.optimizer, torch.optim.RMSprop) and np.isfinite(float(ag.last_loss))
    assert any(not torch.equal(before[k], v) for k, v in ag.network.state_dict().items())


def test_loss_kernel_registers_and_spills():
    """nvcc -Xptxas -v on csrc/losses.cu: the new kernel compiles for sm_90a without spills."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                          os.path.join(ROOT, "deeprl_b200", "csrc", "losses.cu"), "-o", os.devnull],
                         capture_output=True, text=True, check=True)
    lines = out.stderr.splitlines()
    i = next(i for i, ln in enumerate(lines) if "Compiling entry function" in ln and "nstep_q_loss_kernel" in ln)
    block = "\n".join(lines[i:i + 4])
    assert re.search(r"0 bytes spill stores, 0 bytes spill loads", block), block


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


def _run_kernel(q, qb, action, reward, mask, discount):
    from deeprl_b200 import ops
    c = lambda x, dt=torch.float32: torch.as_tensor(x).to(device="cuda", dtype=dt)
    r = ops.nstep_q_loss(c(q), c(qb), c(action, torch.int64), c(reward), c(mask), discount)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in r.items()}


def _f32(x):
    return torch.from_numpy(np.asarray(x, np.float64)).float()


@pytest.mark.gpu
@pytest.mark.parametrize("A", [2, 4, 18])
@pytest.mark.parametrize("N", [1, 16, 37])
@pytest.mark.parametrize("T", [1, 5, 7])
def test_loss_kernel_exact(rl, T, N, A):
    """Integer q and rewards, discount 0.5, 0/1 masks (``small_int_case``): ret, delta and the sum of squares exact, the loss
    and gq correctly rounded quotients -- all equal to float64 rounded once to fp32."""
    q, qb, action, reward, mask = small_int_case(T, N, A, seed=T * 1000 + N * 10 + A)
    got = _run_kernel(q, qb, action, reward, mask, 0.5)
    ret, delta, loss, gq = nstep_q_reference(q, qb, action, reward, mask, 0.5)
    assert np.all(ret == np.round(ret)) and np.sum(delta ** 2) < 2 ** 24
    assert torch.equal(got["ret"], _f32(ret)) and torch.equal(got["delta"], _f32(delta))
    assert torch.equal(got["loss"], _f32([loss])) and torch.equal(got["gq"], _f32(gq))


@pytest.mark.gpu
@pytest.mark.parametrize("T,N,A", [(5, 16, 4), (3, 300, 6)])
def test_loss_kernel_gaussian(rl, T, N, A):
    """Gaussian inputs (N = 300: three CTAs and the last-CTA reduction): float64 within fp32 rounding, and the same bits on
    every launch."""
    g = np.random.RandomState(7)
    q, qb = g.randn(T * N, A).astype(np.float32), g.randn(N, A).astype(np.float32)
    action = g.randint(0, A, size=(T, N))
    reward, mask = g.randn(T, N).astype(np.float32), (g.rand(T, N) > 0.1).astype(np.float32)
    got = _run_kernel(q, qb, action, reward, mask, 0.99)
    ret, delta, loss, gq = nstep_q_reference(q, qb, action, reward, mask, 0.99)
    np.testing.assert_allclose(got["ret"].numpy(), ret, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(got["delta"].numpy(), delta, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(float(got["loss"][0]), loss, rtol=1e-5)
    np.testing.assert_allclose(got["gq"].numpy(), gq, rtol=1e-5, atol=1e-9)
    again = _run_kernel(q, qb, action, reward, mask, 0.99)
    assert all(torch.equal(got[k], again[k]) for k in got)


def _agent(rl, seed=0, **kw):
    np.random.seed(seed), torch.manual_seed(seed)
    ag = _pixel_config(rl, **kw)
    assert ag._graph_ok(), ag.graph_refusal
    return ag


class Recorder:
    """Wraps the agent's GraphedQActor: the stacks and the q of every actor replay."""

    def __init__(self, ag):
        self.actor = ag._graph[1]
        self.inner = self.actor.q_values
        self.states, self.q = [], []
        self.actor.q_values = self

    def __call__(self, states, slot=0):
        self.states.append(np.stack([np.asarray(s) for s in states]))
        q = self.inner(states, slot)
        self.q.append(q)
        return q

    def clear(self):
        self.states, self.q = [], []


def _rollout(ag, rec):
    """One agent step; returns the rollout (states (T+1, N, 4, 84, 84) uint8, actions, rewards, masks (T, N)) it trained on."""
    rec.clear()
    ag.step()
    torch.cuda.synchronize()
    lr = ag._graph[0]
    states = np.stack(rec.states + [np.stack([np.asarray(s) for s in ag.states])])
    return types.SimpleNamespace(states=states, actions=lr.h_action.numpy().copy(), rewards=lr.h_reward.numpy().copy(),
                                 masks=lr.h_mask.numpy().copy(), q=np.concatenate(rec.q))


def _sd64(net):
    return {k: v.detach().double().cpu().clone() for k, v in net.state_dict().items()}


class Oracle:
    """The float64 pixel n-step update (``nstep_q_update``) with its own RMSprop state, following the agent's target syncs."""

    def __init__(self, ag):
        self.sd = agents.leafify(_sd64(ag.network))
        self.tgt = _sd64(ag.target_network)
        self.params = list(self.sd.values())
        o = ag.optimizer
        self.opt = torch.optim.RMSprop(self.params, lr=o.lr, alpha=o.alpha, eps=o.eps, centered=o.centered)
        self.discount, self.clip = ag.config.discount, ag.config.gradient_clip

    def anchor(self, ag):
        """Continue from the agent's online parameters and RMSprop state: float64 and bf16 trajectories part after a few
        updates (RMSprop's first steps move every parameter by about 10 lr whatever the gradient's size), so each rollout is
        compared from the same start.  The oracle's target network stays its own, synchronised on its own schedule."""
        o, named = ag.optimizer, dict(ag.network.named_parameters())
        base = o.flat.data_ptr()
        with torch.no_grad():
            for k, leaf in self.sd.items():
                p = named[k]
                off = (p.data_ptr() - base) // 4
                leaf.copy_(p.detach().double().cpu())
                st = self.opt.state[leaf]
                st["step"] = torch.tensor(float(ag._graph[0].updates))
                st["square_avg"] = o.s1[off:off + p.numel()].view_as(p).double().cpu().clone()
                if o.centered:
                    st["grad_avg"] = o.s2[off:off + p.numel()].view_as(p).double().cpu().clone()

    def update(self, r, sync=False):
        if sync:
            self.tgt = {k: v.detach().clone() for k, v in self.sd.items()}
        s = torch.from_numpy(r.states)
        rew = torch.from_numpy(r.rewards).double().unsqueeze(-1)
        msk = torch.from_numpy(r.masks).double().unsqueeze(-1)
        _, loss = nstep_q_update(self.sd, self.tgt, self.params, self.opt, s, torch.from_numpy(r.actions), rew, msk,
                                 self.discount, self.clip, pixel_body)
        return float(loss)

    def flat(self):
        return torch.cat([v.detach().flatten() for v in self.sd.values()])


def _flat(net):
    return torch.cat([v.detach().double().cpu().flatten() for v in net.state_dict().values()])


def cosine(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


@pytest.mark.gpu
def test_recomputed_q_is_the_actors_q(rl):
    """The batch-80 online q the update recomputes from the arena equals the q the actor's batch-16 replays returned, bit
    for bit (each row's reduction order does not depend on the batch), over two rollouts."""
    ag = _agent(rl, max_steps=0)
    rec = Recorder(ag)
    for _ in range(2):
        r = _rollout(ag, rec)
        assert torch.equal(ag._graph[0].q.cpu(), torch.from_numpy(r.q))


def _eager_rerun(ag, flat0, s10, s20, flat_graph):
    """Rewind to the state before the update and run it eagerly on the same staged rollout: the parameters come out as the
    graph replay left them, to fp32 rounding -- the head's backward (b2rl_head_bwd_relu) sums its weight and bias gradients
    across CTAs with atomics, so two runs of one update agree to rounding, not to the bit.  Returns the reference-layout
    gradient of the eager run."""
    lr = ag._graph[0]
    o = ag.optimizer
    o.flat.copy_(flat0), o.s1.copy_(s10), o.s2.copy_(s20)
    lr.refresh_packed()
    lr._main()
    torch.cuda.synchronize()
    grad = o.grad.clone()
    lr._opt()
    torch.cuda.synchronize()
    err = float((o.flat - flat_graph).abs().max())
    assert err <= 1e-6, "eager run of the update vs its graph replay: %g" % err
    return grad


@pytest.mark.gpu
@pytest.mark.parametrize("game", ["SyntheticAtari-v0", "SyntheticAtari-A18-v0"])
def test_one_update_matches_the_float64_oracle(rl, game):
    """One rollout at the launcher's shape (T 5, N 16): loss within 2e-2 relative, clipped gradient norm and parameter-delta
    norm within 5e-2, gradient and step directions cosine > 0.995 / 0.98, against the float64 oracle on the same frames,
    weights, actions, rewards and masks."""
    ag = _agent(rl, game=game, max_steps=0)
    rec = Recorder(ag)
    orc = Oracle(ag)
    o = ag.optimizer
    flat0, s10, s20 = o.flat.clone(), o.s1.clone(), o.s2.clone()
    before = orc.flat().clone()
    r = _rollout(ag, rec)
    loss_dev = float(ag.last_loss)
    flat1 = o.flat.clone()
    grad = _eager_rerun(ag, flat0, s10, s20, flat1)
    loss_orc = orc.update(r)
    np.testing.assert_allclose(loss_dev, loss_orc, rtol=2e-2)
    g_orc = torch.cat([v.grad.flatten() for v in orc.sd.values()])     # (clipped in place by clip_grad_norm_)
    base = o.flat.data_ptr()
    g_dev = torch.cat([grad[(p.data_ptr() - base) // 4:][:p.numel()].double().cpu() for p in ag.network.parameters()])
    d_dev = _flat(ag.network) - torch.cat([flat0[(p.data_ptr() - base) // 4:][:p.numel()].double().cpu()
                                           for p in ag.network.parameters()])
    d_orc = orc.flat() - before
    assert cosine(g_dev, g_orc) > 0.995, cosine(g_dev, g_orc)
    assert cosine(d_dev, d_orc) > 0.98, cosine(d_dev, d_orc)
    n = float(g_dev.norm())
    np.testing.assert_allclose(n * min(1.0, ag.config.gradient_clip / (n + 1e-6)), float(g_orc.norm()), rtol=5e-2)
    np.testing.assert_allclose(float(d_dev.norm()), float(d_orc.norm()), rtol=5e-2)


@pytest.mark.gpu
def test_consecutive_rollouts_with_target_syncs(rl):
    """Four rollouts with the target synchronised every 7 env steps (in rollouts 2 and 3, mid-rollout): after a sync the target
    equals the online network of that rollout bit for bit, otherwise it is unchanged; the actor's next q equals an eager bf16
    forward of a fresh copy of the updated network; every rollout's loss and step follow the float64 oracle, which keeps its
    own target network on the same schedule (``Oracle.anchor``)."""
    from deeprl_b200.network.fused import frame_scale
    ag = _agent(rl, max_steps=0)
    ag.config.target_network_update_freq = 7
    rec = Recorder(ag)
    orc = Oracle(ag)
    synced = []
    for k in range(4):
        online, target = _flat(ag.network), _flat(ag.target_network)
        steps = [ag.total_steps // N16 + t + 1 for t in range(T5)]
        sync = any(s % 7 == 0 for s in steps)
        orc.anchor(ag)
        r = _rollout(ag, rec)
        assert torch.equal(_flat(ag.target_network), online if sync else target), k
        synced.append(sync)
        np.testing.assert_allclose(float(ag.last_loss), orc.update(r, sync), rtol=2e-2, err_msg="rollout %d" % k)
        d_dev, d_orc = _flat(ag.network) - online, orc.flat() - online
        assert cosine(d_dev, d_orc) > 0.98, (k, cosine(d_dev, d_orc))
        np.testing.assert_allclose(float(d_dev.norm()), float(d_orc.norm()), rtol=5e-2, err_msg="rollout %d" % k)
        # the next actor replay sees theta_{k+1}
        actor = ag._graph[1]
        q_next = rec.inner(ag.states, 0)
        fresh = ag.config.network_fn()
        fresh.load_state_dict(ag.network.state_dict())
        with torch.no_grad(), frame_scale(ag.config.state_normalizer.coef):
            q_ref = fresh(actor.x.permute(0, 3, 1, 2))["q"].float().cpu()
        assert torch.equal(torch.from_numpy(q_next), q_ref), k
    assert synced == [False, True, True, False]


@pytest.mark.gpu
def test_a_step_is_graph_replays_only(rl, monkeypatch):
    """After capture, a step without a target sync makes no C-ABI launch and exactly T + 1 graph replays."""
    from deeprl_b200 import _lib
    ag = _agent(rl, max_steps=0)
    ag.step()                                              # captures the actor's slot graphs
    torch.cuda.synchronize()
    replays = []
    real = torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda g: (replays.append(g), real(g))[1])
    _lib.reset_launch_count()
    ag.step()
    torch.cuda.synchronize()
    assert _lib.launch_count() == 0
    assert len(replays) == T5 + 1 and replays[-1] is ag._graph[0].graph


@pytest.mark.gpu
def test_checkpoint_round_trip(rl, tmp_path):
    """Save after k steps, load into a fresh agent that has already captured its graphs and trained, give it the same
    target, optimizer state and env stream, and step both: the same parameters (load() refreshed the packed operands)."""
    import copy
    a = _agent(rl, seed=1, max_steps=0)
    for _ in range(3):
        a.step()
    torch.cuda.synchronize()
    a.save(str(tmp_path / "ck"))
    b = _agent(rl, seed=2, max_steps=0)
    b.step()                                               # graphs captured and trained from b's own weights
    b.load(str(tmp_path / "ck"))
    assert torch.equal(_flat(a.network), _flat(b.network))
    # what the checkpoint does not hold: the target network, the optimizer state, the envs and the exploration schedule
    b.target_network.load_state_dict(a.target_network.state_dict())
    b._graph[0].refresh_packed()
    b.optimizer.s1.copy_(a.optimizer.s1), b.optimizer.s2.copy_(a.optimizer.s2)
    for ea, eb in zip(a.task.env.envs, b.task.env.envs):
        while hasattr(ea, "env"):                          # the SyntheticAtariEnv under the wrappers
            ea, eb = ea.env, eb.env
        eb.rng.set_state(ea.rng.get_state())
        eb.frames = list(ea.frames)
    b.states, b.total_steps = a.states, a.total_steps
    b.config.random_action_prob = copy.deepcopy(a.config.random_action_prob)
    for _ in range(2):
        for ag in (a, b):
            np.random.seed(11)                             # the same epsilon-greedy draws
            ag.step()
        torch.cuda.synchronize()
        # equal up to the fp32 rounding of the head backward's atomic sums (see _eager_rerun); operands left stale by load()
        # would change the gradients themselves, and the step (about 10 lr = 1e-3 per parameter) with them
        err = float((_flat(a.network) - _flat(b.network)).abs().max())
        assert err <= 1e-6, err


@pytest.mark.gpu
def test_launcher_end_to_end(rl):
    """examples.n_step_dqn_pixel(cuda_graph=True) through run_steps: the graph path runs and the loss is finite."""
    from deeprl_b200.utils.misc import run_steps
    np.random.seed(0), torch.manual_seed(0)
    ag = _pixel_config(rl)
    ag.config.max_steps = 6 * T5 * N16
    ag.config.eval_interval = 0
    run_steps(ag)
    assert ag._graph and ag.total_steps == 6 * T5 * N16
    assert ag.last_loss.is_cuda and np.isfinite(float(ag.last_loss))


@pytest.mark.gpu
def test_fp32_launcher_keeps_the_eager_path(rl):
    """The launcher's default fp32 compute is refused for its dtype and trains on today's eager path."""
    rl.Config.COMPUTE_DTYPE = torch.float32
    try:
        np.random.seed(0), torch.manual_seed(0)
        ag = _pixel_config(rl, max_steps=0)
        ag.step()
        assert ag._graph is False and "compute dtype" in ag.graph_refusal
        assert isinstance(ag.optimizer, torch.optim.RMSprop) and np.isfinite(float(ag.last_loss))
    finally:
        rl.Config.COMPUTE_DTYPE = torch.bfloat16
