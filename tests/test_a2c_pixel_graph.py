"""``a2c_pixel`` on the captured sm_90a path (``config.cuda_graph``; A2CAgent ``_step_graph``): one GraphedQActor replay per
env step running the body and the actor-critic head with the action drawn on the device (``b2rl_ac_head_fwd``), and one
GraphedA2CLearner replay per rollout, whose GAE, objective and head-output gradient are ONE ``b2rl_a2c_rollout_loss`` launch
(csrc/onpolicy.cu) and whose head backward is ``b2rl_head_bwd_geff_relu`` (csrc/head.cu).

CPU: the float64 restatement of the pixel A2C update against oracle/agents.py ``a2c_update``; the float64 reference of the
loss kernel's outputs against autograd; the coverage predicate (``a2c_graph_unsupported``) and the eager path of refused
configurations; the new kernels' registers and spills.
GPU: the loss kernel against ``ops.gae(exact=True)`` (bit for bit) and float64; the head forward / backward against float64;
the device draws against the host Philox; the recomputed batch-(T+1)N head outputs against the actor's; one update and
consecutive updates against the float64 oracle at the tolerances of tests/test_gpu_step_vs_oracle.py (bf16 operands, fp32
accumulation); launch accounting; checkpoints; the launchers."""
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
from oracle import agents, losses, nets, philox  # noqa: E402

T5, N16 = 5, 16                                      # the launcher's rollout length and workers (examples.py a2c_pixel)


# ------------------------------------------------------------------------------------------------ float64 references
def a2c_pixel_update(sd, params, opt, states, actions, rewards, masks, discount, tau, entropy_weight, value_loss_weight,
                     gradient_clip, body, use_gae=True):
    """A2C_agent.py:22-64 for one rollout whose env interaction is given -- the statements of oracle/agents.py ``a2c_update``
    with the trunk a function ``phi = body(sd, x)`` (``pixel_body`` for the NatureConvBody) and DummyBody actor / critic
    bodies.  ``states`` (T+1, N, ...), ``actions`` (T, N), ``rewards`` / ``masks`` (T, N, 1).  Returns (adv, ret, loss)."""
    T = actions.shape[0]

    def ac(x, action):
        phi = body(sd, x)
        dist = torch.distributions.Categorical(logits=F.linear(phi, sd["fc_action.weight"], sd["fc_action.bias"]))
        return dict(log_pi_a=dist.log_prob(action).unsqueeze(-1), entropy=dist.entropy().unsqueeze(-1),
                    v=F.linear(phi, sd["fc_critic.weight"], sd["fc_critic.bias"]))

    preds = [ac(states[t], actions[t]) for t in range(T)]
    last = ac(states[T], actions[T - 1])
    v = torch.stack([p["v"] for p in preds] + [last["v"]])
    adv, ret = losses.gae(rewards, masks, v.detach(), discount, tau, use_gae)
    cat = lambda k: torch.cat([p[k] for p in preds], dim=0)
    loss = losses.a2c_loss(cat("log_pi_a"), cat("v"), ret.reshape(-1, 1), adv.reshape(-1, 1), cat("entropy"),
                           entropy_weight, value_loss_weight)
    opt.zero_grad()
    loss.backward()
    agents.clip_grad_norm(params, gradient_clip)
    opt.step()
    return adv, ret, loss.detach()


def pixel_body(sd, x):
    """ImageNormalizer (x / 255) then the NatureConvBody (network_bodies.py:27-33) on uint8 stacks [N, 4, 84, 84]."""
    return nets.nature_body(sd, x.to(torch.float64) / 255.0, prefix="phi_body.")


def rollout_reference(head, action, reward, mask, discount, tau, use_gae, ew, vw):
    """float64 outputs of ``b2rl_a2c_rollout_loss``: adv, ret [T*N], loss, geff [(T+1)*N, A+1].  ``head`` [(T+1)*N, A+1]
    (logits, v), ``action`` / ``reward`` / ``mask`` [T, N]."""
    h = np.asarray(head, np.float64)
    T, N = np.shape(reward)
    A = h.shape[1] - 1
    r, m = np.asarray(reward, np.float64), np.asarray(mask, np.float64)
    v = h[:, A].reshape(T + 1, N)
    ret, adv = np.zeros((T, N)), np.zeros((T, N))
    x, g = v[T].copy(), np.zeros(N)
    for t in reversed(range(T)):
        x = r[t] + discount * m[t] * x
        g = g * tau * discount * m[t] + (r[t] + discount * m[t] * v[t + 1] - v[t]) if use_gae else x - v[t]
        ret[t], adv[t] = x, g
    R = T * N
    z = h[:R, :A]
    lp = z - z.max(1, keepdims=True)
    lp = lp - np.log(np.exp(lp).sum(1, keepdims=True))
    p = np.exp(lp)
    H = -(p * lp).sum(1)
    a = np.asarray(action).reshape(-1)
    rows = np.arange(R)
    adv, ret = adv.reshape(-1), ret.reshape(-1)
    vr = v[:T].reshape(-1)
    loss = -np.mean(lp[rows, a] * adv) - ew * np.mean(H) + vw * 0.5 * np.mean((ret - vr) ** 2)
    geff = np.zeros(((T + 1) * N, A + 1))
    onehot = np.zeros((R, A))
    onehot[rows, a] = 1.0
    geff[:R, :A] = -(adv / R)[:, None] * (onehot - p) + (ew / R) * p * (lp + H[:, None])
    geff[:R, A] = (vw / R) * (vr - ret)
    return adv, ret, loss, geff


def rollout_case(T, N, A, seed):
    g = np.random.RandomState(seed)
    head = np.concatenate([g.randn((T + 1) * N, A) * 2.0, g.randn((T + 1) * N, 1)], axis=1).astype(np.float32)
    action = g.randint(0, A, size=(T, N)).astype(np.int64)
    reward = g.randint(-1, 2, size=(T, N)).astype(np.float32)
    mask = (g.rand(T, N) > 0.2).astype(np.float32)
    return head, action, reward, mask


# ------------------------------------------------------------------------------------------------ CPU
def test_pixel_oracle_reduces_to_the_fc_oracle():
    """With the FC body, the pixel restatement is oracle/agents.py a2c_update statement for statement: same advantages,
    returns and parameters after the step."""
    g = torch.Generator().manual_seed(3)
    T, N, D, A = 5, 4, 6, 3
    sd = {"phi_body.layers.0.weight": torch.randn(16, D, generator=g, dtype=torch.float64) * 0.3,
          "phi_body.layers.0.bias": torch.randn(16, generator=g, dtype=torch.float64) * 0.1,
          "phi_body.layers.1.weight": torch.randn(16, 16, generator=g, dtype=torch.float64) * 0.3,
          "phi_body.layers.1.bias": torch.randn(16, generator=g, dtype=torch.float64) * 0.1,
          "fc_action.weight": torch.randn(A, 16, generator=g, dtype=torch.float64) * 0.3,
          "fc_action.bias": torch.randn(A, generator=g, dtype=torch.float64) * 0.1,
          "fc_critic.weight": torch.randn(1, 16, generator=g, dtype=torch.float64) * 0.3,
          "fc_critic.bias": torch.randn(1, generator=g, dtype=torch.float64) * 0.1}
    states = torch.randn(T + 1, N, D, generator=g, dtype=torch.float64)
    actions = torch.randint(0, A, (T, N), generator=g)
    rewards = torch.randint(-1, 2, (T, N, 1), generator=g).double()
    masks = (torch.rand(T, N, 1, generator=g) > 0.2).double()
    out = []
    for pixel in (False, True):
        leaves = agents.leafify(sd)
        params = list(leaves.values())
        opt = torch.optim.RMSprop(params, lr=1e-3, alpha=0.99, eps=1e-5)
        if pixel:
            adv, ret, _ = a2c_pixel_update(leaves, params, opt, states, actions, rewards, masks, 0.99, 0.95, 0.01, 1.0, 5.0,
                                           lambda s, x: nets.fc_body(s, x, "phi_body.", torch.tanh))
        else:
            adv, ret = agents.a2c_update(leaves, params, opt, states, actions, rewards, masks, 0.99, 0.95, 0.01, 1.0, 5.0)
        out.append((adv, ret, {k: v.detach().clone() for k, v in leaves.items()}))
    (a0, r0, p0), (a1, r1, p1) = out
    assert torch.equal(a0, a1) and torch.equal(r0, r1)
    assert all(torch.equal(p0[k], p1[k]) for k in p0)


@pytest.mark.parametrize("use_gae", [True, False])
@pytest.mark.parametrize("T,N,A", [(1, 1, 2), (5, 16, 6), (7, 37, 31)])
def test_loss_reference_matches_autograd(T, N, A, use_gae):
    """The float64 reference of adv / ret / loss / geff against autograd on the reference's statements (oracle/losses.py gae
    on detached values, a2c_loss on a Categorical): geff is the gradient of the loss with respect to the head's outputs."""
    head, action, reward, mask = rollout_case(T, N, A, seed=T * 100 + N)
    adv, ret, loss, geff = rollout_reference(head, action, reward, mask, 0.99, 0.95, use_gae, 0.01, 0.5)
    h = torch.tensor(head, dtype=torch.float64, requires_grad=True)
    v = h[:, A].view(T + 1, N, 1)
    ta, tr = losses.gae(torch.tensor(reward).double().unsqueeze(-1), torch.tensor(mask).double().unsqueeze(-1), v.detach(),
                        0.99, 0.95, use_gae)
    dist = torch.distributions.Categorical(logits=h[:T * N, :A])
    a = torch.tensor(action).reshape(-1)
    lt = losses.a2c_loss(dist.log_prob(a).unsqueeze(-1), v[:T].reshape(-1, 1), tr.reshape(-1, 1), ta.reshape(-1, 1),
                         dist.entropy().unsqueeze(-1), 0.01, 0.5)
    lt.backward()
    np.testing.assert_allclose(adv, ta.reshape(-1).numpy(), rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(ret, tr.reshape(-1).numpy(), rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(loss, float(lt.detach()), rtol=1e-12)
    np.testing.assert_allclose(geff, h.grad.numpy(), rtol=1e-10, atol=1e-15)


def _pixel_config(rl, **kw):
    """The configuration ``examples.a2c_pixel`` builds (examples.py), on whatever device is selected.  Built in a temporary
    directory: the launcher's logger opens its file under ./log."""
    import tempfile

    import examples
    got = []
    mp = pytest.MonkeyPatch()
    mp.setattr(examples, "run_steps", got.append)
    mp.chdir(tempfile.mkdtemp(prefix="a2c_pixel_"))
    try:
        examples.a2c_pixel(game=kw.pop("game", "SyntheticAtari-v0"), cuda_graph=True, **kw)
    finally:
        mp.undo()
    return got[0]


def _refusals(rl):
    """(name, config change, network_fn, expected reason) for every refused configuration."""
    ac = lambda A=4, **k: (lambda: rl.CategoricalActorCriticNet(None, A, **k))
    return [
        ("fp32", dict(dtype=torch.float32), None, "compute dtype"),
        ("fc_body", {}, ac(phi_body=rl.FCBody(4 * 84 * 84)), "captured update implements NatureConvBody"),
        ("noisy", {}, ac(phi_body=rl.NatureConvBody(noisy_linear=True)), "NoisyLinear"),
        ("actor_body", {}, ac(phi_body=rl.NatureConvBody(), actor_body=rl.FCBody(512)), "DummyBody"),
        ("actions", {}, ac(32, phi_body=rl.NatureConvBody()), "fewer than 32"),
        ("vanilla", {}, lambda: rl.VanillaNet(4, rl.NatureConvBody()), "implements CategoricalActorCriticNet"),
        ("normalizer", dict(state_normalizer=rl.MeanStdNormalizer()), None, "RescaleNormalizer"),
        ("device_a2c", dict(device_a2c=True), None, "device_a2c"),
        ("no_cuda_graph", dict(cuda_graph=False), None, "cuda_graph is not set"),
        ("sgd", dict(optimizer_fn=lambda p: torch.optim.SGD(p, 1e-3)), None, "optimizer is SGD"),
        ("rmsprop_momentum", dict(optimizer_fn=lambda p: torch.optim.RMSprop(p, 1e-3, momentum=0.9)), None, "optimizer is"),
    ]


def _predicate(rl, cfg, net):
    from deeprl_b200.component.coverage import a2c_graph_unsupported
    opt = cfg.optimizer_fn(net.parameters())
    states = cfg.task_fn().reset()
    return a2c_graph_unsupported(cfg, net, opt, states)


def test_coverage_predicate_on_the_host():
    """Every refusal names its condition; the launcher's configuration is refused on the host for its device only."""
    import deeprl_b200 as rl
    rl.select_device(-1)
    old = rl.Config.COMPUTE_DTYPE
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    try:
        ag = _pixel_config(rl, max_steps=0)
        cfg = ag.config
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


@pytest.mark.parametrize("src,kernel", [("head.cu", "ac_head_fwd_kernel"), ("onpolicy.cu", "a2c_rollout_loss_kernel")])
def test_kernel_registers_and_spills(src, kernel):
    """nvcc -Xptxas -v: every instantiation of the new kernels compiles for sm_90a without spills."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                          os.path.join(ROOT, "deeprl_b200", "csrc", src), "-o", os.devnull],
                         capture_output=True, text=True, check=True)
    lines = out.stderr.splitlines()
    starts = [i for i, ln in enumerate(lines) if "Compiling entry function" in ln and kernel in ln]
    assert starts
    for i in starts:
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


def _cuda(x, dt=torch.float32):
    return torch.as_tensor(x).to(device="cuda", dtype=dt)


def _run_loss(head, action, reward, mask, use_gae):
    from deeprl_b200 import ops
    r = ops.a2c_rollout_loss(_cuda(head), _cuda(action, torch.int64), _cuda(reward), _cuda(mask), 0.99, 0.95, use_gae, 0.01,
                             0.5)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in r.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("use_gae", [True, False])
@pytest.mark.parametrize("A", [2, 6, 18, 31])
@pytest.mark.parametrize("N", [1, 16, 37])
@pytest.mark.parametrize("T", [1, 5, 7])
def test_loss_kernel(rl, T, N, A, use_gae):
    """adv / ret the bits of ops.gae(exact=True) on the head's values; loss and geff float64 within fp32 rounding, zero in the
    final rows; the same bits on a second launch (N = 37: ten CTAs and the last-CTA reduction)."""
    from deeprl_b200 import ops
    head, action, reward, mask = rollout_case(T, N, A, seed=T * 1000 + N * 10 + A)
    got = _run_loss(head, action, reward, mask, use_gae)
    v = _cuda(head[:, A]).view(T + 1, N)
    adv_g, ret_g = ops.gae(_cuda(reward), _cuda(mask), v, 0.99, 0.95, use_gae, exact=True)
    assert torch.equal(got["adv"], adv_g.cpu().view(-1)) and torch.equal(got["ret"], ret_g.cpu().view(-1))
    adv, ret, loss, geff = rollout_reference(head, action, reward, mask, 0.99, 0.95, use_gae, 0.01, 0.5)
    np.testing.assert_allclose(float(got["loss"][0]), loss, rtol=2e-5, atol=1e-6)
    g = got["geff"][:, :A + 1].numpy()
    np.testing.assert_allclose(g, geff, rtol=1e-4, atol=1e-6 * np.abs(geff).max())
    assert not g[T * N:].any()
    again = _run_loss(head, action, reward, mask, use_gae)
    assert all(torch.equal(got[k], again[k]) for k in got)


def _head_case(B, A, seed, zero=False):
    g = torch.Generator().manual_seed(seed)
    phi = torch.relu(torch.randn(B, 512, generator=g)).to(torch.bfloat16)
    fa, fc = torch.nn.Linear(512, A).cuda(), torch.nn.Linear(512, 1).cuda()
    with torch.no_grad():
        for m, s in ((fa, 0.2), (fc, 0.05)):
            m.weight.copy_(torch.randn(m.weight.shape, generator=g) * s * (0.0 if zero else 1.0))
            m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1 * (0.0 if zero else 1.0))
    return phi.cuda(), fa, fc


def _w64(fa, fc):
    return (torch.cat([fa.weight, fc.weight]).detach().double().cpu(), torch.cat([fa.bias, fc.bias]).detach().double().cpu())


@pytest.mark.gpu
@pytest.mark.parametrize("A", [2, 6, 18, 31])
def test_head_forward_and_backward(rl, A):
    """Forward: (logits, v) of bf16 features against float64.  Backward from geff [B, 33]: the bf16 feature gradient masked by
    phi > 0, the weight / bias gradients (accumulated onto what the buffers held) and fc4's column sums against float64."""
    from deeprl_b200 import _lib
    from deeprl_b200.network import fused
    B = 100
    phi, fa, fc = _head_case(B, A, seed=A)
    out = fused.ac_head(phi, fa, fc)
    W, b = _w64(fa, fc)
    x = phi.double().cpu()
    ref = x @ W.T + b
    np.testing.assert_allclose(out.cpu().numpy(), ref.numpy(), rtol=1e-5, atol=1e-5)
    geff = torch.zeros(B, 33, device="cuda")
    geff[:, :A + 1] = torch.randn(B, A + 1, device="cuda") * 1e-2
    grads = [torch.full_like(p, 0.5) for p in (fa.weight, fa.bias, fc.weight, fc.bias)]
    gphi = torch.empty_like(phi)
    colsum = torch.zeros(512, device="cuda")
    _lib.call("b2rl_head_bwd_geff_relu", _lib.ptr(geff), _lib.ptr(phi), _lib.ptr(fa.weight), _lib.ptr(fc.weight), B, 512, A,
              _lib.ptr(gphi), *[_lib.ptr(t) for t in grads], _lib.ptr(colsum), _lib.stream())
    torch.cuda.synchronize()
    ge = geff[:, :A + 1].double().cpu()
    gp = (ge @ W) * (x > 0)
    np.testing.assert_allclose(gphi.double().cpu().numpy(), gp.numpy(), rtol=2 ** -8, atol=1e-7)
    gw, gb = ge.T @ x, ge.sum(0)
    np.testing.assert_allclose(torch.cat([grads[0], grads[2]]).double().cpu().numpy(), gw.numpy() + 0.5, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(torch.cat([grads[1], grads[3]]).double().cpu().numpy(), gb.numpy() + 0.5, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(colsum.double().cpu().numpy(), gphi.double().cpu().sum(0).numpy(), rtol=1e-5, atol=1e-6)


def _draw(phi, fa, fc, counter, ticket, seed):
    from deeprl_b200.network import fused
    act = torch.full((phi.shape[0],), -1, dtype=torch.int64, device="cuda")
    out = fused.ac_head(phi, fa, fc, draw=(seed, counter, act, ticket))
    torch.cuda.synchronize()
    return out.cpu().numpy(), act.cpu().numpy()


SEED, C0 = 0x1234_5678_9ABC_DEF, 1000


@pytest.mark.gpu
@pytest.mark.parametrize("A", [2, 6, 18, 31])
def test_draws_with_zeroed_head(rl, A):
    """Zeroed head weights (uniform softmax): every action is categorical_inverse_cdf of u24(seed, ctr0 + n, 13) bit for bit,
    over two launches of 300 rows (many CTAs); the counter advances by the batch per launch."""
    B = 300
    phi, fa, fc = _head_case(B, A, seed=A, zero=True)
    counter = torch.full((1,), C0, dtype=torch.int64, device="cuda")
    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
    for s in range(2):
        out, act = _draw(phi, fa, fc, counter, ticket, SEED)
        u = philox.u24(SEED, np.uint64(C0 + B * s) + np.arange(B, dtype=np.uint64), 13)
        want, _ = philox.categorical_inverse_cdf(u, out[:, :A])
        assert np.array_equal(act, want)
        assert int(counter) == C0 + B * (s + 1) and int(ticket) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("A", [6, 18])
def test_draws_general_logits(rl, A):
    """Logits of a trained-looking head: the picks equal a float64 inverse CDF on the float64 logits, for every row whose target
    is further than 1e-5 (relative) from a partial-sum boundary; fewer than 1 % are excluded."""
    B = 1024
    phi, fa, fc = _head_case(B, A, seed=100 + A)
    counter = torch.full((1,), C0, dtype=torch.int64, device="cuda")
    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
    _, act = _draw(phi, fa, fc, counter, ticket, SEED)
    W, b = _w64(fa, fc)
    logits = (phi.double().cpu() @ W.T + b)[:, :A].numpy()
    u = philox.u24(SEED, np.uint64(C0) + np.arange(B, dtype=np.uint64), 13)
    want, gap = philox.categorical_inverse_cdf(u, logits, np.float64)
    keep = gap > 1e-5
    assert keep.mean() > 0.99, keep.mean()
    assert np.array_equal(act[keep], want[keep])
    assert len(set(want[keep].tolist())) == A


def _agent(rl, seed=0, **kw):
    np.random.seed(seed), torch.manual_seed(seed)
    ag = _pixel_config(rl, **kw)
    assert ag._graph_ok(), ag.graph_refusal
    return ag


class Recorder:
    """Wraps the agent's GraphedQActor: the stacks, the actions and the head outputs of every actor replay."""

    def __init__(self, ag):
        self.actor = ag._graph[1]
        self.lr = ag._graph[0]
        self.inner = self.actor.q_values
        self.clear()
        self.actor.q_values = self

    def __call__(self, states, slot=0):
        self.states.append(np.stack([np.asarray(s) for s in states]))
        a = self.inner(states, slot)
        self.actions.append(a)
        self.out.append(self.lr.act_out[slot].cpu().clone())
        return a

    def clear(self):
        self.states, self.actions, self.out = [], [], []


def _rollout(ag, rec):
    """One agent step; returns the rollout (states (T+1, N, 4, 84, 84) uint8, actions, rewards, masks (T, N)) it trained on."""
    rec.clear()
    ag.step()
    torch.cuda.synchronize()
    lr = ag._graph[0]
    states = np.stack(rec.states + [np.stack([np.asarray(s) for s in ag.states])])
    return types.SimpleNamespace(states=states, actions=np.stack(rec.actions), rewards=lr.h_reward.numpy().copy(),
                                 masks=lr.h_mask.numpy().copy(), out=torch.stack(rec.out))


def _sd64(net):
    return {k: v.detach().double().cpu().clone() for k, v in net.state_dict().items()}


class Oracle:
    """The float64 pixel A2C update (``a2c_pixel_update``) with its own RMSprop state."""

    def __init__(self, ag):
        self.sd = agents.leafify(_sd64(ag.network))
        self.params = list(self.sd.values())
        o = ag.optimizer
        self.opt = torch.optim.RMSprop(self.params, lr=o.lr, alpha=o.alpha, eps=o.eps, centered=o.centered)
        self.cfg = ag.config

    def anchor(self, ag):
        """Continue from the agent's parameters and RMSprop state: float64 and bf16 trajectories part after a few updates
        (RMSprop's first steps move every parameter by about 10 lr whatever the gradient's size), so each rollout is compared
        from the same start."""
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

    def update(self, r):
        c = self.cfg
        _, _, loss = a2c_pixel_update(self.sd, self.params, self.opt, torch.from_numpy(r.states),
                                      torch.from_numpy(r.actions), torch.from_numpy(r.rewards).double().unsqueeze(-1),
                                      torch.from_numpy(r.masks).double().unsqueeze(-1), c.discount, c.gae_tau,
                                      c.entropy_weight, c.value_loss_weight, c.gradient_clip, pixel_body, c.use_gae)
        return float(loss)

    def flat(self):
        return torch.cat([v.detach().flatten() for v in self.sd.values()])


def _flat(net):
    return torch.cat([v.detach().double().cpu().flatten() for v in net.state_dict().values()])


def cosine(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


@pytest.mark.gpu
def test_recomputed_head_outputs_are_the_actors(rl):
    """The (logits, v) the update recomputes at batch (T+1) N from the arena equal what the actor's batch-N replays computed
    for each slot, bit for bit, over two rollouts; the actions of the update are the ones the actor downloaded."""
    ag = _agent(rl, max_steps=0)
    rec = Recorder(ag)
    lr = ag._graph[0]
    for _ in range(2):
        r = _rollout(ag, rec)
        got = lr.head_out[:T5 * N16].cpu()
        assert torch.equal(got, r.out.reshape(T5 * N16, -1))
        assert np.array_equal(lr.d_action.cpu().numpy(), r.actions)


@pytest.mark.gpu
def test_counter_advances_by_n_per_replay(rl):
    """After capture, each actor replay advances the device counter by N, across slots, and draws from Philox at the counter
    it found (checked on the logits the replay wrote)."""
    ag = _agent(rl, max_steps=0)
    ag.step()                                              # captures the actor's slot graphs
    torch.cuda.synchronize()
    lr, actor = ag._graph
    for slot in (0, 1):
        c0 = int(lr.counter)
        a = actor.q_values(ag.states, slot)
        assert int(lr.counter) == c0 + N16
        u = philox.u24(lr.seed, np.uint64(c0) + np.arange(N16, dtype=np.uint64), 13)
        want, gap = philox.categorical_inverse_cdf(u, lr.act_out[slot, :, :-1].cpu().numpy())
        assert np.array_equal(a[gap > 1e-6], want[gap > 1e-6])


def _eager_rerun(ag, flat0, s10, flat_graph):
    """Rewind to the state before the update and run it eagerly on the same staged rollout: the parameters come out as the
    graph replay left them, to fp32 rounding (the head backward sums its weight and bias gradients across CTAs with atomics).
    Returns the reference-layout gradient of the eager run."""
    lr = ag._graph[0]
    o = ag.optimizer
    o.flat.copy_(flat0), o.s1.copy_(s10)
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
    flat0, s10 = o.flat.clone(), o.s1.clone()
    before = orc.flat().clone()
    r = _rollout(ag, rec)
    loss_dev = float(ag.last_loss)
    flat1 = o.flat.clone()
    grad = _eager_rerun(ag, flat0, s10, flat1)
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
def test_consecutive_rollouts(rl):
    """Four rollouts in a row: every rollout's loss and step follow the float64 oracle continued from the device's parameters
    and RMSprop state (``Oracle.anchor``); the actor's next head outputs equal an eager bf16 forward of a fresh copy of the
    updated network, so the next replay acts with theta_{k+1}."""
    from deeprl_b200.network import fused
    from deeprl_b200.network.fused import frame_scale
    ag = _agent(rl, max_steps=0)
    rec = Recorder(ag)
    orc = Oracle(ag)
    lr, actor = ag._graph
    for k in range(4):
        online = _flat(ag.network)
        orc.anchor(ag)
        r = _rollout(ag, rec)
        np.testing.assert_allclose(float(ag.last_loss), orc.update(r), rtol=2e-2, err_msg="rollout %d" % k)
        d_dev, d_orc = _flat(ag.network) - online, orc.flat() - online
        assert cosine(d_dev, d_orc) > 0.98, (k, cosine(d_dev, d_orc))
        np.testing.assert_allclose(float(d_dev.norm()), float(d_orc.norm()), rtol=5e-2, err_msg="rollout %d" % k)
        rec.inner(ag.states, 0)
        got = lr.act_out[0].cpu()
        fresh = ag.config.network_fn()
        fresh.load_state_dict(ag.network.state_dict())
        with torch.no_grad(), frame_scale(ag.config.state_normalizer.coef):
            phi = fresh.phi_body(actor.x.permute(0, 3, 1, 2))
            ref = fused.ac_head(phi, fresh.fc_action, fresh.fc_critic).cpu()
        assert torch.equal(got, ref), k


@pytest.mark.gpu
def test_a_step_is_graph_replays_only(rl, monkeypatch):
    """After capture, a step makes no C-ABI launch and exactly T + 1 graph replays, the last the update's."""
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
    """Save after 3 steps, load into an agent with the same Philox key that has already captured its graphs and trained one
    step, give it the same optimizer state, Philox counter and env stream, and step both: the same parameters (load()
    refreshed the packed operands)."""
    a = _agent(rl, seed=1, max_steps=0)
    for _ in range(3):
        a.step()
    torch.cuda.synchronize()
    a.save(str(tmp_path / "ck"))
    b = _agent(rl, seed=1, max_steps=0)
    b.step()                                               # graphs captured and trained from b's own weights
    assert a._graph[0].seed == b._graph[0].seed
    assert not torch.equal(_flat(a.network), _flat(b.network))
    b.load(str(tmp_path / "ck"))
    assert torch.equal(_flat(a.network), _flat(b.network))
    # what the checkpoint does not hold: the optimizer state, the Philox counter and the envs
    b.optimizer.s1.copy_(a.optimizer.s1), b.optimizer.s2.copy_(a.optimizer.s2)
    b._graph[0].counter.copy_(a._graph[0].counter)
    for ea, eb in zip(a.task.env.envs, b.task.env.envs):
        while hasattr(ea, "env"):                          # the SyntheticAtariEnv under the wrappers
            ea, eb = ea.env, eb.env
        eb.rng.set_state(ea.rng.get_state())
        eb.frames = list(ea.frames)
    b.states, b.total_steps = a.states, a.total_steps
    for _ in range(2):
        for ag in (a, b):
            ag.step()
        torch.cuda.synchronize()
        # equal up to the fp32 rounding of the head backward's atomic sums (see _eager_rerun); operands left stale by load()
        # would change the actions and gradients themselves, and the step (about 10 lr = 1e-3 per parameter) with them
        err = float((_flat(a.network) - _flat(b.network)).abs().max())
        assert err <= 1e-6, err


@pytest.mark.gpu
def test_launcher_end_to_end(rl):
    """examples.a2c_pixel(cuda_graph=True) through run_steps: the graph path runs and the loss is finite."""
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
