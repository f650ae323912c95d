"""``ppo_pixel`` on the captured sm_90a path (``config.cuda_graph``; PPOAgent ``_step_graph``): one GraphedQActor replay per
env step running the body and the actor-critic head with the action drawn on the device (as ``a2c_pixel``), and one
GraphedPPOPixelLearner replay per rollout: the final states' value, ``b2rl_ppo_rollout_prep`` (old log-probabilities, GAE),
advantage normalisation, then every epoch's minibatch updates unrolled, each with ONE ``b2rl_ppo_cat_loss`` launch
(csrc/onpolicy.cu) and an Adam step at the learning rate the host writes for the rollout (``b2rl_nature_fused_opt_lr``).

CPU: the float64 restatement of the shared-representation PPO update against autograd on the reference's own statements; the
float64 reference of the loss kernel's outputs against autograd (ratios below, inside and above the clip range, ties); the
coverage predicate (``ppo_graph_unsupported``) and the eager path of refused configurations; the learning rate the agent writes
against ``LambdaLR``; the new kernels' registers and spills.
GPU: the kernels against float64 and ``ops.gae(exact=True)``; the update's final-state value against the actor's; the
minibatch rows against ``random_sample``; one update, the launcher's schedule and consecutive rollouts against the float64
oracle; launch accounting; checkpoints; the launchers."""
import gc
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
from oracle import agents, losses, nets  # noqa: E402

CLIP, EW = 0.1, 0.01                                  # the launcher's ppo_ratio_clip and entropy_weight (examples.py ppo_pixel)


# ------------------------------------------------------------------------------------------------ float64 references
def ppo_pixel_update(sd, params, opt, states, actions, rewards, masks, batches, discount, tau, use_gae, clip, entropy_weight,
                     gradient_clip, body):
    """PPO_agent.py:29-99 with ``config.shared_repr`` for one rollout whose env interaction and minibatch rows are given, from
    oracle/nets.py and oracle/losses.py: the trunk is a function ``phi = body(sd, x)`` (``pixel_body`` for the NatureConvBody)
    with DummyBody actor / critic bodies.  ``states`` (T+1, N, ...), ``actions`` (T, N), ``rewards`` / ``masks`` (T, N, 1),
    ``batches``: the rows of every minibatch of every epoch, in order (what ``random_sample`` yielded).  Returns (adv
    normalised, ret, old log pi_a, [(policy_loss, value_loss, approx_kl) per minibatch], [clip_grad_norm_'s total norm])."""
    T, N = actions.shape

    def ac(x, action):
        phi = body(sd, x)
        dist = torch.distributions.Categorical(logits=F.linear(phi, sd["fc_action.weight"], sd["fc_action.bias"]))
        return dict(log_pi_a=dist.log_prob(action).unsqueeze(-1), entropy=dist.entropy().unsqueeze(-1),
                    v=F.linear(phi, sd["fc_critic.weight"], sd["fc_critic.bias"]))

    with torch.no_grad():
        preds = [ac(states[t], actions[t]) for t in range(T)]
        last = ac(states[T], actions[T - 1])
    v = torch.stack([p["v"] for p in preds] + [last["v"]])
    adv, ret = losses.gae(rewards, masks, v, discount, tau, use_gae)
    S = states[:T].reshape(T * N, *states.shape[2:])
    act = actions.reshape(-1)
    lp_old = torch.cat([p["log_pi_a"] for p in preds])
    adv, ret = losses.normalize_advantage(adv.reshape(-1, 1)), ret.reshape(-1, 1)
    stats, norms = [], []
    for idx in batches:
        idx = torch.as_tensor(np.asarray(idx)).long()
        out = ac(S[idx], act[idx])
        pl, vl, kl = losses.ppo_losses(out["log_pi_a"], out["entropy"], out["v"], lp_old[idx], adv[idx], ret[idx], clip,
                                       entropy_weight)
        opt.zero_grad()
        (pl + vl).backward()
        norms.append(float(torch.nn.utils.clip_grad_norm_(params, gradient_clip)))
        opt.step()
        stats.append((float(pl.detach()), float(vl.detach()), float(kl.detach())))
    return adv.reshape(-1), ret.reshape(-1), lp_old.reshape(-1), stats, norms


def pixel_body(sd, x):
    """ImageNormalizer (x / 255) then the NatureConvBody (network_bodies.py:27-33) on uint8 stacks [N, 4, 84, 84]."""
    return nets.nature_body(sd, x.to(torch.float64) / 255.0, prefix="phi_body.")


def cat_loss_reference(head, idx, action, old_logp, adv, ret, clip, ew):
    """float64 outputs of ``b2rl_ppo_cat_loss``: geff [B, A+1] and [policy_loss, value_loss, approx_kl], with
    ppo_loss_kernel's rules: torch.min splits a tie evenly, clamp passes the gradient on the closed interval."""
    h = np.asarray(head, np.float64)
    B, A = h.shape[0], h.shape[1] - 1
    i = np.asarray(idx)
    a = np.asarray(action).reshape(-1)[i]
    olp, ad, rt = (np.asarray(x, np.float64).reshape(-1)[i] for x in (old_logp, adv, ret))
    z = h[:, :A]
    lp = z - z.max(1, keepdims=True)
    lp = lp - np.log(np.exp(lp).sum(1, keepdims=True))
    p = np.exp(lp)
    H = -(p * lp).sum(1)
    rows = np.arange(B)
    lpa = lp[rows, a]
    r = np.exp(lpa - olp)
    obj, objc = r * ad, np.clip(r, 1 - clip, 1 + clip) * ad
    inside = (r >= 1 - clip) & (r <= 1 + clip)
    g = np.where(obj < objc, ad * r, np.where(obj > objc, np.where(inside, ad * r, 0.0), 0.5 * ad * r + np.where(inside, 0.5 * ad * r, 0.0)))
    onehot = np.zeros((B, A))
    onehot[rows, a] = 1.0
    geff = np.zeros((B, A + 1))
    geff[:, :A] = (-g / B)[:, None] * (onehot - p) + (ew / B) * p * (lp + H[:, None])
    v = h[:, A]
    geff[:, A] = (v - rt) / B
    stats = np.array([-np.mean(np.minimum(obj, objc)) - ew * np.mean(H), 0.5 * np.mean((rt - v) ** 2), np.mean(olp - lpa)])
    return geff, stats


RATIOS = np.array([0.3, 0.7, 0.85, 0.95, 1.0, 1.0, 1.04, 1.15, 1.6, 3.0])    # below, inside (ties) and above [0.9, 1.1]


def cat_loss_case(B, A, seed, rows_total=None):
    """Head outputs, minibatch rows of a larger rollout, and rollout arrays whose old log-probabilities put each row's ratio
    at one of ``RATIOS`` (at least 1e-2 from a clip edge, so fp32 and float64 take the same branch); a tenth of the
    advantages are exactly zero."""
    g = np.random.RandomState(seed)
    R = rows_total or 3 * B + 5
    head = np.concatenate([g.randn(B, A) * 2.0, g.randn(B, 1)], axis=1).astype(np.float32)
    idx = g.choice(R, size=B, replace=False).astype(np.int64)
    action = g.randint(0, A, size=R).astype(np.int64)
    adv = g.randn(R).astype(np.float32)
    adv[g.rand(R) < 0.1] = 0.0
    ret = g.randn(R).astype(np.float32)
    h = head.astype(np.float64)
    lp = h[:, :A] - h[:, :A].max(1, keepdims=True)
    lp = lp - np.log(np.exp(lp).sum(1, keepdims=True))
    old = g.randn(R).astype(np.float32)
    old[idx] = (lp[np.arange(B), action[idx]] - np.log(RATIOS[np.arange(B) % len(RATIOS)])).astype(np.float32)
    return head, idx, action, old, adv, ret


# ------------------------------------------------------------------------------------------------ CPU
class _RefNet(torch.nn.Module):
    """CategoricalActorCriticNet with a tanh FC phi_body and DummyBody actor / critic bodies (network_heads.py:173-255)."""

    def __init__(self, sd):
        super().__init__()
        D, H = sd["phi_body.layers.0.weight"].shape[1], sd["phi_body.layers.0.weight"].shape[0]
        A = sd["fc_action.weight"].shape[0]
        self.phi = torch.nn.Sequential(torch.nn.Linear(D, H), torch.nn.Tanh(), torch.nn.Linear(H, H), torch.nn.Tanh())
        self.fc_action, self.fc_critic = torch.nn.Linear(H, A), torch.nn.Linear(H, 1)
        self.double()
        with torch.no_grad():
            for (k, v), p in zip(sd.items(), self.parameters()):
                p.copy_(v)

    def forward(self, obs, action=None):
        phi = self.phi(obs)
        dist = torch.distributions.Categorical(logits=self.fc_action(phi))
        if action is None:
            action = dist.sample()
        return {"action": action, "log_pi_a": dist.log_prob(action).unsqueeze(-1), "entropy": dist.entropy().unsqueeze(-1),
                "v": self.fc_critic(phi)}


def _reference_step(net, opt, states, actions, rewards, masks, config, seed):
    """PPO_agent.py:29-99 statement for statement (shared_repr), with the rollout's env interaction given."""
    T = actions.shape[0]
    st = {k: [] for k in ("state", "action", "log_pi_a", "v", "reward", "mask")}
    for t in range(T):
        prediction = net(states[t], actions[t])
        for k in ("action", "log_pi_a", "v"):
            st[k].append(prediction[k])
        st["reward"].append(rewards[t]), st["mask"].append(masks[t]), st["state"].append(states[t])
    prediction = net(states[T], actions[T - 1])
    st["v"].append(prediction["v"])
    advantages = torch.zeros_like(prediction["v"])
    returns = prediction["v"].detach()
    adv, ret = [None] * T, [None] * T
    for i in reversed(range(T)):
        returns = st["reward"][i] + config.discount * st["mask"][i] * returns
        td_error = st["reward"][i] + config.discount * st["mask"][i] * st["v"][i + 1] - st["v"][i]
        advantages = advantages * config.gae_tau * config.discount * st["mask"][i] + td_error
        adv[i], ret[i] = advantages.detach(), returns.detach()
    cat = lambda x: torch.cat(x, dim=0)
    e = types.SimpleNamespace(state=cat(st["state"]), action=cat(st["action"]), log_pi_a=cat(st["log_pi_a"]).detach(),
                              ret=cat(ret), advantage=cat(adv))
    e.advantage.copy_((e.advantage - e.advantage.mean()) / e.advantage.std())
    np.random.seed(seed)
    for _ in range(config.optimization_epochs):
        for batch_indices in agents.random_sample(np.arange(e.state.size(0)), config.mini_batch_size):
            batch_indices = torch.from_numpy(np.asarray(batch_indices)).long()
            prediction = net(e.state[batch_indices], e.action[batch_indices])
            ratio = (prediction["log_pi_a"] - e.log_pi_a[batch_indices]).exp()
            obj = ratio * e.advantage[batch_indices]
            obj_clipped = ratio.clamp(1.0 - config.ppo_ratio_clip, 1.0 + config.ppo_ratio_clip) * e.advantage[batch_indices]
            policy_loss = -torch.min(obj, obj_clipped).mean() - config.entropy_weight * prediction["entropy"].mean()
            value_loss = 0.5 * (e.ret[batch_indices] - prediction["v"]).pow(2).mean()
            opt.zero_grad()
            (policy_loss + value_loss).backward()
            torch.nn.utils.clip_grad_norm_(net.parameters(), config.gradient_clip)
            opt.step()
    return e


def test_shared_oracle_matches_the_reference_statements():
    """The float64 restatement (``ppo_pixel_update``, built from oracle/nets.py and oracle/losses.py) equals autograd on
    PPO_agent.py's own statements over a torch module: advantages, returns, old log-probabilities and the parameters after
    two epochs of three minibatches of Adam steps, on a tanh FC trunk."""
    g = torch.Generator().manual_seed(5)
    T, N, D, H, A = 6, 4, 7, 16, 5
    sd = {"phi_body.layers.0.weight": torch.randn(H, D, generator=g, dtype=torch.float64) * 0.3,
          "phi_body.layers.0.bias": torch.randn(H, generator=g, dtype=torch.float64) * 0.1,
          "phi_body.layers.1.weight": torch.randn(H, H, generator=g, dtype=torch.float64) * 0.3,
          "phi_body.layers.1.bias": torch.randn(H, generator=g, dtype=torch.float64) * 0.1,
          "fc_action.weight": torch.randn(A, H, generator=g, dtype=torch.float64) * 0.3,
          "fc_action.bias": torch.randn(A, generator=g, dtype=torch.float64) * 0.1,
          "fc_critic.weight": torch.randn(1, H, generator=g, dtype=torch.float64) * 0.3,
          "fc_critic.bias": torch.randn(1, generator=g, dtype=torch.float64) * 0.1}
    states = torch.randn(T + 1, N, D, generator=g, dtype=torch.float64)
    actions = torch.randint(0, A, (T, N), generator=g)
    rewards = torch.randint(-1, 2, (T, N, 1), generator=g).double()
    masks = (torch.rand(T, N, 1, generator=g) > 0.2).double()
    cfg = types.SimpleNamespace(discount=0.99, gae_tau=0.95, optimization_epochs=2, mini_batch_size=8, ppo_ratio_clip=0.1,
                                entropy_weight=0.01, gradient_clip=0.5)
    net = _RefNet(sd)
    opt = torch.optim.Adam(net.parameters(), lr=2.5e-3)
    e = _reference_step(net, opt, states, actions, rewards, masks, cfg, seed=11)

    np.random.seed(11)
    batches = [b for _ in range(cfg.optimization_epochs) for b in agents.random_sample(np.arange(T * N), cfg.mini_batch_size)]
    leaves = agents.leafify(sd)
    params = list(leaves.values())
    adam = torch.optim.Adam(params, lr=2.5e-3)
    adv, ret, lp, stats, _ = ppo_pixel_update(leaves, params, adam, states, actions, rewards, masks, batches, cfg.discount,
                                              cfg.gae_tau, True, cfg.ppo_ratio_clip, cfg.entropy_weight, cfg.gradient_clip,
                                              lambda s, x: nets.fc_body(s, x, "phi_body.", torch.tanh))
    assert len(stats) == 6
    np.testing.assert_allclose(adv.numpy(), e.advantage.reshape(-1).numpy(), rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(ret.numpy(), e.ret.reshape(-1).numpy(), rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(lp.numpy(), e.log_pi_a.reshape(-1).numpy(), rtol=1e-13, atol=1e-13)
    for (k, leaf), p in zip(leaves.items(), net.parameters()):
        np.testing.assert_allclose(leaf.detach().numpy(), p.detach().numpy(), rtol=1e-10, atol=1e-13, err_msg=k)
        assert not torch.equal(leaf.detach(), sd[k]), k


@pytest.mark.parametrize("A", [2, 6, 31])
@pytest.mark.parametrize("B", [1, 37, 256])
def test_loss_reference_matches_autograd(B, A):
    """The float64 reference of geff / stats against autograd on oracle/losses.py ppo_losses over a Categorical of the head's
    logits: ratios below, inside and above the clip range, inside ties (clamp(r) == r) and zero advantages."""
    head, idx, action, old, adv, ret = cat_loss_case(B, A, seed=B * 10 + A)
    geff, stats = cat_loss_reference(head, idx, action, old, adv, ret, CLIP, EW)
    h = torch.tensor(head, dtype=torch.float64, requires_grad=True)
    i = torch.from_numpy(idx)
    dist = torch.distributions.Categorical(logits=h[:, :A])
    lp = dist.log_prob(torch.from_numpy(action)[i]).unsqueeze(-1)
    t = lambda x: torch.from_numpy(np.asarray(x, np.float64))[i].unsqueeze(-1)
    pl, vl, kl = losses.ppo_losses(lp, dist.entropy().unsqueeze(-1), h[:, A:], t(old), t(adv), t(ret), CLIP, EW)
    (pl + vl).backward()
    np.testing.assert_allclose(stats, [float(pl), float(vl), float(kl)], rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(geff, h.grad.numpy(), rtol=1e-10, atol=1e-15)


def _pixel_config(rl, **kw):
    """The configuration ``examples.ppo_pixel`` builds (examples.py), on whatever device is selected; the ``kw`` entries the
    launcher's own table would override (rollout_length, mini_batch_size, optimization_epochs, max_steps) are set on the config
    afterwards (the scheduler reads max_steps when it steps).  Built in
    a temporary directory: the launcher's logger opens its file under ./log."""
    import tempfile

    import examples
    after = {k: kw.pop(k) for k in ("rollout_length", "mini_batch_size", "optimization_epochs", "max_steps") if k in kw}
    got = []
    mp = pytest.MonkeyPatch()
    mp.setattr(examples, "run_steps", got.append)
    mp.chdir(tempfile.mkdtemp(prefix="ppo_pixel_"))
    try:
        examples.ppo_pixel(game=kw.pop("game", "SyntheticAtari-v0"), cuda_graph=True, **kw)
    finally:
        mp.undo()
    ag = got[0]
    for k, v in after.items():
        setattr(ag.config, k, v)
    return ag


def _refusals(rl):
    """(name, config change, network_fn, expected reason) for every refused configuration."""
    ac = lambda A=4, **k: (lambda: rl.CategoricalActorCriticNet(None, A, **k))
    return [
        ("fp32", dict(dtype=torch.float32), None, "compute dtype"),
        ("not_shared", dict(shared_repr=False), None, "shared_repr is not set"),
        ("short_minibatch", dict(mini_batch_size=300), None, "not a multiple of mini_batch_size 300"),
        ("fc_body", {}, ac(phi_body=rl.FCBody(4 * 84 * 84)), "captured update implements NatureConvBody"),
        ("noisy", {}, ac(phi_body=rl.NatureConvBody(noisy_linear=True)), "NoisyLinear"),
        ("actor_body", {}, ac(phi_body=rl.NatureConvBody(), actor_body=rl.FCBody(512)), "DummyBody"),
        ("actions", {}, ac(32, phi_body=rl.NatureConvBody()), "fewer than 32"),
        ("normalizer", dict(state_normalizer=rl.MeanStdNormalizer()), None, "RescaleNormalizer"),
        ("no_cuda_graph", dict(cuda_graph=False), None, "cuda_graph is not set"),
        ("sgd", dict(optimizer_fn=lambda p: torch.optim.SGD(p, 1e-3)), None, "optimizer is SGD"),
        ("adam_amsgrad", dict(optimizer_fn=lambda p: torch.optim.Adam(p, 1e-3, amsgrad=True)), None, "optimizer is Adam"),
    ]


def _predicate(rl, cfg, net):
    from deeprl_b200.component.coverage import ppo_graph_unsupported
    opt = cfg.optimizer_fn(net.parameters())
    states = cfg.task_fn().reset()
    return ppo_graph_unsupported(cfg, net, opt, states)


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
    """The launcher at its default fp32 compute on the host: the agent notes the refusal and its step() is the eager path
    (torch Adam, a learning rate from the scheduler, statistics of the last minibatch)."""
    import deeprl_b200 as rl
    rl.select_device(-1)
    np.random.seed(0), torch.manual_seed(0)
    ag = _pixel_config(rl, max_steps=1000, num_workers=2, rollout_length=2, mini_batch_size=2, optimization_epochs=1)
    before = {k: v.clone() for k, v in ag.network.state_dict().items()}
    ag.step()
    assert ag._graph is None and "compute dtype" in ag.graph_refusal
    assert isinstance(ag.opt, torch.optim.Adam) and ag.opt.param_groups[0]["lr"] == pytest.approx(2.5e-4 * (1 - 4 / 1000))
    assert any(not torch.equal(before[k], v) for k, v in ag.network.state_dict().items())


def test_graph_learning_rate_follows_lambda_lr():
    """What ``graph_lr`` writes for each rollout equals ``LambdaLR``'s learning rate after ``step(total_steps)`` on a
    separate Adam with the launcher's lr, and 2.5e-4 * (1 - total_steps / max_steps)."""
    import deeprl_b200 as rl
    rl.select_device(-1)
    ag = _pixel_config(rl, max_steps=10 * 1024)
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.Adam([p], lr=2.5e-4)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda step: 1 - step / (10 * 1024))
    for k in range(1, 6):
        ag.total_steps = k * 1024
        got = ag.graph_lr()
        sched.step(k * 1024)
        assert got == opt.param_groups[0]["lr"]
        assert got == pytest.approx(2.5e-4 * (1 - k / 10), rel=1e-12)


@pytest.mark.parametrize("src,kernel", [("onpolicy.cu", "ppo_cat_loss_kernel"), ("onpolicy.cu", "ppo_rollout_prep_kernel"),
                                        ("tail.cu", "nature_fused_opt_kernel")])
def test_kernel_registers_and_spills(src, kernel):
    """nvcc -Xptxas -v: the new kernels (and the optimizer kernel with its device learning rate) compile for sm_90a without
    spills."""
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


def _run_cat_loss(head, idx, action, old, adv, ret):
    from deeprl_b200 import ops
    r = ops.ppo_cat_loss(_cuda(head), _cuda(idx, torch.int64), _cuda(action, torch.int64), _cuda(old), _cuda(adv), _cuda(ret),
                         CLIP, EW)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in r.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("A", [2, 6, 18, 31])
@pytest.mark.parametrize("B", [1, 37, 256])
def test_cat_loss_kernel(rl, B, A):
    """geff and [policy_loss, value_loss, approx_kl] against float64 within fp32 rounding, with ratios across both clip edges
    (B = 256: 32 CTAs and the last-CTA reduction); the columns past A stay zero; a second launch gives the same bits."""
    head, idx, action, old, adv, ret = cat_loss_case(B, A, seed=1000 + B * 10 + A)
    got = _run_cat_loss(head, idx, action, old, adv, ret)
    geff, stats = cat_loss_reference(head, idx, action, old, adv, ret, CLIP, EW)
    g = got["geff"].numpy()
    np.testing.assert_allclose(g[:, :A + 1], geff, rtol=1e-4, atol=1e-6 * np.abs(geff).max())
    assert not g[:, A + 1:].any()
    np.testing.assert_allclose(got["stats"].numpy(), stats, rtol=2e-5, atol=1e-6)
    again = _run_cat_loss(head, idx, action, old, adv, ret)
    assert all(torch.equal(got[k], again[k]) for k in got)


@pytest.mark.gpu
@pytest.mark.parametrize("use_gae", [True, False])
@pytest.mark.parametrize("T,N,A", [(1, 2, 2), (128, 8, 6), (7, 37, 31)])
def test_rollout_prep(rl, T, N, A, use_gae):
    """ret / adv before normalisation the bits of ops.gae(exact=True) on the head's values; the old log-probabilities and the
    normalised advantages against float64."""
    from deeprl_b200 import ops
    g = np.random.RandomState(T * 100 + N + A)
    head = np.concatenate([g.randn((T + 1) * N, A) * 2.0, g.randn((T + 1) * N, 1)], axis=1).astype(np.float32)
    action = g.randint(0, A, size=(T, N)).astype(np.int64)
    reward = g.randint(-1, 2, size=(T, N)).astype(np.float32)
    mask = (g.rand(T, N) > 0.2).astype(np.float32)
    r = ops.ppo_rollout_prep(_cuda(head), _cuda(action, torch.int64), _cuda(reward), _cuda(mask), 0.99, 0.95, use_gae)
    v = _cuda(head[:, A]).view(T + 1, N)
    adv_g, ret_g = ops.gae(_cuda(reward), _cuda(mask), v, 0.99, 0.95, use_gae, exact=True)
    torch.cuda.synchronize()
    assert torch.equal(r["adv"].cpu(), adv_g.cpu().view(-1)) and torch.equal(r["ret"].cpu(), ret_g.cpu().view(-1))
    h = head.astype(np.float64)[:T * N]
    lp = h[:, :A] - h[:, :A].max(1, keepdims=True)
    lp = lp - np.log(np.exp(lp).sum(1, keepdims=True))
    np.testing.assert_allclose(r["logp"].cpu().numpy(), lp[np.arange(T * N), action.reshape(-1)], rtol=1e-5, atol=1e-5)
    a64 = r["adv"].cpu().double().numpy()
    ops.normalize_advantage_(r["adv"])
    torch.cuda.synchronize()
    want = (a64 - a64.mean()) / a64.std(ddof=1)
    np.testing.assert_allclose(r["adv"].cpu().numpy(), want, rtol=1e-5, atol=1e-5)


# the examples' shapes: (T 128, N 8, minibatch 256, 4 epochs) is the launcher's; the small one keeps the float64 oracle quick
SMALL = dict(num_workers=8, rollout_length=8, mini_batch_size=32, optimization_epochs=2)


def _agent(rl, seed=0, **kw):
    gc.collect()                                           # the agents of earlier tests, with their graphs and pinned buffers
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
    """One agent step; returns what it trained on: states (T+1, N, 4, 84, 84) uint8, actions, rewards, masks (T, N), the
    minibatch rows of every epoch and the learning rate."""
    rec.clear()
    ag.step()
    torch.cuda.synchronize()
    lr = ag._graph[0]
    states = np.stack(rec.states + [np.stack([np.asarray(s) for s in ag._raw_states])])
    return types.SimpleNamespace(states=states, actions=np.stack(rec.actions), rewards=lr.h_reward.numpy().copy(),
                                 masks=lr.h_mask.numpy().copy(), batches=lr.h_idx.numpy().copy(),
                                 lr=float(lr.h_lr.numpy()[0]), out=torch.stack(rec.out))


def _sd64(net):
    return {k: v.detach().double().cpu().clone() for k, v in net.state_dict().items()}


class Oracle:
    """The float64 pixel PPO update (``ppo_pixel_update``) with its own Adam state."""

    def __init__(self, ag):
        self.sd = agents.leafify(_sd64(ag.network))
        self.params = list(self.sd.values())
        o = ag.flat_opt
        self.opt = torch.optim.Adam(self.params, lr=o.lr, betas=o.betas, eps=o.eps)
        self.cfg = ag.config

    def anchor(self, ag):
        """Continue from the agent's parameters and Adam state (moments and step count)."""
        o, named = ag.flat_opt, dict(ag.network.named_parameters())
        base = o.flat.data_ptr()
        step = float(o.step_dev.item())
        with torch.no_grad():
            for k, leaf in self.sd.items():
                p = named[k]
                off = (p.data_ptr() - base) // 4
                leaf.copy_(p.detach().double().cpu())
                st = self.opt.state[leaf]
                st["step"] = torch.tensor(step)
                st["exp_avg"] = o.s1[off:off + p.numel()].view_as(p).double().cpu().clone()
                st["exp_avg_sq"] = o.s2[off:off + p.numel()].view_as(p).double().cpu().clone()

    def update(self, r):
        c = self.cfg
        for grp in self.opt.param_groups:
            grp["lr"] = r.lr
        return ppo_pixel_update(self.sd, self.params, self.opt, torch.from_numpy(r.states), torch.from_numpy(r.actions),
                                torch.from_numpy(r.rewards).double().unsqueeze(-1),
                                torch.from_numpy(r.masks).double().unsqueeze(-1), list(r.batches), c.discount, c.gae_tau,
                                c.use_gae, c.ppo_ratio_clip, c.entropy_weight, c.gradient_clip, pixel_body)

    def flat(self):
        return torch.cat([v.detach().flatten() for v in self.sd.values()])


def _flat(net):
    return torch.cat([v.detach().double().cpu().flatten() for v in net.state_dict().values()])


def cosine(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


@pytest.mark.gpu
def test_final_value_is_the_actors(rl):
    """The (logits, v) of the final states the update graph computes at batch N (K1 over arena slot T) equal, bit for bit,
    an actor replay's on the same states with the same (pre-update) weights."""
    ag = _agent(rl, max_steps=10 ** 6, **SMALL)
    rec = Recorder(ag)
    lr = ag._graph[0]
    o = ag.flat_opt
    for _ in range(2):
        flat0 = o.flat.clone()
        _rollout(ag, rec)
        vT = lr.act_out[lr.T].cpu().clone()
        flat1 = o.flat.clone()
        o.flat.copy_(flat0)
        lr.refresh_packed()
        rec.inner(ag._raw_states, 0)
        torch.cuda.synchronize()
        assert torch.equal(lr.act_out[0].cpu(), vT)
        o.flat.copy_(flat1)
        lr.refresh_packed()


@pytest.mark.gpu
def test_minibatch_rows_are_random_sample(rl, monkeypatch):
    """The rows of every minibatch the graph used (its device copy of the upload) are what random_sample yields for the same
    numpy state, epoch after epoch; the arena rows are 4 x the rollout rows."""
    import deeprl_b200.agent.PPO_agent as mod
    ag = _agent(rl, max_steps=10 ** 6)
    lr = ag._graph[0]
    seen = []
    real = mod.random_sample
    monkeypatch.setattr(mod, "random_sample", lambda *a: (seen.append(np.random.get_state()) if not seen else None,
                                                          real(*a))[1])
    ag.step()
    torch.cuda.synchronize()
    np.random.set_state(seen[0])
    rows = ag.config.rollout_length * ag.config.num_workers
    want = np.stack([b for _ in range(ag.config.optimization_epochs)
                     for b in agents.random_sample(np.arange(rows), ag.config.mini_batch_size)])
    assert want.shape == (16, 256)
    assert np.array_equal(lr.d_idx.cpu().numpy(), want)
    assert np.array_equal(lr.d_arow.cpu().numpy(), 4 * want)


def _check_against_oracle(ag, orc, r, flat_before, tol_step, tol_stats, tag):
    """Last minibatch's statistics and every minibatch's pre-clip gradient norm (the first against the device's
    clip_grad_norm_ total norm), and the rollout's parameter step, against the float64 oracle."""
    _, _, _, stats, norms = orc.update(r)
    dev_stats = ag.last_stats.cpu().double().numpy()
    np.testing.assert_allclose(dev_stats[:2], stats[-1][:2], rtol=tol_stats, atol=1e-4, err_msg=tag)
    np.testing.assert_allclose(dev_stats[2], stats[-1][2], atol=5e-3, err_msg=tag)
    d_dev, d_orc = _flat(ag.network) - flat_before, orc.flat() - flat_before
    c = cosine(d_dev, d_orc)
    print("%s: stats dev %s oracle %s; step cosine %.5f, norms %.6g / %.6g" % (tag, dev_stats, stats[-1], c,
                                                                              float(d_dev.norm()), float(d_orc.norm())))
    assert c > tol_step[0], (tag, c)
    np.testing.assert_allclose(float(d_dev.norm()), float(d_orc.norm()), rtol=tol_step[1], err_msg=tag)
    return norms


@pytest.mark.gpu
@pytest.mark.parametrize("game", ["SyntheticAtari-v0", "SyntheticAtari-A18-v0"])
def test_one_update_matches_the_float64_oracle(rl, game):
    """E = 1 and rows = mini_batch_size (one Adam step): the policy and value losses within 2e-2 relative, approx_kl within
    5e-3, the pre-clip gradient norm within 5e-2 and the parameter step within cosine 0.98 / norm 5e-2 of the float64
    oracle (tests/test_gpu_step_vs_oracle.py's tolerances) on the same frames, weights, actions, rewards and masks."""
    ag = _agent(rl, game=game, max_steps=10 ** 6, num_workers=8, rollout_length=8, mini_batch_size=64,
                optimization_epochs=1)
    rec = Recorder(ag)
    orc = Oracle(ag)
    before = _flat(ag.network)
    r = _rollout(ag, rec)
    assert r.batches.shape == (1, 64)
    norms = _check_against_oracle(ag, orc, r, before, (0.98, 5e-2), 2e-2, game)
    np.testing.assert_allclose(float(ag.flat_opt.total_norm), norms[0], rtol=5e-2)


@pytest.mark.gpu
def test_launcher_schedule_matches_the_float64_oracle(rl):
    """The launcher's shape (T 128, N 8, 4 epochs x 4 minibatches of 256: 16 dependent Adam steps) for one rollout, at the
    one-step tolerances except the step cosine: > 0.97 (measured 0.989 on an H100), norm within 5e-2, the last minibatch's
    losses within 2e-2.  It holds because Adam moves each coordinate by about lr per step whatever the gradient's size: bf16
    rounding only changes the steps of coordinates whose gradient is near zero, so the 16 steps add their differences on
    those coordinates, not on the ones that carry the step's norm, and 16 steps at lr 2.5e-4 leave the rollout's later
    minibatches' losses within 1e-3 of the oracle's."""
    ag = _agent(rl, max_steps=10 ** 7)
    rec = Recorder(ag)
    orc = Oracle(ag)
    before = _flat(ag.network)
    r = _rollout(ag, rec)
    assert r.batches.shape == (16, 256)
    _check_against_oracle(ag, orc, r, before, (0.97, 5e-2), 2e-2, "launcher")


@pytest.mark.gpu
def test_consecutive_rollouts(rl):
    """Three rollouts with the learning rate decaying between them (max_steps = 4 rollouts): the device learning rate is
    LambdaLR's, and each rollout follows the float64 oracle continued from the device's parameters and Adam state; the next
    actor replay acts with the updated weights (its head outputs equal an eager bf16 forward of a fresh copy)."""
    from deeprl_b200.network import fused
    from deeprl_b200.network.fused import frame_scale
    rows = SMALL["num_workers"] * SMALL["rollout_length"]
    ag = _agent(rl, max_steps=4 * rows, **SMALL)
    rec = Recorder(ag)
    orc = Oracle(ag)
    lr, actor = ag._graph
    for k in range(3):
        online = _flat(ag.network)
        orc.anchor(ag)
        r = _rollout(ag, rec)
        assert float(lr.d_lr.cpu()) == np.float32(ag.opt.param_groups[0]["lr"])
        assert r.lr == np.float32(2.5e-4 * (1 - (k + 1) / 4))
        _check_against_oracle(ag, orc, r, online, (0.98, 5e-2), 2e-2, "rollout %d" % k)
        rec.inner(ag._raw_states, 0)
        got = lr.act_out[0].cpu()
        fresh = ag.config.network_fn()
        fresh.load_state_dict(ag.network.state_dict())
        with torch.no_grad(), frame_scale(ag.config.state_normalizer.coef):
            phi = fresh.phi_body(actor.x.permute(0, 3, 1, 2))
            ref = fused.ac_head(phi, fresh.fc_action, fresh.fc_critic).cpu()
        assert torch.equal(got, ref), k


@pytest.mark.gpu
def test_a_step_is_graph_replays_only(rl, monkeypatch):
    """After capture, a step makes no C-ABI launch and exactly T + 1 graph replays: T actor replays, then the update's (which
    holds the final states' forward)."""
    from deeprl_b200 import _lib
    ag = _agent(rl, max_steps=10 ** 6, **SMALL)
    ag.step()                                              # captures the actor's slot graphs
    torch.cuda.synchronize()
    replays = []
    real = torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda g: (replays.append(g), real(g))[1])
    _lib.reset_launch_count()
    ag.step()
    torch.cuda.synchronize()
    assert _lib.launch_count() == 0
    assert len(replays) == SMALL["rollout_length"] + 1 and replays[-1] is ag._graph[0].graph


@pytest.mark.gpu
def test_checkpoint_round_trip(rl, tmp_path):
    """Save after 3 steps, load into an agent with the same Philox key that has already captured its graphs and trained one
    step, give it the same Adam state, Philox counter, scheduler position, env stream and numpy state, and step both: the
    same parameters to fp32 rounding (the head backward's atomics are not bitwise deterministic), so load() refreshed the
    packed operands."""
    a = _agent(rl, seed=1, max_steps=10 ** 6, **SMALL)
    for _ in range(3):
        a.step()
    torch.cuda.synchronize()
    a.save(str(tmp_path / "ck"))
    b = _agent(rl, seed=1, max_steps=10 ** 6, **SMALL)
    b.step()
    assert a._graph[0].seed == b._graph[0].seed
    assert not torch.equal(_flat(a.network), _flat(b.network))
    b.load(str(tmp_path / "ck"))
    assert torch.equal(_flat(a.network), _flat(b.network))
    for t in ("s1", "s2", "step_dev"):
        getattr(b.flat_opt, t).copy_(getattr(a.flat_opt, t))
    b._graph[0].counter.copy_(a._graph[0].counter)
    for ea, eb in zip(a.task.env.envs, b.task.env.envs):
        while hasattr(ea, "env"):                          # the SyntheticAtariEnv under the wrappers
            ea, eb = ea.env, eb.env
        eb.rng.set_state(ea.rng.get_state())
        eb.frames = list(ea.frames)
    b._raw_states, b.states, b.total_steps = a._raw_states, a.states, a.total_steps
    for _ in range(2):
        state = np.random.get_state()
        a.step()
        np.random.set_state(state)
        b.step()
        torch.cuda.synchronize()
        err = float((_flat(a.network) - _flat(b.network)).abs().max())
        assert err <= 1e-5, err


@pytest.mark.gpu
def test_launcher_end_to_end(rl):
    """examples.ppo_pixel(cuda_graph=True) through run_steps: the graph path runs and the statistics are finite."""
    from deeprl_b200.utils.misc import run_steps
    np.random.seed(0), torch.manual_seed(0)
    ag = _pixel_config(rl)
    ag.config.max_steps = 2 * 128 * 8
    ag.config.eval_interval = 0
    run_steps(ag)
    assert ag._graph and ag.total_steps == 2 * 128 * 8
    assert ag.last_stats.is_cuda and np.isfinite(ag.last_stats.cpu().numpy()).all()


@pytest.mark.gpu
def test_fp32_launcher_and_refused_configuration_keep_the_eager_path(rl):
    """The launcher's default fp32 compute, and a bf16 configuration whose rollout is not whole minibatches, are refused with
    their reasons and train on today's eager path (torch Adam)."""
    rl.Config.COMPUTE_DTYPE = torch.float32
    try:
        np.random.seed(0), torch.manual_seed(0)
        ag = _pixel_config(rl, max_steps=10 ** 6, **SMALL)
        ag.step()
        assert ag._graph is None and "compute dtype" in ag.graph_refusal
        assert isinstance(ag.opt, torch.optim.Adam) and np.isfinite(ag.last_stats.cpu().numpy()).all()
    finally:
        rl.Config.COMPUTE_DTYPE = torch.bfloat16
    np.random.seed(0), torch.manual_seed(0)
    ag = _pixel_config(rl, max_steps=10 ** 6, **dict(SMALL, mini_batch_size=48))
    before = _flat(ag.network)
    ag.step()
    assert ag._graph is None and "mini_batch_size 48" in ag.graph_refusal
    assert isinstance(ag.opt, torch.optim.Adam) and not torch.equal(before, _flat(ag.network))
