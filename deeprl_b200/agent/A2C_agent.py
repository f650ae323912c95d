"""Synchronous advantage actor-critic behind the reference's interface (``deep_rl/agent/A2C_agent.py:13-64``).

The rollout keeps the autograd graph of its T forward passes exactly like the reference (``storage.feed(prediction)``
stores tensors with grad, A2C_agent.py:31) and does ONE backward.  On a CUDA device the GAE recurrence and the
objective (+ its gradient with respect to log-prob / entropy / value) are the kernels of ``csrc/onpolicy.cu``; on
``select_device(-1)`` -- BASELINE configs[0], "a2c_feature CartPole, 8 workers, CPU only, plumbing" -- the same
statements run as torch expressions, which is the reference's own path, not a fallback for a missing library.

``config.device_a2c = True`` (off by default) runs the whole step on the device for the feature launchers' networks: one
``b2rl_a2c_actor_step`` launch per env step and one ``b2rl_a2c_update`` launch per rollout (csrc/a2c.cu, component/actor.py
``DeviceA2C``).  The actions are then drawn from the device's Philox stream, not from torch's generator.  Configurations the
kernels do not cover raise ``NotImplementedError`` naming the unmet condition.

``config.cuda_graph = True`` (off by default) runs each ``step()`` of a CategoricalActorCriticNet on a wgmma NatureConvBody at
bf16 (``a2c_pixel`` with ``Config.COMPUTE_DTYPE = torch.bfloat16``) as captured graphs: one ``GraphedQActor`` replay per env
step (pinned upload of the frame stacks into the rollout arena, the body, the actor-critic head with the action drawn on the
device, the actions down to the host) and one ``GraphedA2CLearner`` replay per rollout (learner.py).  The actions then come
from the device's Philox stream (keyed from torch's seeded generator, as with ``config.device_a2c``), not from torch's
``Categorical.sample``.  The torch optimizer is replaced by a ``FlatOptimizer`` with its hyper-parameters; the network's
parameters become views into its arena, so ``state_dict()`` is always current.  Configurations it does not cover
(``component/coverage.py a2c_graph_unsupported``; the reason is kept in ``graph_refusal``) keep the eager path;
``config.device_a2c`` takes precedence.
"""
import numpy as np
import torch
import torch.nn as nn

from .. import ops
from ..component import Storage
from ..utils import philox_seed, tensor, to_np
from .BaseAgent import BaseAgent


def gae_torch(reward, mask, value, discount, tau, use_gae):
    """A2C_agent.py:43-53 == PPO_agent.py:51-61 (torch statements; CPU device only)."""
    T = len(reward)
    adv = torch.zeros_like(value[0])
    ret = value[T].detach()
    advs, rets = [None] * T, [None] * T
    for i in reversed(range(T)):
        ret = reward[i] + discount * mask[i] * ret
        if not use_gae:
            adv = ret - value[i].detach()
        else:
            td = reward[i] + discount * mask[i] * value[i + 1].detach() - value[i].detach()
            adv = adv * tau * discount * mask[i] + td
        advs[i], rets[i] = adv.detach(), ret.detach()
    return advs, rets


def compute_advantages(storage, config, last_v, exact=True):
    """Fill ``storage.advantage`` / ``storage.ret`` (lists of (N,1) tensors) from reward / mask / v."""
    T = config.rollout_length
    v = [x.detach() for x in storage.v[:T]] + [last_v.detach()]
    if v[0].is_cuda:
        adv, ret = ops.gae(torch.stack(storage.reward[:T]), torch.stack(storage.mask[:T]), torch.stack(v),
                           config.discount, config.gae_tau, config.use_gae, exact=exact)
        storage.advantage, storage.ret = list(adv.unbind(0)), list(ret.unbind(0))
    else:
        storage.advantage, storage.ret = gae_torch(storage.reward[:T], storage.mask[:T], v, config.discount,
                                                   config.gae_tau, config.use_gae)


class A2CAgent(BaseAgent):
    def __init__(self, config):
        BaseAgent.__init__(self, config)
        self.config = config
        self.task = config.task_fn()
        self.network = config.network_fn()
        self.optimizer = config.optimizer_fn(self.network.parameters())
        self.total_steps = 0
        self.states = self.task.reset()
        self.last_loss = None
        self._graph = None                                  # (GraphedA2CLearner, GraphedQActor), False: eager; decided once
        self.graph_refusal = None
        self.device_a2c = None
        if getattr(config, "device_a2c", False):
            from ..component.actor import DeviceA2C
            self.device_a2c = DeviceA2C(self.network, self.optimizer, config, philox_seed())
            self.optimizer = self.device_a2c.opt

    def eval_step(self, state):
        with torch.no_grad():
            prediction = self.network(self.config.state_normalizer(np.asarray([np.asarray(s) for s in state])))
        return to_np(prediction["action"])

    def load(self, filename):
        BaseAgent.load(self, filename)
        if self._graph:
            self._graph[0].refresh_packed()                # the next step trains (and acts) from the loaded weights

    def step(self):
        if self.device_a2c is not None:
            return self._step_device()
        if self._graph_ok():
            return self._step_graph()
        config = self.config
        storage = Storage(config.rollout_length)
        states = self.states
        for _ in range(config.rollout_length):
            prediction = self.network(config.state_normalizer(np.asarray([np.asarray(s) for s in states])))
            next_states, rewards, terminals, info = self.task.step(to_np(prediction["action"]))
            self.record_online_return(info)
            rewards = config.reward_normalizer(rewards)
            storage.feed(prediction)
            storage.feed({"reward": tensor(rewards).unsqueeze(-1), "mask": tensor(1 - terminals).unsqueeze(-1)})
            states = next_states
            self.total_steps += config.num_workers

        self.states = states
        prediction = self.network(config.state_normalizer(np.asarray([np.asarray(s) for s in states])))
        storage.feed(prediction)
        storage.placeholder()
        compute_advantages(storage, config, prediction["v"])

        entries = storage.extract(["log_pi_a", "v", "ret", "advantage", "entropy"])
        self.optimizer.zero_grad()
        if entries.v.is_cuda:
            r = ops.a2c_loss_fused(entries.log_pi_a.detach(), entries.entropy.detach(), entries.v.detach(),
                                   entries.advantage, entries.ret, config.entropy_weight, config.value_loss_weight)
            shape = entries.v.shape
            torch.autograd.backward([entries.log_pi_a, entries.entropy, entries.v],
                                    [r["dlogp"].view(shape), r["dent"].view(shape), r["dv"].view(shape)])
            self.last_loss = r["out"][0]
        else:
            policy_loss = -(entries.log_pi_a * entries.advantage).mean()
            value_loss = 0.5 * (entries.ret - entries.v).pow(2).mean()
            entropy_loss = entries.entropy.mean()
            loss = policy_loss - config.entropy_weight * entropy_loss + config.value_loss_weight * value_loss
            loss.backward()
            self.last_loss = loss.detach()
        nn.utils.clip_grad_norm_(self.network.parameters(), config.gradient_clip)
        self.optimizer.step()

    def _step_device(self):
        """``step()`` with ``config.device_a2c``: T actor launches, each followed by ``task.step`` on the host; rewards and masks
        stay in host arrays until the rollout ends; then the final observations, one upload, and one update launch."""
        config, dev = self.config, self.device_a2c
        dev.begin_rollout()
        states = self.states
        for t in range(config.rollout_length):
            action = dev.act(t, states)
            next_states, rewards, terminals, info = self.task.step(action)
            self.record_online_return(info)
            dev.rewards[t] = np.asarray(config.reward_normalizer(rewards), dtype=np.float32)   # tensor(): float32
            dev.masks[t] = np.asarray(1 - terminals, dtype=np.float32)
            states = next_states
            self.total_steps += config.num_workers
        self.states = states
        self.last_loss = dev.update(config.state_normalizer(np.asarray([np.asarray(s) for s in states])))

    # ------------------------------------------------------------------ config.cuda_graph (opt-in)
    def _graph_ok(self):
        """Decided on the first step: the captured actor + update serve this configuration (``a2c_graph_unsupported``), or the
        eager path runs (the reason is kept in ``graph_refusal``)."""
        if self._graph is None:
            from ..component.actor import GraphedQActor
            from ..component.coverage import a2c_graph_unsupported
            from ..learner import GraphedA2CLearner
            config = self.config
            self.graph_refusal = a2c_graph_unsupported(config, self.network, self.optimizer, self.states)
            self._graph = False
            if self.graph_refusal is None:
                self.optimizer = ops.FlatOptimizer.from_torch(self.optimizer, list(self.network.parameters()))
                coef = config.state_normalizer.coef
                lr = GraphedA2CLearner(self.network, self.optimizer, config.rollout_length, config.num_workers, philox_seed(),
                                       config.discount, config.gae_tau, config.use_gae, config.entropy_weight,
                                       config.value_loss_weight, config.gradient_clip, coef).capture()
                actor = GraphedQActor(self.network, None, config.num_workers, 4, (84, 84), coef, arena=lr.arena, run=lr.act,
                                      body=self.network.phi_body)
                self._graph = (lr, actor)
        return bool(self._graph)

    def _step_graph(self):
        """``step()`` with ``config.cuda_graph``: T actor replays (the action drawn on the device into the learner's action row
        t; its pinned download is the step's only synchronisation), each followed by ``task.step`` on the host, with rewards
        and masks written into the learner's pinned staging buffer; then the final states and one update replay."""
        config = self.config
        lr, actor = self._graph
        states = self.states
        for t in range(config.rollout_length):
            actions = actor.q_values(states, t)
            next_states, rewards, terminals, info = self.task.step(actions)
            self.record_online_return(info)
            lr.h_reward[t].numpy()[...] = np.asarray(config.reward_normalizer(rewards), dtype=np.float32)   # tensor(): float32
            lr.h_mask[t].numpy()[...] = 1 - np.asarray(terminals, dtype=np.float32)
            states = next_states
            self.total_steps += config.num_workers
        self.states = states
        lr.stage_final(states)
        self.last_loss = lr.update()
