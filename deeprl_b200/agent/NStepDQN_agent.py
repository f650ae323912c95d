"""n-step Q-learning behind the reference's interface (``deep_rl/agent/NStepDQN_agent.py:13-70``; SURVEY 8f-4).

``step()``: a ``rollout_length`` rollout with epsilon-greedy actions whose q-values keep their autograd graphs
(NStepDQN_agent.py:33-46), hard target sync on the reference's schedule inside the rollout (:48-49), bootstrap
``max_a target(s_T)`` (:56-57), backward return scan ``ret_t = r_t + discount * mask_t * ret_{t+1}`` (:58-60), loss
``0.5 * mean((q[a] - ret)^2)`` (:63), clip, optimizer step (:64-67).

On a CUDA device the return scan is the K7 scan kernel (``ops.gae``: its ``ret`` output is this recurrence; csrc/onpolicy.cu) and
the loss and its gradient are the fused DQN kernel (``ops.dqn_loss_fused`` with the n-step return as the target: reward = ret, mask = 0;
csrc/losses.cu).  On ``select_device(-1)`` the same statements run as torch expressions -- the reference's own CPU path.

``config.device_nstep_dqn = True`` (off by default) runs the whole step on the device for a VanillaNet on a two-layer FCBody
(``n_step_dqn_feature``): one ``b2rl_nstep_dqn_actor_step`` launch per env step and one ``b2rl_nstep_dqn_update`` launch per
rollout, the target sync included (csrc/a2c.cu, component/actor.py ``DeviceNStepDQN``).  The epsilon-greedy draws then come from
the device's Philox stream, not from numpy's.  Configurations the kernels do not cover raise ``NotImplementedError`` naming the
unmet condition.

``config.cuda_graph = True`` (off by default) runs each ``step()`` of a VanillaNet on a wgmma NatureConvBody at bf16
(``n_step_dqn_pixel`` with ``Config.COMPUTE_DTYPE = torch.bfloat16``) as captured graphs: one ``GraphedQActor`` replay per env
step (pinned upload of the frame stacks into the rollout arena, the network, q down to the host; epsilon-greedy stays in numpy
as in the reference) and one ``GraphedNStepLearner`` replay per rollout (learner.py).  The torch optimizer is replaced by a
``FlatOptimizer`` with its hyper-parameters; the network's parameters become views into its arena, so ``state_dict()`` is
always current.  Configurations it does not cover (``component/coverage.py nstep_q_graph_unsupported``; the reason is kept in
``graph_refusal``) keep the eager path; ``config.device_nstep_dqn`` takes precedence.
"""
import numpy as np
import torch
import torch.nn as nn

from .. import ops
from ..component import Storage
from ..utils import epsilon_greedy, philox_seed, tensor, to_np
from .BaseAgent import BaseAgent


class NStepDQNAgent(BaseAgent):
    def __init__(self, config):
        BaseAgent.__init__(self, config)
        self.config = config
        self.task = config.task_fn()
        self.network = config.network_fn()
        self.target_network = config.network_fn()
        self.optimizer = config.optimizer_fn(self.network.parameters())
        self.target_network.load_state_dict(self.network.state_dict())
        self.total_steps = 0
        self.states = self.task.reset()
        self.last_loss = None
        self._graph = None                                  # (GraphedNStepLearner, GraphedQActor), False: eager; decided once
        self.graph_refusal = None
        self.device_nstep_dqn = None
        if getattr(config, "device_nstep_dqn", False):
            from ..component.actor import DeviceNStepDQN
            self.device_nstep_dqn = DeviceNStepDQN(self.network, self.target_network, self.optimizer, config, philox_seed())
            self.optimizer = self.device_nstep_dqn.opt

    def eval_step(self, state):
        """(the reference defines none for this agent; greedy action, as DQNAgent.eval_step DQN_agent.py:69-75)"""
        with torch.no_grad():
            q = self.network(self.config.state_normalizer(np.asarray([np.asarray(s) for s in state])))["q"]
        return to_np(q.argmax(dim=-1))

    def _obs(self, states):
        return self.config.state_normalizer(np.asarray([np.asarray(s) for s in states]))

    def load(self, filename):
        BaseAgent.load(self, filename)
        if self._graph:
            self._graph[0].refresh_packed()                # the next step trains (and acts) from the loaded weights

    def step(self):
        if self.device_nstep_dqn is not None:
            return self._step_device()
        if self._graph_ok():
            return self._step_graph()
        config = self.config
        T = config.rollout_length
        storage = Storage(T)
        states = self.states
        for _ in range(T):
            q = self.network(self._obs(states))["q"]
            epsilon = config.random_action_prob(config.num_workers)
            actions = epsilon_greedy(epsilon, to_np(q))
            next_states, rewards, terminals, info = self.task.step(actions)
            self.record_online_return(info)
            rewards = config.reward_normalizer(rewards)
            storage.feed({"q": q, "action": tensor(actions).unsqueeze(-1).long(), "reward": tensor(rewards).unsqueeze(-1),
                          "mask": tensor(1 - np.asarray(terminals)).unsqueeze(-1)})
            states = next_states
            self.total_steps += config.num_workers
            if self.total_steps // config.num_workers % config.target_network_update_freq == 0:
                self.target_network.load_state_dict(self.network.state_dict())
        self.states = states
        storage.placeholder()

        with torch.no_grad():
            boot = self.target_network(self._obs(states))["q"].max(dim=1, keepdim=True)[0]
        self.optimizer.zero_grad()
        if boot.is_cuda:
            reward, mask = torch.stack(storage.reward[:T]), torch.stack(storage.mask[:T])
            value = torch.zeros((T + 1,) + tuple(boot.shape), device=boot.device, dtype=torch.float32)
            value[T] = boot
            _, ret = ops.gae(reward, mask, value, config.discount, 1.0, use_gae=False)
            q = torch.cat(storage.q[:T], dim=0)
            rows = q.shape[0]
            # one launch: delta, loss = 0.5 * mean(delta^2) and dloss/dq, with y = ret + 1.0 * q_next * 0
            r = ops.dqn_loss_fused(q.detach(), torch.zeros_like(q), None, torch.cat(storage.action[:T], dim=0).view(-1),
                                   ret.reshape(rows), torch.zeros(rows, device=q.device), 1.0)
            torch.autograd.backward([q], [r["dq"]])
            loss = r["loss"][0]
        else:
            ret = boot
            for i in reversed(range(T)):
                ret = storage.reward[i] + config.discount * storage.mask[i] * ret
                storage.ret[i] = ret
            entries = storage.extract(["q", "action", "ret"])
            loss = 0.5 * (entries.q.gather(1, entries.action) - entries.ret).pow(2).mean()
            loss.backward()
        self.last_loss = loss.detach()
        nn.utils.clip_grad_norm_(self.network.parameters(), config.gradient_clip)
        self.optimizer.step()

    def _step_device(self):
        """``step()`` with ``config.device_nstep_dqn``: T actor launches, each followed by ``task.step`` on the host; rewards and
        masks stay in host arrays until the rollout ends; then the final observations, one upload, and one update launch, which
        also does the target sync when an env step of this rollout reached its schedule (:48-50)."""
        config, dev = self.config, self.device_nstep_dqn
        dev.begin_rollout()
        states = self.states
        sync = False
        for t in range(config.rollout_length):
            action = dev.act(t, states, config.random_action_prob(config.num_workers))
            next_states, rewards, terminals, info = self.task.step(action)
            self.record_online_return(info)
            dev.rewards[t] = np.asarray(config.reward_normalizer(rewards), dtype=np.float32)   # tensor(): float32
            dev.masks[t] = np.asarray(1 - np.asarray(terminals), dtype=np.float32)
            states = next_states
            self.total_steps += config.num_workers
            sync = sync or self.total_steps // config.num_workers % config.target_network_update_freq == 0
        self.states = states
        self.last_loss = dev.update(self._obs(states), sync)

    # ------------------------------------------------------------------ config.cuda_graph (opt-in)
    def _graph_ok(self):
        """Decided on the first step: the captured actor + update serve this configuration (``nstep_q_graph_unsupported``),
        or the eager path runs (the reason is kept in ``graph_refusal``)."""
        if self._graph is None:
            from ..component.actor import GraphedQActor
            from ..component.coverage import nstep_q_graph_unsupported
            from ..learner import GraphedNStepLearner
            config = self.config
            self.graph_refusal = nstep_q_graph_unsupported(config, self.network, self.optimizer, self.states)
            self._graph = False
            if self.graph_refusal is None:
                self.optimizer = ops.FlatOptimizer.from_torch(self.optimizer, list(self.network.parameters()))
                coef = config.state_normalizer.coef
                lr = GraphedNStepLearner(self.network, self.target_network, self.optimizer, config.rollout_length,
                                         config.num_workers, config.discount, config.gradient_clip, coef).capture()
                actor = GraphedQActor(self.network, lambda out: out["q"], config.num_workers, 4, (84, 84), coef, arena=lr.arena)
                self._graph = (lr, actor)
        return bool(self._graph)

    def _step_graph(self):
        """``step()`` with ``config.cuda_graph``: T actor replays, each followed by epsilon-greedy and ``task.step`` on the host,
        with actions / rewards / masks written into the learner's pinned staging buffer; then one update replay, preceded by
        the target sync when an env step of this rollout reached its schedule (:48-50; the online network does not change
        inside the rollout, so syncing at its end is the same)."""
        config = self.config
        lr, actor = self._graph
        states, sync = self.states, False
        for t in range(config.rollout_length):
            q = actor.q_values(states, t)
            epsilon = config.random_action_prob(config.num_workers)
            actions = epsilon_greedy(epsilon, q)
            next_states, rewards, terminals, info = self.task.step(actions)
            self.record_online_return(info)
            lr.h_action[t].numpy()[...] = actions
            lr.h_reward[t].numpy()[...] = np.asarray(config.reward_normalizer(rewards), dtype=np.float32)   # tensor(): float32
            lr.h_mask[t].numpy()[...] = 1 - np.asarray(terminals, dtype=np.float32)
            states = next_states
            self.total_steps += config.num_workers
            sync = sync or self.total_steps // config.num_workers % config.target_network_update_freq == 0
        self.states = states
        lr.stage_final(states)
        self.last_loss = lr.update(sync_target=sync)
