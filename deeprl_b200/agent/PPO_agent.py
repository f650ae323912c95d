"""PPO behind the reference's interface (``deep_rl/agent/PPO_agent.py:13-99``): rollout, GAE, advantage
normalisation, ``optimization_epochs`` x minibatches of the clipped surrogate, KL-gated actor step (non-shared
representation) or one clipped optimizer step (shared representation).

CUDA device: GAE = ``b2rl_gae``, advantage normalisation = ``b2rl_normalize_advantage``, each minibatch's surrogate /
value loss / approx-KL and their gradients = one ``b2rl_ppo_loss`` launch.  ``select_device(-1)``: torch statements
(the reference's own CPU path; see A2C_agent.py docstring).

``config.cuda_graph = True`` (off by default) runs each ``step()`` of a shared-representation CategoricalActorCriticNet on a
wgmma NatureConvBody at bf16 (``ppo_pixel`` with ``Config.COMPUTE_DTYPE = torch.bfloat16``) as captured graphs: one
``GraphedQActor`` replay per env step (pinned upload of the frame stacks into the rollout arena, the body, the actor-critic
head with the action drawn on the device, the actions down to the host) and one ``GraphedPPOPixelLearner`` replay per rollout
(learner.py: the final states' value, GAE and the old log-probabilities from the actor's outputs, advantage normalisation,
then every epoch's minibatch updates unrolled).  The actions then come from the device's Philox stream (keyed from torch's
seeded generator, as in ``a2c_pixel``), not from torch's ``Categorical.sample``; the minibatches are still drawn by
``random_sample`` on the host.  A ``FlatOptimizer`` built from ``self.opt`` takes over the Adam state; ``self.opt`` stays as
the holder of ``lr_scheduler``'s learning rate, which each update reads from the device.  The network's parameters become
views into the optimizer's arena, so ``state_dict()`` is always current.  Configurations it does not cover
(``component/coverage.py ppo_graph_unsupported``; the reason is kept in ``graph_refusal``) keep the eager path.
"""
import numpy as np
import torch
import torch.nn as nn

from .. import ops
from ..component import Storage
from ..utils import philox_seed, random_sample, tensor, to_np
from .A2C_agent import compute_advantages
from .BaseAgent import BaseAgent


class PPOAgent(BaseAgent):
    def __init__(self, config):
        BaseAgent.__init__(self, config)
        self.config = config
        self.task = config.task_fn()
        self.network = config.network_fn()
        if config.shared_repr:
            self.opt = config.optimizer_fn(self.network.parameters())
        else:
            self.actor_opt = config.actor_opt_fn(self.network.actor_params)
            self.critic_opt = config.critic_opt_fn(self.network.critic_params)
        self.total_steps = 0
        self.states = self.task.reset()
        self._raw_states, self._raw_seen = self.states, True      # (device actor: un-normalised copy, already counted below)
        self.states = config.state_normalizer(self.states)
        if config.shared_repr:
            self.lr_scheduler = torch.optim.lr_scheduler.LambdaLR(self.opt, lambda step: 1 - step / config.max_steps)
        self.gae_exact = True
        self.last_stats = None
        self._graph = None                                 # cuda_graph: (GraphedPPOPixelLearner, GraphedQActor)
        self._graph_checked, self.graph_refusal = False, None
        # data parallel under torchrun (parallel.init(), world > 1): rank-local rollout / GAE / advantage normalisation /
        # permutations / state normaliser; every minibatch update is one step on the union of the ranks' minibatches, with the
        # gradients exchanged inside the persistent PPO kernel.  Parameters start as rank 0's.
        import torch.distributed as dist
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        if self.world > 1:
            if config.shared_repr or not getattr(config, "graph_minibatch", False):
                raise NotImplementedError("data-parallel PPO (world size %d) runs on the persistent PPO kernel only: it needs "
                                          "config.shared_repr = False and config.graph_minibatch = True" % self.world)
            with torch.no_grad():
                for p in self.network.parameters():
                    dist.broadcast(p.data, 0)

    def load(self, filename):
        BaseAgent.load(self, filename)
        if self._graph_checked and self.graph_refusal is None:
            self._graph[0].refresh_packed()                # the next step trains (and acts) from the loaded weights

    def eval_step(self, state):
        with torch.no_grad():
            prediction = self.network(self.config.state_normalizer(state))
        return to_np(prediction["action"])

    # ------------------------------------------------------------------ device-side actor (SURVEY 8f-3, component/actor.py)
    def _device_actor(self):
        """One launch per env step for normaliser + network forward + sampling when the network / normaliser are the reference's
        continuous-control configuration (examples.py:496-522) on a CUDA device (``config.device_actor = False`` turns it off)."""
        if getattr(self, "_actor", None) is None:
            from ..component import actor as dev_actor
            cfg = self.config
            ok = (getattr(cfg, "device_actor", True) and dev_actor.supported(self.network, cfg.state_normalizer)
                  and cfg.num_workers <= 64 and type(cfg.reward_normalizer).__name__ == "RescaleNormalizer")
            self._actor = dev_actor.DeviceGaussianActor(self.network, cfg.state_normalizer, cfg.num_workers) if ok else False
        return self._actor or None

    def _rollout_device(self, actor):
        """``_rollout`` with the per-step normaliser / forward / sampling on the device: the raw observations go up through a
        pinned double buffer, the actions come back for the host envs; everything else stays in HBM.  As in the reference, every
        observation batch updates the running moments exactly once -- when it is first seen (the constructor counted the reset
        batch on the host; the batch that ends a rollout is counted by its value forward and re-used, read-only, by the first
        step of the next rollout)."""
        config = self.config
        T = config.rollout_length
        storage = Storage(T)
        raw, seen = self._raw_states, self._raw_seen
        keys = ("action", "log_pi_a", "entropy", "mean", "v")
        if not getattr(config, "device_actor_arena", True):        # one set of output tensors and two small uploads per env step
            for _ in range(T):
                pred = actor.step(raw, update=not seen)
                raw, rewards, terminals, info = self.task.step(to_np(pred["action"]))
                seen = False
                self.record_online_return(info)
                rewards = config.reward_normalizer(rewards)
                storage.feed({k: pred[k] for k in keys})
                storage.feed({"reward": tensor(rewards).unsqueeze(-1), "mask": tensor(1 - terminals).unsqueeze(-1),
                              "state": pred["state"]})
                self.total_steps += config.num_workers
            pred = actor.step(raw, update=True)             # value of the last state (PPO_agent.py:46-47)
            self._raw_states, self._raw_seen = raw, True
            storage.feed({k: pred[k] for k in keys})
            last_v = pred["v"]
        else:
            # the actor's outputs go straight into rollout-sized arenas; rewards / masks stay on the host until the rollout ends
            N = config.num_workers
            actor.begin_rollout(T)
            rew, msk = np.empty((T, N), dtype=np.float32), np.empty((T, N), dtype=np.float32)
            for t in range(T):
                action = actor.step_into(t, raw, update=not seen)
                raw, rewards, terminals, info = self.task.step(action)
                seen = False
                self.record_online_return(info)
                rew[t] = np.asarray(config.reward_normalizer(rewards), dtype=np.float32)     # tensor(): float32 (torch_utils.py:20-25)
                msk[t] = np.asarray(1 - terminals, dtype=np.float32)
                self.total_steps += N
            actor.step_into(T, raw, update=True)            # value of the last state (PPO_agent.py:46-47)
            self._raw_states, self._raw_seen = raw, True
            roll, dev = actor.roll, actor.dev
            for k in keys:
                setattr(storage, k, list(roll[k].unbind(0)))                                  # T + 1 entries, like feed()
            storage.state = list(roll["state"][:T].unbind(0))
            storage.reward = list(torch.from_numpy(rew).to(dev).unsqueeze(-1).unbind(0))
            storage.mask = list(torch.from_numpy(msk).to(dev).unsqueeze(-1).unbind(0))
            last_v = roll["v"][T]
        storage.placeholder()
        compute_advantages(storage, config, last_v, exact=self.gae_exact)
        actor.pull_stats()                                  # the host normaliser object stays current (eval_step, save)
        entries = storage.extract(["state", "action", "log_pi_a", "ret", "advantage"])
        return type(entries)(*[x.detach().contiguous() for x in entries])

    def _rollout(self):
        config = self.config
        actor = self._device_actor()
        if actor is not None:
            return self._rollout_device(actor)
        storage = Storage(config.rollout_length)
        states = self.states
        for _ in range(config.rollout_length):
            with torch.no_grad():
                prediction = self.network(states)
            next_states, rewards, terminals, info = self.task.step(to_np(prediction["action"]))
            self.record_online_return(info)
            rewards = config.reward_normalizer(rewards)
            next_states = config.state_normalizer(next_states)
            storage.feed(prediction)
            storage.feed({"reward": tensor(rewards).unsqueeze(-1), "mask": tensor(1 - terminals).unsqueeze(-1),
                          "state": tensor(states)})
            states = next_states
            self.total_steps += config.num_workers
        self.states = states
        with torch.no_grad():
            prediction = self.network(states)
        storage.feed(prediction)
        storage.placeholder()
        compute_advantages(storage, config, prediction["v"], exact=self.gae_exact)
        entries = storage.extract(["state", "action", "log_pi_a", "ret", "advantage"])
        return type(entries)(*[x.detach().contiguous() for x in entries])

    def _normalize(self, entries):
        adv = entries.advantage
        if adv.is_cuda:
            ops.normalize_advantage_(adv)
        else:
            adv.copy_((adv - adv.mean()) / adv.std())

    def _minibatch(self, entries, batch_indices):
        config = self.config
        batch_indices = tensor(batch_indices).long()
        entry = type(entries)(*[x[batch_indices] for x in entries])
        prediction = self.network(entry.state, entry.action)
        if entry.state.is_cuda:
            r = ops.ppo_loss_fused(prediction["log_pi_a"].detach(), prediction["entropy"].detach(), prediction["v"].detach(),
                                   entry.log_pi_a, entry.advantage, entry.ret, config.ppo_ratio_clip, config.entropy_weight)
            shape = prediction["v"].shape
            g_lp, g_en, g_v = r["dlogp"].view(shape), r["dent"].view(shape), r["dv"].view(shape)
            self.last_stats = r["out"]
            if config.shared_repr:
                self.opt.zero_grad()
                torch.autograd.backward([prediction["log_pi_a"], prediction["entropy"], prediction["v"]], [g_lp, g_en, g_v])
                nn.utils.clip_grad_norm_(self.network.parameters(), config.gradient_clip)
                self.opt.step()
            else:
                approx_kl = r["out"][2]
                if approx_kl <= 1.5 * config.target_kl:          # host decision, as PPO_agent.py:94
                    self.actor_opt.zero_grad()
                    torch.autograd.backward([prediction["log_pi_a"], prediction["entropy"]], [g_lp, g_en])
                    self.actor_opt.step()
                self.critic_opt.zero_grad()
                prediction["v"].backward(g_v)
                self.critic_opt.step()
            return
        ratio = (prediction["log_pi_a"] - entry.log_pi_a).exp()
        obj = ratio * entry.advantage
        obj_clipped = ratio.clamp(1.0 - config.ppo_ratio_clip, 1.0 + config.ppo_ratio_clip) * entry.advantage
        policy_loss = -torch.min(obj, obj_clipped).mean() - config.entropy_weight * prediction["entropy"].mean()
        value_loss = 0.5 * (entry.ret - prediction["v"]).pow(2).mean()
        approx_kl = (entry.log_pi_a - prediction["log_pi_a"]).mean()
        if config.shared_repr:
            self.opt.zero_grad()
            (policy_loss + value_loss).backward()
            nn.utils.clip_grad_norm_(self.network.parameters(), config.gradient_clip)
            self.opt.step()
        else:
            if approx_kl <= 1.5 * config.target_kl:
                self.actor_opt.zero_grad()
                policy_loss.backward()
                self.actor_opt.step()
            self.critic_opt.zero_grad()
            value_loss.backward()
            self.critic_opt.step()

    def step(self):
        if self._graph_ok():
            return self._step_graph()
        config = self.config
        entries = self._rollout()
        self._normalize(entries)
        if config.shared_repr:
            self.lr_scheduler.step(self.total_steps)
        rows = entries.state.size(0)
        # the graphed path keeps the actor's and the critic's parameters in two separate arenas: a shared phi_body (whose
        # parameters the reference gives to BOTH optimizers, network_heads.py:186-189) or discrete (1-D) actions are served
        # by the eager loop below
        shared_phi = len(getattr(self.network, "phi_params", [])) > 0
        if (getattr(config, "graph_minibatch", False) and entries.state.is_cuda and not config.shared_repr
                and rows % config.mini_batch_size == 0 and not shared_phi and entries.action.dim() == 2):
            self._graphed_epochs(entries)                  # same updates, one CUDA-graph replay each (learner.py)
            return
        if self.world > 1:
            raise NotImplementedError("data-parallel PPO needs CUDA rollouts, continuous actions, no shared phi_body and "
                                      "rollout rows divisible by mini_batch_size (the persistent PPO kernel)")
        for _ in range(config.optimization_epochs):
            for batch_indices in random_sample(np.arange(rows), config.mini_batch_size):
                self._minibatch(entries, batch_indices)

    def _graphed_epochs(self, entries):
        """``config.graph_minibatch = True``: the minibatch loop of PPO_agent.py:68-99 through ``GraphedPPOLearner``.  The
        torch optimizers built by ``actor_opt_fn`` / ``critic_opt_fn`` are replaced by flat-arena Adam with the same
        hyper-parameters on first use; the permutations come from ``np.random.permutation`` exactly as ``random_sample``."""
        from ..learner import GraphedPPOLearner, PersistentPPOLearner
        config = self.config
        rows, mb = entries.state.size(0), config.mini_batch_size
        if getattr(self, "_graph", None) is None:
            a = ops.FlatOptimizer.from_torch(self.actor_opt, self.network.actor_params)
            c = ops.FlatOptimizer.from_torch(self.critic_opt, self.network.critic_params)
            # one persistent kernel for the whole loop where the network is the examples' Gaussian MLP pair
            # (config.persistent_minibatch = False keeps the one-graph-replay-per-minibatch form)
            persistent = (getattr(config, "persistent_minibatch", True) and a.kind == "adam" and c.kind == "adam"
                          and PersistentPPOLearner.supported(self.network, mb))
            cls = PersistentPPOLearner if persistent else GraphedPPOLearner
            kw = {}
            if self.world > 1:
                if not persistent:
                    raise NotImplementedError("data-parallel PPO runs on the persistent PPO kernel: Adam for actor and critic "
                                              "and a network PersistentPPOLearner.supported() accepts")
                import torch.distributed as dist
                kw = dict(world=self.world, rank=dist.get_rank())
            self._graph = cls(self.network, a, c, rows, entries.state.shape[1], entries.action.shape[1], mb,
                              config.ppo_ratio_clip, config.entropy_weight, config.target_kl,
                              config.optimization_epochs * (rows // mb), **kw)
            self._graph.load(entries)
            self._graph.capture()
        g = self._graph
        g.load(entries)
        batches = [b for _ in range(config.optimization_epochs) for b in random_sample(np.arange(rows), mb)]
        g.run(g.set_batches(batches))
        self.last_stats = g.stats

    # ------------------------------------------------------------------ config.cuda_graph (opt-in)
    def _graph_ok(self):
        """Decided on the first step: the captured actor + update serve this configuration (``ppo_graph_unsupported``), or the
        eager path runs (the reason is kept in ``graph_refusal``)."""
        if not self._graph_checked:
            from ..component.actor import GraphedQActor
            from ..component.coverage import ppo_graph_unsupported
            from ..learner import GraphedPPOPixelLearner
            config = self.config
            self._graph_checked = True
            self.graph_refusal = ppo_graph_unsupported(config, self.network, getattr(self, "opt", None), self._raw_states)
            if self.graph_refusal is None:
                self.flat_opt = ops.FlatOptimizer.from_torch(self.opt, list(self.network.parameters()))
                coef = config.state_normalizer.coef
                lr = GraphedPPOPixelLearner(self.network, self.flat_opt, config.rollout_length, config.num_workers,
                                            philox_seed(), config.mini_batch_size, config.optimization_epochs,
                                            config.discount, config.gae_tau, config.use_gae, config.ppo_ratio_clip,
                                            config.entropy_weight, config.gradient_clip, coef).capture()
                actor = GraphedQActor(self.network, None, config.num_workers, 4, (84, 84), coef, arena=lr.arena, run=lr.act,
                                      body=self.network.phi_body)
                self._graph = (lr, actor)
        return self.graph_refusal is None

    def graph_lr(self):
        """``lr_scheduler.step(self.total_steps)`` (PPO_agent.py:67) and the learning rate it leaves on ``self.opt``: what the
        update graph's Adam uses for this rollout."""
        self.lr_scheduler.step(self.total_steps)
        return float(self.opt.param_groups[0]["lr"])

    def _step_graph(self):
        """``step()`` with ``config.cuda_graph``: T actor replays (the action drawn on the device into the learner's action row
        t; its pinned download is the step's only synchronisation), each followed by ``task.step`` on the host, with rewards
        and masks written into the learner's pinned staging buffer; then the final states, the learning rate, the minibatches
        of every epoch (``random_sample``, as the eager loop draws them) and one update replay."""
        config = self.config
        lr, actor = self._graph
        states = self._raw_states
        for t in range(config.rollout_length):
            actions = actor.q_values(states, t)
            next_states, rewards, terminals, info = self.task.step(actions)
            self.record_online_return(info)
            lr.h_reward[t].numpy()[...] = np.asarray(config.reward_normalizer(rewards), dtype=np.float32)   # tensor(): float32
            lr.h_mask[t].numpy()[...] = 1 - np.asarray(terminals, dtype=np.float32)
            states = next_states
            self.total_steps += config.num_workers
        self._raw_states = states
        self.states = config.state_normalizer(states)
        lr.stage_final(states)
        rows = config.rollout_length * config.num_workers
        step_lr = self.graph_lr()
        batches = [b for _ in range(config.optimization_epochs) for b in random_sample(np.arange(rows), config.mini_batch_size)]
        lr.stage_batches(batches, step_lr)
        self.last_stats = lr.update()
