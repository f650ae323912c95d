"""DQN / Double-DQN / prioritized / n-step agent behind the reference's interface
(``deep_rl/agent/DQN_agent.py``: ``DQNActor``:14, ``DQNAgent``:48).

One ``step()`` = ``sgd_update_frequency`` actor transitions fed to the HBM replay ring, then (after the
exploration phase) one gradient update: sample -> networks -> ONE fused target/loss/priority/gradient kernel
(``csrc/losses.cu``) -> backward -> ONE fused global-norm clip + optimizer launch pair (``csrc/optim.cu``) ->
sum-tree priority update on the device (``csrc/sumtree.cu``).  Nothing of the update touches the host.

``compute_loss`` / ``reduce_loss`` keep the reference's contract (per-sample tensor, then reduction,
DQN_agent.py:78-99) and differentiate through the same kernel; a subclass that overrides either is served by
the generic autograd path in ``_generic_update``.

``config.device_dqn = True`` (off by default) runs a VanillaNet / DuelingNet on a two-layer FCBody (``dqn_feature``) on the
device: one ``b2rl_nstep_dqn_actor_step`` launch per env step (epsilon-greedy on the device's Philox stream, not numpy's) and
one ``b2rl_dqn_replay_update`` launch per gradient update on the batch ``replay.sample()`` returns (csrc/a2c.cu,
component/actor.py ``DeviceDQN``).  Configurations the kernels do not cover raise ``NotImplementedError`` naming the unmet
condition.  ``CategoricalDQNAgent`` / ``QuantileRegressionDQNAgent`` have their own flags, ``config.device_c51`` /
``config.device_qr``, served by the same ``step()`` with ``DeviceDistDQN`` (csrc/dist_dqn.cu); they also run with
``async_actor``, the actor thread launching its actor steps under ``config.lock``.  ``config.device_rainbow`` does the same for
a ``CategoricalDQNAgent`` on a RainbowNet (``DeviceRainbow``, csrc/rainbow.cu): the NoisyLinear noise is drawn in the kernels,
so the ``reset_noise()`` calls of the eager path do not run.

``config.cuda_graph = True`` with ``ReplayWrapper(..., async_=True)`` over 84x84 uint8 frames (``dqn_pixel``,
``categorical_dqn_pixel``, ``quantile_regression_dqn_pixel`` as written, at ``Config.COMPUTE_DTYPE = torch.bfloat16``): past
exploration each step's transitions are staged in the learner's pinned buffer and fed inside ONE update replay
(``_async_graph_update``; learner.GraphedDQNLearner with ``prefetch`` and ``wrapper_order``), the actor's forward is a
GraphedQActor replay, on the actor thread with ``async_actor`` (component/actor.py ``ParameterOrder``).  Configurations it
does not cover (``component/coverage.py dqn_graph_unsupported``; the reason is kept in ``graph_refusal``) keep their path.
"""
import threading

import numpy as np
import torch
import torch.nn as nn

from .. import ops
from ..component import LazyFrames, PrioritizedTransition
from ..network.fused import frame_scale
from ..utils import Config, RescaleNormalizer, close_obj, epsilon_greedy, philox_seed, tensor, to_np
from .BaseAgent import BaseActor, BaseAgent


class DQNActor(BaseActor):
    def __init__(self, config):
        BaseActor.__init__(self, config)
        self.config = config
        self.start()

    def _q_tensor(self, prediction):
        """Action values [num_envs, A] on the device (what ``compute_q`` converts to numpy)."""
        return prediction["q"]

    def compute_q(self, prediction):
        return to_np(self._q_tensor(prediction))

    _order = None                                          # component/actor.py ParameterOrder: the agent's async captured path

    def _graphed(self):
        """``config.cuda_graph``: the forward pass below as one captured launch sequence (component/actor.py GraphedQActor).
        Not for subclasses that redefine ``compute_q`` itself (they get the statements of the reference)."""
        ga = getattr(self, "_graph_actor", None)
        if ga is None:
            from ..component.actor import GraphedQActor
            from ..component.coverage import q_actor_unsupported
            order = self._order
            ok = (type(self).compute_q is DQNActor.compute_q
                  and q_actor_unsupported(self.config, self._network, self._state, async_ok=order is not None) is None)
            ga = self._graph_actor = GraphedQActor(
                self._network, self._q_tensor, len(self._state), 4, (84, 84), self.config.state_normalizer.coef) if ok else False
            if ga and order is not None and self.config.async_actor:
                ga.capture_error_mode = "thread_local"     # the learner thread may synchronise while this thread captures
        return ga or None

    def _ordered_q_values(self, order):
        """``async_actor`` on the agent's captured path: the GraphedQActor replay on this thread's stream, after the latest
        update replay and before the next one (``ParameterOrder``); ``config.lock`` is held to enqueue (and to capture), not
        while this thread waits for its q values."""
        stream = order.actor_stream()
        with torch.cuda.stream(stream):
            with order.lock:
                ga = self._graphed()
                stream.wait_event(order.updated)
                if ga is None:                             # (a subclass's own compute_q): the eager forward, same order
                    with torch.no_grad():
                        prediction = self._network(self.config.state_normalizer(np.asarray([np.asarray(s) for s in self._state])))
                else:
                    ga.enqueue(self._state)
                order.acted.record(stream)
            return ga.result() if ga is not None else self.compute_q(prediction)

    def _transition(self):
        """DQN_agent.py:24-45: epsilon-greedy on a forward pass of the shared network, one env step."""
        if self._state is None:
            self._state = self._task.reset()
        config = self.config
        dev = getattr(self, "_device_dqn", None)
        if dev is not None:                                # config.device_dqn: rescale + forward + epsilon-greedy, one launch
            if config.noisy_linear:                        # config.device_rainbow: the noise explores (DQN_agent.py:34-35)
                epsilon = 0
            else:
                epsilon = 1 if self._total_steps < config.exploration_steps else config.random_action_prob()
            with config.lock:
                action = dev.act(self._state, epsilon)
            return self._env_step(action)
        if config.noisy_linear:
            self._network.reset_noise()
        order = self._order if config.async_actor else None
        ga = self._graphed() if getattr(config, "cuda_graph", False) and order is None else None
        if order is not None:
            q_values = self._ordered_q_values(order)
        elif ga is not None:
            with config.lock:
                q_values = ga.q_values(self._state)
        else:
            with config.lock, torch.no_grad():
                prediction = self._network(config.state_normalizer(np.asarray([np.asarray(s) for s in self._state])))
            q_values = self.compute_q(prediction)
        if config.noisy_linear:
            epsilon = 0
        elif self._total_steps < config.exploration_steps:
            epsilon = 1
        else:
            epsilon = config.random_action_prob()
        action = epsilon_greedy(epsilon, q_values)
        return self._env_step(action)

    def _env_step(self, action):
        next_state, reward, done, info = self._task.step(action)
        entry = [self._state, action, reward, next_state, done, info]
        self._total_steps += 1
        self._state = next_state
        return entry


def _pre_normalized(config, replay):
    """True when the state normalizer is a pure rescale of a uint8 frame ring, so that the fused
    gather->normalize kernel can produce the network input directly (ImageNormalizer, normalizer.py:64-66)."""
    norm = config.state_normalizer
    inner = getattr(replay, "replay", replay)
    return (isinstance(norm, RescaleNormalizer) and hasattr(inner, "sample_normalized")
            and getattr(inner, "item_dtype", None) == np.uint8 and not getattr(replay, "async_", False))


class DQNAgent(BaseAgent):
    def __init__(self, config):
        BaseAgent.__init__(self, config)
        self.config = config
        config.lock = threading.Lock()
        self._build(DQNActor)

    def _build(self, actor_cls):
        config = self.config
        self.replay = config.replay_fn()
        self.actor = actor_cls(config)
        self.network = config.network_fn()
        self.target_network = config.network_fn()
        self.target_network.load_state_dict(self.network.state_dict())
        self.optimizer = config.optimizer_fn(self.network.parameters())
        self._flat = None
        if next(self.network.parameters()).is_cuda:
            try:
                self._flat = ops.FlatOptimizer.from_torch(self.optimizer, list(self.network.parameters()))
            except NotImplementedError:
                self._flat = None             # exotic optimizer: torch.optim + clip_grad_norm_ (library path)
        self.actor.set_network(self.network)
        self.total_steps = 0
        self.last_loss = None
        self.device_dqn = None
        self._learner = None
        from ..component.actor import DeviceDistDQN, DeviceDQN, DeviceRainbow, ParameterOrder
        flag, device = self._device_flag, None
        if getattr(config, "device_rainbow", False):
            for other in ("device_dqn", flag):
                if other is not None and getattr(config, other, False):
                    raise NotImplementedError("config.device_rainbow and config.%s are both set; a RainbowNet runs on the "
                                              "device with config.device_rainbow alone" % other)
            device = DeviceRainbow
        elif flag is not None and getattr(config, flag, False):
            if getattr(config, "device_dqn", False):
                raise NotImplementedError("config.device_dqn and config.%s are both set; %s runs on the device with "
                                          "config.%s alone" % (flag, type(self).__name__, flag))
            device = DeviceDistDQN
        elif getattr(config, "device_dqn", False):
            device = DeviceDQN
        if device is not None:
            self.device_dqn = self.actor._device_dqn = device(self, philox_seed())
        # config.cuda_graph with async replay: decided once, here, before the actor thread starts
        from ..component.coverage import dqn_graph_unsupported
        self.graph_refusal = dqn_graph_unsupported(config, self)
        self._async_graph = self.graph_refusal is None
        if self._async_graph:
            self._order = ParameterOrder(config.lock)
            self.actor._order = self._order if config.async_actor else None

    def close(self):
        close_obj(self.replay)
        close_obj(self.actor)

    def eval_step(self, state):
        self.config.state_normalizer.set_read_only()
        state = self.config.state_normalizer(np.asarray([np.asarray(s) for s in state]))
        with torch.no_grad():
            q = self.network(state)["q"]
        action = to_np(q.argmax(-1))
        self.config.state_normalizer.unset_read_only()
        return action

    # ------------------------------------------------------------------ reference-shaped loss API
    def reduce_loss(self, loss):
        return loss.pow(2).mul(0.5).mean()

    def _inputs(self, transitions):
        if getattr(transitions, "_normalized", False) or getattr(self, "_batch_is_normalized", False):
            return transitions.state, transitions.next_state
        norm = self.config.state_normalizer
        return norm(transitions.state), norm(transitions.next_state)

    def compute_loss(self, transitions):
        """DQN_agent.py:81-99 -> per-sample ``q_target - q`` (autograd through q)."""
        config = self.config
        states, next_states = self._inputs(transitions)
        with torch.no_grad():
            q_next_t = self.target_network(next_states)["q"]
            q_next_o = self.network(next_states)["q"] if config.double_q else None
        q = self.network(states)["q"]
        return ops.dqn_delta(q, q_next_t, q_next_o, tensor(transitions.action), tensor(transitions.reward),
                             tensor(transitions.mask), config.discount ** config.n_step)

    # ------------------------------------------------------------------ update
    def _fused_forward(self, transitions, per):
        """Network passes + the fused loss kernel.  Returns (output tensor to back-propagate, gradient, result)."""
        config = self.config
        states, next_states = self._inputs(transitions)
        with torch.no_grad():
            q_next_t = self.target_network(next_states)["q"]
            q_next_o = self.network(next_states)["q"] if config.double_q else None
        q = self.network(states)["q"]
        r = ops.dqn_loss_fused(q.detach(), q_next_t, q_next_o, transitions.action, transitions.reward, transitions.mask,
                               config.discount ** config.n_step, **per)
        return q, r["dq"], r

    def _per_args(self, transitions):
        if not isinstance(transitions, PrioritizedTransition):
            return {}
        c = self.config
        return dict(is_prob=tensor(transitions.sampling_prob), beta=c.replay_beta(), eps=c.replay_eps, alpha=c.replay_alpha)

    def _apply_gradients(self):
        config = self.config
        if self._flat is not None:
            with config.lock:
                self._flat.step(max_norm=config.gradient_clip or 0.0)
        else:
            if config.gradient_clip:
                nn.utils.clip_grad_norm_(self.network.parameters(), config.gradient_clip)
            with config.lock:
                self.optimizer.step()

    def _zero_grad(self):
        if self._flat is not None:
            self._flat.zero_grad()
        else:
            self.optimizer.zero_grad()

    def _fused_update(self, transitions):
        per = self._per_args(transitions)
        out, grad, r = self._fused_forward(transitions, per)
        if per:
            self.replay.update_priorities((transitions.idx, r["priority"]))      # DQN_agent.py:120-123, on the device
        self._zero_grad()
        out.backward(grad)
        self._apply_gradients()
        return r["loss"]

    def _generic_update(self, transitions):
        """DQN_agent.py:119-134 verbatim in torch, for subclasses that override compute_loss / reduce_loss."""
        config = self.config
        loss = self.compute_loss(transitions)
        if isinstance(transitions, PrioritizedTransition):
            priorities = loss.detach().abs().add(config.replay_eps).pow(config.replay_alpha)
            self.replay.update_priorities((tensor(transitions.idx).long(), priorities.float().contiguous()))
            sampling_probs = tensor(transitions.sampling_prob)
            weights = sampling_probs.mul(sampling_probs.size(0)).add(1e-6).pow(-config.replay_beta())
            weights = weights / weights.max()
            loss = loss.mul(weights)
        loss = self.reduce_loss(loss)
        self._zero_grad()
        loss.backward()
        self._apply_gradients()
        return loss.detach()

    _fused_methods = ("compute_loss", "reduce_loss")

    def _uses_reference_hooks(self):
        cls = type(self)
        owner = self._fused_owner()
        return any(getattr(cls, m) is not getattr(owner, m) for m in self._fused_methods)

    def _fused_owner(self):
        return DQNAgent

    def _sample(self):
        config = self.config
        inner = getattr(self.replay, "replay", self.replay)
        self._batch_scale = 1.0
        if _pre_normalized(config, self.replay) and len(inner.item_shape) == 2:
            dtype, coef = Config.COMPUTE_DTYPE, config.state_normalizer.coef
            self._batch_is_normalized = True
            if dtype == torch.bfloat16 and inner.item_shape[0] % 4 == 0 and inner.item_shape[1] % 4 == 0:
                # throughput mode: exact integer frames in space-to-depth layout, 1/255 folded into conv1
                self._batch_scale = coef
                return inner.sample_normalized(out_dtype=dtype, scale=None, layout="s2d")
            return inner.sample_normalized(out_dtype=dtype, scale=coef, layout="nchw")     # parity mode: exact LUT
        self._batch_is_normalized = False
        return self.replay.sample()

    def step(self):
        config = self.config
        transitions = self.actor.step()
        feeds = []
        for states, actions, rewards, next_states, dones, info in transitions:
            self.record_online_return(info)
            self.total_steps += 1
            feeds.append(dict(
                state=np.array([s[-1] if isinstance(s, LazyFrames) else s for s in states]),
                action=actions,
                reward=[config.reward_normalizer(r) for r in rewards],
                mask=1 - np.asarray(dones, dtype=np.int32)))
        if self._async_graph and self.total_steps > config.exploration_steps:
            # config.cuda_graph with async replay: the feeds are staged for the learner and fed inside its update graph
            self._async_graph_update(feeds)
        else:
            feed_many = getattr(self.replay, "feed_many", None)
            if feed_many is not None:                      # one staging upload for the env steps of this agent step;
                feed_many(feeds)                           # ring / tree state as after feed(d) for d in feeds (replay.py:75-90)
            else:
                for d in feeds:
                    self.replay.feed(d)

        if self.total_steps <= config.exploration_steps or self._async_graph:
            pass
        elif self.device_dqn is not None:
            self._device_update()                          # config.device_dqn: the whole update is one launch
        elif self._graph_ok():
            self._graph_update()                           # config.cuda_graph: the whole update is one graph replay
        else:
            transitions = self._sample()
            if config.noisy_linear:
                self.target_network.reset_noise()
                self.network.reset_noise()
            with frame_scale(self._batch_scale):
                if self._uses_reference_hooks():
                    self.last_loss = self._generic_update(transitions)
                else:
                    self.last_loss = self._fused_update(transitions)

        if self.total_steps / config.sgd_update_frequency % config.target_network_update_freq == 0:
            if self.device_dqn is not None:
                self.device_dqn.sync_target()              # one copy of the online arena into the target arena
            elif getattr(self, "_learner", None) is not None:
                self._learner.sync_target()                # load_state_dict + re-pack of the target's bf16 operands
            else:
                self.target_network.load_state_dict(self.network.state_dict())

    # ------------------------------------------------------------------ config.device_dqn (opt-in)
    _device_flag = None                                    # the distributional agents' own flag (device_c51 / device_qr)

    def _device_update(self):
        """DQN_agent.py:115-134 for the batch ``replay.sample()`` returns (sync or async wrapper, uniform or prioritized) as
        ONE ``b2rl_dqn_replay_update`` launch; the new priorities go to the tree from the device (:120-123)."""
        config = self.config
        transitions = self.replay.sample()
        per = isinstance(transitions, PrioritizedTransition)
        beta = config.replay_beta() if per else 0.0
        with config.lock:                                  # the actor reads the shared parameters (DQN_agent.py:30,133)
            self.last_loss, priority = self.device_dqn.update(transitions, beta)
        if per:
            self.replay.update_priorities((transitions.idx, priority))

    # ------------------------------------------------------------------ config.cuda_graph (opt-in)
    _graph_kind = "dqn"

    def _graph_ok(self):
        """The captured update (learner.GraphedDQNLearner) serves the stock agents on a CUDA device with a synchronous uint8
        image replay and the fused optimizer; everything else keeps the eager path."""
        config = self.config
        if not getattr(config, "cuda_graph", False) or self._flat is None or self._uses_reference_hooks():
            return False
        if config.noisy_linear or not _pre_normalized(config, self.replay):
            return False
        inner = getattr(self.replay, "replay", self.replay)
        return len(getattr(inner, "item_shape", ())) == 2 and inner.size() >= inner.batch_size + 64

    def _graphed_learner(self, replay, **schedule):
        """The learner.GraphedDQNLearner of ``_graph_update`` and ``_async_learner``, which differ only in ``schedule``:
        ``feeds_per_update``, ``prefetch`` and ``wrapper_order``."""
        from ..learner import GraphedDQNLearner
        config = self.config
        return GraphedDQNLearner(
            self.network, self.target_network, self._flat, replay, kind=self._graph_kind, discount=config.discount,
            n_step=config.n_step, double_q=bool(config.double_q), gradient_clip=config.gradient_clip or 0.0,
            compute_dtype=Config.COMPUTE_DTYPE, state_scale=config.state_normalizer.coef,
            replay_eps=getattr(config, "replay_eps", 0.01), replay_alpha=getattr(config, "replay_alpha", 0.5),
            categorical=(getattr(config, "categorical_v_min", -10.0), getattr(config, "categorical_v_max", 10.0)),
            target_sync_every=0, **schedule)

    def _graph_update(self):
        config = self.config
        lr = getattr(self, "_learner", None)
        if lr is None:
            lr = self._learner = self._graphed_learner(getattr(self.replay, "replay", self.replay), feeds_per_update=0,
                                                       prefetch=False)
            with config.lock:
                lr.capture(warmup=1)                       # NOTE: the warm-up is one real (extra) gradient update
        if lr.per:
            lr.d_beta.fill_(float(config.replay_beta()))
        with config.lock:                                  # the actor reads the shared parameters (DQN_agent.py:30,133)
            lr.update()
            lr.repack_online()                             # the actor's next forward sees theta_k
        self.last_loss = lr.loss

    # ------------------------------------------------------------------ config.cuda_graph with async replay (opt-in)
    def _async_graph_update(self, feeds):
        """``step()`` on the captured path with async replay (``component/coverage.py dqn_graph_unsupported``): this step's
        transitions -- frame ``s[-1]``, action, ``reward_normalizer(r)``, mask -- and PER's ``replay_beta()`` go into the
        learner's pinned staging buffer, then ONE update replay copies them up, trains on the batch the previous replay drew,
        feeds them after that batch's last ring read and draws the next batch (learner.GraphedDQNLearner with ``prefetch``
        and ``wrapper_order``: the graph form of ReplayWrapper(async_=True)).  The first call builds the learner; its eager
        warm-up is this step's own update and its capture executes nothing (``first_update``)."""
        config = self.config
        lr, first = self._learner, self._learner is None
        if first:
            lr = self._learner = self._async_learner(feeds)
        else:
            lr.staged.synchronize()                        # the previous replay's copy node has read the staging buffer
        n = sum(len(d["state"]) for d in feeds)
        if n != lr.feeds:
            raise RuntimeError("%d transitions in this step; the captured update feeds %d" % (n, lr.feeds))
        cat = lambda key, dt: np.concatenate([np.asarray(d[key], dtype=dt).reshape(len(d["state"]), -1) for d in feeds])
        lr.h_frames.numpy()[...] = cat("state", np.uint8)
        lr.h_action.numpy()[...] = cat("action", np.int64).reshape(-1)
        lr.h_reward.numpy()[...] = cat("reward", np.float64).reshape(-1)
        lr.h_mask.numpy()[...] = cat("mask", np.int64).reshape(-1)
        if lr.per:
            lr.h_beta[0] = float(config.replay_beta())     # once per update, as _per_args calls it on the eager path
        order = self._order
        with order.lock:                                   # held to enqueue (and to capture), not across a synchronise
            cur = torch.cuda.current_stream()
            cur.wait_event(order.acted)                    # the actor's latest forward has read (and, before the learner
            if first:                                      # existed, re-packed) the packed operands
                cur.wait_stream(self.replay._side)         # after the feeds the wrapper ran during exploration
                lr.first_update()                          # (its re-pack and warm-up start from this stream)
            else:
                lr.update()
            order.updated.record(cur)
        self.last_loss = lr.loss

    def _async_learner(self, feeds):
        config = self.config
        inner = self.replay.replay
        inner.allocate(np.asarray(feeds[0]["state"][0]))   # (the ring exists once the wrapper has fed it)
        with config.lock:
            lr = self._graphed_learner(inner, feeds_per_update=sum(len(d["state"]) for d in feeds), prefetch=True,
                                       wrapper_order=True)
        if config.async_actor:
            lr.capture_error_mode = "thread_local"         # the actor thread may synchronise its stream during the capture
        return lr
