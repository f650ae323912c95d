"""C51 agent (also Rainbow through ``RainbowNet`` + PER + double-Q + n-step) behind the reference's interface
(``deep_rl/agent/CategoricalDQN_agent.py``: ``CategoricalDQNActor``:14, ``CategoricalDQNAgent``:27).
The categorical projection + KL + gradient run as one kernel (``csrc/losses.cu: c51_loss_kernel``).

``config.device_c51 = True`` (off by default; ``categorical_dqn_feature(game=..., device_c51=True)``) runs a CategoricalNet on a
two-layer FCBody on the device: one ``b2rl_dist_dqn_actor_step`` launch per env step (epsilon-greedy on the device's Philox
stream, not numpy's) and one ``b2rl_dist_dqn_replay_update`` launch per gradient update (csrc/dist_dqn.cu, component/actor.py
``DeviceDistDQN``), also with ``async_actor``.  Configurations the kernels do not cover raise ``NotImplementedError``.

``config.device_rainbow = True`` (off by default; ``rainbow_feature(game=..., device_rainbow=True)``) is the same for a
RainbowNet on a two-layer FCBody, all layers NoisyLinear or all nn.Linear: one ``b2rl_rainbow_actor_step`` launch per env step
and one ``b2rl_rainbow_replay_update`` launch per gradient update (csrc/rainbow.cu, component/actor.py ``DeviceRainbow``), the
factorised noise drawn in the kernels from a Philox stream of its own."""
import threading

import numpy as np
import torch

from .. import ops
from ..utils import range_tensor, tensor, to_np
from .BaseAgent import BaseAgent
from .DQN_agent import DQNActor, DQNAgent


class CategoricalDQNActor(DQNActor):
    def _set_up(self):
        self.config.atoms = tensor(self.config.atoms)

    def _q_tensor(self, prediction):
        return (prediction["prob"] * self.config.atoms).sum(-1)


class CategoricalDQNAgent(DQNAgent):
    def __init__(self, config):
        BaseAgent.__init__(self, config)
        self.config = config
        config.lock = threading.Lock()
        config.atoms = np.linspace(config.categorical_v_min, config.categorical_v_max, config.categorical_n_atoms)
        self._build(CategoricalDQNActor)
        self.batch_indices = range_tensor(config.batch_size)
        self.atoms = tensor(config.atoms)
        self.delta_atom = (config.categorical_v_max - config.categorical_v_min) / float(config.categorical_n_atoms - 1)

    _graph_kind = "c51"
    _device_flag = "device_c51"

    def _fused_owner(self):
        return CategoricalDQNAgent

    def eval_step(self, state):
        self.config.state_normalizer.set_read_only()
        state = self.config.state_normalizer(np.asarray([np.asarray(s) for s in state]))
        with torch.no_grad():
            q = (self.network(state)["prob"] * self.atoms).sum(-1)
        action = to_np(q.argmax(-1))
        self.config.state_normalizer.unset_read_only()
        return action

    def _heads(self, transitions):
        config = self.config
        states, next_states = self._inputs(transitions)
        with torch.no_grad():
            pn_t = self.target_network(next_states)["prob"]
            pn_o = self.network(next_states)["prob"] if config.double_q else None
        log_prob = self.network(states)["log_prob"]
        return log_prob, pn_t, pn_o

    def compute_loss(self, transitions):
        """CategoricalDQN_agent.py:60-86 -> per-sample KL (autograd through log_prob)."""
        c = self.config
        log_prob, pn_t, pn_o = self._heads(transitions)
        return ops.c51_kl(log_prob, pn_t, pn_o, tensor(transitions.action), tensor(transitions.reward),
                          tensor(transitions.mask), c.discount ** c.n_step, c.categorical_v_min, c.categorical_v_max)

    def reduce_loss(self, loss):
        return loss.mean()

    def _fused_forward(self, transitions, per):
        c = self.config
        log_prob, pn_t, pn_o = self._heads(transitions)
        r = ops.c51_loss_fused(log_prob.detach(), pn_t, pn_o, transitions.action, transitions.reward, transitions.mask,
                               c.discount ** c.n_step, c.categorical_v_min, c.categorical_v_max, **per)
        return log_prob, r["dlogp"], r
