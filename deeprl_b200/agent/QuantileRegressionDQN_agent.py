"""QR-DQN agent behind the reference's interface (``deep_rl/agent/QuantileRegressionDQN_agent.py``:
``QuantileRegressionDQNActor``:14, ``QuantileRegressionDQNAgent``:23).  The pairwise quantile-Huber loss
(N x B x N terms, six 82 MB temporaries in the reference at N=200, B=512) is one kernel that never
materialises the pair tensor (``csrc/losses.cu: qr_loss_kernel``).  As in the reference the loss tensor is
indexed by TARGET quantile, shape (N,), so QR-DQN + prioritized replay is not defined (SURVEY 7.3-7).

``config.device_qr = True`` (off by default; ``quantile_regression_dqn_feature(game=..., device_qr=True)``) runs a QuantileNet
on a two-layer FCBody on the device: one ``b2rl_dist_dqn_actor_step`` launch per env step (epsilon-greedy on the device's
Philox stream, not numpy's) and one ``b2rl_dist_dqn_replay_update`` launch per gradient update (csrc/dist_dqn.cu,
component/actor.py ``DeviceDistDQN``), also with ``async_actor``.  Configurations the kernels do not cover raise
``NotImplementedError``."""
import threading

import numpy as np
import torch

from .. import ops
from ..component import PrioritizedTransition
from ..utils import range_tensor, tensor, to_np
from .BaseAgent import BaseAgent
from .DQN_agent import DQNActor, DQNAgent


class QuantileRegressionDQNActor(DQNActor):
    def _q_tensor(self, prediction):
        return prediction["quantile"].mean(-1)


class QuantileRegressionDQNAgent(DQNAgent):
    def __init__(self, config):
        BaseAgent.__init__(self, config)
        self.config = config
        config.lock = threading.Lock()
        self._build(QuantileRegressionDQNActor)
        self.batch_indices = range_tensor(config.batch_size)
        self.quantile_weight = 1.0 / config.num_quantiles
        self.cumulative_density = tensor((2 * np.arange(config.num_quantiles) + 1) / (2.0 * config.num_quantiles)).view(1, -1)

    _graph_kind = "qr"
    _device_flag = "device_qr"

    def _fused_owner(self):
        return QuantileRegressionDQNAgent

    def eval_step(self, state):
        self.config.state_normalizer.set_read_only()
        state = self.config.state_normalizer(np.asarray([np.asarray(s) for s in state]))
        with torch.no_grad():
            q = self.network(state)["quantile"].mean(-1)
        action = np.argmax(to_np(q).flatten())
        self.config.state_normalizer.unset_read_only()
        return [action]

    def _heads(self, transitions):
        states, next_states = self._inputs(transitions)
        with torch.no_grad():
            quantiles_next = self.target_network(next_states)["quantile"]
        return self.network(states)["quantile"], quantiles_next

    def compute_loss(self, transitions):
        """QuantileRegressionDQN_agent.py:55-74 -> vector (N,) indexed by target quantile."""
        c = self.config
        quantiles, quantiles_next = self._heads(transitions)
        return ops.qr_vector(quantiles, quantiles_next, tensor(transitions.action), tensor(transitions.reward),
                             tensor(transitions.mask), c.discount ** c.n_step)

    def reduce_loss(self, loss):
        return loss.mean()

    def _per_args(self, transitions):
        if isinstance(transitions, PrioritizedTransition):
            raise NotImplementedError("QR-DQN with prioritized replay is undefined in the reference: its loss is "
                                      "per target quantile, not per sample (QuantileRegressionDQN_agent.py:74)")
        return {}

    def _fused_forward(self, transitions, per):
        c = self.config
        quantiles, quantiles_next = self._heads(transitions)
        r = ops.qr_loss_fused(quantiles.detach(), quantiles_next, transitions.action, transitions.reward,
                              transitions.mask, c.discount ** c.n_step)
        return quantiles, r["dquant"], r
