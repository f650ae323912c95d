"""Which configurations the accelerated paths cover.  Each path has a predicate that returns ``None`` when a configuration runs
on it and otherwise the first unmet condition: the captured (``config.cuda_graph``) predicates' reason is kept in the agent's
``graph_refusal`` and the agent keeps its eager path, the device (``config.device_*``) predicates' is raised by the ``Device*``
constructors in component/actor.py.  A predicate is an ordered sequence of the checks below, each of which returns ``None`` or
its reason; a condition that more than one path has is written once, here.  Every check of the device is ``on_cuda``."""
import numpy as np
import torch
import torch.nn.functional as F

from .. import _lib
from ..network import nature_tc
from ..network.network_bodies import DummyBody, FCBody, NatureConvBody
from ..network.network_heads import (CategoricalActorCriticNet, CategoricalNet, DuelingNet, GaussianActorCriticNet,
                                     QuantileNet, RainbowNet, VanillaNet)
from ..utils import Config
from ..utils.normalizer import RescaleNormalizer
from .replay import PrioritizedReplay, ReplayWrapper, UniformReplay

CAPTURED = "the captured update implements"               # (the subject of the checks both kinds of path have)
KERNELS = "the device kernels implement"


# ------------------------------------------------------------------------------------------------ checks every path has
def on_cuda(network):
    """Whether the network's parameters are on a CUDA device."""
    return next(network.parameters()).is_cuda


def cuda(network):
    if not on_cuda(network):
        return "the network is not on a CUDA device (select_device(0))"


def network_class(network, cls, subject):
    if type(network) is not cls:
        return "the network is a %s; %s %s" % (type(network).__name__, subject, cls.__name__)


def linear_layers(body, config, subject):
    if body.noisy_linear or config.noisy_linear:
        return "the network has NoisyLinear layers; %s nn.Linear" % subject


# ------------------------------------------------------------------------------------------------ checks of the captured paths
def graph_requested(config, *device_flags):
    """``config.cuda_graph`` is set, and none of the ``device_flags``, which take precedence."""
    if not getattr(config, "cuda_graph", False):
        return "config.cuda_graph is not set"
    for flag in device_flags:
        if getattr(config, flag, False):
            return "config.%s is set; it runs the agent on the device itself" % flag


def nature_conv(body, name):
    if not isinstance(body, NatureConvBody):
        return "the %s is a %s; the captured update implements NatureConvBody" % (name, type(body).__name__)


def four_channels(body):
    if body.conv1.in_channels != 4:
        return "the NatureConvBody takes %d channels; the captured update reads stacks of 4 frames" % body.conv1.in_channels


def bf16_wgmma():
    if Config.COMPUTE_DTYPE != torch.bfloat16 or Config.DENSE_BACKEND != "tcgen05":
        return ("the compute dtype is %s with the %r dense backend; the captured update runs bf16 on the wgmma kernels "
                "(tcgen05)" % (Config.COMPUTE_DTYPE, Config.DENSE_BACKEND))


def fused_tail():
    if not (nature_tc.FUSED_BWD and _lib.CONV_SLAB):
        return "the fused backward epilogues are switched off; the captured update needs the fused update tail"


def fewer_than_32_actions(actions, head):
    if actions >= 32:
        return "%d actions; the %s and loss kernels take fewer than 32" % (actions, head)


def rescale_folded(config):
    if not isinstance(config.state_normalizer, RescaleNormalizer):
        return "the state normalizer is %s; the captured update folds a RescaleNormalizer into conv1" % type(
            config.state_normalizer).__name__


def frame_stacks(states):
    if not all(np.asarray(s).dtype == np.uint8 and np.asarray(s).shape == (4, 84, 84) for s in states):
        return "the envs do not return uint8 4 x 84 x 84 frame stacks"


def fused_optimizer(optimizer):
    """What FlatOptimizer.from_torch turns into a kind the fused tail (NatureTail) takes."""
    g = optimizer.param_groups[0]
    if not ((isinstance(optimizer, torch.optim.RMSprop) and g["momentum"] == 0 and g["weight_decay"] == 0)
            or (isinstance(optimizer, torch.optim.Adam) and g["weight_decay"] == 0 and not g["amsgrad"])):
        return ("the optimizer is %s; the fused update tail implements RMSprop (centered or not) and Adam without momentum, "
                "weight decay or amsgrad" % type(optimizer).__name__)


# ------------------------------------------------------------------------------------------------ checks of the device kernels
def fc_body_class(body):
    if isinstance(body, NatureConvBody):
        return "the body is a NatureConvBody; the device kernels implement a two-layer FCBody"
    if not isinstance(body, FCBody):
        return "the network needs an FCBody body (got %s)" % type(body).__name__


def two_layers(body):
    if len(body.layers) != 2:
        return "the device kernels implement a two-layer FCBody (got %d layers)" % len(body.layers)


def fc_gate(gate):
    if gate not in (torch.tanh, F.relu):
        return "the FCBody gate must be torch.tanh or F.relu"


def fc_widths(body):
    """(state_dim, hidden 1, hidden 2) of a two-layer FCBody."""
    return body.layers[0].in_features, body.layers[0].out_features, body.layers[1].out_features


def kernel_sizes(D, H1, H2, A, K=None, k_name="atoms", min_actions=2):
    """The kernels' limits: state_dim <= 256, hidden widths <= 128, ``min_actions`` <= actions <= 32 and, for the
    distributional heads, 2 <= atoms / quantiles ``K`` <= 256."""
    if D > 256 or H1 > 128 or H2 > 128 or not min_actions <= A <= 32 or (K is not None and not 2 <= K <= 256):
        return ("sizes beyond the kernels' limits: state_dim %d <= 256, hidden %d / %d <= 128, %sactions %d <= 32%s"
                % (D, H1, H2, "2 <= " if min_actions else "", A, "" if K is None else ", 2 <= %s %d <= 256" % (k_name, K)))


def rmsprop(optimizer, flat=True):
    """``flat``: the agent could build its FlatOptimizer (DQNAgent._flat)."""
    if not isinstance(optimizer, torch.optim.RMSprop) or not flat:
        return "the optimizer is %s; the device update implements RMSprop" % type(optimizer).__name__


def rescale_applied(config):
    if type(config.state_normalizer) is not RescaleNormalizer:
        return "the state normalizer is %s; the device actor applies RescaleNormalizer" % type(config.state_normalizer).__name__


def stock_loss(agent, owner):
    if agent._uses_reference_hooks():
        return "%s overrides compute_loss / reduce_loss; the device update implements %s's" % (type(agent).__name__, owner)


def single_states(history_length, accepted):
    if history_length not in accepted:
        return "history_length is %d; the device kernels read single 1-D states, not frame stacks" % history_length


def fits_one_sm(fn, args, what):
    """``fn``: the C ABI's shared-memory size of the launch; ``what``: the rows it holds, for the reason."""
    smem = getattr(_lib.lib(), fn)(*args)
    if not 0 < smem <= 227 * 1024:
        return "%s needs %d bytes of shared memory, more than one SM has (%s)" % (what, smem, fn)


def two_layer_fc_body(network, config):
    """The body checks of ``dqn_unsupported`` and ``dist_dqn_unsupported``: a two-layer, non-noisy FCBody with tanh or ReLU on
    a CUDA device."""
    body = network.body
    return (fc_body_class(body) or linear_layers(body, config, KERNELS) or two_layers(body) or fc_gate(body.gate)
            or cuda(network))


# ------------------------------------------------------------------------------------------------ the captured paths
def q_actor_unsupported(config, network, states, async_ok=False):
    """``None`` when the DQN-family actor's forward is the captured device path (GraphedQActor) under ``config.cuda_graph``:
    a synchronous actor, a bf16 wgmma NatureConvBody on a CUDA device, an ImageNormalizer-style rescale and uint8 frame stacks
    (``states``: the envs' current observations).  ``async_ok``: the agent orders an actor thread's replays against its updates
    (``ParameterOrder``), so ``async_actor`` is no obstacle."""
    why = graph_requested(config)
    if why:
        return why
    if config.async_actor and not async_ok:
        return "config.async_actor is set; the agent does not order the actor thread's replays against its updates"
    body = getattr(network, "body", None)
    return (nature_conv(body, "body") or linear_layers(body, config, CAPTURED) or four_channels(body) or bf16_wgmma()
            or rescale_folded(config) or frame_stacks(states) or cuda(network))


def nstep_q_graph_unsupported(config, network, optimizer, states):
    """``None`` when ``NStepDQNAgent.step()`` runs as captured graphs under ``config.cuda_graph`` (GraphedQActor per env step,
    learner.GraphedNStepLearner per rollout), else the unmet condition; the agent then keeps its eager path.  ``states``: the
    envs' current observations.  (``config.async_actor`` plays no part: this agent steps its envs itself.)"""
    why = graph_requested(config, "device_nstep_dqn") or network_class(network, VanillaNet, CAPTURED)
    if why:
        return why
    body = network.body
    return (nature_conv(body, "body") or linear_layers(body, config, CAPTURED) or four_channels(body) or bf16_wgmma()
            or fused_tail() or fewer_than_32_actions(network.fc_head.out_features, "narrow head") or rescale_folded(config)
            or frame_stacks(states) or fused_optimizer(optimizer) or cuda(network))


def a2c_graph_unsupported(config, network, optimizer, states):
    """``None`` when ``A2CAgent.step()`` runs as captured graphs under ``config.cuda_graph`` (GraphedQActor with
    learner.GraphedA2CLearner.act per env step, GraphedA2CLearner per rollout), else the unmet condition; the agent then keeps
    its eager path.  ``states``: the envs' current observations."""
    why = (graph_requested(config, "device_a2c") or network_class(network, CategoricalActorCriticNet, CAPTURED)
           or nature_conv(network.phi_body, "phi_body"))
    if why:
        return why
    if not (isinstance(network.actor_body, DummyBody) and isinstance(network.critic_body, DummyBody)):
        return ("the actor / critic bodies are %s / %s; the captured update implements DummyBody for both"
                % (type(network.actor_body).__name__, type(network.critic_body).__name__))
    body = network.phi_body
    return (linear_layers(body, config, CAPTURED) or four_channels(body) or bf16_wgmma() or fused_tail()
            or fewer_than_32_actions(network.fc_action.out_features, "actor-critic head") or rescale_folded(config)
            or frame_stacks(states) or fused_optimizer(optimizer) or cuda(network))


def ppo_graph_unsupported(config, network, optimizer, states):
    """``None`` when ``PPOAgent.step()`` runs as captured graphs under ``config.cuda_graph`` (GraphedQActor with
    learner.GraphedPPOPixelLearner.act per env step, GraphedPPOPixelLearner per rollout), else the unmet condition; the agent
    then keeps its eager path.  The conditions of ``a2c_graph_unsupported`` (the same network, optimizer and frames), plus a
    shared representation (one optimizer over the whole network) and rollouts of whole minibatches.  ``states``: the envs'
    current raw observations."""
    why = graph_requested(config)
    if why:
        return why
    if not config.shared_repr:
        return "config.shared_repr is not set; the captured update implements one optimizer over the shared network"
    rows = config.rollout_length * config.num_workers
    if rows < 2 or rows % config.mini_batch_size:
        return ("the rollout's %d rows are not a multiple of mini_batch_size %d; random_sample would yield a short last "
                "minibatch" % (rows, config.mini_batch_size))
    return a2c_graph_unsupported(config, network, optimizer, states)


def dqn_graph_unsupported(config, agent):
    """``None`` when ``DQNAgent.step()`` (or the C51 / QR-DQN agent's) runs on the captured path with async replay under
    ``config.cuda_graph``: the env transitions staged in learner.GraphedDQNLearner's pinned buffer and one update replay per
    step (``prefetch`` = the graph form of ``ReplayWrapper(async_=True)``, ``wrapper_order``), the actor's forward a
    GraphedQActor replay (on its own thread with ``async_actor``, ordered by ``ParameterOrder``).  Else the unmet condition;
    the agent then keeps its eager path.  Reads ``agent.network``, ``agent.optimizer`` (the torch optimizer), ``agent.replay``
    (the wrapper: its class and keyword arguments) and the agent's class."""
    why = graph_requested(config, "device_dqn", "device_c51", "device_qr", "device_rainbow")
    if why:
        return why
    rp = agent.replay
    if not isinstance(rp, ReplayWrapper) or not rp.async_:
        return ("the replay is not ReplayWrapper(..., async_=True); the captured update with async replay implements its "
                "double buffer")
    if rp.replay_cls not in (UniformReplay, PrioritizedReplay):
        return "the replay is a %s; the captured update implements UniformReplay and PrioritizedReplay" % rp.replay_cls.__name__
    kind = agent._graph_kind
    if kind == "qr" and rp.replay_cls is PrioritizedReplay:
        return "QR-DQN with prioritized replay is undefined in the reference (its loss is per target quantile)"
    net = agent.network
    if type(net).__name__ == "RainbowNet" or config.noisy_linear:
        return "the network is a RainbowNet or has NoisyLinear layers; the captured update implements nn.Linear heads"
    want = {"dqn": (VanillaNet, DuelingNet), "c51": (CategoricalNet,), "qr": (QuantileNet,)}[kind]
    if type(net) not in want:
        return "the network is a %s; the captured update implements %s for %s" % (
            type(net).__name__, " / ".join(c.__name__ for c in want), type(agent).__name__)
    body = net.body
    why = (nature_conv(body, "body") or linear_layers(body, config, CAPTURED) or bf16_wgmma() or fused_tail()
           or rescale_folded(config))
    if why:
        return why
    space = getattr(getattr(config, "eval_env", None), "observation_space", None)
    shape = tuple(getattr(space, "shape", ()) or ())
    dtype = np.dtype(getattr(space, "dtype", None) or np.float64)
    hl = int(rp.replay_kwargs.get("history_length", 1))
    if body.conv1.in_channels != 4 or hl != 4 or shape != (4, 84, 84) or dtype != np.uint8:
        return ("the frames are %s %s with history_length %d into %d channels; the captured update reads 84 x 84 uint8 frames "
                "with a history of 4" % (dtype, shape or "unknown", hl, body.conv1.in_channels))
    if config.num_workers != 1:
        return "%d envs per actor step; the staged feeds follow the reference's one-transition feed() calls" % config.num_workers
    why = fused_optimizer(agent.optimizer)
    if why:
        return why
    if agent._uses_reference_hooks():
        return "%s overrides compute_loss / reduce_loss; the captured update runs the stock loss" % type(agent).__name__
    if getattr(rp, "_primed", False):
        return "the replay wrapper has already handed out an eager batch; its pending batch is not handed to the learner"
    return cuda(net)


# ------------------------------------------------------------------------------------------------ the device kernels
def a2c_unsupported(network, optimizer, config):
    """``None`` when ``config.device_a2c``'s kernels (csrc/a2c.cu) cover this agent, else the unmet condition."""
    fc2 = lambda b: isinstance(b, FCBody) and len(b.layers) == 2 and not b.noisy_linear
    if isinstance(network, CategoricalActorCriticNet):
        if not (fc2(network.phi_body) and isinstance(network.actor_body, DummyBody)
                and isinstance(network.critic_body, DummyBody)):
            return ("a CategoricalActorCriticNet needs a two-layer FCBody phi_body and DummyBody actor / critic bodies "
                    "(got %s / %s / %s)" % tuple(type(b).__name__ for b in (network.phi_body, network.actor_body,
                                                                              network.critic_body)))
        trunks = [network.phi_body]
    elif isinstance(network, GaussianActorCriticNet):
        if not (isinstance(network.phi_body, DummyBody) and fc2(network.actor_body) and fc2(network.critic_body)):
            return ("a GaussianActorCriticNet needs a DummyBody phi_body and two-layer FCBody actor / critic bodies "
                    "(got %s / %s / %s)" % tuple(type(b).__name__ for b in (network.phi_body, network.actor_body,
                                                                              network.critic_body)))
        trunks = [network.actor_body, network.critic_body]
    else:
        return "the network is a %s, not a CategoricalActorCriticNet or GaussianActorCriticNet" % type(network).__name__
    widths = [fc_widths(b) for b in trunks]
    if len(set(widths)) != 1 or len(set(id(b.gate) for b in trunks)) != 1:
        return "the actor and critic bodies must have the same widths and gate"
    D, H1, H2 = widths[0]
    A = network.fc_action.out_features
    head = 0 if isinstance(network, CategoricalActorCriticNet) else 1
    T, N = config.rollout_length, config.num_workers
    return (fc_gate(trunks[0].gate) or cuda(network) or kernel_sizes(D, H1, H2, A, min_actions=0) or rmsprop(optimizer)
            or rescale_applied(config)
            or fits_one_sm("b2rl_a2c_smem_bytes", (head, int(head == 0), D, H1, H2, A, N, T),
                           "a rollout of %d x %d rows" % (T + 1, N)))


def nstep_dqn_unsupported(network, optimizer, config):
    """``None`` when ``config.device_nstep_dqn``'s kernels (csrc/a2c.cu, b2rl_nstep_dqn_*) cover this agent, else the unmet
    condition."""
    if not isinstance(network, VanillaNet):
        return "the network is a %s, not a VanillaNet" % type(network).__name__
    body = network.body
    if not isinstance(body, FCBody):
        return "a VanillaNet needs an FCBody body (got %s)" % type(body).__name__
    if body.noisy_linear:
        return "the FCBody has NoisyLinear layers; the device kernels implement nn.Linear"
    why = two_layers(body) or fc_gate(body.gate) or cuda(network)
    if why:
        return why
    D, H1, H2 = fc_widths(body)
    A, T, N = network.fc_head.out_features, config.rollout_length, config.num_workers
    return (kernel_sizes(D, H1, H2, A) or rmsprop(optimizer) or rescale_applied(config)
            or fits_one_sm("b2rl_nstep_dqn_smem_bytes", (D, H1, H2, A, N, T), "a rollout of %d x %d rows" % (T + 1, N)))


def dqn_unsupported(agent):
    """``None`` when ``config.device_dqn``'s kernels (csrc/a2c.cu: b2rl_nstep_dqn_actor_step, b2rl_dqn_replay_update) cover
    this ``DQNAgent``, else the unmet condition."""
    config, network = agent.config, agent.network
    if type(network) not in (VanillaNet, DuelingNet):
        return ("the network is a %s; the device kernels implement VanillaNet and DuelingNet (C51, QR and Rainbow heads are "
                "not covered)" % type(network).__name__)
    why = stock_loss(agent, "DQNAgent") or two_layer_fc_body(network, config)
    if why:
        return why
    D, H1, H2 = fc_widths(network.body)
    A = (network.fc_advantage if isinstance(network, DuelingNet) else network.fc_head).out_features
    why = kernel_sizes(D, H1, H2, A) or rmsprop(agent.optimizer, agent._flat is not None) or rescale_applied(config)
    if why:
        return why
    if config.async_actor:
        return "async_actor is set; the device actor runs in the agent's thread (async_actor=False)"
    return (single_states(config.history_length, (1,))
            or fits_one_sm("b2rl_dqn_replay_smem_bytes", (int(isinstance(network, DuelingNet)), D, H1, H2, A,
                                                          int(config.batch_size), int(bool(config.double_q))),
                           "a batch of %d" % config.batch_size))


def dist_dqn_unsupported(agent):
    """``None`` when ``config.device_c51`` / ``config.device_qr``'s kernels (csrc/dist_dqn.cu: b2rl_dist_dqn_actor_step,
    b2rl_dist_dqn_replay_update) cover this ``CategoricalDQNAgent`` / ``QuantileRegressionDQNAgent``, else the unmet
    condition."""
    from ..agent.CategoricalDQN_agent import CategoricalDQNAgent
    config, network = agent.config, agent.network
    c51 = isinstance(agent, CategoricalDQNAgent)
    if isinstance(network, RainbowNet):
        return "the network is a RainbowNet; the device kernels implement CategoricalNet (RainbowNet / NoisyLinear is not covered)"
    why = (network_class(network, CategoricalNet if c51 else QuantileNet, KERNELS)
           or stock_loss(agent, agent._fused_owner().__name__) or two_layer_fc_body(network, config))
    if why:
        return why
    D, H1, H2 = fc_widths(network.body)
    A, K = network.action_dim, network.num_atoms if c51 else network.num_quantiles
    why = (kernel_sizes(D, H1, H2, A, K, "atoms" if c51 else "quantiles") or rmsprop(agent.optimizer, agent._flat is not None)
           or rescale_applied(config) or single_states(config.history_length, (None, 1)))
    if why:
        return why
    replay_cls = getattr(agent.replay, "replay_cls", type(agent.replay))
    if not c51 and issubclass(replay_cls, PrioritizedReplay):
        return ("QR-DQN with prioritized replay is undefined in the reference: its loss is per target quantile, not per sample "
                "(QuantileRegressionDQN_agent.py:74)")
    return fits_one_sm("b2rl_dist_dqn_smem_bytes", (int(not c51), D, H1, H2, A, K, int(config.batch_size),
                                                    int(bool(config.double_q))), "a batch of %d" % config.batch_size)


def rainbow_unsupported(agent):
    """``None`` when ``config.device_rainbow``'s kernels (csrc/rainbow.cu: b2rl_rainbow_actor_step, b2rl_rainbow_replay_update)
    cover this agent, else the unmet condition."""
    from ..agent.CategoricalDQN_agent import CategoricalDQNAgent
    from ..network.network_utils import NoisyLinear
    from .actor import rainbow_layers
    config, network = agent.config, agent.network
    if not isinstance(agent, CategoricalDQNAgent):
        return "the agent is a %s; Rainbow is a CategoricalDQNAgent on a RainbowNet" % type(agent).__name__
    why = (network_class(network, RainbowNet, KERNELS) or stock_loss(agent, "CategoricalDQNAgent")
           or fc_body_class(network.body) or two_layers(network.body))
    if why:
        return why
    body = network.body
    noisy = [isinstance(m, NoisyLinear) for m in rainbow_layers(network)]
    if len(set(noisy + [bool(network.noisy_linear), bool(body.noisy_linear), bool(config.noisy_linear)])) != 1:
        return ("the body, the head and config.noisy_linear disagree: the device kernels implement all four layers NoisyLinear "
                "or all four nn.Linear, not a mix")
    why = fc_gate(body.gate) or cuda(network)
    if why:
        return why
    D, H1, H2 = fc_widths(body)
    A, K = network.action_dim, network.num_atoms
    return (kernel_sizes(D, H1, H2, A, K) or rmsprop(agent.optimizer, agent._flat is not None) or rescale_applied(config)
            or single_states(config.history_length, (None, 1))
            or fits_one_sm("b2rl_rainbow_smem_bytes", (int(noisy[0]), D, H1, H2, A, K, int(config.batch_size),
                                                       int(bool(config.double_q))), "a batch of %d" % config.batch_size))
