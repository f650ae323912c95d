"""Device-side actor step for the on-policy agents (SURVEY 8f-3): the work ``PPOAgent`` / ``A2CAgent`` do per env step between
two ``task.step()`` calls (PPO_agent.py:45-50) -- ``MeanStdNormalizer`` (normalizer.py:36-51), the ``GaussianActorCriticNet``
forward (network_heads.py:173-214) and the Normal sample / log-prob / entropy -- as ONE launch of ``b2rl_gaussian_actor_step``
(csrc/actor.cu) on a pinned, double-buffered observation upload.  The envs stay on the host (north_star)."""
import ctypes

import numpy as np
import torch

from .. import _lib
from ..network.network_bodies import DummyBody, FCBody
from ..utils.normalizer import MeanStdNormalizer, RunningMoments

_f32, _f64 = torch.float32, torch.float64


def supported(network, normalizer):
    """GaussianActorCriticNet on a CUDA device with DummyBody phi, two-layer tanh FCBody actor / critic bodies and a
    MeanStdNormalizer (or no normaliser state at all)."""
    try:
        from ..network.network_heads import GaussianActorCriticNet
        ok = (isinstance(network, GaussianActorCriticNet) and isinstance(network.phi_body, DummyBody)
              and all(isinstance(b, FCBody) and len(b.layers) == 2 and b.gate is torch.tanh and not b.noisy_linear
                      for b in (network.actor_body, network.critic_body))
              and network.fc_action.weight.is_cuda and network.fc_action.out_features <= 32
              and max(network.actor_body.layers[0].out_features, network.actor_body.layers[1].out_features) <= 128
              and network.actor_body.layers[0].in_features <= 128
              and isinstance(normalizer, MeanStdNormalizer))
        return bool(ok)
    except Exception:                                    # noqa: BLE001
        return False


class DeviceGaussianActor:
    def __init__(self, network, normalizer, num_envs, seed=0):
        self.net, self.norm = network, normalizer
        dev = network.fc_action.weight.device
        self.dev = dev
        self.N, self.D = int(num_envs), network.actor_body.layers[0].in_features
        self.A = network.fc_action.out_features
        if self.N > 64:
            raise _lib.B2RLError("the device actor serves at most 64 workers per launch")
        self.h_obs = [torch.zeros((self.N, self.D), dtype=_f32, pin_memory=True) for _ in range(2)]
        self.d_obs = [torch.zeros((self.N, self.D), dtype=_f32, device=dev) for _ in range(2)]
        self.slot = 0
        self.rm_mean = torch.zeros(self.D, dtype=_f64, device=dev)
        self.rm_var = torch.ones(self.D, dtype=_f64, device=dev)
        self.rm_count = torch.full((1,), 1e-4, dtype=_f64, device=dev)
        self.counter = torch.zeros(1, dtype=torch.int64, device=dev)
        self.seed = int(seed)
        self.push_stats()

    # ---- the host normaliser object stays the checkpointed / evaluated one: moments move between it and the device
    def push_stats(self):
        rms = self.norm.rms
        if rms is not None:
            self.rm_mean.copy_(torch.from_numpy(np.asarray(rms.mean, dtype=np.float64).reshape(-1)))
            self.rm_var.copy_(torch.from_numpy(np.asarray(rms.var, dtype=np.float64).reshape(-1)))
            self.rm_count.fill_(float(rms.count))

    def pull_stats(self):
        if self.norm.rms is None:
            self.norm.rms = RunningMoments(shape=(1, self.D))
        rms = self.norm.rms
        rms.mean = self.rm_mean.cpu().numpy().reshape(np.shape(rms.mean))
        rms.var = self.rm_var.cpu().numpy().reshape(np.shape(rms.var))
        rms.count = float(self.rm_count.item())

    def step(self, raw_obs, z=None, given_action=None, update=None):
        """raw (un-normalised) observations [N, D] from the envs -> dict(state (normalised), action, log_pi_a, entropy, mean,
        v): device tensors shaped like GaussianActorCriticNet.forward's.  ``z``: supplied standard normals (parity mode)."""
        n = self.net
        k = self.slot
        self.slot = 1 - k
        self.h_obs[k].numpy()[...] = np.asarray(raw_obs, dtype=np.float32).reshape(self.N, self.D)
        self.d_obs[k].copy_(self.h_obs[k], non_blocking=True)
        out = dict(state=torch.empty((self.N, self.D), dtype=_f32, device=self.dev),
                   action=torch.empty((self.N, self.A), dtype=_f32, device=self.dev),
                   log_pi_a=torch.empty((self.N, 1), dtype=_f32, device=self.dev),
                   entropy=torch.empty((self.N, 1), dtype=_f32, device=self.dev),
                   mean=torch.empty((self.N, self.A), dtype=_f32, device=self.dev),
                   v=torch.empty((self.N, 1), dtype=_f32, device=self.dev))
        ab, cb = n.actor_body.layers, n.critic_body.layers
        w = lambda m: _lib.ptr(m.weight.detach())
        b = lambda m: _lib.ptr(m.bias.detach())
        ro = int(bool(update)) if update is not None else (0 if self.norm.read_only else 1)
        _lib.call("b2rl_gaussian_actor_step", _lib.ptr(self.d_obs[k]), _lib.ptr(self.rm_mean), _lib.ptr(self.rm_var),
                  _lib.ptr(self.rm_count), ro, float(self.norm.clip), float(self.norm.epsilon),
                  w(ab[0]), b(ab[0]), w(ab[1]), b(ab[1]), w(n.fc_action), b(n.fc_action),
                  w(cb[0]), b(cb[0]), w(cb[1]), b(cb[1]), w(n.fc_critic), b(n.fc_critic), _lib.ptr(n.std.detach()),
                  self.N, self.D, ab[0].out_features, ab[1].out_features, self.A,
                  _lib.ptr(None if z is None else z.contiguous()), self.seed, _lib.ptr(self.counter),
                  _lib.ptr(None if given_action is None else given_action.contiguous()),
                  _lib.ptr(out["state"]), _lib.ptr(out["action"]), _lib.ptr(out["log_pi_a"]), _lib.ptr(out["entropy"]),
                  _lib.ptr(out["mean"]), _lib.ptr(out["v"]), _lib.stream())
        return out


    # ---- rollout form: outputs written straight into rollout-sized arenas, weight addresses looked up once per rollout
    KEYS = ("state", "action", "log_pi_a", "entropy", "mean", "v")

    def begin_rollout(self, T):
        """Arenas [T + 1, N, dim] for the six outputs of T + 1 actor steps (the last one is the bootstrap value forward) and
        the argument block of the launches (the parameters' addresses change when an optimizer re-points them into its flat
        arena, so they are read again at the start of every rollout)."""
        n, N = self.net, self.N
        if getattr(self, "_T", None) != T:
            dims = dict(state=self.D, action=self.A, log_pi_a=1, entropy=1, mean=self.A, v=1)
            self.roll = {k: torch.empty((T + 1, N, d), dtype=_f32, device=self.dev) for k, d in dims.items()}
            self.h_action = torch.empty((N, self.A), dtype=_f32, pin_memory=True)
            self._stride = {k: N * d * 4 for k, d in dims.items()}
            self._T = T
        self._base = {k: self.roll[k].data_ptr() for k in self.KEYS}
        ab, cb = n.actor_body.layers, n.critic_body.layers
        mods = (ab[0], ab[1], n.fc_action, cb[0], cb[1], n.fc_critic)
        self._wptr = [_lib.ptr(t.detach()) for m in mods for t in (m.weight, m.bias)] + [_lib.ptr(n.std.detach())]
        self._dims = (N, self.D, ab[0].out_features, ab[1].out_features, self.A)
        self._obs_ptr = [_lib.ptr(t) for t in self.d_obs]
        self._np_obs = [t.numpy() for t in self.h_obs]
        self._fixed = (_lib.ptr(self.rm_mean), _lib.ptr(self.rm_var), _lib.ptr(self.rm_count))

    def step_into(self, t, raw_obs, update):
        """Actor step ``t`` of the rollout begun with ``begin_rollout``: outputs go to ``roll[key][t]``; returns the actions as
        a host array (pinned download + one stream synchronise)."""
        k = self.slot
        self.slot = 1 - k
        self._np_obs[k][...] = np.asarray(raw_obs, dtype=np.float32).reshape(self.N, self.D)
        self.d_obs[k].copy_(self.h_obs[k], non_blocking=True)
        at = lambda key: ctypes.c_void_p(self._base[key] + t * self._stride[key])
        _lib.call("b2rl_gaussian_actor_step", self._obs_ptr[k], *self._fixed, int(bool(update)), float(self.norm.clip),
                  float(self.norm.epsilon), *self._wptr, *self._dims, None, self.seed, _lib.ptr(self.counter), None,
                  at("state"), at("action"), at("log_pi_a"), at("entropy"), at("mean"), at("v"), _lib.stream())
        self.h_action.copy_(self.roll["action"][t], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self.h_action.numpy().copy()


class GraphedQActor:
    """The DQN-family actor's forward pass (DQN_agent.py:29-31: ``network(state_normalizer(stack(state)))`` at batch
    ``num_envs``, normally 1) as ONE CUDA-graph replay: pinned upload of the uint8 frame stacks -> frame-stack conversion to
    the exact-integer bf16 space-to-depth layout (``b2rl_replay_gather`` on the staging buffer; ImageNormalizer's 1/255 is
    folded into conv1 like in the learner) -> the network on the wgmma kernels -> action values -> pinned download.  The
    epsilon-greedy draw stays on the host (``epsilon_greedy``: the reference's numpy stream, torch_utils.py:51-58).

    The eager form of the same step is ~40 kernel / memcpy launches of Python-driven work per env step; this is one launch and
    one stream synchronise."""

    def __init__(self, network, q_fn, num_envs, history, frame_hw, scale):
        p = next(network.parameters())
        self.net, self.q_fn, self.dev = network, q_fn, p.device
        self.N, self.hl, self.hw, self.scale = int(num_envs), int(history), tuple(frame_hw), float(scale)
        self.row = self.hw[0] * self.hw[1]
        rows = self.N * self.hl + 1                       # (+1: the gather kernel stages history + n_step rows)
        self.h_frames = torch.zeros((rows, self.row), dtype=torch.uint8, pin_memory=True)
        self.d_frames = torch.zeros((rows, self.row), dtype=torch.uint8, device=self.dev)
        self._np_frames = self.h_frames.numpy()[:self.N * self.hl].reshape(self.N, self.hl, self.row)
        self.idx = (torch.arange(self.N, dtype=torch.int64) * self.hl + self.hl - 1).to(self.dev)
        self.d_action = torch.zeros(rows, dtype=torch.int32, device=self.dev)      # (scalar columns of the ring API: unused)
        self.d_reward = torch.zeros(rows, dtype=torch.float64, device=self.dev)
        self.d_mask = torch.ones(rows, dtype=torch.int32, device=self.dev)
        self.x = torch.empty((self.N, self.hw[0] // 4, self.hw[1] // 4, 16 * self.hl), dtype=torch.bfloat16, device=self.dev)
        self.d_q = self.h_q = None
        self.graph, self._sig = None, None
        self.replays = 0

    def _signature(self):
        """What the captured launch sequence depends on besides addresses: who re-packs the body's bf16 operands (the body per
        forward, or the learner's optimizer kernel) and whether the distributional heads have their bf16 operand."""
        body = getattr(self.net, "body", None)
        heads = tuple(getattr(m, "_w16", None) is not None for m in self.net.children() if isinstance(m, torch.nn.Linear))
        return (bool(getattr(body, "auto_repack", True)), heads)

    def _forward(self):
        from ..network.fused import frame_scale
        self.d_frames.copy_(self.h_frames, non_blocking=True)
        _lib.call("b2rl_replay_gather", _lib.ptr(self.d_frames), _lib.ptr(self.d_action), _lib.ptr(self.d_reward),
                  _lib.ptr(self.d_mask), self.d_frames.shape[0], self.row, _lib.ptr(self.idx), self.N, self.hl, 1, 1.0, None,
                  _lib.DTYPE_CODE[torch.bfloat16], 2, self.hw[1], _lib.ptr(self.x), None, None, None, None, _lib.stream())
        with torch.no_grad(), frame_scale(self.scale):
            q = self.q_fn(self.net(self.x.permute(0, 3, 1, 2))).float()
        if self.d_q is None:
            self.d_q = torch.empty_like(q)
            self.h_q = torch.empty(q.shape, dtype=torch.float32, pin_memory=True)
        self.d_q.copy_(q)
        self.h_q.copy_(self.d_q, non_blocking=True)

    def _capture(self):
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):                     # eager warm-up (lazy allocations, cuBLAS workspaces of library heads)
            self._forward()
        cur.wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._forward()
        self._sig = self._signature()

    def q_values(self, states):
        """``states``: ``num_envs`` frame stacks (LazyFrames / uint8 arrays [history, H, W]).  Returns float32 [num_envs, A]."""
        for i, s in enumerate(states):
            a = np.asarray(s)
            if a.dtype != np.uint8 or a.size != self.hl * self.row:
                raise _lib.B2RLError("GraphedQActor expects uint8 frame stacks of %d x %s" % (self.hl, self.hw))
            self._np_frames[i] = a.reshape(self.hl, self.row)
        if self.graph is None or self._sig != self._signature():
            self._capture()
        self.graph.replay()
        self.replays += 1
        torch.cuda.current_stream().synchronize()
        return self.h_q.numpy().copy()


def q_actor_supported(config, network):
    """``config.cuda_graph`` + synchronous actor + bf16 wgmma NatureConvBody on a CUDA device + ImageNormalizer-style rescale
    of uint8 frames: the conditions under which the actor's forward is the captured device path."""
    from ..network.network_bodies import NatureConvBody
    from ..utils import Config
    from ..utils.normalizer import RescaleNormalizer
    body = getattr(network, "body", None)
    return bool(getattr(config, "cuda_graph", False) and not config.async_actor and not config.noisy_linear
                and isinstance(body, NatureConvBody) and not body.noisy_linear and body.conv1.weight.is_cuda
                and body.conv1.in_channels == 4
                and Config.COMPUTE_DTYPE == torch.bfloat16 and Config.DENSE_BACKEND == "tcgen05"
                and isinstance(config.state_normalizer, RescaleNormalizer))
