"""Device-side actor step for the on-policy agents (SURVEY 8f-3): the work ``PPOAgent`` / ``A2CAgent`` do per env step between
two ``task.step()`` calls (PPO_agent.py:45-50) -- ``MeanStdNormalizer`` (normalizer.py:36-51), the ``GaussianActorCriticNet``
forward (network_heads.py:173-214) and the Normal sample / log-prob / entropy -- as ONE launch of ``b2rl_gaussian_actor_step``
(csrc/actor.cu) on a pinned, double-buffered observation upload.  The envs stay on the host (north_star)."""
import contextlib
import ctypes
import gc

import numpy as np
import torch

from .. import _lib
from ..network.network_bodies import DummyBody, FCBody
from ..utils.normalizer import MeanStdNormalizer, RunningMoments
from .coverage import a2c_unsupported, dist_dqn_unsupported, dqn_unsupported, nstep_dqn_unsupported, rainbow_unsupported
# the captured paths' predicates stay importable from here, where callers have always found them
from .coverage import a2c_graph_unsupported, dqn_graph_unsupported, nstep_q_graph_unsupported, ppo_graph_unsupported  # noqa: F401

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
    one stream synchronise.

    ``arena``: a uint8 device tensor [slots * num_envs * history + 1, H * W] that receives the uploaded stacks instead of the
    actor's own one-slot buffer: ``q_values(states, slot)`` uploads them into rows ``slot * num_envs * history ...`` and
    forwards from there (one captured graph per slot), so a learner can read a whole rollout's frame stacks from the arena
    without uploading them again (learner.GraphedNStepLearner).  The last row is padding the gather stages but never uses.

    ``run``: what runs on the gathered batch instead of ``q_fn(network(x))``: ``run(x, slot)`` returns the device tensor that
    ``q_values`` downloads (learner.GraphedA2CLearner.act: the body, the actor-critic head and the action draw, returning the
    actions).  ``body``: the network's NatureConvBody when it is not ``network.body`` (``phi_body`` of an actor-critic net)."""

    def __init__(self, network, q_fn, num_envs, history, frame_hw, scale, arena=None, run=None, body=None):
        p = next(network.parameters())
        self.net, self.q_fn, self.run, self.dev = network, q_fn, run, p.device
        self.body = body if body is not None else getattr(network, "body", None)
        self.N, self.hl, self.hw, self.scale = int(num_envs), int(history), tuple(frame_hw), float(scale)
        self.row = self.hw[0] * self.hw[1]
        rows = self.N * self.hl + 1                       # (+1: the gather kernel stages history + n_step rows)
        self.h_frames = torch.zeros((rows, self.row), dtype=torch.uint8, pin_memory=True)
        if arena is None:
            self.d_frames = torch.zeros((rows, self.row), dtype=torch.uint8, device=self.dev)
        else:
            ok = (arena.dtype == torch.uint8 and arena.device == self.dev and arena.dim() == 2 and arena.shape[1] == self.row
                  and arena.is_contiguous() and (arena.shape[0] - 1) % (self.N * self.hl) == 0 and arena.shape[0] > 1)
            if not ok:
                raise _lib.B2RLError("GraphedQActor: the arena must be a contiguous uint8 tensor [slots * %d + 1, %d] on %s"
                                     % (self.N * self.hl, self.row, self.dev))
            self.d_frames = arena
        self.slots = (self.d_frames.shape[0] - 1) // (self.N * self.hl)
        self._np_frames = self.h_frames.numpy()[:self.N * self.hl].reshape(self.N, self.hl, self.row)
        last = torch.arange(self.N, dtype=torch.int64) * self.hl + self.hl - 1
        self.idxs = [(last + s * self.N * self.hl).to(self.dev) for s in range(self.slots)]
        self.idx = self.idxs[0]
        n = self.d_frames.shape[0]
        self.d_action = torch.zeros(n, dtype=torch.int32, device=self.dev)         # (scalar columns of the ring API: unused)
        self.d_reward = torch.zeros(n, dtype=torch.float64, device=self.dev)
        self.d_mask = torch.ones(n, dtype=torch.int32, device=self.dev)
        self.x = torch.empty((self.N, self.hw[0] // 4, self.hw[1] // 4, 16 * self.hl), dtype=torch.bfloat16, device=self.dev)
        self.d_q = self.h_q = None
        self.graphs, self._sig = [None] * self.slots, None
        self.replays = 0
        self.capture_error_mode = "global"                # "thread_local": captured on an actor thread (ParameterOrder)

    @property
    def graph(self):
        return self.graphs[0]

    def _signature(self):
        """What the captured launch sequence depends on besides addresses: who re-packs the body's bf16 operands (the body per
        forward, or the learner's optimizer kernel) and whether the distributional heads have their bf16 operand."""
        heads = tuple(getattr(m, "_w16", None) is not None for m in self.net.children() if isinstance(m, torch.nn.Linear))
        return (bool(getattr(self.body, "auto_repack", True)), heads)

    def _forward(self, slot=0):
        from ..network.fused import frame_scale
        k = self.N * self.hl
        self.d_frames[slot * k:(slot + 1) * k].copy_(self.h_frames[:k], non_blocking=True)
        _lib.call("b2rl_replay_gather", _lib.ptr(self.d_frames), _lib.ptr(self.d_action), _lib.ptr(self.d_reward),
                  _lib.ptr(self.d_mask), self.d_frames.shape[0], self.row, _lib.ptr(self.idxs[slot]), self.N, self.hl, 1, 1.0, None,
                  _lib.DTYPE_CODE[torch.bfloat16], 2, self.hw[1], _lib.ptr(self.x), None, None, None, None, _lib.stream())
        with torch.no_grad(), frame_scale(self.scale):
            x = self.x.permute(0, 3, 1, 2)
            q = self.run(x, slot) if self.run is not None else self.q_fn(self.net(x)).float()
        if self.d_q is None:
            self.d_q = torch.empty_like(q)
            self.h_q = torch.empty(q.shape, dtype=q.dtype, pin_memory=True)
        self.d_q.copy_(q)
        self.h_q.copy_(self.d_q, non_blocking=True)

    def _capture(self, slot=0):
        if self._sig != self._signature():               # the launch sequence changed: every slot's graph is stale
            self.graphs = [None] * self.slots
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):                     # eager warm-up (lazy allocations, cuBLAS workspaces of library heads)
            self._forward(slot)
        cur.wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        pool = next((h.pool() for h in self.graphs if h is not None), None)     # the slots' graphs replay one at a time
        with no_gc(), torch.cuda.graph(g, pool=pool, capture_error_mode=self.capture_error_mode):
            self._forward(slot)
        self.graphs[slot] = g
        self._sig = self._signature()

    def q_values(self, states, slot=0):
        """``states``: ``num_envs`` frame stacks (LazyFrames / uint8 arrays [history, H, W]).  Returns float32 [num_envs, A]
        (with ``run``: what it returns, on the host).  ``slot``: where in the arena the stacks land (0 without an arena)."""
        self.enqueue(states, slot)
        return self.result()

    def enqueue(self, states, slot=0):
        """The first half of ``q_values``: stage the stacks, capture if needed and replay, on the current stream."""
        for i, s in enumerate(states):
            a = np.asarray(s)
            if a.dtype != np.uint8 or a.size != self.hl * self.row:
                raise _lib.B2RLError("GraphedQActor expects uint8 frame stacks of %d x %s" % (self.hl, self.hw))
            self._np_frames[i] = a.reshape(self.hl, self.row)
        if self.graphs[slot] is None or self._sig != self._signature():
            self._capture(slot)
        self.graphs[slot].replay()
        self.replays += 1

    def result(self):
        """The second half of ``q_values``: wait for the replay (on the current stream) and return its download."""
        torch.cuda.current_stream().synchronize()
        return self.h_q.numpy().copy()


class ParameterOrder:
    """What ``config.lock`` guarantees between the DQN agent's actor thread and its learner (DQN_agent.py:30,133: a forward
    reads one whole parameter version), moved onto the device for the captured path with ``async_actor``.  The actor replays
    on a stream of its own; each actor replay waits for the event recorded after the latest update replay (``updated``) and
    each update replay waits for the one recorded after the latest actor replay (``acted``), so a forward never runs while an
    update's tail rewrites the packed bf16 operands, nor an update while a forward reads them.  The host holds ``lock`` only
    while it enqueues the wait, the replay and the record (and while it captures), never across a synchronise: the learner
    does not wait on the host for the actor's forward, and the actor's wait for its own q values leaves the learner free."""

    def __init__(self, lock):
        self.lock = lock
        self.updated, self.acted = torch.cuda.Event(), torch.cuda.Event()
        self.stream = None                                # the actor's stream, made on the actor thread

    def actor_stream(self):
        if self.stream is None:
            self.stream = torch.cuda.Stream()
        return self.stream


@contextlib.contextmanager
def no_gc():
    """No garbage collection inside a graph capture: collecting unreachable objects that own CUDA resources (pinned buffers,
    graphs, streams of an agent dropped earlier) frees them mid-capture, which invalidates the capture."""
    enabled = gc.isenabled()
    gc.disable()
    try:
        yield
    finally:
        if enabled:
            gc.enable()


# ------------------------------------------------------------------------------------------------ A2C on the device
class _DeviceRollout:
    """What ``DeviceA2C``, ``DeviceNStepDQN`` and ``DeviceDQN`` share: the rollout arenas, the pinned double-buffered float64
    observation upload, rewards / masks (uploaded once per rollout), the action download, the parity-mode actions, the Philox
    counter, the check that the parameters still live in the optimizer's arena and, for the Q agents, the target arena.  The
    subclass sets ``opt``, ``dev``, ``tensors`` (kernel order), ``cfg``, ``N``, ``T``, ``D`` and ``acols`` first."""

    def _adopt_target(self, target_network):
        """The target network's parameters become views into ``target``, a second arena of the online arena's layout (their
        values kept), so the target sync is one device copy and the module's ``state_dict()`` is always current."""
        self.target = torch.zeros_like(self.opt.flat)
        with torch.no_grad():
            for p, o in zip(target_network.parameters(), self.opt.offsets):
                k = p.numel()
                self.target[o:o + k].copy_(p.detach().reshape(-1))
                p.data = self.target[o:o + k].view_as(p)

    def _check_target(self, tensors, owner):
        """``tensors``: the target network's parameters in kernel order, each at its online twin's offset in ``target``."""
        base = self.target.data_ptr()
        for t, o in zip(tensors, self.off.tolist()):
            if t.data_ptr() != base + 4 * o:
                raise _lib.B2RLError("%s: a target parameter no longer lives in the target arena" % owner)

    def _buffers(self, seed):
        N, T, D, acols = self.N, self.T, self.D, self.acols
        self.states = torch.zeros((T + 1, N, D), dtype=_f32, device=self.dev)
        self.actions = torch.zeros((T, N, acols), dtype=_f32, device=self.dev)
        self.rm = torch.zeros((2, T, N), dtype=_f32, device=self.dev)                 # rewards, masks
        self.h_rm = torch.zeros((2, T, N), dtype=_f32, pin_memory=True)
        self.h_obs = [torch.zeros((N, D), dtype=_f64, pin_memory=True) for _ in range(2)]
        self.d_obs = [torch.zeros((N, D), dtype=_f64, device=self.dev) for _ in range(2)]
        self.h_last = torch.zeros((N, D), dtype=_f32, pin_memory=True)
        self.h_action = torch.zeros((N, acols), dtype=_f32, pin_memory=True)
        self.h_given = torch.zeros((N, acols), dtype=_f32, pin_memory=True)
        self.d_given = torch.zeros((N, acols), dtype=_f32, device=self.dev)
        self.counter = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self.seed = int(seed)
        self.off = torch.zeros(len(self.tensors), dtype=torch.int32)
        self.slot = 0
        self.forced = None
        self.rewards, self.masks = self.h_rm[0].numpy(), self.h_rm[1].numpy()

    def _arena_offsets(self):
        """Arena offsets of the parameters, read once per rollout (and checked: a parameter re-pointed out of the arena would
        otherwise be trained in a copy nobody reads), and the launch arguments that follow from them."""
        base, n = self.opt.flat.data_ptr(), self.opt.n
        for i, t in enumerate(self.tensors):
            o = (t.data_ptr() - base) // 4
            if not (0 <= o and o + t.numel() <= n and t.is_contiguous()):
                raise _lib.B2RLError("%s: a parameter no longer lives in the optimizer's arena" % type(self).__name__)
            self.off[i] = o
        self._flat = _lib.ptr(self.opt.flat)
        self._off = _lib.ptr(self.off)
        self._obs = [_lib.ptr(t) for t in self.d_obs]
        self._np_obs = [t.numpy() for t in self.h_obs]
        self._row = self.N * self.D * 4, self.N * self.acols * 4
        self._scale = float(self.cfg.state_normalizer.coef)

    def _stage(self, raw_obs):
        """The env step's raw observations up (pinned, double-buffered) and, in parity mode, the given actions; returns the
        device addresses of both (None: draw)."""
        k = self.slot
        self.slot = 1 - k
        self._np_obs[k][...] = np.asarray([np.asarray(s) for s in raw_obs], dtype=np.float64).reshape(self.N, self.D)
        self.d_obs[k].copy_(self.h_obs[k], non_blocking=True)
        given = None
        if self.forced is not None:
            self.h_given.numpy()[...] = np.asarray(self.forced(), dtype=np.float32).reshape(self.N, self.acols)
            self.d_given.copy_(self.h_given, non_blocking=True)
            given = _lib.ptr(self.d_given)
        return self._obs[k], given

    def _row_ptrs(self, t):
        return (ctypes.c_void_p(self.states.data_ptr() + t * self._row[0]),
                ctypes.c_void_p(self.actions.data_ptr() + t * self._row[1]))

    def _fetch(self, t):
        """Row t of the action arena down to the host (pinned copy + one stream synchronise)."""
        self.h_action.copy_(self.actions[t], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self.h_action.numpy()

    def _stage_last(self, last_states):
        """The final (normalised) observations into row T; rewards / masks (``self.rewards`` / ``self.masks``, filled by the
        caller) up in one copy."""
        self.h_last.numpy()[...] = np.asarray(last_states, dtype=np.float32).reshape(self.N, self.D)
        self.states[self.T].copy_(self.h_last, non_blocking=True)
        self.rm.copy_(self.h_rm, non_blocking=True)


class DeviceA2C(_DeviceRollout):
    """``A2CAgent.step()`` on the device (``config.device_a2c``): the rollout arenas, the pinned upload / download buffers,
    the Philox counter and the arguments of ``b2rl_a2c_actor_step`` (one launch per env step) and ``b2rl_a2c_update`` (one
    launch per rollout).  The torch RMSprop built by ``config.optimizer_fn`` is replaced by a ``FlatOptimizer`` with the same
    hyper-parameters: the module's parameters become views into its arena, so ``state_dict()`` is always current.

    ``forced``: test hook -- a callable returning the actions of the next env step, which the actor step then writes through
    unchanged instead of drawing (parity mode)."""

    def __init__(self, network, optimizer, config, seed):
        import torch.nn.functional as F

        from .. import ops
        from ..network.network_heads import CategoricalActorCriticNet
        why = a2c_unsupported(network, optimizer, config)
        if why is not None:
            raise NotImplementedError("config.device_a2c: " + why)
        n = network
        self.net, self.cfg = n, config
        self.head = 0 if isinstance(n, CategoricalActorCriticNet) else 1
        self.shared = int(self.head == 0)
        trunks = [n.phi_body] if self.shared else [n.actor_body, n.critic_body]
        self.gate = 0 if trunks[0].gate is torch.tanh else 1
        assert trunks[0].gate in (torch.tanh, F.relu)
        self.tensors = [t for b in trunks for m in b.layers for t in (m.weight, m.bias)]
        self.tensors += [n.fc_action.weight, n.fc_action.bias, n.fc_critic.weight, n.fc_critic.bias]
        if self.head == 1:
            self.tensors.append(n.std)
        self.opt = ops.FlatOptimizer.from_torch(optimizer, list(n.parameters()))
        self.dev = self.opt.flat.device
        self.N, self.T = int(config.num_workers), int(config.rollout_length)
        self.D, self.H1, self.H2 = trunks[0].layers[0].in_features, trunks[0].layers[0].out_features, trunks[0].layers[1].out_features
        self.A = n.fc_action.out_features
        self.acols = 1 if self.head == 0 else self.A
        self._buffers(seed)

    def begin_rollout(self):
        self._arena_offsets()
        self._net = (self.head, self.shared, self.gate)
        self._dims = (self.D, self.H1, self.H2, self.A)

    def act(self, t, raw_obs):
        """Env step ``t`` of the rollout: rescale + forward + draw in one launch; returns the actions for ``task.step``."""
        obs, given = self._stage(raw_obs)
        _lib.call("b2rl_a2c_actor_step", *self._net, obs, self._scale, self._flat, self._off, *self._dims, self.N,
                  *self._row_ptrs(t), given, self.seed, _lib.ptr(self.counter), _lib.stream())
        a = self._fetch(t)
        return a[:, 0].astype(np.int64) if self.head == 0 else a.copy()

    def update(self, last_states):
        """The final observations and the rollout's rewards / masks up, then the update launch.  Returns the objective as a
        0-dim device tensor."""
        c = self.cfg
        self._stage_last(last_states)
        loss = torch.empty((), dtype=_f32, device=self.dev)
        o = self.opt
        _lib.call("b2rl_a2c_update", *self._net, _lib.ptr(self.states), _lib.ptr(self.actions), _lib.ptr(self.rm[0]),
                  _lib.ptr(self.rm[1]), self.T, self.N, *self._dims, self._flat, _lib.ptr(o.s1), _lib.ptr(o.s2),
                  _lib.ptr(o.step_dev), self._off, float(o.lr), float(o.alpha), float(o.eps), int(o.centered),
                  float(c.discount), float(c.gae_tau), int(bool(c.use_gae)), float(c.entropy_weight),
                  float(c.value_loss_weight), float(c.gradient_clip), _lib.ptr(loss), _lib.stream())
        return loss


# ------------------------------------------------------------------------------------------------ n-step Q on the device
class DeviceNStepDQN(_DeviceRollout):
    """``NStepDQNAgent.step()`` on the device (``config.device_nstep_dqn``): one ``b2rl_nstep_dqn_actor_step`` launch per env
    step (epsilon-greedy on the device's Philox stream) and one ``b2rl_nstep_dqn_update`` launch per rollout, which also does the
    rollout's target sync.  The torch RMSprop built by ``config.optimizer_fn`` is replaced by a ``FlatOptimizer`` with the same
    hyper-parameters, and the target network's parameters become views into a second arena of the same layout (``target``), so
    both modules' ``state_dict()`` are always current.

    ``forced``: test hook -- a callable returning the actions of the next env step, which the actor step then writes through
    unchanged instead of drawing (parity mode)."""

    def __init__(self, network, target_network, optimizer, config, seed):
        from .. import ops
        why = nstep_dqn_unsupported(network, optimizer, config)
        if why is not None:
            raise NotImplementedError("config.device_nstep_dqn: " + why)
        self.net, self.target_net, self.cfg = network, target_network, config
        body = network.body
        self.gate = 0 if body.gate is torch.tanh else 1
        self.tensors = self.kernel_order(network)
        self.opt = ops.FlatOptimizer.from_torch(optimizer, list(network.parameters()))
        self.dev = self.opt.flat.device
        self._adopt_target(target_network)
        self.N, self.T = int(config.num_workers), int(config.rollout_length)
        self.D, self.H1, self.H2 = body.layers[0].in_features, body.layers[0].out_features, body.layers[1].out_features
        self.A = network.fc_head.out_features
        self.acols = 1
        self._buffers(seed)

    @staticmethod
    def kernel_order(net):
        """A VanillaNet's parameters in the kernels' tensor order: w1 b1 w2 b2 fc_head.w fc_head.b."""
        return [t for m in net.body.layers for t in (m.weight, m.bias)] + [net.fc_head.weight, net.fc_head.bias]

    def begin_rollout(self):
        self._arena_offsets()
        self._check_target(self.kernel_order(self.target_net), "DeviceNStepDQN")
        self._dims = (self.D, self.H1, self.H2, self.A)

    def act(self, t, raw_obs, epsilon):
        """Env step ``t`` of the rollout: rescale + forward + epsilon-greedy in one launch; returns the actions for
        ``task.step``."""
        obs, given = self._stage(raw_obs)
        _lib.call("b2rl_nstep_dqn_actor_step", self.gate, obs, self._scale, self._flat, self._off, *self._dims, self.N,
                  float(epsilon), *self._row_ptrs(t), given, self.seed, _lib.ptr(self.counter), _lib.stream())
        return self._fetch(t)[:, 0].astype(np.int64)

    def update(self, last_states, sync_target):
        """The final observations and the rollout's rewards / masks up, then the update launch; ``sync_target``: an env step of
        this rollout reached the target sync schedule.  Returns the objective as a 0-dim device tensor."""
        c, o = self.cfg, self.opt
        self._stage_last(last_states)
        loss = torch.empty((), dtype=_f32, device=self.dev)
        _lib.call("b2rl_nstep_dqn_update", self.gate, _lib.ptr(self.states), _lib.ptr(self.actions), _lib.ptr(self.rm[0]),
                  _lib.ptr(self.rm[1]), self.T, self.N, *self._dims, self._flat, _lib.ptr(self.target), int(bool(sync_target)),
                  _lib.ptr(o.s1), _lib.ptr(o.s2), _lib.ptr(o.step_dev), self._off, float(o.lr), float(o.alpha), float(o.eps),
                  int(o.centered), float(c.discount), float(c.gradient_clip), _lib.ptr(loss), _lib.stream())
        return loss


# ------------------------------------------------------------------------------------------------ replay DQN on the device
def dqn_kernel_order(net):
    """A VanillaNet's / DuelingNet's / CategoricalNet's / QuantileNet's parameters in the kernels' tensor order: w1 b1 w2 b2,
    then fc_head.w fc_head.b, or fc_advantage.w fc_advantage.b fc_value.w fc_value.b, or fc_categorical.w fc_categorical.b, or
    fc_quantiles.w fc_quantiles.b."""
    from ..network.network_heads import DuelingNet
    body = [t for m in net.body.layers for t in (m.weight, m.bias)]
    if isinstance(net, DuelingNet):
        return body + [net.fc_advantage.weight, net.fc_advantage.bias, net.fc_value.weight, net.fc_value.bias]
    head = next(getattr(net, k) for k in ("fc_head", "fc_categorical", "fc_quantiles") if hasattr(net, k))
    return body + [head.weight, head.bias]


class DeviceDQN(_DeviceRollout):
    """``DQNAgent.step()`` on the device (``config.device_dqn``): one ``b2rl_nstep_dqn_actor_step`` launch per env step
    (rescale, forward, epsilon-greedy on the device's Philox stream) and one ``b2rl_dqn_replay_update`` launch per gradient
    update on the batch ``replay.sample()`` returned.  The update trains ``DQNAgent._flat``'s arena; the target network's
    parameters become views into a second arena of the same layout (``target``), so the target sync is one device copy and both
    modules' ``state_dict()`` are always current.

    ``forced``: test hook -- a callable returning the actions of the next env step, which the actor step then writes through
    unchanged instead of drawing."""

    flag = "config.device_dqn"

    unsupported = staticmethod(dqn_unsupported)

    def __init__(self, agent, seed):
        from ..network.network_heads import DuelingNet
        why = self.unsupported(agent)
        if why is not None:
            raise NotImplementedError(self.flag + ": " + why)
        config, network = agent.config, agent.network
        self.net, self.target_net, self.cfg = network, agent.target_network, config
        body = network.body
        self.head = int(isinstance(network, DuelingNet))
        self.gate = 0 if body.gate is torch.tanh else 1
        self.tensors = self._tensors(network)
        self.opt = agent._flat
        self.dev = self.opt.flat.device
        self._adopt_target(agent.target_network)
        self.N, self.T = int(config.num_workers), 1
        self.D, self.H1, self.H2 = body.layers[0].in_features, body.layers[0].out_features, body.layers[1].out_features
        self.A = self.tensors[4].shape[0]
        self.acols = 1
        self._buffers(seed)
        self._dims = (self.D, self.H1, self.H2, self.A)
        self._offsets()

    @staticmethod
    def _tensors(net):
        return dqn_kernel_order(net)

    def _offsets(self):
        """``_arena_offsets``, and the check that the target parameters still live in the target arena."""
        self._arena_offsets()
        self._check_target(self._tensors(self.target_net), "DeviceDQN")

    def act(self, raw_obs, epsilon):
        """One env step's actions: rescale + forward + epsilon-greedy in one launch, downloaded for ``task.step``."""
        obs, given = self._stage(raw_obs)
        _lib.call("b2rl_nstep_dqn_actor_step", self.gate + 2 * self.head, obs, self._scale, self._flat, self._off, *self._dims,
                  self.N, float(epsilon), None, self._row_ptrs(0)[1], given, self.seed, _lib.ptr(self.counter), _lib.stream())
        return self._fetch(0)[:, 0].astype(np.int64)

    def _check_states(self, s):
        if s.dtype not in (_f32, _f64) or s.dim() != 2 or s.shape[1] != self.D:
            raise NotImplementedError("%s: the replay returned %s states of shape %s; the device update reads 1-D float32 / "
                                      "float64 rows of %d" % (self.flag, s.dtype, tuple(s.shape), self.D))

    def update(self, tr, beta=0.0):
        """One gradient update on a sampled batch (``Transition`` / ``PrioritizedTransition`` of device tensors).  Returns the
        objective (0-dim device tensor) and, for a prioritized batch, the new priorities (float32 device tensor [B])."""
        c, o = self.cfg, self.opt
        s, s2 = tr.state, tr.next_state
        self._check_states(s)
        self._offsets()
        B = s.shape[0]
        per = getattr(tr, "sampling_prob", None) is not None
        loss = torch.empty((), dtype=_f32, device=self.dev)
        prio = torch.empty(B, dtype=_f32, device=self.dev) if per else None
        ptr = lambda t: _lib.ptr(None if t is None else t.contiguous())
        _lib.call("b2rl_dqn_replay_update", self.head, self.gate, ptr(s), ptr(s2), int(s.dtype == _f64), self._scale,
                  ptr(tr.action), ptr(tr.reward), ptr(tr.mask), B, *self._dims, self._flat, _lib.ptr(self.target),
                  _lib.ptr(o.s1), _lib.ptr(o.s2), _lib.ptr(o.step_dev), self._off, float(o.lr), float(o.alpha), float(o.eps),
                  int(o.centered), float(c.discount ** c.n_step), int(bool(c.double_q)), float(c.gradient_clip or 0.0),
                  ptr(tr.sampling_prob if per else None), float(beta), float(getattr(c, "replay_eps", 0.01)),
                  float(getattr(c, "replay_alpha", 0.5)), ptr(prio), None, _lib.ptr(loss), _lib.stream())
        return loss, prio

    def sync_target(self):
        """DQN_agent.py:136-138: the target arena becomes the online arena (one device copy)."""
        self.target.copy_(self.opt.flat)


# ------------------------------------------------------------------------------------------------ C51 / QR-DQN on the device
class DeviceDistDQN(DeviceDQN):
    """``CategoricalDQNAgent.step()`` / ``QuantileRegressionDQNAgent.step()`` on the device (``config.device_c51`` /
    ``config.device_qr``): one ``b2rl_dist_dqn_actor_step`` launch per env step (rescale, forward, the action values,
    epsilon-greedy on the device's Philox stream) and one ``b2rl_dist_dqn_replay_update`` launch per gradient update.  The
    arenas, the target network's parameters as views into the target arena, the staging buffers and the target sync are
    ``DeviceDQN``'s.

    With ``async_actor`` the actor thread calls ``act`` (inside ``config.lock``, as ``DQNActor._transition`` does) and the agent
    calls ``update`` under the same lock; both launch on torch's current stream.  The staging buffers and the Philox counter are
    only touched by ``act``."""

    @property
    def flag(self):
        return "config.device_c51" if self.kind == 0 else "config.device_qr"

    unsupported = staticmethod(dist_dqn_unsupported)

    def __init__(self, agent, seed):
        from ..agent.CategoricalDQN_agent import CategoricalDQNAgent
        self.kind = 0 if isinstance(agent, CategoricalDQNAgent) else 1      # C51, QR
        super().__init__(agent, seed)
        n, c = agent.network, agent.config
        self.A = n.action_dim
        self.K = n.num_atoms if self.kind == 0 else n.num_quantiles
        self.v_min = float(getattr(c, "categorical_v_min", 0.0)) if self.kind == 0 else 0.0
        self.v_max = float(getattr(c, "categorical_v_max", 1.0)) if self.kind == 0 else 1.0
        self._dims = (self.D, self.H1, self.H2, self.A, self.K)

    def act(self, raw_obs, epsilon):
        """One env step's actions: rescale + forward + action values + epsilon-greedy in one launch, downloaded for
        ``task.step``."""
        obs, given = self._stage(raw_obs)
        _lib.call("b2rl_dist_dqn_actor_step", self.kind, self.gate, obs, self._scale, self._flat, self._off, *self._dims, self.N,
                  self.v_min, self.v_max, float(epsilon), self._row_ptrs(0)[1], given, self.seed, _lib.ptr(self.counter),
                  _lib.stream())
        return self._fetch(0)[:, 0].astype(np.int64)

    def update(self, tr, beta=0.0, loss_vec=None):
        """One gradient update on a sampled batch (``Transition`` / ``PrioritizedTransition`` of device tensors; C51 only for
        the latter).  Returns the objective (0-dim device tensor) and, for a prioritized batch, the new priorities (float32
        device tensor [B]).  ``loss_vec``: optional float32 device tensor for the per-sample KL [B] (C51) / the loss vector [K]
        (QR)."""
        c, o = self.cfg, self.opt
        s, s2 = tr.state, tr.next_state
        self._check_states(s)
        self._offsets()
        B = s.shape[0]
        per = getattr(tr, "sampling_prob", None) is not None
        if per and self.kind == 1:
            raise NotImplementedError("config.device_qr: QR-DQN with prioritized replay is undefined in the reference: its loss "
                                      "is per target quantile, not per sample (QuantileRegressionDQN_agent.py:74)")
        loss = torch.empty((), dtype=_f32, device=self.dev)
        prio = torch.empty(B, dtype=_f32, device=self.dev) if per else None
        ptr = lambda t: _lib.ptr(None if t is None else t.contiguous())
        _lib.call("b2rl_dist_dqn_replay_update", self.kind, self.gate, ptr(s), ptr(s2), int(s.dtype == _f64), self._scale,
                  ptr(tr.action), ptr(tr.reward), ptr(tr.mask), B, *self._dims, self._flat, _lib.ptr(self.target),
                  _lib.ptr(o.s1), _lib.ptr(o.s2), _lib.ptr(o.step_dev), self._off, float(o.lr), float(o.alpha), float(o.eps),
                  int(o.centered), float(c.discount ** c.n_step), int(bool(c.double_q)), self.v_min, self.v_max,
                  float(c.gradient_clip or 0.0), ptr(tr.sampling_prob if per else None), float(beta),
                  float(getattr(c, "replay_eps", 0.01)), float(getattr(c, "replay_alpha", 0.5)), ptr(prio), ptr(loss_vec),
                  _lib.ptr(loss), _lib.stream())
        return loss, prio


# ------------------------------------------------------------------------------------------------ Rainbow on the device
RAINBOW_NOISE_BUFFERS = ("noise_in", "noise_out_weight", "noise_out_bias")


def rainbow_layers(net):
    """A RainbowNet's four layers in the kernels' order: body.layers.0, body.layers.1, fc_advantage, fc_value."""
    return list(net.body.layers) + [net.fc_advantage, net.fc_value]


def rainbow_kernel_order(net):
    """A RainbowNet's parameters in the kernels' tensor order: per layer of ``rainbow_layers`` weight_mu weight_sigma bias_mu
    bias_sigma (NoisyLinear) or weight bias (nn.Linear)."""
    names = ("weight_mu", "weight_sigma", "bias_mu", "bias_sigma") if net.noisy_linear else ("weight", "bias")
    return [getattr(m, k) for m in rainbow_layers(net) for k in names]


class DeviceRainbow(DeviceDistDQN):
    """``CategoricalDQNAgent.step()`` for a RainbowNet on the device (``config.device_rainbow``): one ``b2rl_rainbow_actor_step``
    launch per env step and one ``b2rl_rainbow_replay_update`` launch per gradient update (csrc/rainbow.cu).  The arenas, the
    target network's parameters as views into the target arena, the staging buffers, the target sync and the locking with
    ``async_actor`` are ``DeviceDistDQN``'s / ``DeviceDQN``'s.

    NoisyLinear: the kernels draw the factorised noise themselves (Philox stream 29 under the agent's key, position
    ``noise_counter``: an actor step advances it by ``noise_len``, an update by twice that, the target network's vector first),
    so the eager ``reset_noise()`` calls do not run.  The online module's noise buffers become views into ``noise`` (the vectors
    of all layers, then every bias_epsilon, then every weight_epsilon), which every update writes: ``eval_step``, ``save`` and
    any eager code see the noise of the latest update.  The actor steps' noise and the target module's buffers are not written
    back.

    Test hooks: ``forced`` (the actions of the next env step) and ``forced_noise``, a callable ``(count)`` returning the noise
    vector(s) of the next launch: ``count`` is 1 for an actor step (``noise_len`` floats) and 2 for an update (the target's, then
    the online network's); then nothing is drawn and the counter does not move."""

    flag = "config.device_rainbow"

    unsupported = staticmethod(rainbow_unsupported)

    def __init__(self, agent, seed):
        from ..utils import Config
        self.kind = 0
        DeviceDQN.__init__(self, agent, seed)
        n, c = agent.network, agent.config
        self.noisy = int(bool(n.noisy_linear))
        self.A, self.K = n.action_dim, n.num_atoms
        self.v_min, self.v_max = float(c.categorical_v_min), float(c.categorical_v_max)
        self._dims = (self.D, self.H1, self.H2, self.A, self.K)
        self.noise_std = float(Config.NOISY_LAYER_STD)
        self.noise_counter = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self.forced_noise = None
        shapes = [(m.in_features, m.out_features) for m in rainbow_layers(n)]
        self.noise_len = sum(i + 2 * o for i, o in shapes)
        self.noise = torch.zeros(self.noise_len + sum(o + o * i for i, o in shapes), dtype=_f32, device=self.dev)
        self._given_noise = torch.zeros(2 * self.noise_len, dtype=_f32, device=self.dev)
        if self.noisy:
            self._adopt_noise_buffers()

    @staticmethod
    def _tensors(net):
        return rainbow_kernel_order(net)

    def _adopt_noise_buffers(self):
        """The online module's noise buffers as views into ``noise`` (their present values kept)."""
        layers = rainbow_layers(self.net)
        o, views = 0, []
        for m in layers:
            for k in RAINBOW_NOISE_BUFFERS:
                views.append((m, k, o))
                o += getattr(m, k).numel()
        for k in ("bias_epsilon", "weight_epsilon"):
            for m in layers:
                views.append((m, k, o))
                o += getattr(m, k).numel()
        assert o == self.noise.numel()
        with torch.no_grad():
            for m, k, o in views:
                old = getattr(m, k)
                view = self.noise[o:o + old.numel()].view_as(old)
                view.copy_(old)
                setattr(m, k, view)

    def _noise_arg(self, count):
        if self.forced_noise is None or not self.noisy:
            return None
        v = torch.as_tensor(np.asarray(self.forced_noise(count), dtype=np.float32).reshape(count * self.noise_len))
        self._given_noise[:v.numel()].copy_(v)
        return _lib.ptr(self._given_noise)

    def act(self, raw_obs, epsilon, noise_out=None):
        """One env step's actions: fresh noise + rescale + forward + dueling combination + action values + the choice in one
        launch, downloaded for ``task.step``.  ``noise_out``: optional float32 device tensor [noise_len] for the noise used."""
        obs, given = self._stage(raw_obs)
        _lib.call("b2rl_rainbow_actor_step", self.noisy, self.gate, obs, self._scale, self._flat, self._off, *self._dims, self.N,
                  self.v_min, self.v_max, float(epsilon), self._row_ptrs(0)[1], given, self.seed, _lib.ptr(self.counter),
                  self.noise_std, self._noise_arg(1), _lib.ptr(noise_out), _lib.ptr(self.noise_counter), _lib.stream())
        return self._fetch(0)[:, 0].astype(np.int64)

    def update(self, tr, beta=0.0, loss_vec=None, target_noise_out=None):
        """One gradient update on a sampled batch (``Transition`` / ``PrioritizedTransition`` of device tensors).  Returns the
        objective (0-dim device tensor) and, for a prioritized batch, the new priorities (float32 device tensor [B]).
        ``loss_vec``: optional float32 device tensor [B] for the per-sample KL; ``target_noise_out``: optional [noise_len] for
        the target network's noise."""
        c, o = self.cfg, self.opt
        s, s2 = tr.state, tr.next_state
        self._check_states(s)
        self._offsets()
        B = s.shape[0]
        per = getattr(tr, "sampling_prob", None) is not None
        loss = torch.empty((), dtype=_f32, device=self.dev)
        prio = torch.empty(B, dtype=_f32, device=self.dev) if per else None
        ptr = lambda t: _lib.ptr(None if t is None else t.contiguous())
        _lib.call("b2rl_rainbow_replay_update", self.noisy, self.gate, ptr(s), ptr(s2), int(s.dtype == _f64), self._scale,
                  ptr(tr.action), ptr(tr.reward), ptr(tr.mask), B, *self._dims, self._flat, _lib.ptr(self.target),
                  _lib.ptr(o.s1), _lib.ptr(o.s2), _lib.ptr(o.step_dev), self._off, float(o.lr), float(o.alpha), float(o.eps),
                  int(o.centered), float(c.discount ** c.n_step), int(bool(c.double_q)), self.v_min, self.v_max,
                  float(c.gradient_clip or 0.0), ptr(tr.sampling_prob if per else None), float(beta),
                  float(getattr(c, "replay_eps", 0.01)), float(getattr(c, "replay_alpha", 0.5)), ptr(prio), ptr(loss_vec),
                  _lib.ptr(loss), self.seed, self.noise_std, self._noise_arg(2),
                  _lib.ptr(self.noise) if self.noisy else None, ptr(target_noise_out), _lib.ptr(self.noise_counter),
                  _lib.stream())
        return loss, prio
