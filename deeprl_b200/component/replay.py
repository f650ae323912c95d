"""Replay store / sample path, resident in HBM, behind the reference's interface
(``deep_rl/component/replay.py``: ``Storage``:20, ``UniformReplay``:57, ``PrioritizedReplay``:152,
``ReplayWrapper``:199).

What lives where
* ``Storage`` (on-policy rollouts) keeps the reference's list-of-tensors design: it holds a handful
  of device tensors per step and is not a bandwidth problem.
* ``UniformReplay`` / ``PrioritizedReplay`` keep the ring in device memory: ``frames`` uint8
  ``[capacity][row_bytes]`` (7.06 GB for 1M 84x84 frames), ``action`` int32, ``reward`` float64,
  ``mask`` int32, and for PER the float64 sum tree.  ``feed`` stages the host items in pinned memory,
  copies them once and runs the feed kernel; ``sample`` runs index selection + the TMA gather
  kernel (``csrc/replay.cu``) and returns DEVICE tensors in a ``Transition`` namedtuple with the
  reference's field names.  No CPU fallback exists: constructing a replay on a CPU device raises.
* ``ReplayWrapper(replay_cls, replay_kwargs, async_=True)``: the reference's ``async`` keyword is a
  reserved word since Python 3.7 (replay.py:205), hence ``async_`` (third positional argument, as
  examples.py passes it).  ``async_=True`` keeps the reference's double-buffer semantics
  (replay.py:246-254: the batch handed out was drawn BEFORE the previous ``update_priorities``)
  with two device batch buffers filled on a side stream instead of a subprocess and a pipe.

RNG: the reference draws indices with ``np.random.randint`` / ``random.uniform`` on the host.  In
production mode the kernels draw from Philox4x32-10 on the device (seed = ``seed`` argument, counter in
``ring_state[4]``); in parity mode ``sample(candidates=...)`` / ``sample(uniforms=..., fills=...)`` take
the host stream so that results are bit-identical to the reference's (tests/test_replay_gpu.py).
"""
from collections import namedtuple

import numpy as np
import torch

from .. import _lib
from ..utils.config import Config
from ..utils.sum_tree import SumTree

Transition = namedtuple("Transition", ["state", "action", "reward", "next_state", "mask"])
PrioritizedTransition = namedtuple("Transition",
                                   ["state", "action", "reward", "next_state", "mask", "sampling_prob", "idx"])


class Storage:
    """replay.py:20-54 -- per-rollout lists keyed by name; ``extract`` concatenates over time."""

    def __init__(self, memory_size, keys=None):
        if keys is None:
            keys = []
        keys = keys + ["state", "action", "reward", "mask", "v", "q", "pi", "log_pi", "entropy", "advantage", "ret",
                       "q_a", "log_pi_a", "mean", "next_state"]
        self.keys = keys
        self.memory_size = memory_size
        self.reset()

    def feed(self, data):
        for k, v in data.items():
            if k not in self.keys:
                raise RuntimeError("Undefined key")
            getattr(self, k).append(v)

    def placeholder(self):
        for k in self.keys:
            if len(getattr(self, k)) == 0:
                setattr(self, k, [None] * self.memory_size)

    def reset(self):
        for key in self.keys:
            setattr(self, key, [])
        self.pos = 0
        self._size = 0

    def extract(self, keys):
        data = [torch.cat(getattr(self, k)[:self.memory_size], dim=0) for k in keys]
        return namedtuple("Entry", keys)(*data)


class UniformReplay:
    TransitionCLS = Transition

    def __init__(self, memory_size, batch_size, n_step=1, discount=1, history_length=1, keys=None, device=None,
                 seed=0, reference_feed_quirk=True):
        self.device = _lib.require_cuda(device if device is not None else Config.DEVICE)
        self.memory_size, self.batch_size = int(memory_size), int(batch_size)
        self.n_step, self.discount, self.history_length = int(n_step), float(discount), int(history_length)
        self.keys = ["state", "action", "reward", "mask"] + list(keys or [])
        self.seed = int(seed)
        self.quirk = bool(reference_feed_quirk)
        self.pos = 0
        self._size = 0
        self.frames = None                     # allocated at first feed (shape / dtype come from the data)
        dev = self.device
        self.ring_state = torch.zeros(8, dtype=torch.int64, device=dev)
        self.ring_state[2] = self.memory_size
        self.action = torch.zeros(self.memory_size, dtype=torch.int32, device=dev)
        self.reward = torch.zeros(self.memory_size, dtype=torch.float64, device=dev)
        self.mask = torch.zeros(self.memory_size, dtype=torch.int32, device=dev)
        self._status = torch.zeros(2, dtype=torch.int32, device=dev)
        self._stage = None
        self._device_cursor = False            # set by a learner whose captured graph feeds the ring: pos / size live on the device
        self._lut_cache = {}
        self._bufs = {}

    # ------------------------------------------------------------------ storage
    def _allocate(self, item):
        item = np.asarray(item)
        self.item_shape, self.item_dtype = tuple(item.shape), item.dtype
        self.row_bytes = int(item.nbytes)
        if self.row_bytes == 0:
            raise ValueError("cannot store empty states")
        self.frames = torch.empty((self.memory_size, self.row_bytes), dtype=torch.uint8, device=self.device)
        self._torch_dtype = torch.from_numpy(np.zeros(1, self.item_dtype)).dtype

    def _staging(self, n):
        """Pinned host + device staging for ``n`` items: the frame rows, and ONE block holding reward (float64) | action (int32)
        | mask (int32) column after column, so that a feed is two host->device copies."""
        if self._stage is None or self._stage["n"] < n:
            cap = max(n, 16)
            hs = torch.empty(16 * cap, dtype=torch.uint8, pin_memory=True)
            ds = torch.empty(16 * cap, dtype=torch.uint8, device=self.device)
            cols = lambda t: (t[:8 * cap].view(torch.float64), t[8 * cap:12 * cap].view(torch.int32), t[12 * cap:].view(torch.int32))
            hr, ha, hm = cols(hs)
            dr, da, dm = cols(ds)
            self._stage = dict(
                n=cap, hs=hs, ds=ds, hr=hr, ha=ha, hm=hm, dr=dr, da=da, dm=dm,
                hf=torch.empty((cap, self.row_bytes), dtype=torch.uint8, pin_memory=True),
                df=torch.empty((cap, self.row_bytes), dtype=torch.uint8, device=self.device))
        return self._stage

    def _stage_rows(self, st, o, data):
        """Write one feed() call's items into the pinned staging rows [o, o + n)."""
        n = len(data["state"])
        arr = np.ascontiguousarray(np.asarray(data["state"], dtype=self.item_dtype)).reshape(n, self.row_bytes // self.item_dtype.itemsize)
        st["hf"][o:o + n].numpy()[...] = arr.view(np.uint8).reshape(n, self.row_bytes)
        st["ha"][o:o + n].numpy()[...] = np.asarray(data["action"]).astype(np.int32).reshape(n)
        st["hr"][o:o + n].numpy()[...] = np.asarray(data["reward"], dtype=np.float64).reshape(n)
        st["hm"][o:o + n].numpy()[...] = np.asarray(data["mask"]).astype(np.int32).reshape(n)
        return n

    def _upload(self, st, total):
        st["df"][:total].copy_(st["hf"][:total], non_blocking=True)
        st["ds"].copy_(st["hs"], non_blocking=True)

    def _feed_staged(self, st, o, n):
        UniformReplay.feed_device(self, st["df"][o:o + n], st["da"][o:o + n], st["dr"][o:o + n], st["dm"][o:o + n], n)

    def feed_many(self, items):
        """Several ``feed()`` calls -- the sgd_update_frequency env steps of one agent step, DQN_agent.py:104-112 -- with ONE
        staging upload and one stream synchronise.  Ring (and, for PrioritizedReplay, tree) semantics are exactly those of
        calling ``feed(d)`` for every ``d`` of ``items`` in order: one ring-write launch per original call (the reference's
        multi-item quirk, replay.py:87, depends on the call boundaries)."""
        for d in items:
            for k in d:
                if k not in self.keys:
                    raise RuntimeError("Undefined key")
        items = [d for d in items if len(d["state"])]
        total = sum(len(d["state"]) for d in items)
        if len(items) <= 1 or total > 1024:
            for d in items:
                self.feed(d)
            return
        if self.frames is None:
            self._allocate(items[0]["state"][0])
        st = self._staging(total)
        o, spans = 0, []
        for d in items:
            n = self._stage_rows(st, o, d)
            spans.append((o, n))
            o += n
        self._upload(st, total)
        for o, n in spans:
            self._feed_staged(st, o, n)
        torch.cuda.current_stream().synchronize()       # the pinned staging buffers are reused by the next call

    def feed(self, data):
        """replay.py:75-90.  ``data``: dict of equal-length sequences for state / action / reward / mask."""
        for k in data:
            if k not in self.keys:
                raise RuntimeError("Undefined key")
        states = data["state"]
        n = len(states)
        if n == 0:
            return
        if n > 1024:                                     # chunked by the BASE implementation: a subclass's feed() bookkeeping
            for s in range(0, n, 1024):                  # (PrioritizedReplay adds ONE tree leaf per feed call) must run once
                UniformReplay.feed(self, {k: v[s:s + 1024] for k, v in data.items()})
            return
        if self.frames is None:
            self._allocate(states[0])
        st = self._staging(n)
        self._stage_rows(st, 0, data)
        self._upload(st, n)
        UniformReplay.feed_device(self, st["df"], st["da"], st["dr"], st["dm"], n)      # (a subclass adds its leaf in feed())
        torch.cuda.current_stream().synchronize()       # the pinned staging buffers are reused by the next call

    def feed_device(self, frames, action, reward, mask, n):
        """Feed ``n`` items already staged on the device (uint8 rows, int32, float64, int32)."""
        if self.frames is None:
            raise RuntimeError("feed_device needs an allocated ring: call feed() once or allocate(item) first")
        _lib.call("b2rl_replay_feed", _lib.ptr(self.frames), _lib.ptr(self.action), _lib.ptr(self.reward),
                  _lib.ptr(self.mask), _lib.ptr(self.ring_state), self.row_bytes, _lib.ptr(frames), _lib.ptr(action),
                  _lib.ptr(reward), _lib.ptr(mask), int(n), int(self.quirk), _lib.stream())
        # host mirror of the cursor (replay.py:80-90)
        pos, size = self.pos, self._size
        for _ in range(n):
            if pos >= size:
                size += 1
            pos = (pos + 1) % self.memory_size
        self.pos, self._size = pos, size

    def allocate(self, item):
        if self.frames is None:
            self._allocate(item)

    def load_synthetic(self, frames, action, reward, mask, pos):
        """Bulk-load a full ring from device tensors (bench / tests): ``frames`` uint8 [capacity, row_bytes]."""
        assert frames.shape[0] == self.memory_size and frames.dtype == torch.uint8
        self.row_bytes = int(frames.shape[1])
        self.item_shape = getattr(self, "item_shape", (self.row_bytes,))
        self.item_dtype = getattr(self, "item_dtype", np.dtype(np.uint8))
        self._torch_dtype = torch.from_numpy(np.zeros(1, self.item_dtype)).dtype
        self.frames = frames
        self.action.copy_(action), self.reward.copy_(reward), self.mask.copy_(mask)
        self.pos, self._size = int(pos), self.memory_size
        self.ring_state[0], self.ring_state[1] = self.pos, self._size

    # ------------------------------------------------------------------ checkpoint (SURVEY 8f-4: absent upstream)
    def state_dict(self):
        """Everything needed to resume: the HBM ring (frames + scalars, host copies), the device cursor / Philox counter and the
        host mirrors.  ``torch.save``-able."""
        if self.frames is None:
            return dict(empty=True)
        self._sync_cursor()
        st = self.ring_state.cpu()
        return dict(empty=False, frames=self.frames.cpu(), action=self.action.cpu(), reward=self.reward.cpu(), mask=self.mask.cpu(),
                    ring_state=st, item_shape=tuple(self.item_shape), item_dtype=np.dtype(self.item_dtype).str,
                    memory_size=self.memory_size, n_step=self.n_step, history_length=self.history_length)

    def load_state_dict(self, sd):
        if sd.get("empty"):
            return
        if sd["memory_size"] != self.memory_size or sd["history_length"] != self.history_length:
            raise ValueError("checkpoint of a different replay geometry")
        self.item_shape, self.item_dtype = tuple(sd["item_shape"]), np.dtype(sd["item_dtype"])
        self.row_bytes = int(sd["frames"].shape[1])
        self._torch_dtype = torch.from_numpy(np.zeros(1, self.item_dtype)).dtype
        self.frames = sd["frames"].to(self.device)
        self.action.copy_(sd["action"]), self.reward.copy_(sd["reward"]), self.mask.copy_(sd["mask"])
        self.ring_state.copy_(sd["ring_state"])
        self.pos, self._size = int(sd["ring_state"][0]), int(sd["ring_state"][1])
        self._bufs = {}

    def _sync_cursor(self):
        """The host mirror of the ring cursor follows host-side feeds only; when a learner feeds the ring inside a captured
        graph (``_device_cursor``) the truth is ``ring_state`` on the device (one small synchronising read)."""
        if self._device_cursor:
            self.pos, self._size = (int(x) for x in self.ring_state[:2].tolist())

    def size(self):
        self._sync_cursor()
        return self._size

    def full(self):
        self._sync_cursor()
        return self._size == self.memory_size

    def valid_index(self, index):
        """replay.py:105-110 (host arithmetic on the mirrored cursor; the kernels apply the same rule)."""
        self._sync_cursor()
        hl, n = self.history_length, self.n_step
        if index - hl + 1 >= 0 and index + n < self.pos:
            return True
        if index - hl + 1 >= self.pos and index + n < self._size:
            return True
        return False

    def compute_valid_indices(self):
        """replay.py:69-73."""
        hl, n = self.history_length, self.n_step
        idx = list(range(hl - 1, self.pos - n)) + list(range(self.pos + hl - 1, self._size - n))
        return np.asarray(idx)

    # ------------------------------------------------------------------ sampling
    LAYOUTS = {"nchw": 0, "nhwc": 1, "s2d": 2, "ring": 3, False: 0, True: 1}

    def _buffers(self, B, out_dtype, layout, tag=0):
        layout = self.LAYOUTS[layout]
        key = (B, out_dtype, layout, tag)
        if key not in self._bufs:
            dev, hl = self.device, self.history_length
            shape = (B, self.row_bytes, hl) if layout else (B, hl, self.row_bytes)     # same byte count for s2d
            if layout == 3:
                shape = (0,)                                                           # the frames stay in the ring
            self._bufs[key] = dict(
                idx=torch.empty(B, dtype=torch.int64, device=dev),
                state=torch.empty(shape, dtype=out_dtype, device=dev), next_state=torch.empty(shape, dtype=out_dtype, device=dev),
                action=torch.empty(B, dtype=torch.int64, device=dev), reward=torch.empty(B, dtype=torch.float32, device=dev),
                mask=torch.empty(B, dtype=torch.float32, device=dev),
                tree_idx=torch.empty(B, dtype=torch.int64, device=dev), prob64=torch.empty(B, dtype=torch.float64, device=dev),
                prob=torch.empty(B, dtype=torch.float32, device=dev))
        return self._bufs[key]

    def lut(self, scale=1.0 / 255):
        """uint8 -> float table ``float32(float64(v) * scale)``: the reference's ImageNormalizer multiplies in
        float64 and ``tensor()`` rounds once to float32 (normalizer.py:58-61, torch_utils.py:23)."""
        if scale not in self._lut_cache:
            t = (np.arange(256, dtype=np.float64) * scale).astype(np.float32)
            self._lut_cache[scale] = torch.from_numpy(t).to(self.device)
        return self._lut_cache[scale]

    def select(self, B, idx_out, candidates=None, scalars=None):
        """Draw B valid indices into ``idx_out``; with ``scalars`` (a buffer set) the same launch also writes their action /
        n-step reward / mask, as ``gather_scalars`` does."""
        n_cand = min(8192, max(2 * B, B + 256)) if candidates is None else min(8192, candidates.numel())
        if scalars is not None:
            _lib.call("b2rl_replay_select_uniform_scalars", _lib.ptr(self.ring_state), _lib.ptr(candidates), int(n_cand), self.seed,
                      self.history_length, self.n_step, int(B), _lib.ptr(idx_out), _lib.ptr(self._status), _lib.ptr(self.action),
                      _lib.ptr(self.reward), _lib.ptr(self.mask), self.discount, _lib.ptr(scalars["action"]),
                      _lib.ptr(scalars["reward"]), _lib.ptr(scalars["mask"]), _lib.stream())
            return
        _lib.call("b2rl_replay_select_uniform", _lib.ptr(self.ring_state), _lib.ptr(candidates), int(n_cand), self.seed,
                  self.history_length, self.n_step, int(B), _lib.ptr(idx_out), _lib.ptr(self._status), _lib.stream())

    def ring_frames(self, idx, which):
        """The (not materialised) frame stacks of ``idx``: ``which`` = 0 state, 1 next state (replay.py:124-125)."""
        from ..network.nature_tc import RingFrames
        hl = self.history_length
        return RingFrames(self.frames, idx, which * self.n_step - (hl - 1), self.row_bytes, self.item_shape[-1], hl)

    def gather_scalars(self, idx, B, bufs):
        """action / n-step reward / mask of ``idx`` only (the frame stacks are read from the ring by the consumer)."""
        _lib.call("b2rl_replay_gather", _lib.ptr(self.frames), _lib.ptr(self.action), _lib.ptr(self.reward),
                  _lib.ptr(self.mask), self.memory_size, self.row_bytes, _lib.ptr(idx), int(B), self.history_length,
                  self.n_step, self.discount, None, _lib.DTYPE_CODE[torch.uint8], 0, 0, None, None, _lib.ptr(bufs["action"]),
                  _lib.ptr(bufs["reward"]), _lib.ptr(bufs["mask"]), _lib.stream())

    def gather(self, idx, B, bufs, out_dtype=torch.uint8, lut=None, layout="nchw"):
        frame_w = self.item_shape[-1] if len(getattr(self, "item_shape", ())) >= 2 else 0
        _lib.call("b2rl_replay_gather", _lib.ptr(self.frames), _lib.ptr(self.action), _lib.ptr(self.reward),
                  _lib.ptr(self.mask), self.memory_size, self.row_bytes, _lib.ptr(idx), int(B), self.history_length,
                  self.n_step, self.discount, _lib.ptr(lut), _lib.DTYPE_CODE[out_dtype], self.LAYOUTS[layout], int(frame_w),
                  _lib.ptr(bufs["state"]), _lib.ptr(bufs["next_state"]), _lib.ptr(bufs["action"]), _lib.ptr(bufs["reward"]),
                  _lib.ptr(bufs["mask"]), _lib.stream())

    def _image_view(self, x, B, layout):
        """Logical [B, C, H, W] view of a gathered batch buffer."""
        hw, hl = tuple(self.item_shape[-2:]), self.history_length
        layout = self.LAYOUTS[layout]
        if layout == 2:
            return x.view(B, hw[0] // 4, hw[1] // 4, 16 * hl).permute(0, 3, 1, 2)       # [B, 16*hl, H/4, W/4], NHWC memory
        if layout == 1:
            return x.view((B,) + hw + (hl,)).permute(0, 3, 1, 2)                        # [B, hl, H, W], NHWC memory
        return x.view((B, hl) + hw)

    def _typed(self, raw, B):
        """uint8 rows -> stored dtype and shape; the frame-stack axis disappears when history_length == 1."""
        x = raw.view(self._torch_dtype) if self._torch_dtype != torch.uint8 else raw
        shape = (B, self.history_length) + self.item_shape if self.history_length > 1 else (B,) + self.item_shape
        return x.view(shape)

    def sample(self, batch_size=None, candidates=None, check=True, tag=0):
        """replay.py:92-103.  Returns ``Transition`` of device tensors: state / next_state in the stored dtype,
        action int64, reward float32, mask float32.  ``candidates`` (int64 tensor / array) replaces the device
        Philox stream by an ``np.random.randint(0, size)`` stream (parity mode)."""
        B = self.batch_size if batch_size is None else int(batch_size)
        if self._size == 0:
            raise ValueError("cannot sample from an empty replay")
        bufs = self._buffers(B, torch.uint8, "nchw", tag)
        if candidates is not None and not isinstance(candidates, torch.Tensor):
            candidates = torch.as_tensor(np.asarray(candidates, dtype=np.int64), device=self.device)
        self.select(B, bufs["idx"], candidates)
        if check:
            acc = int(self._status[0].item())
            if acc < B:
                raise RuntimeError("candidate stream exhausted: %d of %d valid indices found" % (acc, B))
        self.gather(bufs["idx"], B, bufs)
        return Transition(self._typed(bufs["state"], B), bufs["action"], bufs["reward"], self._typed(bufs["next_state"], B),
                          bufs["mask"])

    def sample_normalized(self, batch_size=None, out_dtype=torch.float32, scale=1.0 / 255, layout="nchw", candidates=None,
                          tag=0, channels_last=None, phase=None):
        """Fused gather -> normalize (``ImageNormalizer``) for uint8 frame rings.  state / next_state come back as
        ``out_dtype`` [B, history, H, W] (``layout="nhwc"``: same logical shape, channels_last memory) or, with
        ``layout="s2d"``, as the space-to-depth(4) tensor [B, 16*history, H/4, W/4] (channels_last memory).
        ``scale=None`` emits the exact integers 0..255 (the consumer folds 1/255 into its first layer, see
        ``network.frame_scale``); otherwise ``float32(float64(v) * scale)`` rounded to ``out_dtype``.
        ``layout="ring"`` (K1): nothing is gathered -- state / next_state are ``RingFrames`` (ring + indices) that the wgmma
        ``NatureConvBody`` reads directly; they are valid until the ring rows are overwritten."""
        if channels_last is not None:
            layout = "nhwc" if channels_last else "nchw"
        B = self.batch_size if batch_size is None else int(batch_size)
        if self.item_dtype != np.uint8 or len(self.item_shape) < 2:
            raise TypeError("sample_normalized is for uint8 image rings")
        bufs = self._buffers(B, out_dtype, layout, tag)
        if candidates is not None and not isinstance(candidates, torch.Tensor):
            candidates = torch.as_tensor(np.asarray(candidates, dtype=np.int64), device=self.device)
        # phase "select": draw the indices only; phase "gather": build the batch from the indices drawn before (the learner
        # draws early, on tiny kernels, and gathers late, beside its update tail); None: both.  layout "ring" (K1): no batch
        # is materialised, conv1 reads the ring through the sampled indices, and the draw writes action / reward / mask itself
        ring = layout == "ring"
        if phase != "gather":
            self.select(B, bufs["idx"], candidates, scalars=bufs if ring else None)
        if phase == "select":
            return None
        if ring:
            if phase == "gather":
                self.gather_scalars(bufs["idx"], B, bufs)
            return Transition(self.ring_frames(bufs["idx"], 0), bufs["action"], bufs["reward"], self.ring_frames(bufs["idx"], 1),
                              bufs["mask"])
        self.gather(bufs["idx"], B, bufs, out_dtype, None if scale is None else self.lut(scale), layout)
        return Transition(self._image_view(bufs["state"], B, layout), bufs["action"], bufs["reward"],
                          self._image_view(bufs["next_state"], B, layout), bufs["mask"])

    def construct_transition(self, index):
        """replay.py:112-140 for ONE index (inspection / tests): device gather of a batch of one."""
        if not self.valid_index(index):
            return None
        bufs = self._buffers(1, torch.uint8, "nchw", tag=-1)
        bufs["idx"][0] = int(index)
        self.gather(bufs["idx"], 1, bufs)
        t = Transition(self._typed(bufs["state"], 1)[0].clone(), bufs["action"][0].clone(), bufs["reward"][0].clone(),
                       self._typed(bufs["next_state"], 1)[0].clone(), bufs["mask"][0].clone())
        return t

    def update_priorities(self, info):
        raise NotImplementedError

    def close(self):
        pass


class PrioritizedReplay(UniformReplay):
    TransitionCLS = PrioritizedTransition

    def __init__(self, memory_size, batch_size, n_step=1, discount=1, history_length=1, keys=None, device=None,
                 seed=0, reference_feed_quirk=True):
        super().__init__(memory_size, batch_size, n_step, discount, history_length, keys, device, seed,
                         reference_feed_quirk)
        self.tree = SumTree(memory_size, self.device, ring_state=self.ring_state)
        self.max_priority_dev = torch.ones(1, dtype=torch.float64, device=self.device)    # replay.py:158

    @property
    def max_priority(self):
        return float(self.max_priority_dev.item())

    def feed(self, data):
        """replay.py:160-162 -- NOTE the reference adds ONE leaf per feed() call whatever the item count."""
        super().feed(data)
        if len(data["state"]):
            self.tree.add_n(1, self.max_priority_dev)

    def feed_device(self, frames, action, reward, mask, n, *, add_leaf):
        """``add_leaf`` is explicit: transitions fed without a tree leaf have priority zero and are never sampled -- only a
        caller that adds the leaves itself (the learner: ``tree.add_n(feeds)``) passes False."""
        super().feed_device(frames, action, reward, mask, n)
        if add_leaf:
            self.tree.add_n(1, self.max_priority_dev)

    def _feed_staged(self, st, o, n):
        self.feed_device(st["df"][o:o + n], st["da"][o:o + n], st["dr"][o:o + n], st["dm"][o:o + n], n, add_leaf=True)

    def load_synthetic(self, frames, action, reward, mask, pos, priorities=None):
        super().load_synthetic(frames, action, reward, mask, pos)
        cap = self.memory_size
        leaves = torch.ones(cap, dtype=torch.float64, device=self.device) if priorities is None else priorities.double()
        # initial state only: internal nodes = exact sums of their children, built level by level
        t = self.tree.tree
        t[cap - 1:] = leaves
        depth = (cap - 1).bit_length()
        for d in range(depth, -1, -1):
            lo, hi = 2 ** d - 1, min(2 ** (d + 1) - 1, cap - 1)
            if hi > lo:
                idx = torch.arange(lo, hi, device=self.device)
                t[idx] = t[2 * idx + 1] + t[2 * idx + 2]
        self.ring_state[3] = self.pos
        self.tree.n_entries = cap

    def state_dict(self):
        sd = super().state_dict()
        if not sd.get("empty"):
            sd.update(tree=self.tree.tree.cpu(), pending=self.tree.pending.cpu(), max_priority=self.max_priority_dev.cpu(),
                      n_entries=self.tree.n_entries)
        return sd

    def load_state_dict(self, sd):
        super().load_state_dict(sd)
        if not sd.get("empty"):
            self.tree.tree.copy_(sd["tree"]), self.tree.pending.copy_(sd["pending"])
            self.max_priority_dev.copy_(sd["max_priority"])
            self.tree.n_entries = int(sd["n_entries"])

    def sample(self, batch_size=None, uniforms=None, fills=None, check=True, tag=0):
        """replay.py:164-191 -> ``PrioritizedTransition`` (sampling_prob float32 = tensor(p / total), idx = TREE index)."""
        B = self.batch_size if batch_size is None else int(batch_size)
        bufs = self._buffers(B, torch.uint8, "nchw", tag)
        self._select_per(B, bufs, uniforms, fills, check)
        self.gather(bufs["idx"], B, bufs)
        return PrioritizedTransition(self._typed(bufs["state"], B), bufs["action"], bufs["reward"],
                                     self._typed(bufs["next_state"], B), bufs["mask"], bufs["prob"], bufs["tree_idx"])

    def _select_per(self, B, bufs, uniforms=None, fills=None, check=False):
        as_dev = lambda x, dt: None if x is None else (x if isinstance(x, torch.Tensor) else torch.as_tensor(
            np.asarray(x, dtype=dt), device=self.device))
        self.tree.sample_batch(B, self.history_length, self.n_step, bufs["tree_idx"], bufs["idx"], bufs["prob64"],
                               self._status, as_dev(uniforms, np.float64), as_dev(fills, np.int64), self.seed)
        if check and int(self._status[0].item()) == 0:
            raise IndexError("no valid transition among the stratified draws (random.choice on an empty list)")
        bufs["prob"].copy_(bufs["prob64"])              # tensor(sampling_prob): float64 -> float32, one rounding

    def sample_normalized(self, batch_size=None, out_dtype=torch.float32, scale=1.0 / 255, layout="nchw", uniforms=None,
                          fills=None, tag=0, channels_last=None):
        if channels_last is not None:
            layout = "nhwc" if channels_last else "nchw"
        B = self.batch_size if batch_size is None else int(batch_size)
        bufs = self._buffers(B, out_dtype, layout, tag)
        self._select_per(B, bufs, uniforms, fills)
        if layout == "ring":
            self.gather_scalars(bufs["idx"], B, bufs)
            return PrioritizedTransition(self.ring_frames(bufs["idx"], 0), bufs["action"], bufs["reward"],
                                         self.ring_frames(bufs["idx"], 1), bufs["mask"], bufs["prob"], bufs["tree_idx"])
        self.gather(bufs["idx"], B, bufs, out_dtype, None if scale is None else self.lut(scale), layout)
        return PrioritizedTransition(self._image_view(bufs["state"], B, layout), bufs["action"], bufs["reward"],
                                     self._image_view(bufs["next_state"], B, layout), bufs["mask"], bufs["prob"],
                                     bufs["tree_idx"])

    def update_priorities(self, info):
        """replay.py:193-196.  ``info``: iterable of (tree_idx, priority) pairs (the reference's zip of numpy
        arrays) or a pair of DEVICE tensors ``(idx int64 [B], priority float32 [B])`` (no host round trip)."""
        if isinstance(info, tuple) and len(info) == 2 and isinstance(info[0], torch.Tensor):
            idx, prio = info
        else:
            pairs = list(info)
            if not pairs:
                return
            idx = torch.as_tensor(np.asarray([p[0] for p in pairs], dtype=np.int64), device=self.device)
            prio = torch.as_tensor(np.asarray([p[1] for p in pairs], dtype=np.float32), device=self.device)
        for s in range(0, idx.numel(), 1024):
            self.tree.update_batch(idx[s:s + 1024].contiguous(), prio[s:s + 1024].contiguous(), self.max_priority_dev)


class ReplayWrapper:
    """replay.py:199-278.  ``ReplayWrapper(replay_cls, replay_kwargs, async_)``."""
    FEED, SAMPLE, EXIT, UPDATE_PRIORITIES = 0, 1, 2, 3

    def __init__(self, replay_cls, replay_kwargs, async_=True):
        self.replay_cls, self.replay_kwargs = replay_cls, replay_kwargs
        self.cache_len = 2
        self.replay = replay_cls(**replay_kwargs)
        self.async_ = bool(async_)
        if not self.async_:
            self.sample = self.replay.sample
            self.feed = self.replay.feed
            self.feed_many = self.replay.feed_many
            self.update_priorities = self.replay.update_priorities
        else:
            self._side = torch.cuda.Stream(device=self.replay.device)
            self._ready = [None, None]
            self._cache = [None, None]
            self._cur = 0
            self._primed = False

    # async mode: every replay operation is ordered on the side stream, exactly like the reference's worker
    # processes its pipe messages in order; the learner only waits on the event of the buffer it receives.
    def _on_side(self, fn, *a, **k):
        self._side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self._side):
            return fn(*a, **k)

    def _fill(self, slot):
        with torch.cuda.stream(self._side):
            self._cache[slot] = self.replay.sample(tag=slot, check=False)
            ev = torch.cuda.Event()
            ev.record(self._side)
            self._ready[slot] = ev

    def feed(self, exp):
        self._on_side(self.replay.feed, exp)

    def feed_many(self, exps):
        """The feeds of one agent step with one staging upload (``UniformReplay.feed_many``)."""
        self._on_side(self.replay.feed_many, exps)

    def sample(self):
        self._side.wait_stream(torch.cuda.current_stream())
        if not self._primed:                        # replay.py:227-234: both buffers are filled on first use
            self._fill(0), self._fill(1)
            self._primed = True
        slot = self._cur
        torch.cuda.current_stream().wait_event(self._ready[slot])
        out = self._cache[slot]
        self._cur = (self._cur + 1) % 2
        self._fill(self._cur)                       # replay.py:253-254: refill the OTHER buffer right away
        return out

    def update_priorities(self, info):
        # the tensors were allocated on the caller's stream and may be released as soon as the caller returns: tell the
        # caching allocator that the side stream still reads them
        if isinstance(info, tuple) and len(info) == 2 and isinstance(info[0], torch.Tensor):
            for t in info:
                if t.is_cuda:
                    t.record_stream(self._side)
        self._on_side(self.replay.update_priorities, info)

    def size(self):
        return self.replay.size()

    def full(self):
        return self.replay.full()

    def close(self):
        if self.async_:
            self._side.synchronize()
        self.replay.close()
