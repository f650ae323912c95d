"""CUDA-graph learner for the DQN family: one gradient update of ``DQNAgent.step`` (DQN_agent.py:101-138) --
``sgd_update_frequency`` feeds, sample, target / online forward, fused loss, backward, [gradient all-reduce],
fused clip + optimizer, PER priority update -- replayed as (at most two) captured graphs, with every scalar
that changes between updates (ring cursor, Philox counter, PER beta, Adam step, max priority) living in device
memory.  This is the throughput path of bench.py; ``DQNAgent`` without it runs the same kernels eagerly.

Multi-GPU (SURVEY 8e): one learner per rank, rank-local replay shard, parameters identical on every rank;
gradients are summed with ONE NCCL all-reduce of the flat gradient arena between the two graphs and scaled by
1 / world_size inside the clip kernel.
"""
import contextlib
import dataclasses
import os
import sys

import numpy as np
import torch

from . import _lib, ops, parallel
from .component.replay import PrioritizedReplay
from .network import fused, nature_tc
from .network.fused import frame_scale
from .utils.config import Config


class StepTrace:
    """Timing events recorded INSIDE the captured update (``torch.cuda.Event(external=True)`` -> event-record nodes of the
    graph): the real timeline of one graph replay, with the overlap between the branches, which neither the serialised ncu
    launch list nor eager launches show.  ``scripts/trace_step.py`` prints it."""

    def __init__(self):
        self.marks = []

    def mark(self, name, stream=None):
        e = torch.cuda.Event(enable_timing=True, external=True)
        e.record(stream if stream is not None else torch.cuda.current_stream())
        self.marks.append((name, e))

    def timeline(self):
        t0 = self.marks[0][1]
        return [(n, t0.elapsed_time(e) * 1e3) for n, e in self.marks]


@dataclasses.dataclass(frozen=True)
class UpdatePlan:
    """The layout of one ``GraphedDQNLearner`` update, as decided by ``update_plan``."""
    ring: bool            # K1: conv1 reads the sampled frame stacks from the uint8 ring, no batch is materialised
    tail: bool            # the two-launch fused update tail (network/tail.py) replaces unpack + FlatOptimizer.step
    repack_online: bool   # no fused tail: the online operands are re-packed on the side branch at the start of each update
    dist_head: bool       # C51 / QR: the heads read bf16 weight copies on the wgmma GEMM
    head: str             # "separate" (head_fwd | loss | head_bwd), "fused-two" or "fused-one" (csrc/head.cu on the features)
    forward: str          # "two-branch" (target on the side stream), "dual" (one launch per layer for both) or "one-stream"
    conv1: str            # "pair": online conv1(s) and target conv1(s') in one launch from the ring (K1, n_step 1); "separate"
    single_stream: bool   # the side-branch work (target forward, re-pack, weight gradients) runs on the main stream
    prefetch: object      # where the next batch is sampled: None, "start", "gather-after-bwd" / "-dgrad", "after-ring-read"
    join: object          # where the prefetch branch joins: None, "main" (end of _main) or "opt" (after the optimizer kernels)
    one_graph: bool       # multi-GPU: the all-reduce is captured inside the update graph


def update_plan(kind="dqn", per=False, prefetch=False, dual=False, k1_body=True, dual_body=True, tail=True,
                narrow_head=True, world=1, one_graph=True, env=None, n_step=1):
    """Decide the update schedule from plain values: the learner's options, what the networks support (``k1_body``: a
    wgmma NatureConvBody on a 4 x 84 x 84 uint8 ring; ``dual_body``: both bodies on the wgmma kernels; ``tail``: the fused
    update tail applies; ``narrow_head``: VanillaNet / DuelingNet heads the fused head kernel takes), the replay's
    ``n_step`` and the ``B2RL_*`` switches in ``env``.  ``one_graph=False``: the split-graph form after a failed NCCL
    capture."""
    env = env or {}
    on = lambda name, default: env.get(name, default) != "0"
    fused_env = kind == "dqn" and on("B2RL_FUSED_HEAD", "0")
    # K1 with async replay: the feeds and the index draw of the next batch run after this update's last ring read.
    # Prioritized replay keeps the materialising gather: its draw of the next batch must precede this update's priority
    # update, which comes before the backward pass, while the feeds may only overwrite ring rows after the backward pass.
    # The fused-head switch keeps it as well (whether or not the fused head then applies).
    ring = k1_body and not dual and on("B2RL_K1", "1") and not (prefetch and (per or fused_env))
    tail = tail and on("B2RL_TAIL", "1")
    # the fused head (off by default: the separate kernels run the target head on the side branch, which it gives up)
    head = "separate"
    if fused_env and tail and narrow_head:
        head = "fused-one" if env.get("B2RL_FUSED_HEAD") == "one" else "fused-two"
    single = head == "separate" and env.get("B2RL_SINGLE_STREAM", "0") == "1"       # experiment: no parallel branches
    forward = "dual" if head == "separate" and dual and dual_body else ("one-stream" if single else "two-branch")
    one_graph = one_graph and (world == 1 or env.get("B2RL_NCCL_IN_GRAPH", "1") == "1")
    # with n_step 1 the next state's stacks are the state's shifted by one ring row: one conv1 launch reads each sample's
    # five-frame window once for the online forward on s and the target forward on s' (nature_tc.paired_conv1)
    conv1 = "pair" if ring and forward != "dual" and dual_body and n_step == 1 else "separate"
    # async replay, uniform with the materialising gather: feed + index draw at the start, the gather after the backward
    # pass beside the (small-footprint, L2-bound) update tail -- started beside the forward pass its 512 gather CTAs would
    # hold the shared memory the convolution kernels need.  Prioritized replay keeps the whole branch at the start: the
    # reference's replay worker draws the next batch BEFORE this update's priorities arrive (replay.py:219-261).
    pf = join = None
    if prefetch:
        if ring:
            pf, join = "after-ring-read", "opt" if one_graph else "main"
        elif not per and one_graph and env.get("B2RL_PREFETCH_LATE", "1") == "1":
            # B2RL_PREFETCH_AT=dgrad forks the gather after the last dgrad GEMM, beside the conv2 / conv1 weight gradients,
            # where it slows the conv1 weight gradient and kernel A
            at_dgrad = head == "separate" and env.get("B2RL_PREFETCH_AT", "end") == "dgrad"
            pf, join = "gather-after-dgrad" if at_dgrad else "gather-after-bwd", "opt" if head == "separate" else "main"
        else:
            pf, join = "start", "main"
    return UpdatePlan(ring=ring, tail=tail, repack_online=not tail, head=head, forward=forward, conv1=conv1, single_stream=single,
                      dist_head=kind in ("c51", "qr") and tail and on("B2RL_DIST_HEAD", "1"), prefetch=pf, join=join,
                      one_graph=one_graph)


class _NatureLearner:
    """What the captured learners of a wgmma NatureConvBody network share: the update plan (decided on first use by the
    subclass's ``_resolve_plan``), the fused update tail, and the packed bf16 operands of the online (``net``) and target
    (``tgt``) networks -- re-packed after outside parameter changes and at target sync.

    ``body_attr``: the attribute of the networks that holds the NatureConvBody (``phi_body`` for an actor-critic network)."""

    body_attr = "body"

    def _body(self, net):
        return getattr(net, self.body_attr, None)

    @property
    def plan(self):
        """The ``UpdatePlan`` of this learner, decided on first use (the module flags the fused tail depends on are read
        then, as the tail itself is built lazily)."""
        if self._plan is None:
            self._plan = self._resolve_plan()
        return self._plan

    def tail(self):
        """The two-launch update tail (gradient reduce + clip / optimizer / operand pack) when the online network has a
        wgmma NatureConvBody and the backward epilogues are fused; None otherwise (generic unpack + FlatOptimizer.step)."""
        if self._tail is None:
            from .network.tail import NatureTail
            if self.plan.tail:
                self._repack(self.net)
                self._tail = NatureTail(self.opt, self._body(self.net), self.scale)
                self._tail.max_norm, self._tail.grad_scale = self.clip, 1.0 / self.world
                self._refresh_head_operands(True)
                if self.world > 1:
                    # fc4's gradient is reduced into the arena and all-reduced right after its GEMM (beside the convolution
                    # backward); the small remainder follows the last weight-gradient GEMM
                    self._tail.split = True
                    self._tail.early = self._allreduce_early
            else:
                self._tail = False
        return self._tail or None

    def _repack(self, net):
        """wgmma backend: the learner owns the packed bf16 operands of both networks -- the online body is re-packed
        once per update (one launch), the target body only when it is synchronised."""
        body = self._body(net)
        if body is not None and hasattr(body, "repack") and self.dtype == torch.bfloat16:
            body.auto_repack = False
            body.repack(self.scale)

    def repack_online(self):
        """Bring the online network's packed bf16 operands up to date after ``update()``, for a forward outside the learner
        (the actor).  The fused tail's optimizer kernel writes them itself; without it this is one re-pack launch."""
        if self.tail() is None:
            self._repack(self.net)

    def sync_target(self):
        self.tgt.load_state_dict(self.net.state_dict())        # DQN_agent.py:136-138
        self._repack(self.tgt)
        self._refresh_head_operands(False)

    def refresh_packed(self):
        """Re-derive the packed bf16 operands of both networks from the fp32 parameters (after the parameters were changed
        from outside: load_state_dict, a broadcast, a copied arena)."""
        self._repack(self.net)
        self._repack(self.tgt)
        self._refresh_head_operands(True)

    def _refresh_head_operands(self, online):
        """Distributional heads (C51 / QR-DQN) on the wgmma GEMM: the online head reads its bf16 weight from the optimizer's
        arena-wide bf16 shadow (written by the fused optimizer kernel), the target head from a copy refreshed at target sync."""
        if not self.plan.dist_head or self.tail() is None:
            return
        fa, ft = (getattr(n, "fc_categorical", None) or getattr(n, "fc_quantiles", None) for n in (self.net, self.tgt))
        if not isinstance(fa, torch.nn.Linear) or not isinstance(ft, torch.nn.Linear) or fa.weight.data_ptr() % 16:
            return
        o = self.opt
        if o.shadow is None:
            o.shadow = torch.zeros(o.n, dtype=torch.bfloat16, device=o.flat.device)
        if online:
            o.shadow.copy_(o.flat)
            off = (fa.weight.data_ptr() - o.flat.data_ptr()) // 4
            fa._w16 = o.shadow[off:off + fa.weight.numel()].view_as(fa.weight)
        if getattr(ft, "_w16", None) is None:
            ft._w16 = torch.empty_like(ft.weight, dtype=torch.bfloat16)
        ft._w16.copy_(ft.weight.detach())


class GraphedDQNLearner(_NatureLearner):
    def __init__(self, network, target_network, optimizer, replay, kind="dqn", discount=0.99, n_step=1, double_q=False,
                 gradient_clip=5.0, feeds_per_update=4, compute_dtype=torch.bfloat16, state_scale=1.0 / 255,
                 replay_eps=0.01, replay_alpha=0.5, categorical=(-10.0, 10.0), world_size=1, target_sync_every=10000,
                 prefetch=False, dual=False, wrapper_order=False):
        self.net, self.tgt, self.opt, self.replay = network, target_network, optimizer, replay
        self.kind, self.gamma_n, self.double_q = kind, discount ** n_step, double_q
        self.clip, self.feeds = gradient_clip, feeds_per_update
        self.dtype, self.scale = compute_dtype, state_scale
        self.eps, self.alpha, self.cat = replay_eps, replay_alpha, categorical
        self.world = world_size
        self.per = isinstance(replay, PrioritizedReplay)
        self.sync_every = target_sync_every
        self.dev = dev = replay.device
        self.B = replay.batch_size
        n = max(self.feeds, 1)
        rb = replay.row_bytes
        # ONE packed pinned staging buffer for the env transitions of an update (+ PER beta) and ONE device mirror:
        # [frames n*rb | reward n*8 | action n*4 | mask n*4 | beta 4] -> a single host->device copy node in the graph
        o_r = (n * rb + 7) // 8 * 8
        o_a, o_m, o_b = o_r + 8 * n, o_r + 12 * n, o_r + 16 * n
        total = (o_b + 4 + 15) // 16 * 16
        self.h_pack = torch.zeros(total, dtype=torch.uint8, pin_memory=True)
        self.d_pack = torch.zeros(total, dtype=torch.uint8, device=dev)

        def views(buf):
            return (buf[:n * rb].view(n, rb), buf[o_a:o_a + 4 * n].view(torch.int32), buf[o_r:o_r + 8 * n].view(torch.float64),
                    buf[o_m:o_m + 4 * n].view(torch.int32), buf[o_b:o_b + 4].view(torch.float32))

        self.h_frames, self.h_action, self.h_reward, self.h_mask, self.h_beta = views(self.h_pack)
        self.d_frames, self.d_action, self.d_reward, self.d_mask, self.d_beta = views(self.d_pack)
        self.h_mask.fill_(1), self.h_beta.fill_(0.4)
        self.d_pack.copy_(self.h_pack)
        self.h_loss = torch.zeros(1, dtype=torch.float32, pin_memory=True)
        self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
        self.g_main = self.g_opt = None
        self._side = None
        # prefetch = the graph form of ReplayWrapper(async_=True) (replay.py:214-262: the worker hands out the batch it
        # sampled right after the previous request and immediately samples the next one into the other cache): update k
        # trains on the batch sampled during update k-1 while a third branch of the graph feeds + samples batch k+1
        # into the other buffer set.  Two graphs (one per buffer parity) are captured and replayed alternately.
        self.prefetch = bool(prefetch)
        # dual: one launch per body layer for online(s) + target(s') (nature_tc.forward_dual): 27 instead of 33 launches per
        # update; off by default (the two-stream fork of the prefetch branch already hides the per-launch fixed cost).
        self.dual = bool(dual)
        # wrapper_order (async replay with feeds, for an agent): the first update feeds ONCE and draws the batch it trains on
        # and the one the next update trains on after those feeds, like ReplayWrapper's first sample() (three draws: both
        # buffers, then the refill of the second); the h2d copy node is followed by ``staged``, an event the host waits on
        # before it rewrites the pinned staging buffer (no synchronise per update)
        self.wrapper_order = bool(wrapper_order)
        self.staged = torch.cuda.Event(external=True) if self.wrapper_order else None
        self.capture_error_mode = "global"
        self._batch = [None, None]
        self._parity = 0
        self.updates = 0
        self.with_h2d = False
        self._tail = None                 # network/tail.py NatureTail (built on first use), False = not applicable
        self._overlap = False             # multi-GPU: NCCL captured inside the update graph, fc4's all-reduce beside the backward
        self._early_work = None
        self._env = {k: v for k, v in os.environ.items() if k.startswith("B2RL_")}     # update_plan's switches, as constructed
        self._plan = None
        self.opt.zero_grad()              # the fused tail writes / re-zeroes the gradient arena itself: start from zeros

    def _resolve_plan(self, one_graph=True):
        body, rp = getattr(self.net, "body", None), self.replay
        wgmma = self.dtype == torch.bfloat16 and Config.DENSE_BACKEND == "tcgen05" and hasattr(body, "repack")
        plain = wgmma and not getattr(body, "noisy_linear", False)
        return update_plan(
            self.kind, self.per, self.prefetch, self.dual, world=self.world, one_graph=one_graph, env=self._env,
            k1_body=plain and rp.history_length == 4 and tuple(getattr(rp, "item_shape", ())) == (84, 84),
            dual_body=wgmma and hasattr(getattr(self.tgt, "body", None), "repack"),
            tail=plain and nature_tc.FUSED_BWD and bool(_lib.CONV_SLAB) and self.opt.kind in ("rmsprop", "adam"),
            narrow_head=self._heads() is not None, n_step=rp.n_step)

    @property
    def ring(self):
        return self.plan.ring

    def _heads(self):
        """(online head modules, target head modules) when the heads fit the fused head + loss + backward kernel: narrow,
        16-byte aligned VanillaNet / DuelingNet heads."""
        out = []
        for n in (self.net, self.tgt):
            fa = getattr(n, "fc_head", None) or getattr(n, "fc_advantage", None)
            fv = getattr(n, "fc_value", None) if hasattr(n, "fc_advantage") else None
            if not isinstance(fa, torch.nn.Linear) or fa.out_features >= 32 or (fv is not None and not isinstance(fv, torch.nn.Linear)):
                return None
            if any(m is not None and m.weight.data_ptr() % 16 for m in (fa, fv)):
                return None
            out.append((fa, fv))
        return out

    # ------------------------------------------------------------------ the update, as eager code
    def _h2d(self):
        self.d_pack.copy_(self.h_pack, non_blocking=True)
        if self.staged is not None:
            self.staged.record()

    def _sample(self, tag=0, phase=None, feed=True):
        """feeds of this update + one sampled batch into buffer set ``tag`` (on the current stream).  ``phase`` "select" =
        feed + index draw only, "gather" = the batch from those indices (uniform replay), None = everything."""
        rp = self.replay
        # DQN_agent.py:104-112 calls feed() once per env transition; `feeds` single-item calls are exactly one multi-item
        # call with each item in its own slot (reference_feed_quirk off) plus `feeds` tree.add(max_priority) -- one launch
        if self.feeds and feed and phase != "gather":
            quirk, rp.quirk = rp.quirk, False
            rp._device_cursor = True                     # (a captured feed advances the device cursor only)
            if self.per:
                rp.feed_device(self.d_frames, self.d_action, self.d_reward, self.d_mask, self.feeds, add_leaf=False)
                rp.tree.add_n(self.feeds, rp.max_priority_dev)
            else:
                rp.feed_device(self.d_frames, self.d_action, self.d_reward, self.d_mask, self.feeds)
            rp.quirk = quirk
        kw = dict(phase=phase) if phase else {}
        if self.dtype == torch.bfloat16:
            # exact integer frames, space-to-depth layout; ImageNormalizer's scale is folded into conv1's weights.
            # K1 (self.ring): no batch at all -- conv1 reads the sampled stacks from the uint8 ring; the frames of a batch are
            # those of the ring until the next feed, which _main orders after the batch's last read
            return rp.sample_normalized(out_dtype=self.dtype, scale=None, layout="ring" if self.ring else "s2d", tag=tag, **kw)
        return rp.sample_normalized(out_dtype=self.dtype, scale=self.scale, layout="nchw", tag=tag, **kw)

    def _main(self, parity=None):
        plan = self.plan
        cur = torch.cuda.current_stream()
        nature_tc.mark("start")
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.dev)
            self._pre = torch.cuda.Stream(device=self.dev)
            self._packed_ev, self._sampled_ev = torch.cuda.Event(), torch.cuda.Event()
        side, pre = cur if plan.single_stream else self._side, self._pre
        fs = self.scale if self.dtype == torch.bfloat16 else 1.0
        tail = self.tail()
        if plan.repack_online:
            # online weights changed in the previous optimizer step: re-pack them on the side branch, next to feed + sample
            # (with the fused tail the optimizer kernel itself writes the packed bf16 operands)
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                self._repack(self.net)
                self._packed_ev.record(side)
        # async replay: the batch of the NEXT update is fed + sampled on a parallel branch.  K1: this update's batch is read
        # from the ring by both conv1 forwards and, last, by conv1's weight gradient.  The whole prefetch branch -- this
        # update's feeds, the index draw and the action / reward / mask gather of the next batch into the other buffer set --
        # forks after that last read, so every batch sees the ring exactly as the materialising form gathers it (after the
        # previous update's feeds, before this update's)
        feed = True
        if self.prefetch:
            eager = parity is None
            if eager:
                parity = self._parity
            if self._batch[parity] is None:                              # very first update: nothing prefetched yet
                self._batch[parity] = self._sample(parity)
                if self.wrapper_order:
                    self._sample(1 - parity, feed=False)                 # the wrapper's first fill of its second buffer
                    feed = False                                         # this update's feeds ran above
            t = self._batch[parity]
            if plan.prefetch == "start":
                self._prefetch_branch(parity, feed=feed)
            elif plan.prefetch != "after-ring-read":
                self._prefetch_branch(parity, "select", feed=feed)  # feed + index draw now (two one-CTA kernels), the gather later
            if eager:
                self._parity = 1 - parity
        else:
            t = self._sample(0)
        per = dict(is_prob=t.sampling_prob, eps=self.eps, alpha=self.alpha, beta_dev=self.d_beta) if self.per else {}
        # the fused head takes the features of the bodies: the forward fork below runs the bodies only
        fused = plan.head != "separate"
        net, tgt = (self.net.body, self.tgt.body) if fused else (self.net, self.tgt)
        if plan.forward == "dual":
            # online(s) and target(s') share every launch of the convolutional body (nature_tc.forward_dual): the grid of
            # each kernel is split between the two networks, so the per-launch fixed cost is paid once
            if tail is None:
                cur.wait_event(self._packed_ev)
            with nature_tc.dual_forward(net.body, tgt.body, t.next_state), frame_scale(fs):
                out = net(t.state)
                with torch.no_grad():
                    nxt_t = tgt(t.next_state)
                    nxt_o = net(t.next_state) if self.double_q else None
        else:
            # the target forward on s' and the online forward on s are independent: fork them onto two streams (two
            # parallel branches of the captured graph) so that the prologue / tail of one chain overlaps the other.  With
            # the paired conv1 both conv1s run first, as one launch on this stream; the branches continue from its outputs
            pair = contextlib.nullcontext()
            if plan.conv1 == "pair":
                if tail is None:
                    cur.wait_event(self._packed_ev)
                pair = nature_tc.paired_conv1(self.net.body, self.tgt.body, t.state, t.next_state, fs)
                nature_tc.mark("conv1_pair")
            with pair:
                side.wait_stream(cur)
                with torch.cuda.stream(side), frame_scale(fs), torch.no_grad():
                    nxt_t = tgt(t.next_state)
                if tail is None:
                    cur.wait_event(self._packed_ev)
                with frame_scale(fs):
                    with torch.no_grad():
                        nxt_o = net(t.next_state) if self.double_q else None
                    out = net(t.state)
                cur.wait_stream(side)
        nature_tc.mark("fwd_joined")
        if fused:
            # ONE launch for the online / target [/ double-Q] head forwards + target / loss / PER block + head backward
            heads = self._heads()
            r = ops.dqn_head_fused(out.detach(), nxt_t, nxt_o, heads[0], heads[1], t.action, t.reward, t.mask, self.gamma_n,
                                   tail.db4, two=plan.head == "fused-two", **per)
            root, grad = out, r["gphi"]
        elif self.kind == "dqn":
            root = out["q"]
            r = ops.dqn_loss_fused(root.detach(), nxt_t["q"], nxt_o["q"] if nxt_o else None, t.action, t.reward, t.mask,
                                   self.gamma_n, **per)
            grad = r["dq"]
        elif self.kind == "c51":
            root = out["log_prob"]
            r = ops.c51_loss_fused(root.detach(), nxt_t["prob"], nxt_o["prob"] if nxt_o else None, t.action, t.reward,
                                   t.mask, self.gamma_n, self.cat[0], self.cat[1], **per)
            grad = r["dlogp"]
        else:
            root = out["quantile"]
            r = ops.qr_loss_fused(root.detach(), nxt_t["quantile"], t.action, t.reward, t.mask, self.gamma_n)
            grad = r["dquant"]
        if self.per:
            if self.prefetch:                            # the sum tree is read by the prefetch branch: update after it
                cur.wait_event(self._sampled_ev)
            self.replay.update_priorities((t.idx, r["priority"]))
        nature_tc.mark("head" if fused else "loss")
        if fused:
            nature_tc.premask(grad, tail.db4)            # already masked by relu(fc4); its column sums are in the tail's db4
        if tail is None:
            self.opt.zero_grad()
        # the late prefetch fork: after conv1's weight gradient from the ring (beside the rest of the backward pass and the
        # update tail), after the last dgrad GEMM, or -- the fallback when neither fired -- after the backward pass
        fired, phase = [], None if plan.prefetch == "after-ring-read" else "gather"
        fork = lambda after=None: fired or (self._prefetch_branch(parity, phase, after, feed), fired.append(1))
        nature_tc.AFTER_RING_READ = fork if plan.prefetch == "after-ring-read" else None
        nature_tc.AFTER_DGRAD = fork if plan.prefetch == "gather-after-dgrad" else None
        try:
            with nature_tc.wgrad_stream(None if side is cur else side), nature_tc.grad_sink(tail):   # weight-gradient GEMMs on the side branch
                root.backward(grad)
        finally:
            nature_tc.AFTER_DGRAD = nature_tc.AFTER_RING_READ = None
        if not fused:
            nature_tc.mark("bwd_done")
        self.loss.copy_(r["loss"])
        if plan.prefetch not in (None, "start"):
            fork()
        if plan.join == "main":
            cur.wait_stream(pre)

    def _prefetch_branch(self, parity, phase=None, after=None, feed=True):
        cur, pre = torch.cuda.current_stream(), self._pre
        pre.wait_stream(cur)                                             # after the host->device copy of this update's feeds
        if after is not None:
            pre.wait_stream(after)                                       # and after the ring read launched there
        with torch.cuda.stream(pre):
            b = self._sample(1 - parity, phase, feed)
            if phase != "select":
                self._batch[1 - parity] = b
                self._sampled_ev.record(pre)
                nature_tc.mark("sampled")

    def _opt(self):
        tail = self.tail()
        if tail is not None:
            tail.step(max_norm=self.clip, grad_scale=1.0 / self.world, reduced_elsewhere=self.world > 1)
        else:
            self.opt.step(max_norm=self.clip, grad_scale=1.0 / self.world)
        nature_tc.mark("opt")
        if self.plan.join == "opt":                      # the late prefetch branch ran beside the update tail
            torch.cuda.current_stream().wait_stream(self._pre)

    # ------------------------------------------------------------------ capture / replay
    def capture(self, warmup=3, with_h2d=False):
        """Warm up eagerly on a side stream (cuDNN autotune, lazy allocations), then capture."""
        self.with_h2d = with_h2d
        self.refresh_packed()
        # multi GPU, default: the collectives are captured INSIDE the update graph -- fc4's slice of the gradient arena (95 % of
        # the bytes) is all-reduced asynchronously right after its weight-gradient GEMM, beside the convolution backward, the
        # small remainder after the last GEMM.  B2RL_NCCL_IN_GRAPH=0: [sample..backward] graph | eager all-reduce of the whole
        # arena | [clip + optimizer] graph (the older form; it exposes the whole all-reduce).
        self._overlap = self.world > 1 and self.plan.one_graph and self.tail() is not None
        s = torch.cuda.Stream(device=self.dev)
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                if with_h2d:
                    self._h2d()
                self._main()
                self._allreduce()
                self._opt()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.g_main, self.g_opt = [], None
        tree = getattr(self.replay, "tree", None)
        n_entries = tree.n_entries if tree is not None else None     # a capture's tree.add_n adds no leaf on the device
        try:
            self._capture_main(with_h2d)
        except Exception as e:                            # noqa: BLE001 -- any capture error: use the split form
            if self.world == 1 or not self.plan.one_graph:
                raise
            print("b2rl: NCCL capture failed (%s); using the split-graph form" % str(e).splitlines()[0], file=sys.stderr)
            torch.cuda.synchronize()
            self._plan = self._resolve_plan(one_graph=False)
            self._overlap = False
            self.g_main = []
            self._capture_main(with_h2d)
        if not self.plan.one_graph:                      # [sample..backward] | NCCL all-reduce | [clip+opt]
            self.g_opt = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.g_opt):
                self._opt()
        # host mirrors of the ring cursor advanced during warm-up / capture calls; re-derive from the device
        st = self.replay.ring_state.cpu()
        self.replay.pos, self.replay._size = int(st[0]), int(st[1])
        if tree is not None:
            tree.n_entries = n_entries
        self.launches_per_update = None
        return self

    def _capture_main(self, with_h2d):
        for parity in ((0, 1) if self.prefetch else (None,)):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=self.g_main[0].pool() if self.g_main else None,
                                  capture_error_mode=self.capture_error_mode):
                if with_h2d:
                    self._h2d()
                self._main(parity)
                if self.plan.one_graph:
                    self._allreduce()
                    self._opt()
            self.g_main.append(g)

    def _allreduce_early(self):
        """fc4's slice of the gradient arena, asynchronously (called on the weight-gradient branch right after kernel A4): the
        convolution backward proceeds while NCCL runs; ``_allreduce`` waits for it."""
        self._early_work = None
        if self._overlap:
            lo, hi = self._tail.early_slice
            self._early_work = parallel.allreduce_gradients(self.opt.grad[lo:hi], async_op=True)

    def _allreduce(self):
        if self.world <= 1:
            return
        tail = self.tail()
        if tail is not None and self._overlap:
            for lo, hi in tail.late_slices:
                parallel.allreduce_gradients(self.opt.grad[lo:hi])
            if self._early_work is not None:
                self._early_work.wait()
                self._early_work = None
        else:
            parallel.allreduce_gradients(self.opt.grad)

    def update(self):
        """One gradient update (graph replay).  Returns the device loss tensor (no sync)."""
        if self.prefetch:
            self.g_main[self._parity].replay()
            self._parity = 1 - self._parity
        else:
            self.g_main[0].replay()
        if self.g_opt is not None:
            self._allreduce()
            self.g_opt.replay()
        if self.per and self.feeds:                      # the replay's tree.add_n: its host count (state_dict saves it)
            tree = self.replay.tree
            tree.n_entries = min(tree.n_entries + self.feeds, tree.capacity)
        self.updates += 1
        if self.sync_every and self.updates % self.sync_every == 0:
            self.sync_target()
        return self.loss

    def first_update(self):
        """An agent's first update, then the capture (``wrapper_order``; the caller has staged this update's feeds and beta):
        the eager warm-up of ``capture(warmup=1, with_h2d=True)`` IS this update -- its own feeds, both batches drawn after
        them (ReplayWrapper's first sample), one optimizer step -- and the capture that follows executes nothing, so the
        agent ends exactly one update further on.  The next ``update()`` replays the other parity.  Returns the loss."""
        assert self.wrapper_order and self.prefetch and self.feeds and self.updates == 0
        self.capture(warmup=1, with_h2d=True)
        self.updates = 1
        return self.loss

    def update_from_host(self, frames, action, reward, mask, beta=None):
        """End-to-end update through HOST buffers: the env transitions of this update are written to the pinned
        staging area, copied host->device inside the captured graph, and the loss is read back."""
        assert self.with_h2d, "capture(with_h2d=True) first"
        self.h_frames.numpy()[...] = frames
        self.h_action.numpy()[...] = action
        self.h_reward.numpy()[...] = reward
        self.h_mask.numpy()[...] = mask
        if beta is not None:
            self.h_beta[0] = beta
        self.update()
        self.h_loss.copy_(self.loss, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return float(self.h_loss[0])

    @property
    def h2d_bytes(self):
        return self.h_pack.numel()


class _RolloutLearner(_NatureLearner):
    """What the captured rollout learners (``GraphedNStepLearner``, ``GraphedA2CLearner``) share: the uint8 arena of the
    rollout's frame stacks -- slot t (rows t N 4 .. (t + 1) N 4 - 1) the states of env step t, which the actor's upload writes
    there (component/actor.py ``GraphedQActor(arena=...)``), slot T the final states, plus one padding row --, the final states'
    pinned staging buffer, the fused update tail as the optimizer, and a capture that leaves the parameters untrained."""

    def _init_rollout(self, network, optimizer, rollout_length, num_envs, gradient_clip, state_scale, history, frame_hw):
        """Common state; returns the arena row of each of the (T + 1) N stacks (``idx[i] = 4 i``, rows t-major)."""
        self.net, self.opt = network, optimizer
        self.T, self.N, self.hl = int(rollout_length), int(num_envs), int(history)
        self.clip, self.scale = float(gradient_clip or 0.0), float(state_scale)
        self.dtype, self.world = torch.bfloat16, 1
        self.dev = dev = optimizer.flat.device
        self._plan, self._tail, self._side = None, None, None
        if not self.plan.tail:
            raise _lib.B2RLError("%s needs the fused update tail: a wgmma NatureConvBody with the fused backward epilogues, "
                                 "and RMSprop or Adam" % type(self).__name__)
        T, N, hl = self.T, self.N, self.hl
        row = frame_hw[0] * frame_hw[1]
        k = N * hl
        self.arena = torch.zeros(((T + 1) * k + 1, row), dtype=torch.uint8, device=dev)
        self.h_final = torch.zeros((k, row), dtype=torch.uint8, pin_memory=True)
        self._np_final = self.h_final.numpy().reshape(N, hl, row)
        self.graph = None
        self.updates = 0
        self.opt.zero_grad()              # the fused tail writes / re-zeroes the gradient arena itself: start from zeros
        return torch.arange((T + 1) * N, dtype=torch.int64, device=dev) * hl

    def _tail_applies(self):
        return (hasattr(self._body(self.net), "repack") and nature_tc.FUSED_BWD and bool(_lib.CONV_SLAB)
                and self.opt.kind in ("rmsprop", "adam"))

    def stage_final(self, states):
        """The final states' frame stacks (uint8 [history, H, W] each) into the pinned buffer the update uploads to slot T."""
        for i, s in enumerate(states):
            self._np_final[i] = np.asarray(s).reshape(self.hl, -1)

    def _opt(self):
        self.tail().step(max_norm=self.clip)

    def _state(self):
        o = self.opt
        return [o.flat, o.s1, o.s2, o.step_dev]

    def capture(self, warmup=1):
        """Warm up eagerly on a side stream (lazy allocations, kernel attributes), then capture.  The warm-up updates are
        undone: parameters and optimizer state are restored and the online operands re-packed from them."""
        saved = [t.clone() for t in self._state()]
        self.refresh_packed()
        s = torch.cuda.Stream(device=self.dev)
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                self._main()
                self._opt()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        from .component.actor import no_gc
        with no_gc(), torch.cuda.graph(self.graph):
            self._main()
            self._opt()
        for t, v in zip(self._state(), saved):
            t.copy_(v)
        self.opt.grad.zero_()
        self.refresh_packed()
        torch.cuda.synchronize()
        return self


class GraphedNStepLearner(_RolloutLearner):
    """The update of ``NStepDQNAgent.step()`` (NStepDQN_agent.py:52-67) for a VanillaNet on a wgmma NatureConvBody as ONE
    captured graph per rollout: the rollout's actions / rewards / masks up in one packed copy and the final states' stacks up
    into the arena, the online body at batch T N on the rollout's stacks beside the target body at batch N on the final ones
    (two branches), both heads (``b2rl_head_fwd``), the n-step target and loss (``b2rl_nstep_q_loss``), the head backward
    with fc4's ReLU (``b2rl_head_bwd_relu``), the fused body backward and the two-launch update tail (gradient reduce,
    ``clip_grad_norm_``, RMSprop / Adam, bf16 operand writes).

    ``arena`` holds the rollout's uint8 frame stacks: slot t (rows t N 4 .. (t + 1) N 4 - 1) the states of env step t, which
    the actor's upload writes there (component/actor.py ``GraphedQActor(arena=...)``), slot T the final states, plus one
    padding row.  Conv1's forward and weight gradient read the stacks from it (K1: ``RingFrames`` with ``idx[i] = 4 i``); no
    bf16 batch is built.  The online q of the rollout is recomputed rather than kept from the actor: the parameters do not
    change during a rollout, so it is the q the actor saw.

    The target sync (NStepDQN_agent.py:48-49) is the caller's ``sync_target()`` before ``update()``: the online parameters do
    not change inside a rollout, so syncing at its end gives the same target."""

    def __init__(self, network, target_network, optimizer, rollout_length, num_envs, discount=0.99, gradient_clip=5.0,
                 state_scale=1.0 / 255, history=4, frame_hw=(84, 84)):
        self.tgt, self.discount = target_network, float(discount)
        idx = self._init_rollout(network, optimizer, rollout_length, num_envs, gradient_clip, state_scale, history, frame_hw)
        T, N, dev = self.T, self.N, self.dev
        row = frame_hw[0] * frame_hw[1]
        self.states = nature_tc.RingFrames(self.arena, idx[:T * N], 0, row, frame_hw[1], self.hl)
        self.final = nature_tc.RingFrames(self.arena, idx[T * N:], 0, row, frame_hw[1], self.hl)
        # ONE packed pinned staging buffer for the rollout's scalars and ONE device mirror -> a single host->device copy node:
        # [action int64 T*N | reward float32 T*N | mask float32 T*N]
        rows = T * N
        self.h_pack = torch.zeros(16 * rows, dtype=torch.uint8, pin_memory=True)
        self.d_pack = torch.zeros(16 * rows, dtype=torch.uint8, device=dev)

        def views(buf):
            return (buf[:8 * rows].view(torch.int64).view(T, N), buf[8 * rows:12 * rows].view(torch.float32).view(T, N),
                    buf[12 * rows:].view(torch.float32).view(T, N))

        self.h_action, self.h_reward, self.h_mask = views(self.h_pack)
        self.d_action, self.d_reward, self.d_mask = views(self.d_pack)
        A = network.fc_head.out_features
        self.out = dict(ret=torch.zeros(rows, dtype=torch.float32, device=dev),
                        delta=torch.zeros(rows, dtype=torch.float32, device=dev),
                        loss=torch.zeros(1, dtype=torch.float32, device=dev),
                        gq=torch.zeros((rows, A), dtype=torch.float32, device=dev))
        self.loss = self.out["loss"]
        self.q = None                     # the online q of the last update [T*N, A] (a buffer of the captured graph)

    def _resolve_plan(self):
        tail = self._tail_applies()
        return UpdatePlan(ring=True, tail=tail, repack_online=not tail, dist_head=False, head="separate", forward="two-branch",
                          conv1="separate", single_stream=False, prefetch=None, join=None, one_graph=True)

    def _main(self):
        cur = torch.cuda.current_stream()
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.dev)
        side, tail = self._side, self.tail()
        k = self.N * self.hl
        self.arena[self.T * k:(self.T + 1) * k].copy_(self.h_final, non_blocking=True)
        self.d_pack.copy_(self.h_pack, non_blocking=True)
        # the target forward on the final states and the online forward on the rollout's states: two parallel branches
        side.wait_stream(cur)
        with torch.cuda.stream(side), frame_scale(self.scale), torch.no_grad():
            q_boot = self.tgt(self.final)["q"]
        with frame_scale(self.scale):
            q = self.net(self.states)["q"]
        cur.wait_stream(side)
        r = ops.nstep_q_loss(q.detach(), q_boot, self.d_action, self.d_reward, self.d_mask, self.discount, out=self.out)
        with nature_tc.wgrad_stream(side), nature_tc.grad_sink(tail):     # weight-gradient GEMMs on the side branch
            q.backward(r["gq"])
        self.q = q.detach()

    def update(self, sync_target=False):
        """One rollout's update (graph replay) on what the caller staged: ``h_action`` / ``h_reward`` / ``h_mask`` [T, N],
        the rollout's stacks in arena slots 0..T-1 and the final states (``stage_final``).  ``sync_target``: an env step of
        the rollout reached the target sync schedule; the target becomes the online network first.  Returns the device loss
        tensor (no sync)."""
        if sync_target:
            self.sync_target()
        self.graph.replay()
        self.updates += 1
        return self.loss


class GraphedA2CLearner(_RolloutLearner):
    """The update of ``A2CAgent.step()`` (A2C_agent.py:92-115) for a CategoricalActorCriticNet whose ``phi_body`` is a wgmma
    NatureConvBody (DummyBody actor / critic bodies) as ONE captured graph per rollout: the rollout's rewards / masks up in one
    packed copy and the final states' stacks up into arena slot T; the body at batch (T + 1) N on every stack of the arena
    (K1); the actor-critic head (``b2rl_ac_head_fwd``: logits and v); GAE, the objective and its gradient with respect to the
    head's outputs (``b2rl_a2c_rollout_loss``); the head backward with fc4's ReLU (``b2rl_head_bwd_geff_relu``); the fused
    body backward with its weight gradients on the side branch; and the two-launch update tail (gradient reduce,
    ``clip_grad_norm_``, RMSprop / Adam, bf16 operand writes, which the next actor replay reads).

    One forward covers the final states too: the reference's bootstrap value comes from the same (online) network
    (A2C_agent.py:93-96), and the final rows' zero gradient costs about 1 / (T + 1) of the backward.  The rollout's logits and
    values are recomputed rather than kept from the actor: the parameters do not change during a rollout.

    The actions are drawn on the device by the actor's replays (``act``, run by ``GraphedQActor(run=...)``) straight into
    ``d_action`` row t: the inverse CDF of the softmax on Philox ``u24(seed, counter + n, 13)`` with a device-resident counter,
    the stream ``config.device_a2c`` uses -- not torch's ``Categorical.sample``."""

    body_attr = "phi_body"

    def __init__(self, network, optimizer, rollout_length, num_envs, seed, discount=0.99, gae_tau=1.0, use_gae=True,
                 entropy_weight=0.01, value_loss_weight=1.0, gradient_clip=5.0, state_scale=1.0 / 255, history=4,
                 frame_hw=(84, 84)):
        self.tgt = None
        self.discount, self.gae_tau, self.use_gae = float(discount), float(gae_tau), bool(use_gae)
        self.ew, self.vw = float(entropy_weight), float(value_loss_weight)
        idx = self._init_rollout(network, optimizer, rollout_length, num_envs, gradient_clip, state_scale, history, frame_hw)
        T, N, dev = self.T, self.N, self.dev
        self.states = nature_tc.RingFrames(self.arena, idx, 0, frame_hw[0] * frame_hw[1], frame_hw[1], self.hl)
        # ONE packed pinned staging buffer for the rollout's scalars and ONE device mirror: [reward float32 T*N | mask float32 T*N]
        rows = T * N
        self.h_pack = torch.zeros(2 * rows, dtype=torch.float32, pin_memory=True)
        self.d_pack = torch.zeros(2 * rows, dtype=torch.float32, device=dev)
        self.h_reward, self.h_mask = self.h_pack[:rows].view(T, N), self.h_pack[rows:].view(T, N)
        self.d_reward, self.d_mask = self.d_pack[:rows].view(T, N), self.d_pack[rows:].view(T, N)
        A = network.fc_action.out_features
        self.d_action = torch.zeros((T, N), dtype=torch.int64, device=dev)          # row t: the actor replay of env step t
        self.seed = int(seed)
        self.counter = torch.zeros(1, dtype=torch.int64, device=dev)               # Philox position of the next draw
        self.ticket = torch.zeros(1, dtype=torch.int32, device=dev)
        self.act_out = torch.zeros((T, N, A + 1), dtype=torch.float32, device=dev)  # the actor's (logits, v) per slot
        self.head_out = torch.zeros(((T + 1) * N, A + 1), dtype=torch.float32, device=dev)
        self.out = dict(adv=torch.zeros(rows, dtype=torch.float32, device=dev),
                        ret=torch.zeros(rows, dtype=torch.float32, device=dev),
                        loss=torch.zeros(1, dtype=torch.float32, device=dev),
                        geff=torch.zeros(((T + 1) * N, ops.AC_GEFF_LD), dtype=torch.float32, device=dev))
        self.loss = self.out["loss"]

    def _resolve_plan(self):
        tail = self._tail_applies()
        return UpdatePlan(ring=True, tail=tail, repack_online=not tail, dist_head=False, head="separate", forward="one-stream",
                          conv1="separate", single_stream=False, prefetch=None, join=None, one_graph=True)

    def act(self, x, slot):
        """The actor's work on its gathered batch ``x`` (bf16 space-to-depth stacks of env step ``slot``; run by GraphedQActor
        under no_grad and the frame scale): the body, then the head with the draw into ``d_action[slot]``.  Returns that row."""
        net = self.net
        fused.ac_head(self._body(net)(x), net.fc_action, net.fc_critic, out=self.act_out[slot],
                      draw=(self.seed, self.counter, self.d_action[slot], self.ticket))
        return self.d_action[slot]

    def _main(self):
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.dev)
        side, tail, net = self._side, self.tail(), self.net
        k = self.N * self.hl
        self.arena[self.T * k:(self.T + 1) * k].copy_(self.h_final, non_blocking=True)
        self.d_pack.copy_(self.h_pack, non_blocking=True)
        with frame_scale(self.scale):
            phi = self._body(net)(self.states)
        fused.ac_head(phi.detach(), net.fc_action, net.fc_critic, out=self.head_out)
        r = ops.a2c_rollout_loss(self.head_out, self.d_action, self.d_reward, self.d_mask, self.discount, self.gae_tau,
                                 self.use_gae, self.ew, self.vw, out=self.out)
        with nature_tc.wgrad_stream(side), nature_tc.grad_sink(tail):     # weight-gradient GEMMs on the side branch
            phi.backward(fused.ac_head_backward(phi, r["geff"], net.fc_action, net.fc_critic))

    def update(self):
        """One rollout's update (graph replay) on what the caller staged: ``h_reward`` / ``h_mask`` [T, N], the rollout's stacks
        in arena slots 0..T-1 and its actions in ``d_action`` (the actor replays), and the final states (``stage_final``).
        Returns the device loss tensor (no sync)."""
        self.graph.replay()
        self.updates += 1
        return self.loss


class GraphedPPOPixelLearner(_RolloutLearner):
    """The update of ``PPOAgent.step()`` with ``config.shared_repr`` (PPO_agent.py:44-99) for a CategoricalActorCriticNet whose
    ``phi_body`` is a wgmma NatureConvBody (DummyBody actor / critic bodies) as ONE captured graph per rollout, in order:

    * one packed upload: the minibatch rows of all E epochs x M minibatches (drawn on the host by ``random_sample``, so numpy's
      stream is consumed as on the eager path), the rollout's rewards / masks, and this rollout's learning rate; and the final
      states' stacks up into arena slot T;
    * the body at batch N on the final states (K1) and the head without a draw -> ``act_out[T]`` (the reference's
      ``self.network(states)`` after the loop);
    * ``b2rl_ppo_rollout_prep``: the old log-probabilities at the taken actions, and ``ret`` / ``adv`` by GAE, from the
      (logits, v) rows the actor's replays stored in ``act_out`` -- the pre-update policy, not recomputed; then
      ``b2rl_normalize_advantage``;
    * E M minibatch updates, unrolled: the body at batch ``mini_batch_size`` on the minibatch's arena rows (K1: conv1's
      forward and weight gradient read the uint8 frames), the head, ``b2rl_ppo_cat_loss``, the head backward with fc4's ReLU,
      the fused body backward (weight gradients on the side branch) and the update tail (gradient reduce,
      ``clip_grad_norm_``, Adam at the device learning rate, bf16 operand writes that the next minibatch and the next actor
      replay read).

    The actions are drawn by the actor's replays (``act``, as ``GraphedA2CLearner``) into ``d_action`` row t: the inverse CDF
    of the softmax on Philox ``u24(seed, counter + n, 13)`` -- not torch's ``Categorical.sample``."""

    body_attr = "phi_body"
    act = GraphedA2CLearner.act

    def __init__(self, network, optimizer, rollout_length, num_envs, seed, mini_batch_size, optimization_epochs,
                 discount=0.99, gae_tau=0.95, use_gae=True, ppo_ratio_clip=0.1, entropy_weight=0.01, gradient_clip=0.5,
                 state_scale=1.0 / 255, history=4, frame_hw=(84, 84)):
        self.tgt = None
        self.discount, self.gae_tau, self.use_gae = float(discount), float(gae_tau), bool(use_gae)
        self.ratio_clip, self.ew = float(ppo_ratio_clip), float(entropy_weight)
        idx = self._init_rollout(network, optimizer, rollout_length, num_envs, gradient_clip, state_scale, history, frame_hw)
        T, N, hl, dev = self.T, self.N, self.hl, self.dev
        rows = T * N
        self.mb, self.epochs = int(mini_batch_size), int(optimization_epochs)
        if rows % self.mb or rows < 2:
            raise _lib.B2RLError("GraphedPPOPixelLearner: the rollout's %d rows must be at least 2 and a multiple of "
                                 "mini_batch_size %d" % (rows, self.mb))
        self.n_batches = self.epochs * (rows // self.mb)
        K = self.n_batches * self.mb
        row = frame_hw[0] * frame_hw[1]
        self.final = nature_tc.RingFrames(self.arena, idx[T * N:], 0, row, frame_hw[1], hl)
        # ONE packed pinned staging buffer and ONE device mirror -> a single host->device copy node:
        # [rollout row int64 K | arena row int64 K | reward float32 T*N | mask float32 T*N | lr float32 (+ pad)]
        nbytes = 16 * K + 8 * rows + 8
        self.h_pack = torch.zeros(nbytes, dtype=torch.uint8, pin_memory=True)
        self.d_pack = torch.zeros(nbytes, dtype=torch.uint8, device=dev)

        def views(buf):
            o = [0, 8 * K, 16 * K, 16 * K + 4 * rows, 16 * K + 8 * rows]
            return (buf[o[0]:o[1]].view(torch.int64).view(self.n_batches, self.mb),
                    buf[o[1]:o[2]].view(torch.int64).view(self.n_batches, self.mb),
                    buf[o[2]:o[3]].view(torch.float32).view(T, N), buf[o[3]:o[4]].view(torch.float32).view(T, N),
                    buf[o[4]:o[4] + 4].view(torch.float32))

        self.h_idx, self.h_arow, self.h_reward, self.h_mask, self.h_lr = views(self.h_pack)
        self.d_idx, self.d_arow, self.d_reward, self.d_mask, self.d_lr = views(self.d_pack)
        self.batches = [nature_tc.RingFrames(self.arena, self.d_arow[j], 0, row, frame_hw[1], hl) for j in range(self.n_batches)]
        A = network.fc_action.out_features
        self.d_action = torch.zeros((T, N), dtype=torch.int64, device=dev)          # row t: the actor replay of env step t
        self.seed = int(seed)
        self.counter = torch.zeros(1, dtype=torch.int64, device=dev)               # Philox position of the next draw
        self.ticket = torch.zeros(1, dtype=torch.int32, device=dev)
        # the actor's (logits, v) per slot; slot T: the final states' (written by the update)
        self.act_out = torch.zeros((T + 1, N, A + 1), dtype=torch.float32, device=dev)
        self.roll = {k: torch.zeros(rows, dtype=torch.float32, device=dev) for k in ("logp", "adv", "ret")}
        self.head_mb = torch.zeros((self.mb, A + 1), dtype=torch.float32, device=dev)
        self.geff = torch.zeros((self.mb, ops.AC_GEFF_LD), dtype=torch.float32, device=dev)
        self.stats = torch.zeros((self.n_batches, 3), dtype=torch.float32, device=dev)    # per minibatch: [pl, vl, kl]
        self.tail().lr_dev = self.d_lr

    def _resolve_plan(self):
        tail = self._tail_applies()
        return UpdatePlan(ring=True, tail=tail, repack_online=not tail, dist_head=False, head="separate", forward="one-stream",
                          conv1="separate", single_stream=False, prefetch=None, join=None, one_graph=True)

    def stage_batches(self, batches, lr):
        """The E M minibatches' rollout rows (``random_sample``'s arrays, in order) and this rollout's learning rate into the
        pinned buffer the update uploads."""
        b = np.asarray(batches, dtype=np.int64).reshape(self.n_batches, self.mb)
        self.h_idx.numpy()[...] = b
        self.h_arow.numpy()[...] = b * self.hl
        self.h_lr.numpy()[0] = lr

    def _main(self):
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.dev)
        side, tail, net = self._side, self.tail(), self.net
        body = self._body(net)
        T, k = self.T, self.N * self.hl
        self.arena[T * k:(T + 1) * k].copy_(self.h_final, non_blocking=True)
        self.d_pack.copy_(self.h_pack, non_blocking=True)
        with torch.no_grad(), frame_scale(self.scale):
            fused.ac_head(body(self.final), net.fc_action, net.fc_critic, out=self.act_out[T])
        r = ops.ppo_rollout_prep(self.act_out.view((T + 1) * self.N, -1), self.d_action, self.d_reward, self.d_mask,
                                 self.discount, self.gae_tau, self.use_gae, out=self.roll)
        ops.normalize_advantage_(r["adv"])
        for j in range(self.n_batches):
            with frame_scale(self.scale):
                phi = body(self.batches[j])
            fused.ac_head(phi.detach(), net.fc_action, net.fc_critic, out=self.head_mb)
            ops.ppo_cat_loss(self.head_mb, self.d_idx[j], self.d_action, r["logp"], r["adv"], r["ret"], self.ratio_clip,
                             self.ew, geff=self.geff, stats=self.stats[j])
            with nature_tc.wgrad_stream(side), nature_tc.grad_sink(tail):     # weight-gradient GEMMs on the side branch
                phi.backward(fused.ac_head_backward(phi, self.geff, net.fc_action, net.fc_critic))
            tail.step(max_norm=self.clip)

    def _opt(self):
        """(The optimizer steps run inside ``_main``, one per minibatch.)"""

    def update(self):
        """One rollout's update (graph replay) on what the caller staged: ``h_reward`` / ``h_mask`` [T, N], the rollout's stacks
        in arena slots 0..T-1 with their actions in ``d_action`` and (logits, v) in ``act_out`` (the actor replays), the final
        states (``stage_final``), and the minibatches and learning rate (``stage_batches``).  Returns the device statistics
        [policy_loss, value_loss, approx_kl] of the last minibatch (no sync)."""
        self.graph.replay()
        self.updates += 1
        return self.stats[-1]


class _PPOLearner:
    """What both PPO learners share: the rollout rows in persistent device buffers (``load``), the minibatch index rows of
    ALL epochs of an iteration uploaded once (``set_batches``) and the statistics of the last update."""

    KEYS = ("state", "action", "log_pi_a", "ret", "advantage")

    def __init__(self, network, actor_opt, critic_opt, rows, state_dim, action_dim, mini_batch_size, ppo_ratio_clip,
                 entropy_weight, target_kl, max_batches):
        self.net, self.actor_opt, self.critic_opt = network, actor_opt, critic_opt
        self.mb, self.clip, self.ent_w, self.target_kl = int(mini_batch_size), ppo_ratio_clip, entropy_weight, target_kl
        dev = self.dev = actor_opt.flat.device
        f = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)
        self.buf = dict(state=f(rows, state_dim), action=f(rows, action_dim), log_pi_a=f(rows, 1), ret=f(rows, 1),
                        advantage=f(rows, 1))
        self.perm = torch.zeros((max_batches, self.mb), dtype=torch.int64, device=dev)
        self.stats = torch.zeros(4, dtype=torch.float32, device=dev)      # policy loss, value loss, approx KL of the last update

    def load(self, entries):
        for k in self.KEYS:
            self.buf[k].copy_(getattr(entries, k).reshape(self.buf[k].shape))

    def set_batches(self, index_rows):
        rows = np.stack([np.asarray(r, dtype=np.int64) for r in index_rows])
        assert rows.shape[1] == self.mb and rows.shape[0] <= self.perm.shape[0]
        self.perm[:rows.shape[0]].copy_(torch.from_numpy(rows), non_blocking=False)
        return rows.shape[0]


class GraphedPPOLearner(_PPOLearner):
    """The PPO minibatch update (PPO_agent.py:73-99, non-shared representation) as ONE captured graph replayed once per
    minibatch: row gather by a device-resident index matrix, network forward, ``b2rl_ppo_loss`` (clipped surrogate, value
    loss, approx-KL and their gradients in one launch), backward, KL-GATED actor Adam step (``b2rl_clip_adam_gated``: the
    reference's ``if approx_kl <= 1.5 * target_kl`` decided on the device) and the critic Adam step.  An iteration of
    examples.py:496-522 is 5 120 such updates of an 11 k-parameter MLP: eager, each is dominated by Python and launch
    latency; as a graph replay the host cost is one ``cudaGraphLaunch``.  The minibatch index rows (``set_batches``) are
    consumed through a device cursor."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.cursor = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self.graph = None

    def set_batches(self, index_rows):
        n = super().set_batches(index_rows)
        self.cursor.zero_()
        return n

    def _step(self):
        idx = self.perm.index_select(0, self.cursor).view(-1)
        e = {k: v.index_select(0, idx) for k, v in self.buf.items()}
        pred = self.net(e["state"], e["action"])
        r = ops.ppo_loss_fused(pred["log_pi_a"].detach(), pred["entropy"].detach(), pred["v"].detach(), e["log_pi_a"],
                               e["advantage"], e["ret"], self.clip, self.ent_w)
        shape = pred["v"].shape
        self.actor_opt.zero_grad()
        torch.autograd.backward([pred["log_pi_a"], pred["entropy"]], [r["dlogp"].view(shape), r["dent"].view(shape)])
        self.actor_opt.step(gate=r["out"][2:3], gate_max=1.5 * self.target_kl)        # PPO_agent.py:94-97
        self.critic_opt.zero_grad()
        pred["v"].backward(r["dv"].view(shape))
        self.critic_opt.step()                                                        # PPO_agent.py:98-99
        self.stats.copy_(r["out"])
        self.cursor.add_(1)

    def _state(self):
        return [t for o in (self.actor_opt, self.critic_opt) for t in (o.flat, o.s1, o.s2, o.step_dev)]

    def capture(self, warmup=3):
        """Warm-up + capture run on whatever is in the buffers; parameters and optimizer state are restored afterwards."""
        saved = [t.clone() for t in self._state()]
        validate = torch.distributions.Distribution._validate_args
        torch.distributions.Distribution.set_default_validate_args(False)     # argument checks synchronise: not capturable
        try:
            s = torch.cuda.Stream(device=self.dev)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(warmup):
                    self.cursor.zero_()
                    _lib.reset_launch_count()
                    self._step()
                    self.launches_per_update = _lib.launch_count()     # of OUR kernels (the MLP itself is torch / cuBLAS)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            self.cursor.zero_()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._step()
        finally:
            torch.distributions.Distribution.set_default_validate_args(validate)
        for t, v in zip(self._state(), saved):
            t.copy_(v)
        self.cursor.zero_()
        torch.cuda.synchronize()
        return self

    def run(self, n_batches):
        for _ in range(n_batches):
            self.graph.replay()


class PersistentPPOLearner(_PPOLearner):
    """The whole minibatch loop of a PPO iteration (PPO_agent.py:68-99, non-shared representation) as ONE launch of one
    persistent thread block (``b2rl_ppo_minibatch_updates``, csrc/ppo_persistent.cu): weights in shared memory, Adam moments in
    L2, the rows of the next minibatch fetched during the current update, the KL gate decided on the device.  Same interface as
    ``GraphedPPOLearner`` (which replays ~45 small kernels per update and remains the path for every network this kernel does
    not cover)."""

    A_NAMES = ("actor_body.layers.0.weight", "actor_body.layers.0.bias", "actor_body.layers.1.weight",
               "actor_body.layers.1.bias", "fc_action.weight", "fc_action.bias", "std")
    C_NAMES = ("critic_body.layers.0.weight", "critic_body.layers.0.bias", "critic_body.layers.1.weight",
               "critic_body.layers.1.bias", "fc_critic.weight", "fc_critic.bias")

    @staticmethod
    def supported(network, mini_batch_size):
        """GaussianActorCriticNet with DummyBody phi and two-layer tanh FCBody actor / critic bodies of equal widths."""
        from .network.network_bodies import DummyBody, FCBody
        from .network.network_heads import GaussianActorCriticNet
        if not isinstance(network, GaussianActorCriticNet) or not isinstance(network.phi_body, DummyBody):
            return False
        ab, cb = network.actor_body, network.critic_body
        if not all(isinstance(b, FCBody) and len(b.layers) == 2 and b.gate is torch.tanh and not b.noisy_linear for b in (ab, cb)):
            return False
        dims = lambda b: (b.layers[0].in_features, b.layers[0].out_features, b.layers[1].out_features)
        D, H1, H2 = dims(ab)
        A = network.fc_action.out_features
        if not (dims(cb) == (D, H1, H2) and D <= 256 and H1 <= 128 and H2 <= 128 and A <= 32 and 4 <= mini_batch_size <= 128
                and mini_batch_size % 4 == 0 and network.fc_action.weight.is_cuda):
            return False
        # weights + double-buffered rows + both networks' activations must fit the shared memory of one SM
        # (examples.py:496-522: D = 17, hidden 64, A = 6, mini batch 64 -> 205 KB)
        return int(_lib.lib().b2rl_ppo_minibatch_smem_bytes(D, A, H1, H2, int(mini_batch_size))) <= 227 * 1024

    def __init__(self, network, actor_opt, critic_opt, rows, state_dim, action_dim, mini_batch_size, ppo_ratio_clip,
                 entropy_weight, target_kl, max_batches, world=1, rank=0, exchange_timeout_s=5.0):
        if actor_opt.kind != "adam" or critic_opt.kind != "adam":
            raise NotImplementedError("the persistent PPO kernel implements Adam (examples.py:508-509)")
        super().__init__(network, actor_opt, critic_opt, rows, state_dim, action_dim, mini_batch_size, ppo_ratio_clip,
                         entropy_weight, target_kl, max_batches)
        self.world, self.rank, self.rows = int(world), int(rank), int(rows)
        named = dict(network.named_parameters())
        self.a_off = self._offsets(actor_opt, [named[n] for n in self.A_NAMES])
        self.c_off = self._offsets(critic_opt, [named[n] for n in self.C_NAMES])
        ab = network.actor_body
        self.D, self.H1, self.H2 = ab.layers[0].in_features, ab.layers[0].out_features, ab.layers[1].out_features
        self.A = network.fc_action.out_features
        self.launches_per_update = 0.0
        self.n = 0
        if self.world > 1:
            # data parallel (one process per GPU): every update exchanges the ranks' gradients inside the kernel, through
            # exchange regions mapped into every peer (parallel.ExchangeRegions); seq = updates exchanged so far
            a_n, c_n = actor_opt.flat.numel(), critic_opt.flat.numel()
            self.exchange = parallel.ExchangeRegions(int(_lib.lib().b2rl_ppo_dp_region_bytes(a_n, c_n)), self.dev)
            self.status = torch.zeros(1, dtype=torch.int64, device=self.dev)
            self.seq = 0
            self.timeout_ns = int(exchange_timeout_s * 1e9)

    def check_exchange(self):
        """Raise if a data-parallel launch gave up waiting for a peer (synchronises with the device)."""
        if self.world > 1:
            code = int(self.status[0])
            if code:
                peer, k = (code - 1) % 16, (code - 1) // 16
                raise _lib.B2RLError("PPO data-parallel exchange: rank %d did not publish update %d" % (peer, self.seq_last + k))

    @staticmethod
    def _offsets(opt, params):
        """Element offsets of ``params`` inside the optimizer's arena (host int32 array for the kernel's argument block)."""
        base = opt.flat.data_ptr()
        offs = []
        for p in params:
            off = (p.data_ptr() - base) // 4
            if not (0 <= off and off + p.numel() <= opt.n) or getattr(p, "_b2rl_flat_owner", None) != id(opt):
                raise _lib.B2RLError("PersistentPPOLearner: a parameter does not live in the optimizer's arena")
            offs.append(off)
        return torch.tensor(offs, dtype=torch.int32)

    def capture(self, warmup=0):
        return self

    def run(self, n_batches):
        a, c, b = self.actor_opt, self.critic_opt, self.buf
        if self.world > 1:
            self.check_exchange()                      # (the previous iteration's launch)
            n_batches = parallel.agree(n_batches, self.dev, "PPO minibatches per iteration")
        args = (*[_lib.ptr(b[k]) for k in self.KEYS], self.D, self.A, self.H1, self.H2, self.mb, _lib.ptr(self.perm),
                int(n_batches), *[_lib.ptr(t) for t in (a.flat, a.s1, a.s2, a.step_dev, self.a_off)],
                *[_lib.ptr(t) for t in (c.flat, c.s1, c.s2, c.step_dev, self.c_off)],
                *[float(x) for x in (a.lr, a.betas[0], a.betas[1], a.eps, c.lr, c.betas[0], c.betas[1], c.eps)],
                float(self.clip), float(self.ent_w), float(1.5 * self.target_kl), _lib.ptr(self.stats))
        if self.world > 1:
            _lib.call("b2rl_ppo_minibatch_updates_dp", *args, self.rows, a.flat.numel(), c.flat.numel(), self.world, self.rank,
                      self.exchange.table, self.seq, self.timeout_ns, _lib.ptr(self.status), 1, _lib.stream())
            self.seq_last = self.seq
            self.seq += int(n_batches)
        else:
            _lib.call("b2rl_ppo_minibatch_updates", *args, _lib.stream())
        self.n = int(n_batches)         # (the one launch is counted by _lib.call itself; launches_per_update stays 0)

