"""``dqn_pixel``, ``categorical_dqn_pixel`` and ``quantile_regression_dqn_pixel`` as written, on the captured agent path
(``DQNAgent._async_graph_update`` -> ``GraphedDQNLearner(prefetch=True, wrapper_order=True)``), step by step.

Real agents, built from the launchers at bf16 with ``cuda_graph``, a 300-row ring that wraps during the sequence and
epsilon = 1 (the actions do not depend on Q), step through exploration and then take STEPS captured steps.  As in
test_gpu_update_sequence.py nothing compares a trajectory: after every step each check starts from the device's own state.

Exact, after every agent step k (the first captured step included):
1. the pinned staging buffer holds this step's transitions -- frame ``s[-1]``, action, ``SignNormalizer(r)``, ``1 - done``
   and, with PER, float32 of the beta schedule's value for this update -- and the device copy equals it;
2. ring rows (pos + i) % cap hold them and no other row changed; the device cursor is the mirror's;
3. the draws follow ReplayWrapper.sample(): the first update feeds once, then draws A (trained on), B (discarded) and C
   (the refill, trained on by update 2); every later update trains on the batch drawn during the previous one, after that
   update's feeds, and draws one batch.  The Philox counter advances by exactly those draws; the trained and the next
   batch (indices, action, n-step reward and mask; PER: tree indices and sampling probabilities) are the mirror's;
4. PER: the float64 sum tree, ``max_priority``, the pending flags, the write cursor and ``n_entries`` equal
   oracle/replay.PrioritizedReplay driven in the plan's order with the device's own priorities;
5. from the exact tensors the loss kernel read (online output, target and double-Q outputs on s'), the TD target with
   ``gamma_n = discount ** n_step``, the per-sample loss, the PER weights with this update's beta, the priorities and the
   loss recomputed in float64 within fp32 reduction error;
6. the gradient arena is zero, Adam's step counts the updates, the optimizer state is finite, the packed bf16 operands
   (and the distributional head's bf16 weight) are those of the fp32 weights, and the target is unchanged except at a
   sync, where it is the online network bit for bit, re-packed at the same addresses.

Teacher-forced on the first step, the first after a target sync and one later step: oracle.agents.DQNFamilyOracle from the
snapshot before the step, on the batch as the ring held it when the update read it, with the tolerances of
test_gpu_update_sequence.py (the global gradient cosine above 0.99; Adam's first step compared globally only).  With ``async_actor`` every actor forward reads one whole parameter version: the one left by
the updates enqueued before it."""
import itertools
import os
import sys
import threading
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)
from test_dqn_pixel_graph import _launch, _small_replay  # noqa: E402
from test_gpu_losses_exact import c51_atoms, qr_tau32  # noqa: E402
from test_gpu_tail_exact import packed_ref  # noqa: E402
from test_gpu_update_sequence import (Mirror, assert_equal, batch_bufs, check_oracle_step, dist_fc, host_sd,  # noqa: E402
                                      oracle_batch, seed_optimizer, spy_losses)

CAP = 300              # ring rows: not full at the first update (n_entries still counts), wrapped by step 5
EXPLORATION = 280
STEPS = 12
SYNC_EVERY = 3         # target_network_update_freq: syncs after steps 2, 5, 8 and 11
NUMERIC = (1, 3, 7)    # teacher-forced: the first step, the first after a sync, a later one
REWARD_SCALE = 2.5     # the envs' rewards are scaled so that SignNormalizer changes them
P_DONE = 0.05          # n-step rows: episode ends inside sampled windows
PER_STEPS = 100        # PER rows: the beta schedule moves 0.006 per update (a stale call shows in float32)

# (id, launcher, launcher arguments, changes after the launcher, plan: ring, conv1, prefetch, dist_head)
ROWS = [
    ("dqn", "dqn_pixel", {}, {}, (True, "pair", "after-ring-read", False)),
    ("dqn-double", "dqn_pixel", dict(game="SyntheticAtari-A18-v0"), dict(double_q=True),
     (True, "pair", "after-ring-read", False)),
    ("dqn-nstep3", "dqn_pixel", dict(n_step=3), dict(p_done=P_DONE), (True, "separate", "after-ring-read", False)),
    ("dqn-per", "dqn_pixel", dict(replay_cls="per"), {}, (False, "separate", "start", False)),
    ("dqn-per-nstep3", "dqn_pixel", dict(replay_cls="per", n_step=3), dict(p_done=P_DONE), (False, "separate", "start", False)),
    ("c51", "categorical_dqn_pixel", dict(game="SyntheticAtari-A18-v0"), {}, (True, "pair", "after-ring-read", True)),
    ("c51-per", "categorical_dqn_pixel", {}, dict(per=True), (False, "separate", "start", True)),
    ("qr", "quantile_regression_dqn_pixel", {}, {}, (True, "pair", "after-ring-read", True)),
    ("dqn-async-actor", "dqn_pixel", {}, dict(async_actor=True), (True, "pair", "after-ring-read", False)),
]
KIND = {"dqn_pixel": "dqn", "categorical_dqn_pixel": "c51", "quantile_regression_dqn_pixel": "qr"}
HEAD = {"VanillaNet": "vanilla", "CategoricalNet": "categorical", "QuantileNet": "quantile"}


# ------------------------------------------------------------------------------------------------ wrapper order
def wrapper_draws(k):
    """What update k (1-based) does after its feeds, in ReplayWrapper.sample()'s order: the draws it makes, each
    "train" (the batch this update trains on), "discard" or "next" (the batch the next update trains on)."""
    return ("train", "discard", "next") if k == 1 else ("next",)


def mirror_step(mirror, k, pending, staged):
    """The mirror through update k's feeds and draws; returns (trained batch, next batch)."""
    mirror.feed(*staged)
    drawn = {role: mirror.draw() for role in wrapper_draws(k)}
    return drawn.get("train", pending), drawn["next"]


# ------------------------------------------------------------------------------------------------ CPU premises
@pytest.mark.parametrize("case,name,kw,after,plan", ROWS, ids=[r[0] for r in ROWS])
def test_update_plan_of_each_row(case, name, kw, after, plan):
    """The agent builds its learner with prefetch and wrapper_order on a wgmma NatureConvBody and a 4 x 84 x 84 uint8 ring;
    from those plain values update_plan gives each row's plan."""
    from deeprl_b200.learner import update_plan
    kind = KIND[name]
    per = kw.get("replay_cls") == "per" or after.get("per", False)
    p = update_plan(kind, per, prefetch=True, narrow_head=kind == "dqn", n_step=kw.get("n_step", 1))
    assert (p.ring, p.conv1, p.prefetch, p.dist_head) == plan, p
    assert p.tail and p.head == "separate" and p.forward == "two-branch" and p.one_graph, p


def test_wrapper_order_is_the_async_wrappers_fill_sequence(monkeypatch):
    """On a stub replay that numbers its draws, ReplayWrapper(async_=True) hands out draw 0 on the first sample() after the
    step's feed, draws 1 (discarded) and 2 (handed out next), then one draw per sample(), each after that step's feed:
    the sequence ``wrapper_draws`` gives the mirror."""
    from deeprl_b200.component.replay import ReplayWrapper
    log, count = [], iter(range(100))

    class Stub:
        def sample(self, tag=0, check=True):
            log.append("draw")
            return next(count)

        def feed(self, exp):
            log.append("feed")

    class NoStream:
        def wait_stream(self, s):
            pass

        def wait_event(self, e):
            pass

    class NoEvent:
        def record(self, stream=None):
            pass

    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: NoStream())
    monkeypatch.setattr(torch.cuda, "Event", NoEvent)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: __import__("contextlib").nullcontext())
    w = ReplayWrapper.__new__(ReplayWrapper)
    w.replay, w.async_, w._side = Stub(), True, NoStream()
    w._ready, w._cache, w._cur, w._primed = [None, None], [None, None], 0, False
    got, want = [], []
    pending, draws = None, 0
    for k in range(1, 6):
        log.clear()
        w.feed({})
        got.append((tuple(log[:1]) + ("sample",), w.sample(), tuple(log[1:])))
        roles = wrapper_draws(k)
        numbered = dict(zip(roles, range(draws, draws + len(roles))))
        draws += len(roles)
        trained = numbered.get("train", pending)
        pending = numbered["next"]
        want.append((("feed", "sample"), trained, ("draw",) * len(roles)))
    assert got == want


def test_raised_p_done_gives_nstep_windows_across_episode_ends():
    """At p_done = 0.05 the ring of the n-step rows holds windows whose n-step mask is 0 (at the launcher's 1e-3 a ring of
    this size would almost surely hold none): a wrong mask or a wrong n-step reward there changes the loss."""
    from deeprl_b200.component.envs import SyntheticAtariEnv
    from oracle.replay import UniformReplay as OU
    env = SyntheticAtariEnv(4, p_done=P_DONE)
    env.seed(0)
    env.reset()
    o = OU(CAP, 32, 3, 0.99, 4)
    for t in range(EXPLORATION + 4 * STEPS):
        _, r, done, _ = env.step(0)
        if done:
            env.reset()
        o.feed(dict(state=[np.array([t])], action=[0], reward=[np.sign(r * REWARD_SCALE)], mask=[1 - int(done)]))
    masks = [o.construct_transition(i).mask for i in range(CAP) if o.valid_index(i)]
    assert len(masks) > 200 and 0.05 < 1 - np.mean(masks) < 0.5, np.mean(masks)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def rl():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import deeprl_b200 as rl
    rl.select_device(0)
    old = rl.Config.COMPUTE_DTYPE
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    yield rl
    rl.Config.COMPUTE_DTYPE = old


def _tweak_envs(task, p_done):
    """Scale the synthetic envs' rewards (so that the sign normalizer is visible) and, for the n-step rows, raise p_done."""
    for e in task.env.envs:
        while not hasattr(e, "p_done"):
            e = e.env
        if p_done is not None:
            e.p_done = p_done
        e.step = lambda a, _step=e.step: (lambda o, r, d, i: (o, REWARD_SCALE * r, d, i))(*_step(a))


def _build(rl, name, kw, after):
    import examples
    kw = dict(kw)
    if kw.get("replay_cls") == "per":
        kw["replay_cls"] = examples.PrioritizedReplay
    cls, cfg = _launch(name, **kw)
    _small_replay(name, cfg, CAP)
    if after.get("per"):
        examples._replay(cfg, examples.PrioritizedReplay, True, memory_size=CAP, history_length=4)
    cfg.max_steps = PER_STEPS
    examples._per_schedule(cfg)
    cfg.double_q = after.get("double_q", cfg.double_q)
    cfg.async_actor = after.get("async_actor", False)
    cfg.exploration_steps = EXPLORATION
    cfg.target_network_update_freq = SYNC_EVERY
    cfg.random_action_prob = rl.LinearSchedule(1.0, 1.0, 1)
    np.random.seed(0), torch.manual_seed(0)
    ag = cls(cfg)
    if cfg.async_actor:                                   # the actor thread builds its task on its first step
        task_fn = cfg.task_fn
        cfg.task_fn = lambda: (lambda t: (_tweak_envs(t, after.get("p_done")), t)[1])(task_fn())
    else:
        _tweak_envs(ag.actor._task, after.get("p_done"))
    return ag


def _close(got, want, scale, what):
    """|got - want| <= 1e-5 scale elementwise (fp32 reductions of float64-exact inputs)."""
    got, want = np.asarray(got, np.float64).reshape(-1), np.asarray(want, np.float64).reshape(-1)
    bad = np.abs(got - want) > 1e-5 * np.asarray(scale, np.float64).reshape(-1) + 1e-30
    assert not bad.any(), "%s: %d of %d differ, e.g. %r vs %r" % (what, bad.sum(), bad.size, got[bad][:3], want[bad][:3])


def _choices(values):
    """Per row, the actions whose float64 value is within fp32 summation error of the maximum (normally one): the device
    picks the first maximum of its own fp32 sums, which a near-tie may resolve either way."""
    v = values.astype(np.float64)
    top = v.max(1, keepdims=True)
    near = v >= top - 1e-5 * (1 + np.abs(v).max(1, keepdims=True))
    return [np.nonzero(r)[0].tolist() for r in near]


def check_loss64(ag, sp, bufs, beta, what):
    """The loss kernel's outputs from its exact inputs, in float64: TD target with gamma_n = discount ** n_step, per-sample
    loss, PER weights with ``beta``, priorities and the reduced loss."""
    cfg, lr = ag.config, ag._learner
    gamma_n = cfg.discount ** cfg.n_step
    a = bufs["action"].cpu().numpy()
    r, m = bufs["reward"].cpu().double().numpy(), bufs["mask"].cpu().double().numpy()
    B = a.shape[0]
    rows = np.arange(B)
    out = sp["out"].float().cpu().double().numpy()
    nt = sp["next_t"].float().cpu().double().numpy()
    no = None if sp["next_o"] is None else sp["next_o"].float().cpu().double().numpy()
    res = {k: (None if v is None else v.float().cpu().double().numpy()) for k, v in sp["r"].items()}
    kind = lr.kind
    if lr.per:
        prob = bufs["prob"].cpu().double().numpy()
        w = (prob * B + 1e-6) ** -float(np.float32(beta))
        w = w / w.max()
    else:
        w = np.ones(B)

    def per_sample(a_star):
        if kind == "dqn":
            target = r + gamma_n * nt[rows, a_star] * m
            return target - out[rows, a], np.abs(target) + np.abs(out[rows, a])
        if kind == "c51":
            z = c51_atoms(lr.cat[0], lr.cat[1], nt.shape[-1]).double().numpy()
            dz = (lr.cat[1] - lr.cat[0]) / (z.size - 1)
            tz = np.clip(r[:, None] + gamma_n * m[:, None] * z[None], lr.cat[0], lr.cat[1])
            proj = np.clip(1 - np.abs(tz[:, None, :] - z[None, :, None]) / dz, 0, 1)        # [B, j, k]
            mm = (proj * nt[rows, a_star][:, None, :]).sum(-1)
            lpa = out[rows, a]
            terms = mm * np.log(mm + float(np.float32(1e-5))) - mm * lpa
            return terms.sum(-1), np.abs(terms).sum(-1)
        N = nt.shape[-1]
        tau = qr_tau32(N).double().numpy()
        T = r[:, None] + gamma_n * m[:, None] * nt[rows, a_star]                               # [B, j]
        u = T[:, :, None] - out[rows, a][:, None, :]                                          # [B, j, i]
        hub = np.where(np.abs(u) < 1.0, 0.5 * u * u, np.abs(u) - 0.5)
        terms = hub * np.abs(tau[None, None, :] - (u < 0))
        return terms.sum((1, 2)) / N, np.abs(terms).sum((1, 2)) / N

    if kind == "dqn":
        sel = no if no is not None else nt
        options = [[int(i)] for i in np.argmax(sel, 1)]             # the fp32 values themselves: the first maximum, exactly
    else:
        z = c51_atoms(lr.cat[0], lr.cat[1], nt.shape[-1]).double().numpy() if kind == "c51" else None
        sel = no if no is not None else nt
        options = _choices((sel * z).sum(-1) if kind == "c51" else sel.sum(-1))
    ambiguous = [i for i, o in enumerate(options) if len(o) > 1]
    assert len(ambiguous) <= 3, what + ": near-tied next actions in %d rows" % len(ambiguous)
    errors = []
    for pick in itertools.product(*[options[i] for i in ambiguous]):
        a_star = np.asarray([o[0] for o in options])
        a_star[ambiguous] = pick
        d, scale = per_sample(a_star)
        try:
            if kind == "dqn":
                _close(res["delta"], d, scale, what + ": delta (TD target - Q)")
                loss, lscale = np.mean(0.5 * (d * w) ** 2), np.mean(0.5 * (scale * w) ** 2)
            elif kind == "c51":
                _close(res["kl"], d, scale, what + ": per-sample KL")
                loss, lscale = np.mean(d * w), np.mean(scale * w)
            else:
                loss, lscale = np.mean(d), np.mean(scale)
            _close(res["loss"], loss, lscale, what + ": loss")
            if lr.per:
                _close(res["priority"], (np.abs(d) + lr.eps) ** lr.alpha, (scale + lr.eps) ** lr.alpha, what + ": priorities")
            return
        except AssertionError as e:
            errors.append(str(e))
    raise AssertionError("; ".join(errors))


def _staged(rec):
    """This step's transitions as the agent stages them: frame s[-1], action, SignNormalizer(r), 1 - done."""
    frames = np.stack([np.asarray(t[0][0])[-1].reshape(-1) for t in rec]).astype(np.uint8)
    action = np.asarray([int(t[1][0]) for t in rec], np.int32)
    reward = np.asarray([np.sign(float(t[2][0])) for t in rec], np.float64)
    mask = np.asarray([1 - int(t[4][0]) for t in rec], np.int32)
    return frames, action, reward, mask


def _oracle(ag, snap, beta):
    from oracle import agents
    cfg, lr = ag.config, ag._learner
    head = HEAD[type(ag.network).__name__]
    orc = agents.DQNFamilyOracle(
        snap["online"], head, "nature", cfg.action_dim, cfg.optimizer_fn, cfg.discount, cfg.n_step, double_q=bool(cfg.double_q),
        gradient_clip=cfg.gradient_clip, state_coef=1.0 / 255,
        atoms=np.linspace(lr.cat[0], lr.cat[1], cfg.categorical_n_atoms) if head == "categorical" else None,
        v_min=lr.cat[0], v_max=lr.cat[1], num_quantiles=getattr(cfg, "num_quantiles", None),
        replay_eps=lr.eps, replay_alpha=lr.alpha, replay_beta=lambda: float(np.float32(beta)))
    for k, v in snap["target"].items():
        orc.target_sd[k].copy_(v)
    seed_optimizer(orc, lr, snap["s1"], snap["s2"], snap["step"])
    return orc


def _record_forwards(ag):
    """async_actor: every actor forward's input and q values, with the number of updates enqueued before it."""
    seen, pending = [], []
    actor = ag.actor
    graphed = actor._graphed

    def wrapped():
        ga = graphed()
        if ga and not getattr(ga, "_recording", False):
            ga._recording = True
            enqueue, result = ga.enqueue, ga.result

            def enq(states, slot=0):                 # under ParameterOrder.lock, as the updates are enqueued
                lr = ag._learner
                pending.append(lr.updates if lr is not None else 0)
                return enqueue(states, slot)

            def res():
                q = result()
                seen.append((pending.pop(), ga.x.clone(), q.copy()))
                return q
            ga.enqueue, ga.result = enq, res
        return ga
    actor._graphed = wrapped
    return seen


def _eager_q(ag, sd, x):
    from deeprl_b200.network.fused import frame_scale
    fresh = ag.config.network_fn()
    fresh.load_state_dict(sd)
    with torch.no_grad(), frame_scale(ag.config.state_normalizer.coef):
        return ag.actor._q_tensor(fresh(x.permute(0, 3, 1, 2))).float().cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("case,name,kw,after,plan", ROWS, ids=[r[0] for r in ROWS])
def test_agent_sequence(rl, monkeypatch, case, name, kw, after, plan):
    from deeprl_b200 import ops
    ag = _build(rl, name, kw, after)
    cfg = ag.config
    assert ag.graph_refusal is None, ag.graph_refusal
    got = []
    inner_step = ag.actor.step
    ag.actor.step = lambda: (lambda out: (got.append(out), out)[1])(inner_step())
    forwards = _record_forwards(ag) if cfg.async_actor else None
    while ag.total_steps < EXPLORATION:
        ag.step()
    torch.cuda.synchronize()
    assert ag._learner is None and ag.total_steps == EXPLORATION
    rp = ag.replay.replay
    per = hasattr(rp, "tree")
    seen = spy_losses(monkeypatch, ops)
    sched = rl.LinearSchedule(0.4, 1.0, PER_STEPS)            # what config.replay_beta returns, call by call
    mirror = Mirror(types.SimpleNamespace(replay=rp, per=per))
    if per:
        assert rp.tree.n_entries == rp.size() == EXPLORATION
        mirror.o.tree.n_entries = rp.tree.n_entries
    o = ag._flat
    versions = [{k: v.detach().clone() for k, v in ag.network.state_dict().items()}]
    tgt_prev, pending, ptrs, zero_masks = host_sd(ag.target_network), None, None, 0
    # async_actor: the checks hold config.lock, so the actor thread enqueues (and captures) nothing while they read the
    # device; it runs its forwards beside every update
    lock = cfg.lock if cfg.async_actor else threading.Lock()
    lock.acquire()
    try:
        for k in range(1, STEPS + 1):
            what = "%s step %d" % (case, k)
            lr = ag._learner
            par = lr._parity if lr is not None else 0
            ring0 = {n: getattr(rp, n).clone() for n in ("frames", "action", "reward", "mask")}
            st0 = rp.ring_state.cpu().tolist()
            assert st0[4] == mirror.ctr, what + ": Philox counter before the step"
            snap = dict(online=host_sd(ag.network), target=tgt_prev, flat=o.flat.clone(), s1=o.s1.cpu(), s2=o.s2.cpu(),
                        step=int(o.step_dev.item()) if o.kind == "adam" else k - 1)
            beta = sched() if per else None
            n_got = len(got)
            lock.release()
            try:
                ag.step()
            finally:
                lock.acquire()
            torch.cuda.synchronize()
            lr = ag._learner
            assert lr is not None and lr.updates == k and len(got) == n_got + 1
            if k == 1:
                p = lr.plan
                assert (p.ring, p.conv1, p.prefetch, p.dist_head) == plan, p
                assert p.tail and lr.wrapper_order and lr.prefetch and lr.per == per
                assert len(seen) == 3, "the first update (eager) and one capture per parity: %d loss launches" % len(seen)
            # 1. staging
            staged = _staged(got[-1])
            assert np.array_equal(lr.h_frames.numpy(), staged[0]), what + ": staged frames"
            for n, want in zip(("action", "reward", "mask"), staged[1:]):
                assert np.array_equal(getattr(lr, "h_" + n).numpy(), want), "%s: staged %s" % (what, n)
            if per:
                assert lr.h_beta.numpy()[0] == np.float32(beta), "%s: staged beta %r, schedule %r" % (what, lr.h_beta[0], beta)
            assert torch.equal(lr.d_pack.cpu(), lr.h_pack), what + ": device copy of the staging buffer"
            # 3. draws in wrapper order, against the mirror
            trained, nxt = mirror_step(mirror, k, pending, staged[1:])
            bufs = batch_bufs(lr, par)
            mirror.check_batch(bufs, trained, what)
            mirror.check_batch(batch_bufs(lr, 1 - par), nxt, what + " (next batch)")
            pending = nxt
            zero_masks += int((bufs["mask"] == 0).sum())
            sp = seen[0] if k == 1 else seen[1 + par]
            # 4. PER: the tree after the device's own priorities of this update
            if per:
                mirror.o.update_priorities(zip(bufs["tree_idx"].cpu().numpy(), sp["r"]["priority"].cpu().numpy()))
                mirror.check_tree(what)
                assert rp.tree.n_entries == mirror.o.tree.n_entries, what + ": n_entries %d, mirror %d" % (
                    rp.tree.n_entries, mirror.o.tree.n_entries)
            # 2. ring: cursor, counter, rows
            st = rp.ring_state.cpu().tolist()
            size = rp.size()                              # (re-reads the host cursor from the device)
            assert (st[0], st[1]) == (mirror.o.pos, mirror.o._size) == (rp.pos, size), (what, st[:2])
            assert st[4] == mirror.ctr, what + ": Philox counter advanced by %d, want %d" % (st[4] - st0[4], mirror.ctr - st0[4])
            rows = torch.as_tensor((int(st0[0]) + np.arange(lr.feeds)) % CAP, device=rp.device)
            for n, want in ring0.items():
                old = want[rows].clone()
                want[rows] = torch.from_numpy(staged[("frames", "action", "reward", "mask").index(n)]).to(want.device, want.dtype)
                assert_equal(getattr(rp, n), want, what + ": ring " + n)
                want[rows] = old                              # the ring before the step's feeds
            # 5. loss outputs from the loss kernel's inputs, in float64
            if per:
                assert lr.d_beta.cpu().numpy()[0] == np.float32(beta), what + ": device beta"
            check_loss64(ag, sp, bufs, beta, what)
            # 6. bookkeeping
            assert int((o.grad != 0).sum()) == 0, what + ": gradient arena not re-zeroed"
            if o.kind == "adam":
                assert int(o.step_dev.item()) == k, what + ": Adam step"
            for n in ("flat", "s1", "s2"):
                assert bool(torch.isfinite(getattr(o, n)).all()), what + ": non-finite " + n
            nets = {"online": ag.network, "target": ag.target_network}
            for w, net in nets.items():
                for n, g, want in zip(("w1f", "w2f", "w2d", "w3f", "w3d", "w4p"), net.body._packed.tensors(),
                                      packed_ref(net.body, lr.scale)):
                    assert_equal(g.cpu(), want, "%s: %s packed %s" % (what, w, n))
                if lr.plan.dist_head:
                    fc = dist_fc(net)
                    assert_equal(fc._w16, fc.weight.detach().to(torch.bfloat16), "%s: %s head _w16" % (what, w))
            synced = ag.total_steps // cfg.sgd_update_frequency % SYNC_EVERY == 0
            tgt_now = host_sd(ag.target_network)
            want_t = host_sd(ag.network) if synced else tgt_prev
            for n, v in tgt_now.items():
                assert_equal(v, want_t[n], "%s: target %s (%s)" % (what, n, "synced" if synced else "unchanged"))
            now = {w: [t.data_ptr() for t in net.body._packed.tensors()] for w, net in nets.items()}
            if lr.plan.dist_head:
                now.update({w + "_w16": dist_fc(net)._w16.data_ptr() for w, net in nets.items()})
            ptrs = ptrs or now
            assert now == ptrs, what + ": a packed operand moved away from the address the graphs read"
            tgt_prev = tgt_now
            versions.append({k2: v.detach().clone() for k2, v in ag.network.state_dict().items()})
            # teacher-forced: the first update read the ring after its own feeds; every later one reads the ring before them
            if k in NUMERIC:
                frames = rp.frames if k == 1 else ring0["frames"]
                tr = oracle_batch(frames, bufs, 4, cfg.n_step)
                if per:
                    tr.sampling_prob = bufs["prob"].cpu().numpy()
                # global gradient cosine above 0.99, not 0.995: measured 0.9948 once at 18 actions with double-Q.  Adam's
                # first step moves each element by about lr * sign(g), so a bias element whose gradient is within bf16
                # noise of zero flips its whole step: that step's delta is compared globally only
                check_oracle_step(_oracle(ag, snap, beta), lr, tr, snap, sp, float(sp["r"]["loss"].item()), what,
                                  grad_cos=0.99, delta_per_tensor=not (o.kind == "adam" and snap["step"] == 0))
    finally:
        lock.release()
        ag.close()                                        # (async_actor: the actor thread is gone, nothing more is recorded)
    if cfg.n_step > 1:
        assert zero_masks > 0, "premise: some trained n-step windows cross an episode end"
    if forwards is not None:
        checked = [f for f in forwards if f[0] >= 1]
        assert len(checked) >= STEPS, len(checked)
        for u, x, q in checked:
            assert torch.equal(torch.from_numpy(q), _eager_q(ag, versions[u], x)), \
                "a forward after %d updates does not read parameter version %d" % (u, u)
