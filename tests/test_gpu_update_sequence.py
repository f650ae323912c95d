"""The captured DQN-family update (``GraphedDQNLearner.update()``, the path bench.py times) across consecutive graph replays.

A replay leaves state behind for the next one: the online network's packed bf16 operands and the bf16 head weight written
by the fused optimizer, the target network re-packed in place by ``sync_target`` between replays, the ring cursor and the
Philox counter, the feeds staged through the pinned upload, the batch the async branch drew for the next replay, the sum tree
and ``max_priority``.  Whole trajectories are not comparable (fp32 atomics in the bias / head gradients change the last bits
from run to run, and with PER those bits change the priorities, the tree and the next batch), so nothing here compares a
trajectory.  After every replay each transition is checked EXACTLY against host mirrors advanced from the device's own
state, and the numerics of some replays are checked TEACHER-FORCED: ``oracle.agents.DQNFamilyOracle`` starts from the
snapshot taken before the replay (online and target parameters, optimizer moments and step) and runs the batch the replay
trained on, with the tolerances of test_gpu_step_vs_oracle.py.

Exact, after every replay k:
1. the online body's six packed operands = the host re-pack of its fp32 parameters (1/255 folded into conv1); C51 / QR:
   the online head's ``_w16`` = bf16 of its weight;
2. the target's fp32 parameters are unchanged, except after the replay that makes ``updates % 3 == 0``, when they equal the
   online parameters; its packed operands = the re-pack of its parameters, its head's ``_w16`` = bf16 of its weight, and
   no packed tensor or ``_w16`` moves (the graph captured their addresses);
3. the gradient arena is all zeros, Adam's step counter = updates since the reset, every optimizer element is finite;
4. the ring cursor = the host mirror advanced by the feeds; ring rows (pos + i) % cap hold the staged transitions and no
   other row changed; the Philox counter advanced by exactly one draw;
5. the indices replay k trained on, and their action / reward / mask, are those oracle/philox.py and oracle/replay.py draw
   from the counter and the ring mirror where the plan draws: after this update's feeds (sync replay) or after the previous
   update's feeds (async replay);
6. PER: the float64 tree, ``max_priority`` and the pending flags = oracle/replay.PrioritizedReplay driven in the plan's
   order (the feeds' adds, the stratified draws from Philox streams 2 / 3, ``update_priorities`` with the device's own
   priorities of the update).

Teacher-forced, on the first replay, the first after the target sync and the one after it: the online and target (and
double-Q online) outputs the loss kernel read are within the bf16 tolerance of test_gpu_q_actor.py of the oracle's forward;
loss 2e-2 relative; the device's clipped gradient, recovered from its new and old optimizer moments, and its parameter delta
have cosine above 0.98 with the oracle's per tensor (0.995 and 0.98 globally); clipped norm and step length within 5e-2.
A stale operand shows up exactly in checks 1-2 and here as a wrong forward and loss; since every update starts from the
device's own state, bf16 rounding does not compound across replays."""
import dataclasses
import os
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)
from oracle import philox  # noqa: E402
from test_gpu_philox_exact import _check_scalars, _oracle_ring  # noqa: E402
from test_gpu_tail_exact import packed_ref  # noqa: E402

pytestmark = pytest.mark.gpu

REPLAYS = 6
SYNC_EVERY = 3
NUMERIC = (0, 3, 4)          # the first replay, the first after the target sync at update 3, and the one after it
FEEDS = 4

# (id, workload, prefetch, conv1 forced, the plan the row is meant to run: ring, conv1, prefetch, head, dist_head; every
# row also runs the fused tail)
ROWS = [
    ("dqn-sync", "dqn", False, None, (True, "pair", None, "separate", False)),
    ("dqn-async", "dqn", True, None, (True, "pair", "after-ring-read", "separate", False)),
    ("dqn-async-conv1-separate", "dqn", True, "separate", (True, "separate", "after-ring-read", "separate", False)),
    ("per-sync", "per", False, None, (True, "pair", None, "separate", False)),
    ("per-async", "per", True, None, (False, "separate", "start", "separate", False)),
    ("c51-sync", "c51", False, None, (True, "pair", None, "separate", True)),
    ("c51-async", "c51", True, None, (True, "pair", "after-ring-read", "separate", True)),
    ("qr-sync", "qr", False, None, (True, "pair", None, "separate", True)),
    ("qr-async", "qr", True, None, (True, "pair", "after-ring-read", "separate", True)),
]


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import bench
    import deeprl_b200 as rl
    rl.select_device(0)
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    bench.CAP = 30_000
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    return bench, rl


def cosine(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def assert_equal(got, want, what):
    assert got.shape == want.shape and torch.equal(got, want), \
        "%s: %d of %d elements differ" % (what, int((got != want).sum()) if got.shape == want.shape else -1, want.numel())


def batch_bufs(lr, parity):
    rp = lr.replay
    return rp._bufs[(rp.batch_size, torch.bfloat16, rp.LAYOUTS["ring" if lr.ring else "s2d"], parity)]


def dist_fc(net):
    return getattr(net, "fc_categorical", None) or getattr(net, "fc_quantiles", None)


def host_sd(net):
    return {k: v.detach().float().cpu().clone() for k, v in net.state_dict().items()}


def spy_losses(monkeypatch, ops):
    """Keep the device tensors every loss launch reads and writes: online output, target (and double-Q online) next-state
    output, and the result dict with the priorities.  Captured graphs replay into the same tensors."""
    seen = []
    for name, n_in in (("dqn_loss_fused", 3), ("c51_loss_fused", 3), ("qr_loss_fused", 2)):
        fn = getattr(ops, name)

        def spy(*args, _fn=fn, _n=n_in, **kw):
            r = _fn(*args, **kw)
            seen.append(dict(out=args[0], next_t=args[1], next_o=args[2] if _n == 3 else None, r=r))
            return r
        monkeypatch.setattr(ops, name, spy)
    return seen


class Mirror:
    """Host mirror of the ring's scalars, cursor and Philox counter (and, with PER, the sum tree) advanced in the plan's
    order from the device's state after capture."""

    def __init__(self, lr):
        rp = self.rp = lr.replay
        st = rp.ring_state.cpu().tolist()
        self.cap, self.B, self.seed = rp.memory_size, rp.batch_size, rp.seed
        self.per = lr.per
        from oracle.replay import PrioritizedReplay as OP, UniformReplay as OU
        self.o = _oracle_ring(OP if self.per else OU, self.cap, self.B, rp.history_length, rp.n_step, int(st[0]), int(st[1]),
                              rp.action.cpu().numpy(), rp.reward.cpu().numpy(), rp.mask.cpu().numpy())
        self.o.discount = rp.discount
        self.ctr = int(st[4])
        if self.per:
            t = self.o.tree
            t.tree[:] = rp.tree.tree.cpu().numpy()
            t.write, t.n_entries = int(st[3]), self.cap
            t.pending = set((np.nonzero(rp.tree.pending.cpu().numpy())[0] + self.cap - 1).tolist())
            self.o.max_priority = float(rp.max_priority_dev.item())

    def feed(self, action, reward, mask):
        o = self.o
        for i in range(FEEDS):
            row = o.pos
            o.data["action"][row], o.data["reward"][row], o.data["mask"][row] = int(action[i]), float(reward[i]), int(mask[i])
            if o.pos >= o._size:
                o._size += 1
            o.pos = (o.pos + 1) % self.cap
            if self.per:
                o.tree.add(o.max_priority)

    def draw(self):
        """The batch the device draws at the current counter: dict(idx, [tree_idx, prob64,] tr)."""
        o, B, ctr = self.o, self.B, self.ctr
        if self.per:
            u = philox.u53(self.seed, np.uint64(ctr) + np.arange(B, dtype=np.uint64), 2)
            seg = o.tree.total() / B
            n_valid = sum(o.valid_index(int(o.tree.get(seg * i + (seg * (i + 1) - seg * i) * u[i])[2])) for i in range(B))
            k = np.arange(B - n_valid, dtype=np.uint64)
            fills = philox.below(self.seed, np.uint64(ctr + B) + k, 3, np.uint64(n_valid) + k).astype(np.int64)
            tr = o.sample(uniforms=u, fills=fills)
            self.ctr += 2 * B
            return dict(idx=np.asarray(tr.idx, np.int64) - self.cap + 1, tree_idx=np.asarray(tr.idx, np.int64),
                        prob64=np.asarray(tr.sampling_prob, np.float64), tr=tr)
        n_cand = min(8192, max(2 * B, B + 256))
        cand = philox.below(self.seed, np.uint64(ctr) + np.arange(n_cand, dtype=np.uint64), 1, o._size).astype(np.int64)
        tr, taken, _ = o.sample(B, candidates=cand)
        self.ctr += n_cand
        return dict(idx=taken, tr=tr)

    def check_batch(self, bufs, want, what):
        assert np.array_equal(bufs["idx"].cpu().numpy(), want["idx"]), what + ": trained-on indices"
        _check_scalars(bufs, want["tr"])
        if self.per:
            assert np.array_equal(bufs["tree_idx"].cpu().numpy(), want["tree_idx"]), what + ": tree indices"
            assert np.array_equal(bufs["prob64"].cpu().numpy(), want["prob64"]), what + ": sampling probabilities"

    def check_tree(self, what):
        rp, t = self.rp, self.o.tree
        assert np.array_equal(rp.tree.tree.cpu().numpy(), t.tree), what + ": sum tree"
        assert rp.max_priority == float(self.o.max_priority), what + ": max_priority"
        pend = np.zeros(self.cap, bool)
        pend[np.asarray(sorted(t.pending), np.int64) - self.cap + 1] = True
        assert np.array_equal(rp.tree.pending.cpu().numpy() != 0, pend), what + ": pending flags"
        assert int(rp.ring_state[3]) == t.write, what + ": tree write cursor"


def seed_optimizer(orc, lr, s1, s2, step):
    """The oracle's torch.optim state = the device's moments and step before the replay."""
    base = lr.opt.flat.data_ptr()
    for n, p in lr.net.named_parameters():
        off, k = (p.data_ptr() - base) // 4, p.numel()
        m1, m2 = s1[off:off + k].view_as(p).clone(), s2[off:off + k].view_as(p).clone()
        st = dict(step=torch.tensor(float(step)))
        if lr.opt.kind == "adam":
            st.update(exp_avg=m1, exp_avg_sq=m2)
        else:
            st.update(square_avg=m1, grad_avg=m2)
        orc.opt.state[orc.sd[n]] = st


def oracle_batch(frames, bufs, hl, n_step):
    """The batch of ``bufs`` (indices, action, reward, mask) with its state / next-state stacks read from ``frames``."""
    idx = bufs["idx"]
    rows = idx.view(-1, 1) + torch.arange(-(hl - 1), 1, device=idx.device).view(1, -1)
    fr = frames.view(-1, 84, 84)
    return types.SimpleNamespace(state=fr[rows.view(-1)].view(-1, hl, 84, 84).cpu().numpy(),
                                 next_state=fr[(rows + n_step).view(-1)].view(-1, hl, 84, 84).cpu().numpy(),
                                 action=bufs["action"].cpu().numpy(), reward=bufs["reward"].cpu().numpy(),
                                 mask=bufs["mask"].cpu().numpy())


def teacher_forced(bench, lr, workload, snap, frames, bufs, spied, loss_dev, beta, what):
    """One oracle update from the snapshot taken before the replay, on the batch it trained on, against the device."""
    from oracle import agents
    tr = oracle_batch(frames, bufs, lr.replay.history_length, lr.replay.n_step)
    head = {"dqn": "vanilla", "per": "dueling", "c51": "categorical", "qr": "quantile"}[workload]
    if workload in ("dqn", "per"):
        opt_fn = lambda p: torch.optim.RMSprop(p, lr=0.00025, alpha=0.95, eps=0.01, centered=True)
    elif workload == "c51":
        opt_fn = lambda p: torch.optim.Adam(p, lr=0.00025, eps=0.01 / 32)
    else:
        opt_fn = lambda p: torch.optim.Adam(p, lr=0.00005, eps=0.01 / 32)
    orc = agents.DQNFamilyOracle(snap["online"], head, "nature", bench.ACTIONS, opt_fn, 0.99, 1, double_q=(workload == "per"),
                                 gradient_clip=5, state_coef=1.0 / 255,
                                 atoms=np.linspace(-10, 10, 51) if workload == "c51" else None, v_min=-10, v_max=10,
                                 num_quantiles=200 if workload == "qr" else None, replay_beta=lambda: beta)
    for k, v in snap["target"].items():
        orc.target_sd[k].copy_(v)
    seed_optimizer(orc, lr, snap["s1"], snap["s2"], snap["step"])
    if workload == "per":
        tr.sampling_prob = bufs["prob"].cpu().numpy()
    check_oracle_step(orc, lr, tr, snap, spied, loss_dev, what)


OUTPUT_KEYS = {"vanilla": ("q", "q"), "dueling": ("q", "q"), "categorical": ("log_prob", "prob"),
               "quantile": ("quantile", "quantile")}


def check_oracle_step(orc, lr, tr, snap, spied, loss_dev, what, grad_cos=0.995, delta_per_tensor=True):
    """The device's update from ``snap`` against ``orc`` (a DQNFamilyOracle seeded with the same parameters, target and
    optimizer state) on the batch ``tr``: the forwards the loss kernel read, the loss, the clipped gradient recovered from
    the optimizer moments (``grad_cos``: the bound of its global cosine) and the parameter delta (``delta_per_tensor``:
    its direction per tensor too, not only globally)."""
    key = OUTPUT_KEYS[orc.head]
    with torch.no_grad():
        s, s2 = orc.normalize(tr.state), orc.normalize(tr.next_state)
        pairs = [(spied["out"], orc.forward(orc.sd, s)[key[0]], "online(s)"),
                 (spied["next_t"], orc.forward(orc.target_sd, s2)[key[1]], "target(s')")]
        if spied["next_o"] is not None:
            pairs.append((spied["next_o"], orc.forward(orc.sd, s2)[key[1]], "online(s')"))
    for dev_out, ref, name in pairs:
        got = dev_out.float().cpu().reshape(ref.shape).numpy()
        ref = ref.double().numpy()
        np.testing.assert_allclose(got, ref, rtol=0, atol=3e-2 * max(1.0, float(np.abs(ref).max())),
                                   err_msg="%s: %s" % (what, name))
    # ---- the update.  The device's clipped gradient is recovered from its moments: Adam's exp_avg (RMSprop's grad_avg) is
    # beta1 m + (1 - beta1) g (alpha a + (1 - alpha) g) of the one before the replay
    before = {k: v.detach().clone() for k, v in orc.sd.items()}
    loss_orc = float(orc.update(tr))
    bad = []
    if abs(loss_dev - loss_orc) > 2e-2 * abs(loss_orc):
        bad.append("loss %.6g, oracle %.6g" % (loss_dev, loss_orc))
    o = lr.opt
    if o.kind == "adam":
        w, new, old = o.betas[0], o.s1.cpu(), snap["s1"]
    else:
        w, new, old = o.alpha, o.s2.cpu(), snap["s2"]
    base = o.flat.data_ptr()
    g_dev, g_orc, d_dev, d_orc = [], [], [], []
    for n, p in lr.net.named_parameters():
        off, k = (p.data_ptr() - base) // 4, p.numel()
        gd = (new[off:off + k].double() - w * old[off:off + k].double()) / (1 - w)
        go = orc.sd[n].grad.flatten()
        dd = (o.flat[off:off + k] - snap["flat"][off:off + k]).float().cpu()
        do = (orc.sd[n].detach() - before[n]).flatten()
        if go.norm() > 1e-8 and cosine(gd, go) <= 0.98:
            bad.append("gradient direction of %s: %.5f" % (n, cosine(gd, go)))
        if delta_per_tensor and do.norm() > 0 and cosine(dd, do) <= 0.98:
            bad.append("parameter-delta direction of %s: %.5f" % (n, cosine(dd, do)))
        g_dev.append(gd), g_orc.append(go), d_dev.append(dd), d_orc.append(do)
    g_dev, g_orc, d_dev, d_orc = (torch.cat(x) for x in (g_dev, g_orc, d_dev, d_orc))
    if cosine(g_dev, g_orc) <= grad_cos:
        bad.append("gradient direction %.5f" % cosine(g_dev, g_orc))
    if cosine(d_dev, d_orc) <= 0.98:
        bad.append("parameter-delta direction %.5f" % cosine(d_dev, d_orc))
    if abs(float(g_dev.norm()) - float(g_orc.norm())) > 5e-2 * float(g_orc.norm()):
        bad.append("clipped gradient norm %.6g, oracle %.6g" % (float(g_dev.norm()), float(g_orc.norm())))
    if abs(float(d_dev.norm()) - float(d_orc.norm())) > 5e-2 * float(d_orc.norm()):
        bad.append("step length %.6g, oracle %.6g" % (float(d_dev.norm()), float(d_orc.norm())))
    assert not bad, "%s: %s" % (what, "; ".join(bad))


@pytest.mark.parametrize("case,workload,prefetch,conv1,plan", ROWS, ids=[r[0] for r in ROWS])
def test_update_sequence(env, monkeypatch, case, workload, prefetch, conv1, plan):
    bench, rl = env
    from deeprl_b200 import ops
    lr = bench.build_learner(rl, workload, torch.device("cuda", 0), 0, 1, prefetch=prefetch)
    lr.sync_every = SYNC_EVERY                           # bench builds with target_sync_every=0
    if conv1 is not None:
        lr._plan = dataclasses.replace(lr.plan, conv1=conv1)
    p = lr.plan
    assert (p.ring, p.conv1, p.prefetch, p.head, p.dist_head) == plan, p
    # every row runs the fused update tail bench.py times (it writes the online operands and re-zeroes the gradient arena);
    # its plan depends on module switches such as nature_tc.FUSED_BWD, which a test must not leave changed
    assert p.tail and not p.repack_online, p
    seen = spy_losses(monkeypatch, ops)
    lr.capture(warmup=3, with_h2d=True)
    graphs = 2 if prefetch else 1
    spied = seen[-graphs:]                               # the captured launches, one per graph (parity 0, 1)
    assert len(spied) == graphs
    rp, opt = lr.replay, lr.opt
    # a clean optimizer state: Adam's step then counts the updates of this sequence
    opt.s1.zero_(), opt.s2.zero_(), opt.step_dev.zero_()
    torch.cuda.synchronize()
    assert lr.updates == 0

    nets = {"online": lr.net, "target": lr.tgt}
    ptrs = {w: [t.data_ptr() for t in n.body._packed.tensors()] for w, n in nets.items()}
    if p.dist_head:
        ptrs.update({w + "_w16": dist_fc(n)._w16.data_ptr() for w, n in nets.items()})
    mirror = Mirror(lr)
    pending = None                                       # async: the batch the previous replay drew for this one
    rng = np.random.default_rng(sum(map(ord, case)))
    tgt_prev = host_sd(lr.tgt)
    for k in range(REPLAYS):
        what = "%s replay %d" % (case, k)
        par = lr._parity if prefetch else 0
        bufs = batch_bufs(lr, par)
        # ---- this update's transitions, all different; PER: a different beta
        frames = rng.integers(0, 256, (FEEDS, rp.row_bytes), dtype=np.uint8)
        action = rng.integers(0, bench.ACTIONS, FEEDS).astype(np.int32)
        reward = rng.normal(size=FEEDS)
        mask = (rng.random(FEEDS) > 0.3).astype(np.int32)
        beta = float(np.float32(0.4 + 0.1 * k)) if lr.per else None
        # ---- snapshot before the replay
        ring0 = {n: getattr(rp, n).clone() for n in ("frames", "action", "reward", "mask")}
        st0 = rp.ring_state.cpu().tolist()
        assert int(st0[4]) == mirror.ctr, what + ": Philox counter before the replay"
        snap = dict(online=host_sd(lr.net), target=tgt_prev, flat=opt.flat.clone(), s1=opt.s1.cpu(), s2=opt.s2.cpu(),
                    step=int(opt.step_dev.item()))
        if prefetch and pending is None:
            pending = dict(idx=bufs["idx"].cpu().numpy())       # drawn before the sequence: checked to stay put
        # ---- the mirror, in the plan's order: feeds, the draw, (after the replay) the priorities of the trained batch
        mirror.feed(action, reward, mask)
        drawn = mirror.draw()
        trained = pending if prefetch else drawn
        loss = lr.update_from_host(frames, action, reward, mask, beta=beta)
        torch.cuda.synchronize()
        sp = spied[par]
        # 5. batch identity (and the batch the async branch drew for the next replay)
        if "tr" in trained:
            mirror.check_batch(bufs, trained, what)
        else:
            assert np.array_equal(bufs["idx"].cpu().numpy(), trained["idx"]), what + ": prefetched batch overwritten"
        if prefetch:
            mirror.check_batch(batch_bufs(lr, 1 - par), drawn, what + " (next batch)")
            pending = drawn
        # 6. PER: the tree after the device's own priorities of this update
        if lr.per:
            prio = sp["r"]["priority"].cpu().numpy()
            tree_idx = bufs["tree_idx"].cpu().numpy()
            mirror.o.update_priorities(zip(tree_idx, prio))
            mirror.check_tree(what)
        # 4. ring: cursor, rows, counter
        o = mirror.o
        st = rp.ring_state.cpu().tolist()
        assert (st[0], st[1]) == (o.pos, o._size), (what, st[:2], o.pos, o._size)
        assert st[4] == mirror.ctr, what + ": Philox counter advanced by %d, want %d" % (st[4] - st0[4], mirror.ctr - st0[4])
        rows = torch.as_tensor((int(st0[0]) + np.arange(FEEDS)) % mirror.cap, device=rp.device)
        staged = dict(frames=torch.from_numpy(frames), action=torch.from_numpy(action), reward=torch.from_numpy(reward),
                      mask=torch.from_numpy(mask))
        for n, want in ring0.items():
            old = want[rows].clone()
            want[rows] = staged[n].to(want.device, want.dtype)
            assert_equal(getattr(rp, n), want, what + ": ring " + n)
            want[rows] = old                             # the snapshot again: the ring as the async batch read it
        # 3. optimizer bookkeeping
        assert int((opt.grad != 0).sum()) == 0, what + ": gradient arena not re-zeroed"
        if opt.kind == "adam":
            assert int(opt.step_dev.item()) == k + 1, what + ": Adam step"
        for n in ("flat", "s1", "s2"):
            assert bool(torch.isfinite(getattr(opt, n)).all()), what + ": non-finite " + n
        # 1. online operands
        for n, got, want in zip(("w1f", "w2f", "w2d", "w3f", "w3d", "w4p"), lr.net.body._packed.tensors(),
                                packed_ref(lr.net.body, lr.scale)):
            assert_equal(got.cpu(), want, what + ": online packed " + n)
        if p.dist_head:
            fc = dist_fc(lr.net)
            assert_equal(fc._w16, fc.weight.detach().to(torch.bfloat16), what + ": online head _w16")
        # 2. target
        tgt_now, synced = host_sd(lr.tgt), lr.updates % SYNC_EVERY == 0
        assert lr.updates == k + 1
        want_t = host_sd(lr.net) if synced else tgt_prev
        for n, v in tgt_now.items():
            assert_equal(v, want_t[n], "%s: target %s (%s)" % (what, n, "synced" if synced else "unchanged"))
        for n, got, want in zip(("w1f", "w2f", "w2d", "w3f", "w3d", "w4p"), lr.tgt.body._packed.tensors(),
                                packed_ref(lr.tgt.body, lr.scale)):
            assert_equal(got.cpu(), want, what + ": target packed " + n)
        if p.dist_head:
            fc = dist_fc(lr.tgt)
            assert_equal(fc._w16, fc.weight.detach().to(torch.bfloat16), what + ": target head _w16")
        now = {w: [t.data_ptr() for t in n.body._packed.tensors()] for w, n in nets.items()}
        if p.dist_head:
            now.update({w + "_w16": dist_fc(n)._w16.data_ptr() for w, n in nets.items()})
        assert now == ptrs, what + ": a packed operand moved away from the address the graph reads"
        tgt_prev = tgt_now
        # teacher-forced numerics from the snapshot, on the frames as the update read them: a sync replay reads the ring
        # after its own feeds, an async one before them (its batch was drawn after the previous update's feeds)
        if k in NUMERIC:
            teacher_forced(bench, lr, workload, snap, ring0["frames"] if prefetch else rp.frames, bufs, sp, loss, beta, what)
