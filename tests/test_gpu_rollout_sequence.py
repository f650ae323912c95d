"""The captured rollout updates (``GraphedPPOPixelLearner``, ``GraphedA2CLearner``, ``GraphedNStepLearner``) checked step by
step, in the shape of test_gpu_update_sequence.py: every hand-off is checked EXACTLY against a host restatement advanced from
the device's own state, and the numerics TEACHER-FORCED, one update at a time from a snapshot.

A ppo_pixel replay unrolls all E M minibatch updates of a rollout; minibatch j + 1 reads what step j wrote (the packed bf16
body operands, the fp32 head weights, Adam's moments and step counter), its own arena rows (``d_arow[j + 1]``) and the
device learning rate.  None of that survives the replay, so the test makes it observable: before the learner captures, the
tail's ``step`` is wrapped so that the captured graph also copies, right after each step and on the stream that already
orders step j before forward j + 1, the optimizer arenas, the step counter, the clip scratch, the six packed operands and the
minibatch's head outputs and loss gradient into per-minibatch buffers (memcpy nodes; the product's kernel order is unchanged).
An instrumented and a plain replay from the same state agree to the head backward's fp32 atomics: asserted within 1e-6 on
the parameters; measured on one H100 SXM (700 W), SMALL: 2.9e-10 on the parameters, 8.4e-11 on exp_avg, 2.7e-15 on
exp_avg_sq.

PPO, exact, for every minibatch j of one replay (SMALL: E 2 x M 2; the launcher's E 4 x M 4):
1. the packed operands after step j = the host re-pack of ``flat_j`` (1/255 folded into conv1), at unchanged addresses;
2. ``head_mb_j`` = bit for bit an eager bf16 forward of the body and ``fused.ac_head`` on arena rows ``4 d_idx[j]`` (rows
   from the host's ``random_sample``, not from the learner's views) with the operands and head weights of ``flat_{j-1}``;
3. ``stats[j]`` and ``geff_j`` = ``ops.ppo_cat_loss`` re-run on the snapshotted ``head_mb_j`` (deterministic reduction);
4. after every step the gradient arena is zero, Adam's step = the step before the replay + j + 1, the optimizer state is
   finite, and ``flat_j`` = the fused Adam applied to ``flat_{j-1}`` from the device's post-step moments, the device
   learning rate and ``t = step`` in float64, within the first-order fp32 bound of test_gpu_tail_exact.py's Adam contract;
   one case stages half the optimizer's learning rate, so a step at ``opt.lr`` fails;
5. the rollout prep: ``ret`` = ``ops.gae(exact=True)`` on the stored values, ``adv`` = its normalisation (both bitwise),
   ``logp`` = the kernel on the stored rows and float64's log-softmax at the taken action; the actions are the host Philox
   inverse-CDF draws; ``act_out[T]`` = an actor replay on the final states.

PPO, teacher-forced, at the first minibatch, the second (the first to read tail-written operands), the first of epoch 2 and the
last: one float64 minibatch step from snapshot j - 1 (parameters, Adam moments and step) on the device's logp / adv / ret.
Head outputs within test_gpu_q_actor.py's bf16 tolerance, policy / value loss within 2e-2 relative, approx_kl within 5e-3,
the clipped gradient recovered from the moments, (s1_j - beta1 s1_{j-1}) / (1 - beta1), cosine > 0.98 per tensor and > 0.995
overall, its norm and the pre-clip norm within 5e-2, and the step's direction cosine > 0.98.  Measured on one H100 SXM
(700 W), the worst over the picked minibatches: SMALL gradient cosine 0.99999 overall and 0.9982 per tensor, step cosine
0.9988, head outputs within 1.5e-4, pre-clip norm within 3e-4 relative; the launcher's shape 0.999996 / 0.99999 / 0.99997,
1.5e-3 and 4e-3.  The Adam write of check 4 came within 0.998 of its bound (the final rounding, U |p|, is the term that
binds).  n_step_dqn_pixel after the sync: loss within 7e-4 relative, step cosine 0.998, step length within 1.2e-3.

a2c_pixel and n_step_dqn_pixel, after each of 4 consecutive replays: online operands = the re-pack, gradient arena zero,
RMSprop's first step from a zero square average equal to lr |g| / (sqrt(sq) + eps) with g^2 = sq / (1 - alpha), later square
averages finite, non-negative and changed wherever the step is non-zero; arena slots 0..T-1 = the stacks the actor uploaded,
slot T = the final states, the padding row untouched.  a2c: the actions = the host Philox draws at counters c0 + t N + n, the
ticket back at 0, adv / ret = ``ops.gae(exact=True)``, the final rows of geff zero.  n-step: the target's parameters change
only at a sync (then = the online ones), its operands = its re-pack at the captured addresses; the replay after the first
sync is teacher-forced against the float64 restatement of test_nstep_pixel_graph.py.

K1 over the rollout arena: conv1's forward and weight gradient at the launchers' batches (N, T N, (T + 1) N, the minibatch),
contiguous and permuted rows, the last stack next to a padding row of 255s, exactly; the slab schedule each batch reaches is
asserted."""
import ctypes
import math
import os
import sys
import types
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)
from oracle import losses, philox  # noqa: E402
import test_a2c_pixel_graph as a2c_t  # noqa: E402
import test_gpu_conv_exact as conv_t  # noqa: E402
import test_nstep_pixel_graph as nstep_t  # noqa: E402
import test_ppo_pixel_graph as ppo_t  # noqa: E402
from test_gpu_tail_exact import U, f32, packed_ref  # noqa: E402

pytestmark = pytest.mark.gpu

PK = ("w1f", "w2f", "w2d", "w3f", "w3d", "w4p")
REPLAYS = 4
SYNC_EVERY = 12              # n-step: after the warm-up rollout (env steps 1-5), replays 1 and 3 reach a target sync


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


def assert_equal(got, want, what):
    assert got.shape == want.shape and torch.equal(got, want), \
        "%s: %d of %d elements differ" % (what, int((got != want).sum()) if got.shape == want.shape else -1, want.numel())


def cosine(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def offsets(lr):
    """(name, offset, numel, shape) of every parameter of the online network in the optimizer's arena."""
    base = lr.opt.flat.data_ptr()
    return [(n, (p.data_ptr() - base) // 4, p.numel(), p.shape) for n, p in lr.net.named_parameters()]


def body_at(lr, flat):
    """A stand-in for the online body whose weights are the arena snapshot ``flat`` (for ``packed_ref``)."""
    base, body = lr.opt.flat.data_ptr(), lr._body(lr.net)

    def mod(m):
        off = (m.weight.data_ptr() - base) // 4
        return types.SimpleNamespace(weight=flat[off:off + m.weight.numel()].view_as(m.weight))
    return types.SimpleNamespace(**{k: mod(getattr(body, k)) for k in ("conv1", "conv2", "conv3", "fc4")})


def check_operands(lr, body, got, what):
    for n, g, w in zip(PK, got, packed_ref(body, lr.scale)):
        assert_equal(g.cpu(), w, "%s: packed %s" % (what, n))


def stacks(arena, first_row, count, hl=4):
    """The ``count`` frame stacks of the arena from row ``first_row`` on, as [count, hl, 84, 84] uint8 (host)."""
    return arena[first_row:first_row + count * hl].cpu().numpy().reshape(count, hl, 84, 84)


# ------------------------------------------------------------------------------------------------ float64 restatements
def adam_from_moments(p_prev, m1, v1, step, lr, betas, eps):
    """The fused Adam's parameter write (csrc/tail.cu nature_fused_opt_kernel) from its own post-step moments, in float64
    with the float32 hyperparameters, and the first-order bound of the kernel's fp32 sequence on it: adam_bounds of
    test_gpu_tail_exact.py with exact moments (powf within 4 ulp in the bias corrections).  Returns (param, bound)."""
    b1, b2, eps, lr = f32(betas[0]), f32(betas[1]), f32(eps), f32(lr)
    p_prev, m1, v1 = p_prev.double(), m1.double(), v1.double()
    pw1, pw2 = b1 ** step, b2 ** step
    bc1, bc2 = 1 - pw1, 1 - pw2
    ss, bc2s = lr / bc1, math.sqrt(bc2)
    root = torch.sqrt(v1)
    q = root / bc2s
    denom = q + eps
    ratio = m1 / denom
    p = p_prev - ss * ratio
    ebc1, ebc2 = 8 * U * pw1 + U * bc1, 8 * U * pw2 + U * bc2
    ess = ss * (ebc1 / bc1 + U)
    ebc2s = ebc2 / (2 * bc2s) + U * bc2s
    eq = U * root / bc2s + q * (ebc2s / bc2s + U)
    ed = eq + U * denom
    r = ratio.abs()
    er = r * (ed / denom + U)
    return p, ess * r + ss * er + U * ss * r + U * p.abs()


def rmsprop_first_step(p_prev, p_new, sq, lr, alpha, eps, what):
    """RMSprop (not centered) from a zero square average: sq = (1 - alpha) g^2, so |g| = sqrt(sq / (1 - alpha)) and
    |p_new - p_prev| = lr |g| / (sqrt(sq) + eps), within the fp32 rounding of the kernel's sequence (the recovery of g from
    sq's two products, sqrt, add, divide, multiply: 8 U relative) plus the final subtraction's (U |p_new|); the last term
    covers gradients whose square underflows."""
    w, lr, eps = float(np.float32(1) - np.float32(alpha)), f32(lr), f32(eps)
    sq, p_prev, p_new = sq.double(), p_prev.double(), p_new.double()
    assert bool((sq >= 0).all()), what + ": negative square average"
    g = torch.sqrt(sq / w)
    d_ref = lr * g / (torch.sqrt(sq) + eps)
    d_dev = (p_new - p_prev).abs()
    bound = 8 * U * d_ref + U * p_new.abs() + lr * 2.0 ** -60 / eps
    err = (d_dev - d_ref).abs()
    bad = ~(err <= bound)
    assert not bool(bad.any()), "%s: %d of %d steps differ from lr |g| / (sqrt(sq) + eps) (worst err %.3g)" % (
        what, int(bad.sum()), bad.numel(), float(err.max()))
    return float(d_ref.max())


def rmsprop_later_step(p_prev, p_new, sq_prev, sq, lr, alpha, eps, what):
    """A later RMSprop step, whose gradient the zeroed arena no longer holds: since sq >= (1 - alpha) g^2, every step is at
    most lr / sqrt(1 - alpha); and the square average changes wherever the step is not zero, except where g^2 = sq_prev
    (then alpha sq_prev + (1 - alpha) g^2 rounds back to sq_prev), where the step must be lr sqrt(sq) / (sqrt(sq) + eps)
    within the rounding of g^2 (about U / (1 - alpha) relative) and of the parameter write (U |p|)."""
    w, lr, eps = float(np.float32(1) - np.float32(alpha)), f32(lr), f32(eps)
    d = (p_new.double() - p_prev.double()).abs()
    top = lr / math.sqrt(w) * (1 + 8 * U) + U * p_new.double().abs()
    assert bool((d <= top).all()), "%s: a step above lr / sqrt(1 - alpha) (%.3g)" % (what, float(d.max()))
    stuck = (d > 0) & (sq == sq_prev)
    s = sq[stuck].double()
    want = lr * torch.sqrt(s) / (torch.sqrt(s) + eps)
    bound = want * (4 * U / w + 8 * U) + 2 * U * p_new[stuck].double().abs()
    err = (d[stuck] - want).abs()
    assert bool((err <= bound).all()), "%s: %d parameters moved with an unchanged square average, steps off by %.3g" % (
        what, int(stuck.sum()), float((err / bound).max()))


# ------------------------------------------------------------------------------------------------ PPO: the instrument
class Instrument:
    """Wraps the learner's ``NatureTail.step`` before capture: after the real step, the graph copies the state each minibatch
    leaves behind into per-minibatch device buffers (``buf[name][j]``).  The copies are captured on the current stream,
    between step j and forward j + 1, which that stream already orders."""

    def __init__(self, lr):
        self.lr = lr
        o, tail = lr.opt, lr.tail()
        pk = tail.packed()
        self.src = dict(flat=o.flat, s1=o.s1, s2=o.s2, grad=o.grad, step=o.step_dev, scratch=o.scratch[:2], head=lr.head_mb,
                        geff=lr.geff, **{n: getattr(pk, n) for n in PK})
        J = lr.n_batches
        self.buf = {k: torch.zeros((J,) + tuple(v.shape), dtype=v.dtype, device=v.device) for k, v in self.src.items()}
        self.calls = 0
        self.inner = tail.step
        tail.step = self

    def __call__(self, *args, **kw):
        self.inner(*args, **kw)
        j = self.calls % self.lr.n_batches
        self.calls += 1
        for k, v in self.src.items():
            self.buf[k][j].copy_(v)

    def remove(self):
        del self.lr.tail().step                            # the class's step again

    def ops(self, j):
        return [self.buf[n][j] for n in PK]


def ppo_agent(rl, monkeypatch, **kw):
    """A ppo_pixel agent whose update graph is captured with the instrument, plus a plain graph of the same update (the
    learner replays the instrumented one).  One step has run (the actor's slot graphs are captured), then the agent is as
    after a rollout."""
    from deeprl_b200.learner import GraphedPPOPixelLearner as L
    real = L.capture
    made = []

    def capture(self, warmup=1):
        made.append(Instrument(self))
        return real(self, warmup)
    monkeypatch.setattr(L, "capture", capture)
    ag = ppo_t._agent(rl, **kw)
    monkeypatch.setattr(L, "capture", real)
    lr, ins = ag._graph[0], made[0]
    ins.remove()
    g_ins = lr.graph
    lr.capture()
    g_plain, lr.graph = lr.graph, g_ins
    ag.step()
    torch.cuda.synchronize()
    return ag, ins, g_plain


def ppo_state(lr):
    o = lr.opt
    return dict(flat=o.flat.clone(), s1=o.s1.clone(), s2=o.s2.clone(), step=int(o.step_dev.item()))


def check_rollout_prep(ag, lr, r, c0, what):
    """Section 5: the graph's rollout prep from the stored actor rows, the actions, and the final states' value."""
    from deeprl_b200 import ops
    c = ag.config
    T, N = lr.T, lr.N
    A = lr.act_out.shape[2] - 1
    v = lr.act_out[:, :, A].contiguous()
    adv_g, ret_g = ops.gae(lr.d_reward, lr.d_mask, v, c.discount, c.gae_tau, c.use_gae, exact=True)
    assert_equal(lr.roll["ret"], ret_g.reshape(-1), what + ": ret")
    a = adv_g.reshape(-1).clone()
    ops.normalize_advantage_(a)
    assert_equal(lr.roll["adv"], a, what + ": normalised adv")
    a64 = adv_g.reshape(-1).double().cpu().numpy()
    np.testing.assert_allclose(lr.roll["adv"].cpu().numpy(), (a64 - a64.mean()) / a64.std(ddof=1), rtol=1e-5, atol=1e-5,
                               err_msg=what + ": adv normalisation")
    eager = ops.ppo_rollout_prep(lr.act_out.view((T + 1) * N, -1), lr.d_action, lr.d_reward, lr.d_mask, c.discount, c.gae_tau,
                                 c.use_gae)
    assert_equal(lr.roll["logp"], eager["logp"], what + ": logp")
    h = lr.act_out[:T].reshape(T * N, -1).double().cpu().numpy()[:, :A]
    lp = h - h.max(1, keepdims=True)
    lp = lp - np.log(np.exp(lp).sum(1, keepdims=True))
    act = lr.d_action.cpu().numpy().reshape(-1)
    np.testing.assert_allclose(lr.roll["logp"].cpu().numpy(), lp[np.arange(T * N), act], rtol=1e-5, atol=1e-5,
                               err_msg=what + ": logp against float64")
    check_draws(lr, r.actions, c0, what)


def check_draws(lr, host_actions, c0, what):
    """``d_action`` row t = the actions the actor replay of env step t downloaded = the inverse CDF of the softmax of the
    logits it stored on Philox u24(seed, c0 + t N + n, 13) (rows off a partial-sum boundary by more than 1e-6); the
    counter advanced by T N and the ticket is back at 0."""
    T, N = lr.T, lr.N
    d = lr.d_action.cpu().numpy()
    assert np.array_equal(d, np.asarray(host_actions).reshape(T, N)), what + ": d_action against the downloads"
    for t in range(T):
        u = philox.u24(lr.seed, np.uint64(c0 + t * N) + np.arange(N, dtype=np.uint64), 13)
        want, gap = philox.categorical_inverse_cdf(u, lr.act_out[t, :, :-1].cpu().numpy())
        keep = gap > 1e-6
        assert np.array_equal(d[t][keep], want[keep]), "%s: Philox draws of env step %d" % (what, t)
    assert int(lr.counter) == c0 + T * N, what + ": Philox counter"
    assert int(lr.ticket) == 0, what + ": ticket"


def eager_head(lr, flat, rows):
    """The body (K1 from the arena at ``rows``) and the actor-critic head with the weights of ``flat``, as the graph's
    minibatch forward runs them (autograd on, same batch)."""
    from deeprl_b200.network import fused, nature_tc
    from deeprl_b200.network.fused import frame_scale
    lr.opt.flat.copy_(flat)
    lr.refresh_packed()
    rf = nature_tc.RingFrames(lr.arena, rows, 0, 84 * 84, 84, lr.hl)
    with frame_scale(lr.scale):
        phi = lr._body(lr.net)(rf)
    out = fused.ac_head(phi.detach(), lr.net.fc_action, lr.net.fc_critic)
    torch.cuda.synchronize()
    return out


def ppo_teacher_forced(ag, lr, ins, prev, j, rows, what):
    """One float64 minibatch step (PPO_agent.py:77-92 with shared_repr, float64 on the GPU) from snapshot j - 1 on the
    device's logp / adv / ret; returns the measured agreement."""
    from test_ppo_pixel_graph import pixel_body
    c, o = ag.config, lr.opt
    dev = o.flat.device
    lr_j = float(lr.d_lr.item())
    sd = {n: prev["flat"][off:off + k].view(shape).double().clone().requires_grad_(True) for n, off, k, shape in offsets(lr)}
    params = list(sd.values())
    adam = torch.optim.Adam(params, lr=lr_j, betas=o.betas, eps=o.eps, foreach=False)
    for (n, off, k, shape), leaf in zip(offsets(lr), params):
        adam.state[leaf] = dict(step=torch.tensor(float(prev["step"])), exp_avg=prev["s1"][off:off + k].view(shape).double().clone(),
                                exp_avg_sq=prev["s2"][off:off + k].view(shape).double().clone())
    idx = torch.as_tensor(rows, device=dev)
    x = lr.arena[(4 * idx).view(-1, 1) + torch.arange(4, device=dev).view(1, -1)].view(-1, 4, 84, 84)
    phi = pixel_body(sd, x)
    logits = F.linear(phi, sd["fc_action.weight"], sd["fc_action.bias"])
    v = F.linear(phi, sd["fc_critic.weight"], sd["fc_critic.bias"])
    dist = torch.distributions.Categorical(logits=logits)
    act = lr.d_action.view(-1)[idx]
    g = lambda t: t[idx].double().unsqueeze(-1)
    pl, vl, kl = losses.ppo_losses(dist.log_prob(act).unsqueeze(-1), dist.entropy().unsqueeze(-1), v, g(lr.roll["logp"]),
                                   g(lr.roll["adv"]), g(lr.roll["ret"]), c.ppo_ratio_clip, c.entropy_weight)
    # the head outputs the loss kernel read
    ref = torch.cat([logits, v], 1).detach()
    got = ins.buf["head"][j].double()
    err = float((got - ref).abs().max())
    assert err <= 3e-2 * max(1.0, float(ref.abs().max())), "%s: head outputs, max |err| %.3g" % (what, err)
    adam.zero_grad()
    (pl + vl).backward()
    norm = float(torch.nn.utils.clip_grad_norm_(params, c.gradient_clip))
    before = [p.detach().clone() for p in params]
    adam.step()
    bad = []
    st = lr.stats[j].double().cpu().numpy()
    for name, d_, o_, rtol, atol in (("policy_loss", st[0], float(pl.detach()), 2e-2, 1e-4),
                                     ("value_loss", st[1], float(vl.detach()), 2e-2, 1e-4),
                                     ("approx_kl", st[2], float(kl.detach()), 0.0, 5e-3)):
        if abs(d_ - o_) > atol + rtol * abs(o_):
            bad.append("%s %.6g, float64 %.6g" % (name, d_, o_))
    b1 = f32(o.betas[0])
    s1_j, s1_p, flat_j = ins.buf["s1"][j].double(), prev["s1"].double(), ins.buf["flat"][j].double()
    g_dev, g_orc, d_dev, d_orc, per = [], [], [], [], {}
    for (n, off, k, shape), p, p0 in zip(offsets(lr), params, before):
        gd = (s1_j[off:off + k] - b1 * s1_p[off:off + k]) / (1 - b1)
        go = p.grad.flatten()
        if float(go.norm()) > 1e-8:
            per[n] = cosine(gd, go)
            if per[n] <= 0.98:
                bad.append("gradient direction of %s: %.5f" % (n, per[n]))
        g_dev.append(gd), g_orc.append(go)
        d_dev.append(flat_j[off:off + k] - prev["flat"][off:off + k].double()), d_orc.append((p.detach() - p0).flatten())
    g_dev, g_orc, d_dev, d_orc = (torch.cat(t) for t in (g_dev, g_orc, d_dev, d_orc))
    m = dict(grad=cosine(g_dev, g_orc), step=cosine(d_dev, d_orc), grad_tensor_min=min(per.values()), head=err,
             clipped_norm=(float(g_dev.norm()), float(g_orc.norm())), norm=(float(ins.buf["scratch"][j][0]), norm))
    if m["grad"] <= 0.995:
        bad.append("gradient direction %.5f" % m["grad"])
    if m["step"] <= 0.98:
        bad.append("step direction %.5f" % m["step"])
    for name, (d_, o_) in (("clipped gradient norm", m["clipped_norm"]), ("pre-clip norm", m["norm"])):
        if abs(d_ - o_) > 5e-2 * o_:
            bad.append("%s %.6g, float64 %.6g" % (name, d_, o_))
    print("%s: teacher-forced %s" % (what, m))
    assert not bad, "%s: %s" % (what, "; ".join(bad))
    return m


PPO_CASES = {"small": (ppo_t.SMALL, 1.0), "small-half-lr": (ppo_t.SMALL, 0.5), "launcher": ({}, 1.0)}


@pytest.mark.parametrize("case", list(PPO_CASES))
def test_ppo_replay_minibatch_by_minibatch(rl, monkeypatch, case):
    shape, lr_factor = PPO_CASES[case]
    ag, ins, _ = ppo_agent(rl, monkeypatch, max_steps=10 ** 7, **shape)
    lr, o = ag._graph[0], ag.flat_opt
    if lr_factor != 1.0:                                   # a staged learning rate that is not the optimizer's
        real = ag.graph_lr
        monkeypatch.setattr(ag, "graph_lr", lambda: lr_factor * real())
    J, M = lr.n_batches, lr.n_batches // lr.epochs
    assert (lr.epochs, M) == ((2, 2) if shape else (4, 4)), (lr.epochs, M)
    rec = ppo_t.Recorder(ag)
    pk = lr.tail().packed()
    ptrs = [t.data_ptr() for t in pk.tensors()]
    prev0 = ppo_state(lr)
    c0 = int(lr.counter)
    r = ppo_t._rollout(ag, rec)
    what = "ppo %s" % case
    d_lr = float(lr.d_lr.item())
    assert d_lr == np.float32(lr_factor * ag.opt.param_groups[0]["lr"]) and (lr_factor == 1.0 or d_lr != np.float32(o.lr))
    assert [t.data_ptr() for t in pk.tensors()] == ptrs, what + ": a packed operand moved"
    assert np.array_equal(lr.d_idx.cpu().numpy(), r.batches), what + ": minibatch rows"
    check_rollout_prep(ag, lr, r, c0, what)
    final = o.flat.clone()
    snaps = [prev0] + [dict(flat=ins.buf["flat"][j], s1=ins.buf["s1"][j], s2=ins.buf["s2"][j],
                            step=int(ins.buf["step"][j].item())) for j in range(J)]
    assert torch.equal(snaps[-1]["flat"], final), what + ": the last snapshot is the replay's result"
    A = lr.act_out.shape[2] - 1
    worst = 0.0
    for j in range(J):
        wj = "%s minibatch %d" % (what, j)
        prev, cur = snaps[j], snaps[j + 1]
        # 4. tail
        assert int((ins.buf["grad"][j] != 0).sum()) == 0, wj + ": gradient arena not re-zeroed"
        assert cur["step"] == prev0["step"] + j + 1, wj + ": Adam step %d" % cur["step"]
        for n in ("flat", "s1", "s2"):
            assert bool(torch.isfinite(cur[n]).all()), wj + ": non-finite " + n
        want, bound = adam_from_moments(prev["flat"], cur["s1"], cur["s2"], cur["step"], d_lr, o.betas, o.eps)
        err = (cur["flat"].double() - want).abs()
        bad = ~(err <= bound)
        assert not bool(bad.any()), "%s: %d parameters off the Adam write from the moments (worst err %.3g, bound there %.3g)" % (
            wj, int(bad.sum()), float(err.max()), float(bound[int(err.argmax())]))
        worst = max(worst, float((err / (bound + 1e-45)).max()))
        # 1. operands
        check_operands(lr, body_at(lr, cur["flat"]), ins.ops(j), wj)
        # 3. loss
        from deeprl_b200 import ops
        res = ops.ppo_cat_loss(ins.buf["head"][j], lr.d_idx[j], lr.d_action, lr.roll["logp"], lr.roll["adv"], lr.roll["ret"],
                               lr.ratio_clip, lr.ew)
        torch.cuda.synchronize()
        assert_equal(lr.stats[j], res["stats"], wj + ": stats")
        assert_equal(ins.buf["geff"][j][:, :A + 1], res["geff"][:, :A + 1], wj + ": geff")
    print("%s: worst Adam error / bound %.3f" % (what, worst))
    # 2. the forward's inputs: operands, head weights and rows of minibatch j are those of flat_{j-1} and 4 d_idx[j]
    for j in range(J):
        rows = torch.as_tensor(4 * r.batches[j], device=o.flat.device)
        got = eager_head(lr, snaps[j]["flat"], rows)
        assert_equal(ins.buf["head"][j], got, "%s minibatch %d: head outputs of the forward" % (what, j))
    # teacher-forced numerics
    picks = sorted({0, 1, M, J - 1})
    for j in picks:
        ppo_teacher_forced(ag, lr, ins, snaps[j], j, r.batches[j], "%s minibatch %d" % (what, j))
    # act_out[T] = an actor replay on the final states with the pre-replay weights
    vT = lr.act_out[lr.T].clone()
    saved = (lr.d_action.clone(), lr.counter.clone(), lr.act_out[0].clone())
    o.flat.copy_(prev0["flat"])
    lr.refresh_packed()
    rec.inner(ag._raw_states, 0)
    torch.cuda.synchronize()
    assert_equal(lr.act_out[0], vT, what + ": final states' value")
    lr.d_action.copy_(saved[0]), lr.counter.copy_(saved[1]), lr.act_out[0].copy_(saved[2])
    o.flat.copy_(final)
    lr.refresh_packed()
    torch.cuda.synchronize()


def test_ppo_instrument_is_neutral(rl, monkeypatch):
    """An instrumented and a plain replay of the same staged rollout from the same state: parameters within 1e-6, moments
    within the fp32 noise the head backward's atomics leave (the replays differ in nothing else)."""
    ag, ins, g_plain = ppo_agent(rl, monkeypatch, max_steps=10 ** 7, **ppo_t.SMALL)
    lr, o = ag._graph[0], ag.flat_opt
    rec = ppo_t.Recorder(ag)
    before = ppo_state(lr)
    ppo_t._rollout(ag, rec)
    inst = ppo_state(lr)
    o.flat.copy_(before["flat"]), o.s1.copy_(before["s1"]), o.s2.copy_(before["s2"]), o.step_dev.fill_(before["step"])
    lr.refresh_packed()
    assert int((o.grad != 0).sum()) == 0
    g_plain.replay()
    torch.cuda.synchronize()
    plain = ppo_state(lr)
    assert plain["step"] == inst["step"]
    d = {n: float((plain[n] - inst[n]).abs().max()) for n in ("flat", "s1", "s2")}
    print("instrumented vs plain replay, max |difference|: %s" % d)
    assert d["flat"] <= 1e-6, d
    assert d["s1"] <= 1e-6 and d["s2"] <= 1e-9, d


# ------------------------------------------------------------------------------------------------ a2c_pixel / n_step_dqn_pixel
def check_rollout_arena(lr, r, what):
    """Slots 0..T-1 hold the stacks the actor replays uploaded, slot T the staged final states; the padding row is zero."""
    T, N, hl = lr.T, lr.N, lr.hl
    for t in range(T + 1):
        got = stacks(lr.arena, t * N * hl, N, hl)
        assert np.array_equal(got, r.states[t].reshape(N, hl, 84, 84)), "%s: arena slot %d" % (what, t)
    assert np.array_equal(lr.h_final.numpy().reshape(N, hl, 84, 84), r.states[T].reshape(N, hl, 84, 84)), what + ": staged"
    assert int(lr.arena[-1].count_nonzero()) == 0, what + ": padding row written"


def check_rmsprop(o, before, k, what):
    """First replay from a zero square average: the step restated from the square average; later replays: the square
    average finite, non-negative and changed wherever the step is not zero."""
    assert not o.centered and o.kind == "rmsprop"
    flat, sq = o.flat, o.s1
    assert bool(torch.isfinite(flat).all()) and bool(torch.isfinite(sq).all()), what + ": non-finite optimizer state"
    assert bool((sq >= 0).all()), what + ": negative square average"
    if k == 0:
        assert int(before["s1"].count_nonzero()) == 0
        rmsprop_first_step(before["flat"], flat, sq, o.lr, o.alpha, o.eps, what)
    else:
        rmsprop_later_step(before["flat"], flat, before["s1"], sq, o.lr, o.alpha, o.eps, what)


def rollout_agent(mod, rl, **kw):
    """An agent of the launcher whose actor graphs are captured (one step), with a clean RMSprop state."""
    ag = mod._agent(rl, max_steps=0, **kw)
    ag.step()
    torch.cuda.synchronize()
    o = ag.optimizer
    o.s1.zero_(), o.s2.zero_()
    return ag


def test_a2c_consecutive_replays(rl):
    from deeprl_b200 import ops
    ag = rollout_agent(a2c_t, rl)
    rec = a2c_t.Recorder(ag)
    lr, o, c = ag._graph[0], ag.optimizer, ag.config
    T, N = lr.T, lr.N
    A = lr.act_out.shape[2] - 1
    pk = lr._body(lr.net)._packed
    ptrs = [t.data_ptr() for t in pk.tensors()]
    for k in range(REPLAYS):
        what = "a2c replay %d" % k
        before = dict(flat=o.flat.clone(), s1=o.s1.clone())
        c0 = int(lr.counter)
        r = a2c_t._rollout(ag, rec)
        check_operands(lr, lr._body(lr.net), pk.tensors(), what)
        assert [t.data_ptr() for t in pk.tensors()] == ptrs, what + ": a packed operand moved"
        assert int((o.grad != 0).sum()) == 0, what + ": gradient arena not re-zeroed"
        check_rmsprop(o, before, k, what)
        check_rollout_arena(lr, r, what)
        check_draws(lr, r.actions, c0, what)
        v = lr.head_out[:, A].view(T + 1, N)
        adv, ret = ops.gae(lr.d_reward, lr.d_mask, v, c.discount, c.gae_tau, c.use_gae, exact=True)
        torch.cuda.synchronize()
        assert_equal(lr.out["adv"], adv.reshape(-1), what + ": adv")
        assert_equal(lr.out["ret"], ret.reshape(-1), what + ": ret")
        assert int(lr.out["geff"][T * N:].count_nonzero()) == 0, what + ": the final rows' gradient"


def test_nstep_consecutive_replays_with_target_sync(rl):
    ag = rollout_agent(nstep_t, rl)
    ag.config.target_network_update_freq = SYNC_EVERY
    rec = nstep_t.Recorder(ag)
    orc = nstep_t.Oracle(ag)
    lr, o = ag._graph[0], ag.optimizer
    N = lr.N
    nets = {"online": lr.net, "target": lr.tgt}
    ptrs = {w: [t.data_ptr() for t in n.body._packed.tensors()] for w, n in nets.items()}
    synced = []
    for k in range(REPLAYS):
        what = "n-step replay %d" % k
        online, target = nstep_t._flat(ag.network), nstep_t._flat(ag.target_network)
        sync = any((ag.total_steps // N + t + 1) % SYNC_EVERY == 0 for t in range(lr.T))
        before = dict(flat=o.flat.clone(), s1=o.s1.clone())
        orc.anchor(ag)
        r = nstep_t._rollout(ag, rec)
        synced.append(sync)
        for w, n in nets.items():
            check_operands(lr, n.body, n.body._packed.tensors(), "%s: %s" % (what, w))
        now = {w: [t.data_ptr() for t in n.body._packed.tensors()] for w, n in nets.items()}
        assert now == ptrs, what + ": a packed operand moved away from the address the graph reads"
        assert torch.equal(nstep_t._flat(ag.target_network), online if sync else target), what + ": target parameters"
        assert int((o.grad != 0).sum()) == 0, what + ": gradient arena not re-zeroed"
        check_rmsprop(o, before, k, what)
        check_rollout_arena(lr, r, what)
        assert np.array_equal(lr.d_action.cpu().numpy(), r.actions), what + ": actions"
        if sync and synced.count(True) == 1:                # teacher-forced: the first replay after a sync
            loss = orc.update(r, sync=True)
            d_dev, d_orc = nstep_t._flat(ag.network) - online, orc.flat() - online
            m = dict(loss=(float(ag.last_loss), loss), step=cosine(d_dev, d_orc), norm=(float(d_dev.norm()), float(d_orc.norm())))
            print("%s: teacher-forced %s" % (what, m))
            assert abs(m["loss"][0] - loss) <= 2e-2 * abs(loss), m
            assert m["step"] > 0.98 and abs(m["norm"][0] - m["norm"][1]) <= 5e-2 * m["norm"][1], m
    assert synced == [False, True, False, True]


# ------------------------------------------------------------------------------------------------ K1 over the rollout arena
def launcher_batches(rl):
    """conv1's batches on the rollout arena, from the launchers' configurations: (what, batch, (T + 1) N stacks)."""
    out = []
    for name, mod in (("a2c_pixel", a2c_t), ("n_step_dqn_pixel", nstep_t)):
        cfg = mod._pixel_config(rl, max_steps=0).config
        T, N = cfg.rollout_length, cfg.num_workers
        out += [(name + " final", N, T, N), (name + " rollout", T * N, T, N)]
        if name == "a2c_pixel":
            out.append((name + " rollout + final", (T + 1) * N, T, N))
    cfg = ppo_t._pixel_config(rl, max_steps=0).config
    T, N = cfg.rollout_length, cfg.num_workers
    out += [("ppo_pixel final", N, T, N), ("ppo_pixel minibatch", cfg.mini_batch_size, T, N)]
    return out


def k1_rows(B, T, N, kind, gen):
    """Arena rows of ``B`` stacks: ``contiguous`` ends with the last stack of the arena (next to the padding row), ``permuted``
    is a random subset of the arena's (T + 1) N stacks that includes the last one."""
    S = (T + 1) * N
    if kind == "contiguous":
        first = S - B
        return 4 * torch.arange(first, S, device="cuda")
    perm = torch.randperm(S, generator=gen, device="cuda")[:B]
    if not bool((perm == S - 1).any()):
        perm[B // 2] = S - 1
    return 4 * perm


@pytest.mark.parametrize("kind", ["contiguous", "permuted"])
def test_k1_on_the_rollout_arena(rl, kind):
    """b2rl_conv1_u8_fwd and b2rl_conv1_u8_wgrad_partials over a rollout arena (ring pixels 0..15, padding row 255) at the
    launchers' batches, against test_gpu_conv_exact.py's fp64 reference built from the arena's own frames."""
    from deeprl_b200 import _lib
    from deeprl_b200.network import nature_tc as tc
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    k = types.SimpleNamespace(rl=rl, lib=_lib, tc=tc, sms=sms)
    cases = launcher_batches(rl)
    assert sorted({B for _, B, _, _ in cases}) == [8, 16, 80, 96, 256], cases
    sched = {B: conv_t.slab_schedule(B * 441, sms) for _, B, _, _ in cases}
    partial = {B: (B * 441) % 128 != 0 for B in sched}
    # what the batches cover: one CTA holding a single tile (small batches), warpgroup 1 with several tiles, a slab ring that
    # wraps, and a partial last tile
    assert sched[8] == (1, 0) and sched[16] == (1, 0), sched
    assert any(wg1 >= 2 for _, wg1 in sched.values()), sched
    assert any(per > conv_t.MAX_STAGES for per, _ in sched.values()), sched
    assert partial[8] and partial[80] and partial[96] and not partial[256], partial
    lib = _lib
    for name, B, T, N in cases:
        what = "%s B=%d %s" % (name, B, kind)
        gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(what.encode()))
        S = (T + 1) * N
        arena = torch.randint(0, 16, (S * 4 + 1, 84 * 84), dtype=torch.uint8, generator=gen, device="cuda")
        arena[-1] = 255                                    # an over-read of the padding row changes the result
        idx = k1_rows(B, T, N, kind, gen)
        rf = tc.RingFrames(arena, idx, 0, 84 * 84, 84, 4)
        x0 = conv_t.ring_grid(arena, idx, 0)
        w1f = conv_t.draw(gen, (32, 256), "int", -1, 1)
        b1 = conv_t.draw(gen, (32,), "int", -20, 20).float()
        v = conv_t.row_conv(x0, w1f.double(), 4, 2, 21) + b1.double()
        conv_t.exact_ok(conv_t.row_conv(x0, w1f.double().abs(), 4, 2, 21) + b1.double().abs(), what)
        ref = conv_t.place(torch.relu(v), 1, (B * 100, 128), conv_t.SENT, 21, 20)
        x1 = conv_t.sentinel((B * 100, 128))
        lib.call("b2rl_conv1_u8_fwd", *rf.args(), lib.ptr(w1f), 32, lib.ptr(x1), x1.stride(0), lib.ptr(b1), 1, 1, 20, lib.stream())
        g1 = conv_t.draw(gen, (B * 441, 32), "int", -1, 1)
        buf = conv_t.nan_partials(k, 32, 256)
        cnt = ctypes.c_int32(0)
        lib.call("b2rl_conv1_u8_wgrad_partials", *rf.args(), lib.ptr(g1), 32, lib.ptr(buf), ctypes.byref(cnt), lib.stream())
        torch.cuda.synchronize()
        conv_t.assert_bf16_equal(x1, ref, what + " forward")
        wref = conv_t.row_wgrad(x0, g1.double(), 4, 2, 21)
        conv_t.exact_ok(conv_t.row_wgrad(x0, g1.double().abs(), 4, 2, 21), what + " wgrad")
        conv_t.check_partials(k, buf, int(cnt.value), wref, what + " wgrad")
