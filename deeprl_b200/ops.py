"""Python face of the fused loss / recurrence kernels in ``libb2rl.so`` (no CPU path).

Two levels:
* ``*_fused`` functions: one launch -> per-sample loss, PER priorities, reduced scalar AND the gradient with
  respect to the network output (what the agents' ``step`` uses: ``out.backward(gradient)``).
* ``torch.autograd.Function`` wrappers that return the reference's per-sample loss tensors so that code written
  against ``agent.compute_loss`` / ``reduce_loss`` (DQN_agent.py:78-99) differentiates through the kernels.
"""
import torch

from . import _lib

_f32 = torch.float32


def _c(x, dtype=None):
    if x is None:
        return None
    if dtype is not None and x.dtype != dtype:
        x = x.to(dtype)
    return x.contiguous()


class _Scratch:
    """Per-device reusable scratch (zero-initialised counters the kernels re-arm themselves).

    Every tensor handed out stays alive for the life of the process, also after a larger request replaced it: a CUDA graph
    captured while it was current keeps using its address, and freeing it would let the caching allocator give that memory
    to another tensor that every replay then overwrites."""
    _store = {}
    _retired = []

    @classmethod
    def get(cls, device, name, numel, dtype):
        key = (str(device), name, dtype)
        t = cls._store.get(key)
        if t is None or t.numel() < numel:
            if t is not None:
                cls._retired.append(t)
            t = torch.zeros(numel, dtype=dtype, device=device)
            cls._store[key] = t
        return t


# ------------------------------------------------------------------------------------------------- DQN
def dqn_loss_fused(q, q_next_target, q_next_online, action, reward, mask, gamma_n, is_prob=None, beta=0.0, eps=0.0,
                   alpha=0.0, want_grad=True, out=None, beta_dev=None):
    """DQN_agent.py:78-99 (+ PER block :120-127 when ``is_prob`` is given).  Returns dict(delta, priority, loss, dq)."""
    q, qt, qo = _c(q, _f32), _c(q_next_target, _f32), _c(q_next_online, _f32)
    B, A = q.shape
    dev = q.device
    o = out if out is not None else {}
    delta = o.get("delta") if "delta" in o else torch.empty(B, dtype=_f32, device=dev)
    prio = (o.get("priority") if "priority" in o else torch.empty(B, dtype=_f32, device=dev)) if is_prob is not None else None
    loss = o.get("loss") if "loss" in o else torch.empty(1, dtype=_f32, device=dev)
    dq = (o.get("dq") if "dq" in o else torch.empty(B, A, dtype=_f32, device=dev)) if want_grad else None
    _lib.call("b2rl_dqn_loss", _lib.ptr(q), _lib.ptr(qt), _lib.ptr(qo), _lib.ptr(_c(action, torch.int64)),
              _lib.ptr(_c(reward, _f32)), _lib.ptr(_c(mask, _f32)), float(gamma_n), B, A, _lib.ptr(_c(is_prob, _f32)),
              float(beta), float(eps), float(alpha), _lib.ptr(delta), _lib.ptr(prio), _lib.ptr(loss), _lib.ptr(dq),
              _lib.ptr(beta_dev), _lib.stream())
    return dict(delta=delta, priority=prio, loss=loss, dq=dq)


def dqn_head_fused(phi, phi_t, phi_o, head, head_t, action, reward, mask, gamma_n, relu_colsum, is_prob=None, beta=0.0,
                   eps=0.0, alpha=0.0, beta_dev=None, want_q=False, two=True):
    """Head forward (online on s, target on s' [, online on s' for double-Q]) + ``dqn_loss_fused`` + head backward in TWO
    launches (``two``: a row kernel + the head backward, csrc/head.cu dqn_head_loss_kernel) or ONE (dqn_head_fused_kernel).  ``head`` / ``head_t`` = (fc_action_or_head, fc_value_or_None) modules of
    the online / target network (VanillaNet / DuelingNet, network_heads.py:11-37); their weight and bias gradients are
    accumulated into ``.grad`` (which must be fp32 contiguous tensors), ``relu_colsum`` [K] receives fc4's bias gradient.
    Returns dict(gphi = dLoss/dphi masked by phi > 0 (bf16), delta, priority, loss, q)."""
    B, K = phi.shape
    fa, fv = head
    ta, tv = head_t
    A = fa.weight.shape[0]
    dev = phi.device
    assert phi.dtype == torch.bfloat16 and phi.is_contiguous() and phi_t.is_contiguous() and (phi_o is None or phi_o.is_contiguous())
    for m in (fa, fv):
        if m is not None:
            assert all(p.grad is not None and p.grad.dtype == _f32 and p.grad.is_contiguous() for p in (m.weight, m.bias))
    gphi = torch.empty_like(phi)
    delta = torch.empty(B, dtype=_f32, device=dev)
    prio = torch.empty(B, dtype=_f32, device=dev) if is_prob is not None else None
    loss = torch.empty(1, dtype=_f32, device=dev)
    q = torch.empty(B, A, dtype=_f32, device=dev) if want_q else None
    scratch = _Scratch.get(dev, "dqn_head_scratch2" if two else "dqn_head_scratch", (B + 3) // 4 + 8, _f32)
    w = lambda m: None if m is None else m.weight.detach()
    b = lambda m: None if m is None else m.bias.detach()
    g = lambda t: None if t is None else t.grad
    extra = (_lib.ptr(_Scratch.get(dev, "dqn_head_geff", B * 33, _f32)),) if two else ()
    _lib.call("b2rl_dqn_head_two" if two else "b2rl_dqn_head_fused", _lib.ptr(phi), _lib.ptr(phi_t), _lib.ptr(phi_o), _lib.ptr(w(fa)), _lib.ptr(b(fa)),
              _lib.ptr(w(fv)), _lib.ptr(b(fv)), _lib.ptr(w(ta)), _lib.ptr(b(ta)), _lib.ptr(w(tv)), _lib.ptr(b(tv)),
              _lib.ptr(_c(action, torch.int64)), _lib.ptr(_c(reward, _f32)), _lib.ptr(_c(mask, _f32)), float(gamma_n), B, K, A,
              _lib.ptr(_c(is_prob, _f32)), float(beta), _lib.ptr(beta_dev), float(eps), float(alpha), _lib.ptr(gphi),
              _lib.ptr(g(fa.weight)), _lib.ptr(g(fa.bias)), _lib.ptr(None if fv is None else g(fv.weight)),
              _lib.ptr(None if fv is None else g(fv.bias)), _lib.ptr(relu_colsum), _lib.ptr(q), _lib.ptr(delta), _lib.ptr(prio),
              _lib.ptr(loss), _lib.ptr(scratch), *extra, _lib.stream())
    return dict(gphi=gphi, delta=delta, priority=prio, loss=loss, q=q)


def nstep_q_loss(q, q_boot, action, reward, mask, discount, out=None):
    """NStepDQN_agent.py:56-63 in one launch (``b2rl_nstep_q_loss``): ``q`` [T*N, A] of the rollout's states (rows t-major),
    ``q_boot`` [N, A] of the final states (target network), ``action`` / ``reward`` / ``mask`` [T*N] or [T, N].  Returns
    dict(ret, delta [T*N], loss [1], gq [T*N, A] = dloss/dq).  ``out``: a dict of preallocated outputs to write instead
    (persistent buffers of a captured graph)."""
    q, qb = _c(q, _f32), _c(q_boot, _f32)
    rows, A = q.shape
    N = qb.shape[0]
    if rows % N or qb.shape[1] != A:
        raise _lib.B2RLError("nstep_q_loss: q has %d rows of %d actions, q_boot %s" % (rows, A, tuple(qb.shape)))
    dev = q.device
    o = out if out is not None else {}
    e = lambda k, *shape: o[k] if k in o else torch.empty(shape, dtype=_f32, device=dev)
    r = dict(ret=e("ret", rows), delta=e("delta", rows), loss=e("loss", 1), gq=e("gq", rows, A))
    ctas = int(_lib.lib().b2rl_nstep_q_loss_ctas(N))
    partial = _Scratch.get(dev, "nstep_q_partial", max(ctas, 1), _f32)
    counter = _Scratch.get(dev, "nstep_q_counter", 1, torch.int32)
    _lib.call("b2rl_nstep_q_loss", _lib.ptr(q), _lib.ptr(qb), _lib.ptr(_c(action, torch.int64)), _lib.ptr(_c(reward, _f32)),
              _lib.ptr(_c(mask, _f32)), float(discount), rows // N, N, A, _lib.ptr(r["ret"]), _lib.ptr(r["delta"]),
              _lib.ptr(r["loss"]), _lib.ptr(r["gq"]), _lib.ptr(partial), _lib.ptr(counter), _lib.stream())
    return r


AC_GEFF_LD = 33                              # row stride of the head backward's effective gradients (csrc/head.cu HEAD_MAX_OUT + 1)


def a2c_rollout_loss(head, action, reward, mask, discount, gae_tau, use_gae, entropy_weight, value_loss_weight, out=None):
    """A2C_agent.py:43-62 in one launch (``b2rl_a2c_rollout_loss``): ``head`` [(T+1)*N, A+1] = (logits, v) of the rollout's
    states and, in rows T*N.., the final states (rows t-major); ``action`` int64 / ``reward`` / ``mask`` [T*N] or [T, N].
    Returns dict(adv, ret [T*N] (the bits of ``gae(exact=True)``), loss [1], geff [(T+1)*N, 33] = dloss / d(head outputs) in
    columns 0..A, the final rows zero).  ``out``: a dict of preallocated outputs to write instead (persistent buffers of a
    captured graph)."""
    head = _c(head, _f32)
    T, N = reward.shape[0], reward.numel() // reward.shape[0]
    A = head.shape[1] - 1
    if head.shape[0] != (T + 1) * N or reward.numel() != T * N:
        raise _lib.B2RLError("a2c_rollout_loss: head has %d rows, reward %s" % (head.shape[0], tuple(reward.shape)))
    dev = head.device
    o = out if out is not None else {}
    e = lambda k, *shape: o[k] if k in o else torch.empty(shape, dtype=_f32, device=dev)
    r = dict(adv=e("adv", T * N), ret=e("ret", T * N), loss=e("loss", 1))
    # (the kernel writes geff's columns 0..A; the rest stay zero)
    r["geff"] = o["geff"] if "geff" in o else torch.zeros(((T + 1) * N, AC_GEFF_LD), dtype=_f32, device=dev)
    ctas = int(_lib.lib().b2rl_a2c_rollout_loss_ctas(N))
    partial = _Scratch.get(dev, "a2c_rollout_partial", max(3 * ctas, 1), _f32)
    counter = _Scratch.get(dev, "a2c_rollout_counter", 1, torch.int32)
    _lib.call("b2rl_a2c_rollout_loss", _lib.ptr(head), _lib.ptr(_c(action, torch.int64)), _lib.ptr(_c(reward, _f32)),
              _lib.ptr(_c(mask, _f32)), float(discount), float(gae_tau), int(bool(use_gae)), float(entropy_weight),
              float(value_loss_weight), T, N, A, _lib.ptr(r["adv"]), _lib.ptr(r["ret"]), _lib.ptr(r["loss"]),
              _lib.ptr(r["geff"]), _lib.ptr(partial), _lib.ptr(counter), _lib.stream())
    return r


def ppo_rollout_prep(head, action, reward, mask, discount, gae_tau, use_gae, out=None):
    """PPO_agent.py:44-61 (shared_repr) from the actor's stored head outputs in one launch (``b2rl_ppo_rollout_prep``):
    ``head`` [(T+1)*N, A+1] = (logits, v) of the rollout's states and, in rows T*N.., the final states (rows t-major);
    ``action`` int64 / ``reward`` / ``mask`` [T*N] or [T, N].  Returns dict(logp = log pi(action) [T*N], adv, ret [T*N] (the
    bits of ``gae(exact=True)``, adv not yet normalised)).  ``out``: preallocated outputs to write instead."""
    head = _c(head, _f32)
    T, N = reward.shape[0], reward.numel() // reward.shape[0]
    A = head.shape[1] - 1
    if head.shape[0] != (T + 1) * N or reward.numel() != T * N:
        raise _lib.B2RLError("ppo_rollout_prep: head has %d rows, reward %s" % (head.shape[0], tuple(reward.shape)))
    o = out if out is not None else {}
    r = {k: o[k] if k in o else torch.empty(T * N, dtype=_f32, device=head.device) for k in ("logp", "adv", "ret")}
    _lib.call("b2rl_ppo_rollout_prep", _lib.ptr(head), _lib.ptr(_c(action, torch.int64)), _lib.ptr(_c(reward, _f32)),
              _lib.ptr(_c(mask, _f32)), float(discount), float(gae_tau), int(bool(use_gae)), T, N, A, _lib.ptr(r["logp"]),
              _lib.ptr(r["adv"]), _lib.ptr(r["ret"]), _lib.stream())
    return r


def ppo_cat_loss(head, idx, action, old_logp, adv, ret, clip, entropy_weight, geff=None, stats=None):
    """PPO_agent.py:77-92 (shared_repr) for one minibatch of a categorical actor-critic head in one launch
    (``b2rl_ppo_cat_loss``): ``head`` [B, A+1] = (logits, v) of the minibatch, ``idx`` int64 [B] its rows of the rollout
    arrays ``action`` / ``old_logp`` / ``adv`` / ``ret``.  Returns dict(geff [B, 33] = d(policy_loss + value_loss) /
    d(head outputs) in columns 0..A, stats [3] = policy_loss, value_loss, approx_kl).  ``geff`` / ``stats``: preallocated
    outputs (persistent buffers of a captured graph)."""
    head = _c(head, _f32)
    B, A = head.shape[0], head.shape[1] - 1
    dev = head.device
    geff = geff if geff is not None else torch.zeros((B, AC_GEFF_LD), dtype=_f32, device=dev)
    stats = stats if stats is not None else torch.empty(3, dtype=_f32, device=dev)
    ctas = int(_lib.lib().b2rl_ppo_cat_loss_ctas(B))
    partial = _Scratch.get(dev, "ppo_cat_partial", max(4 * ctas, 1), _f32)
    counter = _Scratch.get(dev, "ppo_cat_counter", 1, torch.int32)
    _lib.call("b2rl_ppo_cat_loss", _lib.ptr(head), _lib.ptr(_c(idx, torch.int64)), _lib.ptr(_c(action, torch.int64)),
              _lib.ptr(_c(old_logp, _f32)), _lib.ptr(_c(adv, _f32)), _lib.ptr(_c(ret, _f32)), float(clip),
              float(entropy_weight), B, A, _lib.ptr(geff), _lib.ptr(stats), _lib.ptr(partial), _lib.ptr(counter), _lib.stream())
    return dict(geff=geff, stats=stats)


class _DQNDelta(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, q_next_target, q_next_online, action, reward, mask, gamma_n):
        r = dqn_loss_fused(q, q_next_target, q_next_online, action, reward, mask, gamma_n, want_grad=False)
        ctx.save_for_backward(action)
        ctx.shape = q.shape
        return r["delta"]

    @staticmethod
    def backward(ctx, g):
        (action,) = ctx.saved_tensors
        dq = torch.zeros(ctx.shape, dtype=g.dtype, device=g.device)
        dq.scatter_(1, action.long().unsqueeze(1), (-g).unsqueeze(1))       # delta = target - q[a]
        return dq, None, None, None, None, None, None


def dqn_delta(q, q_next_target, q_next_online, action, reward, mask, gamma_n):
    """Per-sample ``q_target - q`` with autograd through ``q`` (what DQNAgent.compute_loss returns)."""
    return _DQNDelta.apply(q, q_next_target, q_next_online, action, reward, mask, gamma_n)


# ------------------------------------------------------------------------------------------------- C51
def c51_loss_fused(log_prob, prob_next_target, prob_next_online, action, reward, mask, gamma_n, v_min, v_max,
                   is_prob=None, beta=0.0, eps=0.0, alpha=0.0, want_grad=True, want_target=False, beta_dev=None):
    """CategoricalDQN_agent.py:60-89.  Returns dict(kl, priority, loss, dlogp, target_prob)."""
    lp, pt, po = _c(log_prob, _f32), _c(prob_next_target, _f32), _c(prob_next_online, _f32)
    B, A, N = lp.shape
    dev = lp.device
    kl = torch.empty(B, dtype=_f32, device=dev)
    prio = torch.empty(B, dtype=_f32, device=dev) if is_prob is not None else None
    loss = torch.empty(1, dtype=_f32, device=dev)
    dlogp = torch.empty(B, A, N, dtype=_f32, device=dev) if want_grad else None
    tp = torch.empty(B, N, dtype=_f32, device=dev) if want_target else None
    counter = _Scratch.get(dev, "c51_counter", 1, torch.int32)
    _lib.call("b2rl_c51_loss", _lib.ptr(lp), _lib.ptr(pt), _lib.ptr(po), _lib.ptr(_c(action, torch.int64)),
              _lib.ptr(_c(reward, _f32)), _lib.ptr(_c(mask, _f32)), float(gamma_n), float(v_min), float(v_max), B, A, N,
              _lib.ptr(_c(is_prob, _f32)), float(beta), float(eps), float(alpha), _lib.ptr(kl), _lib.ptr(prio),
              _lib.ptr(loss), _lib.ptr(dlogp), _lib.ptr(tp), _lib.ptr(counter), _lib.ptr(beta_dev), _lib.stream())
    return dict(kl=kl, priority=prio, loss=loss, dlogp=dlogp, target_prob=tp)


class _C51KL(torch.autograd.Function):
    @staticmethod
    def forward(ctx, log_prob, prob_next_target, prob_next_online, action, reward, mask, gamma_n, v_min, v_max):
        r = c51_loss_fused(log_prob, prob_next_target, prob_next_online, action, reward, mask, gamma_n, v_min, v_max,
                           want_grad=False, want_target=True)
        ctx.save_for_backward(action, r["target_prob"])
        ctx.shape = log_prob.shape
        return r["kl"]

    @staticmethod
    def backward(ctx, g):
        action, tp = ctx.saved_tensors
        B, A, N = ctx.shape
        d = torch.zeros(ctx.shape, dtype=g.dtype, device=g.device)
        d[torch.arange(B, device=g.device), action.long()] = -(g.unsqueeze(1) * tp)     # KL = sum m log(m+eps) - m logp
        return d, None, None, None, None, None, None, None, None


def c51_kl(log_prob, prob_next_target, prob_next_online, action, reward, mask, gamma_n, v_min, v_max):
    return _C51KL.apply(log_prob, prob_next_target, prob_next_online, action, reward, mask, gamma_n, v_min, v_max)


# ------------------------------------------------------------------------------------------------- QR-DQN
def qr_loss_fused(quantile, quantile_next, action, reward, mask, gamma_n, kappa=1.0, want_grad=True, grad_weight=None,
                  grad_only=False):
    """QuantileRegressionDQN_agent.py:55-77.  Returns dict(vec [N], loss, dquant)."""
    qv, qn = _c(quantile, _f32), _c(quantile_next, _f32)
    B, A, N = qv.shape
    dev = qv.device
    vec = None if grad_only else torch.empty(N, dtype=_f32, device=dev)
    loss = None if grad_only else torch.empty(1, dtype=_f32, device=dev)
    dq = torch.empty(B, A, N, dtype=_f32, device=dev) if want_grad else None
    partial = None if grad_only else _Scratch.get(dev, "qr_partial", B * N, _f32)
    counter = None if grad_only else _Scratch.get(dev, "qr_counter", 1, torch.int32)
    _lib.call("b2rl_qr_loss", _lib.ptr(qv), _lib.ptr(qn), _lib.ptr(_c(action, torch.int64)), _lib.ptr(_c(reward, _f32)),
              _lib.ptr(_c(mask, _f32)), float(gamma_n), float(kappa), B, A, N, _lib.ptr(vec), _lib.ptr(loss), _lib.ptr(dq),
              _lib.ptr(partial), _lib.ptr(counter), _lib.ptr(_c(grad_weight, _f32)), _lib.stream())
    return dict(vec=vec, loss=loss, dquant=dq)


class _QRVec(torch.autograd.Function):
    @staticmethod
    def forward(ctx, quantile, quantile_next, action, reward, mask, gamma_n, kappa):
        r = qr_loss_fused(quantile, quantile_next, action, reward, mask, gamma_n, kappa, want_grad=False)
        ctx.save_for_backward(quantile, quantile_next, action, reward, mask)
        ctx.gamma_n, ctx.kappa = gamma_n, kappa
        return r["vec"]

    @staticmethod
    def backward(ctx, g):
        quantile, quantile_next, action, reward, mask = ctx.saved_tensors
        r = qr_loss_fused(quantile, quantile_next, action, reward, mask, ctx.gamma_n, ctx.kappa, want_grad=True,
                          grad_weight=g / quantile.shape[0], grad_only=True)
        return r["dquant"], None, None, None, None, None, None


def qr_vector(quantile, quantile_next, action, reward, mask, gamma_n, kappa=1.0):
    return _QRVec.apply(quantile, quantile_next, action, reward, mask, gamma_n, kappa)


# ------------------------------------------------------------------------------------------------- on-policy
def gae(reward, mask, value, discount, tau, use_gae=True, exact=True):
    """A2C_agent.py:43-53 / PPO_agent.py:51-61.  reward, mask [T,N,1]|[T,N]; value [T+1,N,1]|[T+1,N].
    ``exact`` = sequential kernel (bit-identical to the reference loop); else warp segmented scan."""
    shape = reward.shape
    T, N = shape[0], shape[1]
    r, m, v = _c(reward, _f32).view(T, N), _c(mask, _f32).view(T, N), _c(value, _f32).view(T + 1, N)
    adv, ret = torch.empty_like(r), torch.empty_like(r)
    _lib.call("b2rl_gae", _lib.ptr(r), _lib.ptr(m), _lib.ptr(v), float(discount), float(tau), T, N, int(bool(use_gae)),
              0 if exact else 1, _lib.ptr(adv), _lib.ptr(ret), _lib.stream())
    return adv.view(shape), ret.view(shape)


def normalize_advantage_(adv):
    """PPO_agent.py:66, in place."""
    assert adv.is_contiguous() and adv.dtype == _f32
    _lib.call("b2rl_normalize_advantage", _lib.ptr(adv), adv.numel(), _lib.stream())
    return adv


def ppo_loss_fused(log_pi_a, entropy, v, old_log_pi_a, advantage, ret, clip, entropy_weight, want_grad=True):
    """PPO_agent.py:77-86 -> dict(out=[policy_loss, value_loss, approx_kl, _], dlogp, dent, dv)."""
    M = log_pi_a.numel()
    dev = log_pi_a.device
    out = torch.empty(4, dtype=_f32, device=dev)
    g = [torch.empty(M, dtype=_f32, device=dev) if want_grad else None for _ in range(3)]
    _lib.call("b2rl_ppo_loss", _lib.ptr(_c(log_pi_a, _f32)), _lib.ptr(_c(entropy, _f32)), _lib.ptr(_c(v, _f32)),
              _lib.ptr(_c(old_log_pi_a, _f32)), _lib.ptr(_c(advantage, _f32)), _lib.ptr(_c(ret, _f32)), float(clip),
              float(entropy_weight), M, _lib.ptr(out), _lib.ptr(g[0]), _lib.ptr(g[1]), _lib.ptr(g[2]), _lib.stream())
    return dict(out=out, dlogp=g[0], dent=g[1], dv=g[2])


def a2c_loss_fused(log_pi_a, entropy, v, advantage, ret, entropy_weight, value_loss_weight, want_grad=True):
    """A2C_agent.py:55-62 -> dict(out=[objective, policy, value, entropy], dlogp, dent, dv)."""
    M = log_pi_a.numel()
    dev = log_pi_a.device
    out = torch.empty(4, dtype=_f32, device=dev)
    g = [torch.empty(M, dtype=_f32, device=dev) if want_grad else None for _ in range(3)]
    _lib.call("b2rl_a2c_loss", _lib.ptr(_c(log_pi_a, _f32)), _lib.ptr(_c(entropy, _f32)), _lib.ptr(_c(v, _f32)),
              _lib.ptr(_c(advantage, _f32)), _lib.ptr(_c(ret, _f32)), float(entropy_weight), float(value_loss_weight), M,
              _lib.ptr(out), _lib.ptr(g[0]), _lib.ptr(g[1]), _lib.ptr(g[2]), _lib.stream())
    return dict(out=out, dlogp=g[0], dent=g[1], dv=g[2])


# ------------------------------------------------------------------------------------------------- optimizer
class FlatOptimizer:
    """Global-norm clip + RMSprop(centered) / Adam over ONE flat arena holding every parameter
    (DQN_agent.py:132-134).  ``FlatOptimizer.from_torch(opt, params)`` reads lr/alpha/eps/betas off a
    ``torch.optim.RMSprop`` / ``Adam`` instance built by the reference's ``config.optimizer_fn``."""

    def __init__(self, params, kind, lr, alpha=0.99, eps=1e-8, centered=False, betas=(0.9, 0.999), shadow_dtype=None):
        self.params = [p for p in params]
        dev = self.params[0].device
        _lib.require_cuda(dev)
        for p in self.params:
            # a parameter re-pointed into a second arena would leave the first optimizer with a stale copy and send its gradient
            # to the wrong arena (e.g. the shared phi_body of an actor-critic network given to two FlatOptimizers)
            if getattr(p, "_b2rl_flat_owner", None) is not None:
                raise _lib.B2RLError("FlatOptimizer: a parameter already lives in another FlatOptimizer's arena")
        # every parameter starts on a 16-byte boundary of the arena (vector loads in the consumers); the padding
        # elements have zero gradient for ever, so they do not change the global norm or anything else
        offs, n = [], 0
        for p in self.params:
            offs.append(n)
            n += (p.numel() + 3) // 4 * 4
        self.n = n
        pad = n
        self.flat = torch.zeros(pad, dtype=_f32, device=dev)
        self.grad = torch.zeros(pad, dtype=_f32, device=dev)
        self.offsets = offs
        for p, off in zip(self.params, offs):         # re-point every parameter and its .grad into the arenas
            k = p.numel()
            self.flat[off:off + k].copy_(p.detach().reshape(-1))
            p.data = self.flat[off:off + k].view_as(p)
            p.grad = self.grad[off:off + k].view_as(p)
            p._b2rl_flat_owner = id(self)
        self.kind, self.lr, self.alpha, self.eps, self.centered, self.betas = kind, lr, alpha, eps, centered, betas
        self.s1 = torch.zeros(pad, dtype=_f32, device=dev)      # square_avg / exp_avg
        self.s2 = torch.zeros(pad, dtype=_f32, device=dev)      # grad_avg   / exp_avg_sq
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=dev)
        self.scratch = torch.zeros(512, dtype=_f32, device=dev)
        self.shadow = torch.zeros(pad, dtype=torch.bfloat16, device=dev) if shadow_dtype == torch.bfloat16 else None

    @classmethod
    def from_torch(cls, opt, params=None, **kw):
        g = opt.param_groups[0]
        params = list(params) if params is not None else [p for grp in opt.param_groups for p in grp["params"]]
        if isinstance(opt, torch.optim.RMSprop):
            if g["momentum"] != 0 or g["weight_decay"] != 0:
                raise NotImplementedError("RMSprop momentum / weight decay are not on the reference's path")
            return cls(params, "rmsprop", g["lr"], alpha=g["alpha"], eps=g["eps"], centered=g["centered"], **kw)
        if isinstance(opt, torch.optim.Adam):
            if g["weight_decay"] != 0 or g["amsgrad"]:
                raise NotImplementedError("Adam weight decay / amsgrad are not on the reference's path")
            return cls(params, "adam", g["lr"], eps=g["eps"], betas=tuple(g["betas"]), **kw)
        raise NotImplementedError("optimizer %s has no fused kernel" % type(opt).__name__)

    def zero_grad(self):
        self.grad.zero_()

    def step(self, max_norm=0.0, grad_scale=1.0, gate=None, gate_max=0.0):
        """clip_grad_norm_(max_norm) (0 = no clip) then the update; ``grad_scale`` pre-multiplies the gradient
        (1/world_size after an all-reduce sum).  ``gate`` (Adam only): a float32 DEVICE scalar; the step is taken only if
        ``gate <= gate_max`` (PPO's ``if approx_kl <= 1.5 * target_kl`` without a host round trip)."""
        sh = _lib.ptr(self.shadow)
        if gate is not None:
            if self.kind != "adam":
                raise NotImplementedError("gated steps are implemented for Adam (the PPO actor optimizer)")
            _lib.call("b2rl_clip_adam_gated", _lib.ptr(self.flat), _lib.ptr(self.grad), _lib.ptr(self.s1), _lib.ptr(self.s2),
                      self.n, float(max_norm or 0.0), float(self.lr), float(self.betas[0]), float(self.betas[1]),
                      float(self.eps), _lib.ptr(self.step_dev), float(grad_scale), _lib.ptr(self.scratch), sh, _lib.ptr(gate),
                      float(gate_max), _lib.stream())
            return
        if self.kind == "rmsprop":
            _lib.call("b2rl_clip_rmsprop", _lib.ptr(self.flat), _lib.ptr(self.grad), _lib.ptr(self.s1), _lib.ptr(self.s2),
                      self.n, float(max_norm or 0.0), float(self.lr), float(self.alpha), float(self.eps), int(self.centered),
                      float(grad_scale), _lib.ptr(self.scratch), sh, _lib.stream())
        else:
            _lib.call("b2rl_clip_adam", _lib.ptr(self.flat), _lib.ptr(self.grad), _lib.ptr(self.s1), _lib.ptr(self.s2),
                      self.n, float(max_norm or 0.0), float(self.lr), float(self.betas[0]), float(self.betas[1]),
                      float(self.eps), _lib.ptr(self.step_dev), float(grad_scale), _lib.ptr(self.scratch), sh,
                      _lib.stream())

    @property
    def total_norm(self):
        return self.scratch[0]


# ------------------------------------------------------------------------------------------------- wgmma GEMM
def gemm_bf16(a, b, a_major="k", b_major="k", bias=None, relu=False, out_dtype=torch.bfloat16, out=None, splits=1,
              block_n=None, accumulate=False, stream=None):
    """``D[M,N] (+)= A B^T`` on the tensor cores (csrc/gemm.cu: TMA -> wgmma -> register accumulators).

    ``a_major="k"``: ``a`` is [M, K] row-major; ``"mn"``: ``a`` is [K, M] row-major (its transpose is what is
    multiplied, without being materialised).  Same for ``b`` ([N, K] or [K, N]).  ``splits > 1`` or ``accumulate``
    accumulate into a fp32 ``out`` with atomics (``out`` is zeroed first unless ``accumulate``)."""
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and a.dim() == 2 and b.dim() == 2
    a_mn, b_mn = a_major == "mn", b_major == "mn"
    M, K = (a.shape[1], a.shape[0]) if a_mn else a.shape
    N, Kb = (b.shape[1], b.shape[0]) if b_mn else b.shape
    assert K == Kb, "inner dimensions differ"
    assert a.stride(1) == 1 and b.stride(1) == 1
    if block_n is None:
        block_n = 128 if N >= 128 else (64 if (N > 32 or b_mn) else 32)
    atomic = splits > 1 or accumulate
    if atomic:
        out_dtype = torch.float32
    if out is None:
        out = (torch.zeros if atomic else torch.empty)((M, N), dtype=out_dtype, device=a.device)
    elif atomic and not accumulate:
        out.zero_()
    assert out.dtype == out_dtype and out.stride(1) == 1
    mode = 2 if atomic else (0 if out_dtype == torch.bfloat16 else 1)
    _lib.call("b2rl_gemm_bf16", _lib.ptr(a), int(a_mn), a.stride(0), _lib.ptr(b), int(b_mn), b.stride(0), _lib.ptr(out),
              out.stride(0), int(M), int(N), int(K), _lib.ptr(bias), int(relu), mode, int(splits), int(block_n),
              stream if stream is not None else _lib.stream())
    return out


def gemm_splitk_bf16(a, b, bias=None, relu=False, splits=4, block_n=64, out=None):
    """``act(a @ b.T + bias)`` in bf16, ONE launch: K split over the ``splits`` CTAs (1, 2, 4 or 8; 0: the launcher picks the
    size from the shape) of a thread-block cluster per output tile, whose partials are summed in distributed shared memory
    in a fixed order, so every launch gives the same bits (csrc/gemm.cu dense_gemm_kernel).  ``a`` [M, K] and ``b`` [N, K]
    bf16 row-major."""
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and a.dim() == 2 and b.dim() == 2
    assert a.stride(1) == 1 and b.stride(1) == 1 and a.shape[1] == b.shape[1]
    M, K = a.shape
    N = b.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.bfloat16, device=a.device)
    _lib.call("b2rl_gemm_splitk_bf16", _lib.ptr(a), a.stride(0), _lib.ptr(b), b.stride(0), _lib.ptr(out), out.stride(0), int(M),
              int(N), int(K), _lib.ptr(bias), int(relu), int(splits), int(block_n), _lib.stream())
    return out
