"""The loss kernels between the heads and the update tail compared EXACTLY with a float64 reference: csrc/losses.cu
(b2rl_dqn_loss, b2rl_c51_loss with its projection and last-CTA PER reduction, b2rl_qr_loss with its 8-way last-CTA sum,
the custom upstream gradient and the gradient-only call) and csrc/onpolicy.cu (b2rl_gae in both modes,
b2rl_normalize_advantage, b2rl_ppo_loss, b2rl_a2c_loss), plus the self-re-arming counters across launches and graph
replays, and the scratch buffers a captured graph keeps using (ops._Scratch).

Exactness by choice of data: C51 atoms on v = +-8 with N in {17, 33, 65} (delta_z = 1, 1/2, 1/4), rewards -2..2, gamma_n in
{1/2, 1} and next-state probabilities in multiples of 1/64 put projected atoms exactly on atoms and past the v_min / v_max
clamp; QR quantiles are integers in -4..4 with N a power of two (dyadic tau), so u == 0 and |u| == kappa occur; GAE runs on
integers with discount = tau = 1 (1/2 for short rollouts); PPO / A2C on integers with ratios exactly 1 or far outside the
clip interval.  While the magnitudes of a sum's terms, scaled to integers, add up to less than 2**24, fp32 accumulation is
exact in ANY order, so each output has one correct value; every case asserts that premise on its own data.  Where a kernel
rounds on purpose (explicit _rn intrinsics: the float64 atoms rounded once, the projection weights, the targets, 1/B for
ragged B) a float32 emulation in the kernel's order is bit-exact.  logf, expf, powf and sums of rounded terms are held to
first-order bounds derived from the data (CUDA Math API ulp table: logf 1 ulp, expf 2 ulp, powf 4 ulp).

Outputs start as NaN; the rows of the actions not taken in dlogp / dquant / dq must come back exactly 0.  The CPU tests at
the end pin the reference against oracle/losses.py and autograd in float64 and the float32 emulation against float64."""
import math

import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu

F64, F32 = torch.float64, torch.float32
EXACT = 2.0 ** 24           # sum |terms| (scaled to integers) below this: fp32 accumulation is exact in any order
U = 2.0 ** -24              # unit roundoff of fp32
ULP_LOGF, ULP_EXPF, ULP_POWF = 1, 2, 4   # CUDA Math API, single-precision maximum ulp errors
EPS_PER, EPS_KL = 0.01, 1e-5


def f32(x):
    return torch.tensor(x, dtype=F32)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def ints(g, shape, lo, hi, dtype=F32):
    return torch.randint(lo, hi + 1, shape, generator=g).to(dtype)


def dev(t):
    return None if t is None else t.cuda()


def nan_like(shape):
    return torch.full(shape, float("nan"), dtype=F32, device="cuda")


def grid(x):
    """The smallest power of two 2**s such that every element of x is a multiple of 2**-s (x dyadic)."""
    y, s = x.to(F64), 1.0
    while not torch.equal(y * s, (y * s).round()):
        s *= 2.0
        assert s < 2.0 ** 60, "not a dyadic rational"
    return s


def assert_exact_premise(terms, what):
    """Every term is a multiple of 1/grid and the magnitudes of each sum's terms (a row of a 2-D ``terms``: one sum per
    row) add up to less than 2**24 / grid."""
    t = terms.to(F64)
    t = t.reshape(1, -1) if t.dim() < 2 else t
    worst = float(t.abs().sum(-1).max()) * grid(t)
    assert worst < EXACT, "%s: sum |terms| * grid = %g is not below 2**24, fp32 accumulation could round" % (what, worst)


def assert_within(got, ref, bound, what):
    got, ref = got.to(F64).cpu(), ref.to(F64).cpu()
    bound = torch.as_tensor(bound, dtype=F64).cpu()
    assert not bool(got.isnan().any()), "%s: NaN left (a store is missing)" % what
    err = (got - ref).abs()
    bad = err > bound
    assert not bool(bad.any()), "%s: %d of %d elements beyond the bound (worst err %.3g, its bound %.3g)" % (
        what, int(bad.sum()), bad.numel(), float(err.max()), float(bound.expand_as(err).reshape(-1)[int(err.argmax())]))


def assert_equal(got, ref, what):
    got = got.cpu()
    assert not bool(got.isnan().any()), "%s: NaN left (a store is missing)" % what
    diff = got.to(F64) != ref.to(F64).cpu()
    assert not bool(diff.any()), "%s: %d of %d elements differ (first at %s: %r vs %r)" % (
        what, int(diff.sum()), diff.numel(), tuple(int(i) for i in diff.nonzero()[0]),
        float(got.reshape(-1)[int(diff.reshape(-1).nonzero()[0])]), float(ref.reshape(-1)[int(diff.reshape(-1).nonzero()[0])]))


def rl_lib():
    from deeprl_b200 import _lib
    return _lib


@pytest.fixture
def rl():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import deeprl_b200 as rl
    rl.select_device(0)
    return rl


# ================================================================================================= PER importance weights
def pow_like_torch32(x, e):
    """pow_like_torch of csrc/losses.cu in float32 (the exponents at::pow special-cases); None for a general exponent."""
    if e == 0.5:
        return x.sqrt()
    if e == 1.0:
        return x.clone()
    if e == 2.0:
        return x * x
    if e == -0.5:
        return f32(1.0) / x.sqrt()
    if e == -1.0:
        return f32(1.0) / x
    return None


def per_base32(prob, B):
    """(P * B + 1e-6) in float32, the kernel's two roundings."""
    return prob.float() * f32(float(B)) + f32(1e-6)


def per_weights(prob, B, beta):
    """(w32 or None, w64, relative bound of the device weight).  beta = 1 (1 / x, two correctly rounded operations): the
    float32 emulation is bit-exact.  beta = 1/2: 1.0f / sqrtf(x) on the device is within 1 ulp of the emulation's
    correctly rounded sqrt and division, not bit-equal to it (the compiler's reciprocal square root), so it is bounded like
    a general beta: the raw weight and the maximum within n ulp, one rounding of the division."""
    x = per_base32(prob, B)
    w64 = x.to(F64) ** -beta
    w64 = w64 / w64.max()
    e = -float(np.float32(beta))
    if e == -1.0:
        raw = pow_like_torch32(x, e)
        return raw / raw.max(), w64, 4 * U
    n = 2 if e == -0.5 else ULP_POWF
    return None, w64, (4 * n + 1) * U


def assert_priority(got, x, alpha):
    """(|x| + eps) ** alpha: exact for alpha = 1; sqrtf within 1 ulp of the correctly rounded float32 square root."""
    p = pow_like_torch32(x.float().abs() + f32(EPS_PER), alpha)
    assert p is not None, "alpha in {0.5, 1}"
    if alpha == 1.0:
        assert_equal(got, p, "priority")
    else:
        assert_within(got, p, 2 * U * p.to(F64).abs(), "priority (1 ulp)")


# ================================================================================================= DQN
def dqn_emulate(q, qt, qo, action, reward, mask, gamma_n):
    """float32 target and delta in the kernel's order: target = r + (gamma_n * q_next) * mask, delta = target - q[a];
    q_next = max_a qt, or qt at the FIRST maximum of qo (double-Q)."""
    qnext = qt.gather(1, torch.argmax(qo, 1, keepdim=True))[:, 0] if qo is not None else qt.max(1).values
    target = reward + (f32(gamma_n) * qnext) * mask
    return target - q.gather(1, action[:, None])[:, 0]


def run_dqn(c, beta_dev=None, beta=None):
    L = rl_lib()
    B, A = c.q.shape
    o = {k: nan_like(s) for k, s in (("delta", (B,)), ("prio", (B,)), ("loss", (1,)), ("dq", (B, A)))}
    per = c.is_prob is not None
    d = [dev(t) for t in (c.q, c.qt, c.qo, c.action, c.reward, c.mask, c.is_prob)]     # alive until the kernel is done
    L.call("b2rl_dqn_loss", *[L.ptr(t) for t in d[:6]], float(c.gamma_n), B, A, L.ptr(d[6]), float(c.beta if beta is None else beta),
           float(EPS_PER), float(c.alpha), L.ptr(o["delta"]), L.ptr(o["prio"] if per else None), L.ptr(o["loss"]),
           L.ptr(o["dq"]), L.ptr(beta_dev), L.stream())
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


class Case(dict):
    __getattr__ = dict.__getitem__
    __setattr__ = dict.__setitem__


def dqn_case(seed, B, A, double_q, gamma_n, per=False, beta=0.5, alpha=0.5):
    g = _gen(seed)
    c = Case(B=B, A=A, gamma_n=gamma_n, beta=beta, alpha=alpha)
    c.q, c.qt = ints(g, (B, A), -4, 4), ints(g, (B, A), -4, 4)
    c.qo = ints(g, (B, A), -2, 2) if double_q else None
    c.action = torch.randint(0, A, (B,), generator=g)
    c.reward, c.mask = ints(g, (B,), -2, 2), ints(g, (B,), 0, 1)
    c.is_prob = (torch.rand(B, generator=g) + 0.25) / B if per else None
    return c


@gpu
@pytest.mark.parametrize("B", [1, 7, 37, 1024, 1025, 4096])
@pytest.mark.parametrize("double_q", [False, True])
def test_dqn_loss_exact(rl, B, double_q):
    """b2rl_dqn_loss in its single CTA (thread count rounded up to a warp, the strided loop past 1024): delta, the loss
    and dq exact; dq is zero outside the taken action."""
    A = 6
    c = dqn_case(B + int(double_q), B, A, double_q, 0.5 if B % 2 else 1.0)
    o = run_dqn(c)
    delta = dqn_emulate(c.q, c.qt, c.qo, c.action, c.reward, c.mask, c.gamma_n)
    assert_equal(o["delta"], delta, "delta")
    invB = f32(1.0) / f32(float(B))
    terms = (delta * delta) * f32(0.5)
    assert_exact_premise(terms, "loss")
    assert_equal(o["loss"], (terms.to(F64).sum().float() * invB).reshape(1), "loss")
    dq = torch.zeros(B, A)
    dq[torch.arange(B), c.action] = ((-delta) * f32(1.0)) * invB
    assert_equal(o["dq"], dq, "dq")


@gpu
@pytest.mark.parametrize("B", [7, 512, 1025])
@pytest.mark.parametrize("beta,alpha,from_dev", [(0.5, 0.5, False), (1.0, 1.0, False), (0.4, 0.5, True), (0.6, 1.0, False)])
def test_dqn_loss_per(rl, B, beta, alpha, from_dev):
    """PER: priorities exact for alpha = 1 (sqrtf within 1 ulp for alpha = 1/2); importance weights exact for beta = 1,
    within their bound for beta = 1/2 and within powf's bound for a general beta (taken from beta_dev when given: the scalar argument is then wrong on purpose); loss and dq follow the
    weights in the kernel's order."""
    A = 5
    c = dqn_case(100 + B, B, A, True, 1.0, per=True, beta=beta, alpha=alpha)
    bd = torch.tensor([beta], dtype=F32, device="cuda") if from_dev else None
    o = run_dqn(c, beta_dev=bd, beta=7.0 if from_dev else beta)
    delta = dqn_emulate(c.q, c.qt, c.qo, c.action, c.reward, c.mask, c.gamma_n)
    assert_equal(o["delta"], delta, "delta")
    assert_priority(o["prio"], delta, alpha)
    w32, w64, rel = per_weights(c.is_prob, B, beta)
    invB = f32(1.0) / f32(float(B))
    rows = torch.arange(B)
    dq_taken = o["dq"][rows, c.action]
    off = o["dq"].clone()
    off[rows, c.action] = 0.0
    assert_equal(off, torch.zeros(B, A), "dq outside the taken action")
    if w32 is not None:
        wl = delta * w32
        assert_equal(dq_taken, ((-wl) * w32) * invB, "dq")
        terms = (wl * wl) * f32(0.5)
        loss_ref, bound = terms.to(F64).sum() / B, (B + 2) * U * terms.to(F64).abs().sum() / B
    else:
        d64 = delta.to(F64)
        assert_within(dq_taken, -d64 * w64 * w64 / B, (2 * rel + 4 * U) * (d64 * w64 * w64).abs() / B, "dq")
        loss_ref = (0.5 * (d64 * w64) ** 2).sum() / B
        bound = (2 * rel + (B + 4) * U) * (0.5 * (d64 * w64) ** 2).sum() / B
    assert_within(o["loss"], loss_ref.reshape(1), bound, "loss")


# ================================================================================================= C51
def c51_atoms(vmin, vmax, N):
    """np.linspace in float64 rounded once to float32 (the kernel: k * step + start in double, the last atom v_max)."""
    return torch.tensor(np.linspace(vmin, vmax, N), dtype=F32)


def c51_emulate(lp, pt, po, action, reward, mask, gamma_n, vmin, vmax):
    """float32 in the kernel's order: expected values summed sequentially over atoms, the FIRST maximum, tz = clamp(r +
    (gamma_n * m) z), m_j = sum_k clamp(1 - |tz_k - z_j| / delta_z, 0, 1) p_k sequentially over k.  Returns (target_prob,
    a_star, z)."""
    B, A, N = pt.shape
    z = c51_atoms(vmin, vmax, N)
    dz = f32((float(vmax) - float(vmin)) / (N - 1))
    sel = po if po is not None else pt
    qa = torch.zeros(B, A, dtype=F32)
    for k in range(N):
        qa = qa + sel[:, :, k] * z[k]
    a_star = torch.argmax(qa, 1)
    pn = pt[torch.arange(B), a_star]
    gm = f32(gamma_n) * mask
    tz = torch.clamp(reward[:, None] + gm[:, None] * z[None], f32(vmin), f32(vmax))
    m = torch.zeros(B, N, dtype=F32)
    for k in range(N):
        c = torch.clamp(f32(1.0) - (tz[:, k:k + 1] - z[None]).abs() / dz, f32(0.0), f32(1.0))
        m = m + c * pn[:, k:k + 1]
    return m, a_star, z


def c51_ref64(lp, pt, po, action, reward, mask, gamma_n, vmin, vmax):
    """float64 reference (CategoricalDQN_agent.py:60-86) on the kernel's float32 atoms: (target_prob, kl)."""
    B, A, N = pt.shape
    z = c51_atoms(vmin, vmax, N).to(F64)
    dz = (float(vmax) - float(vmin)) / (N - 1)
    sel = (po if po is not None else pt).to(F64)
    a_star = torch.argmax((sel * z).sum(-1), 1)
    rows = torch.arange(B)
    pn = pt.to(F64)[rows, a_star]
    tz = (reward.to(F64)[:, None] + gamma_n * mask.to(F64)[:, None] * z[None]).clamp(vmin, vmax)
    w = (1 - (tz[:, None, :] - z[None, :, None]).abs() / dz).clamp(0, 1)           # [B, j, k]
    m = (w * pn[:, None, :]).sum(-1)
    lpa = lp.to(F64)[rows, action]
    kl = (m * torch.log(m + float(np.float32(EPS_KL))) - m * lpa).sum(-1)
    return m, kl


def kl_bound(m, lpa, N):
    """First order, per sample: m + 1e-5 rounds (U absolute in the log), logf 1 ulp (2U relative), two products and the
    difference round once each, and the sum of N such terms in any order adds N - 1 roundings of sum |terms|."""
    m, lpa = m.to(F64), lpa.to(F64)
    L = torch.log(m + float(np.float32(EPS_KL)))
    t = (m * L - m * lpa).abs()
    per = m * (U + 2 * ULP_LOGF * U * L.abs()) + U * (m * L).abs() + U * (m * lpa).abs() + U * t
    return per.sum(-1) + (N - 1) * U * t.sum(-1)


def c51_case(seed, B, A, N, vmin, vmax, gamma_n, double_q, exact=True, per=False):
    g = _gen(seed)
    c = Case(B=B, A=A, N=N, vmin=vmin, vmax=vmax, gamma_n=gamma_n)
    if exact:                                          # next-state distributions in multiples of 1/64
        def dist(n):
            cnt = torch.zeros(n, A, N)
            idx = torch.randint(0, N, (n, A, 64), generator=g)
            cnt.scatter_add_(2, idx, torch.ones(n, A, 64))
            return cnt / 64.0
        c.pt = dist(B)
        c.po = dist(B) if double_q else None
        c.reward = ints(g, (B,), -2, 2)
    else:
        c.pt = torch.softmax(torch.randn(B, A, N, generator=g) * 2, -1)
        c.po = torch.softmax(torch.randn(B, A, N, generator=g) * 2, -1) if double_q else None
        c.reward = torch.randn(B, generator=g)
    c.lp = torch.log_softmax(torch.randn(B, A, N, generator=g), -1)
    c.action = torch.randint(0, A, (B,), generator=g)
    c.mask = ints(g, (B,), 0, 1)
    c.is_prob = (torch.rand(B, generator=g) + 0.25) / B if per else None
    return c


def run_c51(c, counter=None, beta=0.0, alpha=0.5, beta_dev=None, beta_arg=None):
    L = rl_lib()
    B, A, N = c.lp.shape
    per = c.is_prob is not None
    o = dict(kl=nan_like((B,)), prio=nan_like((B,)), loss=nan_like((1,)), dlogp=nan_like((B, A, N)), tp=nan_like((B, N)))
    counter = counter if counter is not None else torch.zeros(1, dtype=torch.int32, device="cuda")
    d = [dev(t) for t in (c.lp, c.pt, c.po, c.action, c.reward, c.mask, c.is_prob)]      # alive until the kernel is done
    L.call("b2rl_c51_loss", *[L.ptr(t) for t in d[:6]], float(c.gamma_n), float(c.vmin), float(c.vmax), B, A, N, L.ptr(d[6]),
           float(beta if beta_arg is None else beta_arg), float(EPS_PER), float(alpha), L.ptr(o["kl"]),
           L.ptr(o["prio"] if per else None), L.ptr(o["loss"]), L.ptr(o["dlogp"]), L.ptr(o["tp"]), L.ptr(counter),
           L.ptr(beta_dev), L.stream())
    torch.cuda.synchronize()
    out = {k: v.cpu() for k, v in o.items()}
    out["counter"] = int(counter.cpu()[0])
    return out


def check_c51(c, o, beta=None, alpha=0.5):
    """Every output of one b2rl_c51_loss call: target_prob and dlogp bit-exact with the float32 emulation, KL within its
    bound of float64, priorities exact from the device KL, the loss within the bound of the weighted mean."""
    B, A, N = c.lp.shape
    m32, a_star, z = c51_emulate(c.lp, c.pt, c.po, c.action, c.reward, c.mask, c.gamma_n, c.vmin, c.vmax)
    assert_equal(o["tp"], m32, "target_prob")
    rows = torch.arange(B)
    lpa = c.lp[rows, c.action]
    m64, kl64 = c51_ref64(c.lp, c.pt, c.po, c.action, c.reward, c.mask, c.gamma_n, c.vmin, c.vmax)
    # the KL of the device's own (exact-emulated) target distribution
    L = torch.log(m32.to(F64) + float(np.float32(EPS_KL)))
    kl_dev_ref = (m32.to(F64) * L - m32.to(F64) * lpa.to(F64)).sum(-1)
    assert_within(o["kl"], kl_dev_ref, kl_bound(m32, lpa, N), "kl")
    if c.is_prob is not None:
        w32, w64, rel = per_weights(c.is_prob, B, beta)
        assert_priority(o["prio"], o["kl"], alpha)
    else:
        w32, w64, rel = torch.ones(B, dtype=F32), torch.ones(B, dtype=F64), 0.0
    dl = torch.zeros(B, A, N)
    if w32 is not None:
        scale = w32 / f32(float(B))
        dl[rows, c.action] = -(m32 * scale[:, None])
        assert_equal(o["dlogp"], dl, "dlogp")
    else:
        dl64 = torch.zeros(B, A, N, dtype=F64)
        dl64[rows, c.action] = -(m32.to(F64) * w64[:, None] / B)
        assert_within(o["dlogp"], dl64, (rel + 2 * U) * dl64.abs(), "dlogp")
    kd = o["kl"].to(F64)
    t = (kd * w64).abs()
    assert_within(o["loss"], ((kd * w64).sum() / B).reshape(1), (rel * t.sum() + (B + 2) * U * t.sum()) / B, "loss")
    assert o["counter"] == 0, "the last CTA re-arms the counter"
    return m32, a_star


C51_EXACT = [(B, A, N) for B, A, N in ((1, 4, 17), (7, 18, 33), (9, 4, 65), (37, 6, 17), (512, 18, 33), (1025, 4, 65),
                                       (2048, 6, 17))]


@gpu
@pytest.mark.parametrize("B,A,N", C51_EXACT)
@pytest.mark.parametrize("double_q", [False, True])
def test_c51_exact(rl, B, A, N, double_q):
    """C51 on v = +-8: projected atoms on atoms, between atoms and beyond the clamp; target_prob equals the float64
    projection exactly, dlogp is exact, rows of the other actions are 0."""
    gamma_n = 0.5 if (B + N) % 2 else 1.0
    c = c51_case(B * 7 + N + int(double_q), B, A, N, -8.0, 8.0, gamma_n, double_q)
    o = run_c51(c)
    m32, _ = check_c51(c, o)
    m64, _ = c51_ref64(c.lp, c.pt, c.po, c.action, c.reward, c.mask, gamma_n, -8.0, 8.0)
    assert torch.equal(m32.to(F64), m64), "premise: the emulation is the float64 projection on this data"
    tz = c.reward[:, None] + gamma_n * c.mask[:, None] * c51_atoms(-8.0, 8.0, N)[None]
    if B >= 37 and gamma_n == 1.0:
        assert bool((tz.abs() > 8).any()), "some projected atoms lie beyond the clamp"


@gpu
@pytest.mark.parametrize("B", [7, 512, 1025])
@pytest.mark.parametrize("beta,alpha,from_dev", [(0.5, 0.5, False), (1.0, 1.0, False), (0.4, 0.5, True), (0.5, 1.0, True)])
@pytest.mark.parametrize("double_q", [False, True])
def test_c51_per(rl, B, beta, alpha, from_dev, double_q):
    """C51 with PER: the weights the per-sample CTA uses for dlogp and those the last CTA re-derives for the loss (a weight
    left out of the last-CTA sum moves the loss far beyond its bound); beta from beta_dev overrides a wrong scalar."""
    c = c51_case(300 + B + int(double_q), B, 6, 33, -8.0, 8.0, 0.5, double_q, per=True)
    c.is_prob = c.is_prob * (1 + 3 * torch.rand(B, generator=_gen(B)))       # weights spread over [~0.3, 1]
    bd = torch.tensor([beta], dtype=F32, device="cuda") if from_dev else None
    o = run_c51(c, beta=beta, alpha=alpha, beta_dev=bd, beta_arg=9.0 if from_dev else None)
    check_c51(c, o, beta=beta, alpha=alpha)
    _, w64, _ = per_weights(c.is_prob, B, beta)
    if B >= 512:
        assert float(w64.min()) < 0.8, "premise: the weights differ enough to matter in the loss"


@gpu
@pytest.mark.parametrize("B,A", [(1, 4), (37, 6), (512, 18)])
def test_c51_production_shape(rl, B, A):
    """N = 51 on v = +-10 (delta_z = 0.4 is not dyadic) with softmax probabilities: bit-exact with the float32 emulation."""
    c = c51_case(500 + B, B, A, 51, -10.0, 10.0, 0.99, True, exact=False)
    check_c51(c, run_c51(c))


# ================================================================================================= QR-DQN
def qr_tau32(N):
    return torch.tensor((2.0 * np.arange(N) + 1.0) / (2.0 * N), dtype=F32)


def qr_ref64(quant, qn, action, reward, mask, gamma_n, kappa, gw=None):
    """float64 reference of QuantileRegressionDQN_agent.py:55-77 on float32 targets: (vec [N], loss, dquant [B, A, N],
    |terms| for the bounds).  T_j = r + (gamma_n m) qn[a*, j] in float32 as the kernel; a* is the first maximum of the
    next-state quantile sums.  dquant of mean_j(vec): -sum_j gw_j hp(u_ji) |tau_i - 1{u_ji < 0}|, gw_j = 1/(B N) unless
    a custom upstream gradient is given."""
    B, A, N = quant.shape
    rows = torch.arange(B)
    a_star = torch.argmax(qn.to(F64).sum(-1), 1)
    T = reward[:, None] + (f32(gamma_n) * mask)[:, None] * qn[rows, a_star]            # float32, as the kernel
    th = quant[rows, action].to(F64)
    tau = qr_tau32(N).to(F64)
    u = T.to(F64)[:, :, None] - th[:, None, :]                                         # [B, j, i]
    wq = (tau[None, None, :] - (u < 0).to(F64)).abs()
    hub = torch.where(u.abs() < kappa, 0.5 * u * u, kappa * (u.abs() - 0.5 * kappa))
    terms = hub * wq
    vec = terms.sum(-1).mean(0)
    hp = u.clamp(-kappa, kappa)
    gwj = (torch.full((N,), 1.0 / (B * N), dtype=F64) if gw is None else gw.to(F64))
    gt = gwj[None, :, None] * hp * wq                                                  # [B, j, i]
    dq = torch.zeros(B, A, N, dtype=F64)
    dq[rows, action] = -gt.sum(1)
    return vec, vec.mean(), dq, terms, gt, a_star


def qr_case(seed, B, A, N, gamma_n, exact=True):
    g = _gen(seed)
    c = Case(B=B, A=A, N=N, gamma_n=gamma_n)
    if exact:
        c.quant, c.qn = ints(g, (B, A, N), -4, 4), ints(g, (B, A, N), -4, 4)
        c.reward = ints(g, (B,), -2, 2)
    else:
        c.quant, c.qn = torch.randn(B, A, N, generator=g), torch.randn(B, A, N, generator=g)
        c.reward = torch.randn(B, generator=g)
    c.action = torch.randint(0, A, (B,), generator=g)
    c.mask = ints(g, (B,), 0, 1)
    return c


def run_qr(c, kappa, counter=None, grad_only=False, gw=None, partial=None):
    L = rl_lib()
    B, A, N = c.quant.shape
    vec, loss, dq = nan_like((N,)), nan_like((1,)), nan_like((B, A, N))
    if partial is None:
        partial = nan_like((B * N,))
    counter = counter if counter is not None else torch.zeros(1, dtype=torch.int32, device="cuda")
    d = [dev(t) for t in (c.quant, c.qn, c.action, c.reward, c.mask, gw)]                 # alive until the kernel is done
    L.call("b2rl_qr_loss", *[L.ptr(t) for t in d[:5]], float(c.gamma_n), float(kappa), B, A, N,
           L.ptr(None if grad_only else vec), L.ptr(None if grad_only else loss), L.ptr(dq),
           L.ptr(None if grad_only else partial), L.ptr(None if grad_only else counter), L.ptr(d[5]), L.stream())
    torch.cuda.synchronize()
    return dict(vec=vec.cpu(), loss=loss.cpu(), dq=dq.cpu(), counter=int(counter.cpu()[0]))


def check_qr(c, o, kappa, exact, gw=None, grad_only=False):
    B, A, N = c.quant.shape
    vec, loss, dq, terms, gt, a_star = qr_ref64(c.quant, c.qn, c.action, c.reward, c.mask, c.gamma_n, kappa, gw)
    rows = torch.arange(B)
    off = o["dq"].clone()
    off[rows, c.action] = 0.0
    assert_equal(off, torch.zeros(B, A, N), "dquant outside the taken action")
    gscale_exact = gw is not None or float(f32(1.0) / (f32(float(B)) * f32(float(N)))) == 1.0 / (B * N)
    if exact and gscale_exact:
        for b in range(0, B, max(1, B // 16)):
            assert_exact_premise(gt[b].t(), "dquant row %d (one sum over j per quantile i)" % b)
        assert_equal(o["dq"], dq, "dquant")
    else:                  # gscale rounds once (ragged B), each term two products, N - 1 roundings of the sum
        assert_within(o["dq"], dq, torch.zeros_like(dq).index_put_((rows, c.action), (N + 3) * U * gt.abs().sum(1)),
                      "dquant")
    if grad_only:
        assert bool(o["vec"].isnan().all() and o["loss"].isnan().all()), "the gradient-only call writes no loss"
        return
    assert o["counter"] == 0, "the last CTA re-arms the counter"
    if exact:
        assert_exact_premise(terms.permute(1, 0, 2).reshape(N, -1), "vec sums (one per target quantile)")
        S = terms.sum(-1).sum(0)                                     # exact
        vec32 = S.float() / f32(float(B))
        assert_equal(o["vec"], vec32, "vec")
        v64 = vec32.to(F64)
        if float(v64.abs().sum()) * grid(v64) < EXACT:               # the sum of the rounded vec is exact too
            assert_equal(o["loss"], (f32(float(v64.sum())) / f32(float(N))).reshape(1), "loss")
        else:
            assert_within(o["loss"], v64.mean().reshape(1), (N + 1) * U * v64.abs().sum() / N, "loss")
    else:
        # per term: u rounds (hp |u| U), huber up to 3 roundings, tau once, the product once; the row sum of N terms and
        # the sum over B partials add N + B roundings; the division by B one more
        tb = terms.abs().sum(-1).sum(0)
        b_vec = (N + B + 8) * U * tb / B
        assert_within(o["vec"], vec, b_vec, "vec")
        assert_within(o["loss"], loss.reshape(1), (b_vec.sum() + (N + 1) * U * vec.abs().sum()) / N, "loss")


QR_EXACT = [(1, 4, 8), (7, 4, 32), (8, 6, 2), (9, 3, 1), (8, 4, 256), (37, 18, 8), (512, 6, 32), (1024, 4, 32),
            (1025, 4, 8), (2048, 4, 8)]


@gpu
@pytest.mark.parametrize("B,A,N", QR_EXACT)
@pytest.mark.parametrize("kappa", [1.0, 2.0])
def test_qr_exact(rl, B, A, N, kappa):
    """Integer quantiles, dyadic tau: u == 0 and |u| == kappa occur; vec exact (the 8-way last-CTA sum and its scalar tail
    for B % 8 != 0), dquant exact for B a power of two, zero outside the taken action."""
    c = qr_case(B * 3 + N + int(kappa), B, A, N, 0.5 if B % 2 else 1.0)
    o = run_qr(c, kappa)
    check_qr(c, o, kappa, True)
    _, _, _, _, _, a_star = qr_ref64(c.quant, c.qn, c.action, c.reward, c.mask, c.gamma_n, kappa)
    T = c.reward[:, None] + (f32(c.gamma_n) * c.mask)[:, None] * c.qn[torch.arange(B), a_star]
    u = T[:, :, None] - c.quant[torch.arange(B), c.action][:, None, :]
    if B * N >= 64:
        assert bool((u == 0).any()) and bool((u.abs() == kappa).any()), "premise: ties at u = 0 and |u| = kappa"


@gpu
@pytest.mark.parametrize("B,N", [(7, 32), (512, 8), (1025, 2)])
def test_qr_grad_weight_and_grad_only(rl, B, N):
    """The autograd backward's launch: a custom upstream gradient gw (dyadic: exact) and no partial / counter, so the
    kernel writes dquant only (vec and loss keep their NaN)."""
    A = 4
    c = qr_case(700 + B, B, A, N, 1.0)
    gw = ints(_gen(B), (N,), -3, 3) / 64.0
    o = run_qr(c, 1.0, grad_only=True, gw=gw)
    check_qr(c, o, 1.0, True, gw=gw, grad_only=True)


@gpu
@pytest.mark.parametrize("B,A", [(1, 4), (37, 6), (512, 18)])
def test_qr_production_shape(rl, B, A):
    """N = 200 on Gaussian data within the first-order bounds; the greedy action is not a near tie (premise)."""
    c = qr_case(800 + B, B, A, 200, 0.99, exact=False)
    s = c.qn.to(F64).sum(-1).sort(1, descending=True).values
    assert bool(((s[:, 0] - s[:, 1]) > 200 * U * c.qn.to(F64).abs().sum(-1).max(1).values).all()), "no near tie"
    check_qr(c, run_qr(c, 1.0), 1.0, False)


# ================================================================================================= shapes at the limit
@gpu
@pytest.mark.parametrize("kind", ["c51", "qr"])
def test_largest_accepted_shape_runs_and_next_is_refused(rl, kind):
    """N = A = 4096 is the largest shape the C ABI accepts ((3N + A) * 4 = 64 KiB of dynamic shared memory, past the 48 KiB
    default): it must run and be right.  N = 4097 or A = 4097 must be refused by the host check (B2RL_ERR_ARG) without a
    launch."""
    L = rl_lib()
    B, A, N = 1, 4096, 4096
    if kind == "c51":
        c = c51_case(900, B, A, N, -8.0, 8.0, 1.0, False, exact=False)
        o = run_c51(c)
        m32, _, _ = c51_emulate(c.lp, c.pt, c.po, c.action, c.reward, c.mask, 1.0, -8.0, 8.0)
        assert_equal(o["tp"], m32, "target_prob")
        assert o["counter"] == 0
    else:
        c = qr_case(901, B, A, N, 1.0, exact=False)
        o = run_qr(c, 1.0)
        vec, _, dq, terms, gt, _ = qr_ref64(c.quant, c.qn, c.action, c.reward, c.mask, 1.0, 1.0)
        assert_within(o["vec"], vec, (N + B + 8) * U * terms.abs().sum(-1).sum(0), "vec")
        assert_within(o["dq"][0, c.action[0]], dq[0, c.action[0]], (N + 3) * U * gt.abs().sum(1)[0], "dquant")
    for shape in ((B, A, N + 1), (B, A + 1, N)):
        before = L.launch_count()
        x = torch.zeros(shape, device="cuda")
        act = torch.zeros(B, dtype=torch.int64, device="cuda")
        r = torch.zeros(B, device="cuda")
        kl, out = torch.zeros(B, device="cuda"), torch.zeros(shape[2], device="cuda")
        cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
        name = "b2rl_c51_loss" if kind == "c51" else "b2rl_qr_loss"
        with pytest.raises(L.B2RLError, match=r"\(-1\).*bad shape"):
            if kind == "c51":
                L.call(name, L.ptr(x), L.ptr(x), None, L.ptr(act), L.ptr(r), L.ptr(r), 1.0, -8.0, 8.0, *shape, None, 0.0, 0.0,
                       0.0, L.ptr(kl), None, L.ptr(out), None, None, L.ptr(cnt), None, L.stream())
            else:
                L.call(name, L.ptr(x), L.ptr(x), L.ptr(act), L.ptr(r), L.ptr(r), 1.0, 1.0, *shape, L.ptr(out), L.ptr(out),
                       None, L.ptr(out), L.ptr(cnt), None, L.stream())
        assert L.launch_count() == before, "nothing was launched"
    torch.cuda.synchronize()


# ================================================================================================= counters across launches
@gpu
@pytest.mark.parametrize("kind", ["c51", "qr"])
def test_counter_across_batch_sizes(rl, kind):
    """Five consecutive launches at B = 512, 37, 1, 2048, 64 on ONE counter: each result is that of its own batch and the
    counter reads 0 after each (the last CTA re-arms it)."""
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    for i, B in enumerate((512, 37, 1, 2048, 64)):
        if kind == "c51":
            c = c51_case(1000 + i, B, 6, 33, -8.0, 8.0, 0.5, i % 2 == 0)
            check_c51(c, run_c51(c, counter=counter))
        else:
            c = qr_case(1000 + i, B, 4, 8, 0.5)
            check_qr(c, run_qr(c, 1.0, counter=counter), 1.0, True)
        assert int(counter.cpu()[0]) == 0


def _head_case(B, K, A, seed):
    g = _gen(seed)
    fa, ta = torch.nn.Linear(K, A).cuda(), torch.nn.Linear(K, A).cuda()
    with torch.no_grad():
        for m in (fa, ta):
            m.weight.copy_(ints(g, (A, K), -2, 2))
            m.bias.copy_(ints(g, (A,), -3, 3))
    for p in fa.parameters():
        p.grad = torch.zeros_like(p)
    phi, phi_t = ints(g, (B, K), 0, 3).to(torch.bfloat16).cuda(), ints(g, (B, K), 0, 3).to(torch.bfloat16).cuda()
    action = torch.randint(0, A, (B,), generator=g).cuda()
    reward, mask = ints(g, (B,), -1, 1).cuda(), ints(g, (B,), 0, 1).cuda()
    return fa, ta, phi, phi_t, action, reward, mask


@gpu
def test_graph_replay_after_eager_warmup(rl):
    """c51_loss_fused, qr_loss_fused and dqn_head_fused captured after the learner's pattern (eager warm-up on a side
    stream, then capture): every replay, also after eager calls at other batch sizes on the same counters, equals an eager
    call on the same inputs."""
    from deeprl_b200 import ops
    c51 = c51_case(1100, 64, 6, 51, -10.0, 10.0, 0.99, True, exact=False)
    qr = qr_case(1101, 64, 4, 32, 0.5)
    fa, ta, phi, phi_t, action, reward, mask = _head_case(64, 512, 6, 1102)
    colsum = torch.zeros(512, device="cuda")
    c51d = {k: dev(v) for k, v in c51.items() if torch.is_tensor(v)}
    qrd = {k: dev(v) for k, v in qr.items() if torch.is_tensor(v)}

    def step():
        for p in fa.parameters():
            p.grad.zero_()
        colsum.zero_()
        a = ops.c51_loss_fused(c51d["lp"], c51d["pt"], c51d["po"], c51d["action"], c51d["reward"], c51d["mask"], 0.99, -10.0,
                               10.0, want_target=True)
        b = ops.qr_loss_fused(qrd["quant"], qrd["qn"], qrd["action"], qrd["reward"], qrd["mask"], 0.5)
        h = ops.dqn_head_fused(phi, phi_t, None, (fa, None), (ta, None), action, reward, mask, 0.5, colsum)
        return [a["kl"], a["loss"], a["dlogp"], a["target_prob"], b["vec"], b["loss"], b["dquant"], h["gphi"], h["delta"],
                h["loss"], fa.weight.grad, fa.bias.grad, colsum]

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    torch.cuda.synchronize()
    want = [t.clone() for t in step()]
    for other in (37, 1, 512):                     # eager calls at other batch sizes between replays
        oc = c51_case(1200 + other, other, 6, 51, -10.0, 10.0, 0.99, False, exact=False)
        ops.c51_loss_fused(*[dev(oc[k]) for k in ("lp", "pt", "po", "action", "reward", "mask")], 0.99, -10.0, 10.0)
        oq = qr_case(1200 + other, other, 4, 32, 0.5)
        ops.qr_loss_fused(*[dev(oq[k]) for k in ("quant", "qn", "action", "reward", "mask")], 0.5)
        graph.replay()
        torch.cuda.synchronize()
        for i, (g_, w_) in enumerate(zip(captured, want)):
            assert torch.equal(g_, w_), "replay output %d differs from the eager call" % i
    check_c51(c51, dict(kl=want[0].cpu(), loss=want[1].cpu(), dlogp=want[2].cpu(), tp=want[3].cpu(), counter=0))
    check_qr(qr, dict(vec=want[4].cpu(), loss=want[5].cpu(), dq=want[6].cpu(), counter=0), 1.0, True)


def _block_state(addr):
    """State of the caching-allocator block that holds device address ``addr`` ("active_allocated", "inactive", ...), None
    if no segment of the allocator holds it."""
    for seg in torch.cuda.memory_snapshot():
        a = seg["address"]
        for blk in seg["blocks"]:
            if a <= addr < a + blk["size"]:
                return blk["state"]
            a += blk["size"]
    return None


@gpu
def test_scratch_growth_keeps_captured_buffers(rl, monkeypatch):
    """A graph captured after an eager warm-up holds the address of qr_loss_fused's partial-sum scratch.  A later eager call
    at a larger B * N replaces that scratch; the old buffer must stay allocated.  Were it freed, the caching allocator would
    hand its memory to the next allocations of its size on the warm-up stream (premise, asserted for that case) and every
    replay would write QR partials into them.  Checked by allocating such tensors until one covers the old address (or 64
    of them), replaying, and requiring them intact and the replay equal to the eager call."""
    from deeprl_b200 import ops
    monkeypatch.setattr(ops._Scratch, "_store", {})
    monkeypatch.setattr(ops._Scratch, "_retired", [], raising=False)
    B0, N0, B1, N1 = 48, 32, 96, 64
    nbytes = B0 * N0 * 4
    small, big = qr_case(1300, B0, 4, N0, 0.5), qr_case(1301, B1, 4, N1, 0.5)
    sd = {k: dev(v) for k, v in small.items() if torch.is_tensor(v)}
    bd = {k: dev(v) for k, v in big.items() if torch.is_tensor(v)}
    call = lambda d: ops.qr_loss_fused(d["quant"], d["qn"], d["action"], d["reward"], d["mask"], 0.5)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                      # the learner's warm-up: eager, on a side stream
        call(sd)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    old = ops._Scratch._store[(str(sd["quant"].device), "qr_partial", F32)].data_ptr()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = call(sd)
    torch.cuda.synchronize()
    want = {k: v.clone() for k, v in call(sd).items()}
    call(bd)                                        # grows the scratch
    torch.cuda.synchronize()
    state = _block_state(old)
    victims, covered = [], False
    with torch.cuda.stream(s):
        while not covered and len(victims) < 64:
            v = torch.full((B0 * N0,), 7.0, device="cuda")
            victims.append(v)
            covered = v.data_ptr() < old + nbytes and old < v.data_ptr() + nbytes
    s.synchronize()
    if state != "active_allocated":
        assert covered, "premise: the freed scratch goes to later allocations of its size on the warm-up stream"
    graph.replay()
    torch.cuda.synchronize()
    for i, v in enumerate(victims):
        assert bool((v == 7.0).all()), "the replay wrote into tensor %d of %d allocated after the scratch grew (old scratch " \
            "block %s, covered: %s)" % (i, len(victims), state, covered)
    for k in ("vec", "loss", "dquant"):
        assert torch.equal(captured[k], want[k]), k
    assert state == "active_allocated", "the scratch a captured graph uses is still allocated after it was replaced"
    assert not covered


# ================================================================================================= GAE
def gae_ref64(reward, mask, value, discount, tau, use_gae):
    """float64 backward recurrence (A2C_agent.py:43-53) on [T, N] / [T + 1, N]; also the magnitude sums that bound
    the scan's reassociation: |ret_t| <= R_t = |r_t| + |gm| R_{t+1}, |adv_t| <= D_t = |td_t| + |tau gm| D_{t+1} with
    |td_t| <= |r| + |gm v_{t+1}| + |v_t|."""
    r, m, v = reward.to(F64), mask.to(F64), value.to(F64)
    T = r.shape[0]
    ret, adv = v[T].clone(), torch.zeros_like(v[0])
    R, D = v[T].abs(), torch.zeros_like(v[0])
    advs, rets, Rs, Ds = [None] * T, [None] * T, [None] * T, [None] * T
    for t in reversed(range(T)):
        gm = discount * m[t]
        ret = r[t] + gm * ret
        R = r[t].abs() + gm.abs() * R
        if use_gae:
            td = r[t] + gm * v[t + 1] - v[t]
            adv = adv * tau * gm + td
            D = (r[t].abs() + (gm * v[t + 1]).abs() + v[t].abs()) + (tau * gm).abs() * D
        else:
            adv = ret - v[t]
            D = R + v[t].abs()
        advs[t], rets[t], Rs[t], Ds[t] = adv, ret, R, D
    return torch.stack(advs), torch.stack(rets), torch.stack(Rs), torch.stack(Ds)


def gae_case(seed, T, N, exact=True):
    g = _gen(seed)
    if exact:
        reward, value = ints(g, (T, N), -2, 2), ints(g, (T + 1, N), -3, 3)
    else:
        reward, value = torch.randn(T, N, generator=g), torch.randn(T + 1, N, generator=g)
    mask = (torch.rand(T, N, generator=g) > 0.1).float()
    C = (T + 31) // 32
    for lane in (1, 7, 16, 31):                     # masks of 0 on the scan's chunk boundaries, on every other env
        for t in (lane * C - 1, lane * C):
            if t < T:
                mask[t, ::2] = 0.0
    mask[T - 1, 1::3] = 0.0
    return reward, mask, value


def run_gae(reward, mask, value, discount, tau, use_gae, mode):
    L = rl_lib()
    T, N = reward.shape
    adv, ret = nan_like((T, N)), nan_like((T, N))
    d = [dev(t) for t in (reward, mask, value)]                                            # alive until the kernel is done
    L.call("b2rl_gae", *[L.ptr(t) for t in d], float(discount), float(tau), T, N,
           int(use_gae), int(mode), L.ptr(adv), L.ptr(ret), L.stream())
    torch.cuda.synchronize()
    return adv.cpu(), ret.cpu()


GAE_T = [1, 2, 31, 32, 33, 63, 64, 65, 1024, 2049]
GAE_N = [1, 3, 4, 5, 130]


@gpu
@pytest.mark.parametrize("T", GAE_T)
@pytest.mark.parametrize("N", GAE_N)
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("use_gae", [True, False])
def test_gae_exact(rl, T, N, mode, use_gae):
    """discount = tau = 1 on integers (and 1/2 for T <= 2): both modes equal the float64 recurrence exactly, with masks of 0
    on the scan's chunk boundaries and at t = T - 1."""
    discount = 0.5 if T <= 2 else 1.0
    reward, mask, value = gae_case(T * 131 + N, T, N)
    adv64, ret64, R, D = gae_ref64(reward, mask, value, discount, discount, use_gae)
    assert float(R.max()) * grid(ret64) < EXACT and float(D.max()) * grid(adv64) < EXACT, "premise: exact in fp32"
    adv, ret = run_gae(reward, mask, value, discount, discount, use_gae, mode)
    assert_equal(ret, ret64, "returns")
    assert_equal(adv, adv64, "advantages")


@gpu
@pytest.mark.parametrize("T", [5, 12])
@pytest.mark.parametrize("mode", [0, 1])
def test_gae_half_discount_exact(rl, T, mode):
    """discount = tau = 1/2, T <= 12: every value is dyadic with few bits, so both modes are exact."""
    reward, mask, value = gae_case(T, T, 5)
    adv64, ret64, R, D = gae_ref64(reward, mask, value, 0.5, 0.5, True)
    assert float(D.max()) * grid(adv64) < EXACT and float(R.max()) * grid(ret64) < EXACT
    adv, ret = run_gae(reward, mask, value, 0.5, 0.5, True, mode)
    assert_equal(ret, ret64, "returns")
    assert_equal(adv, adv64, "advantages")


@gpu
@pytest.mark.parametrize("T,N", [(5, 3), (128, 16), (1000, 5), (2049, 130)])
@pytest.mark.parametrize("use_gae", [True, False])
def test_gae_production_constants(rl, T, N, use_gae):
    """discount 0.99, tau 0.95 on Gaussian data.  Mode 0 is the reference loop in float32 (bit-identical to
    oracle.gae in float32); mode 1 within the scan's first-order association bound: a chain of C = ceil(T / 32) steps in
    each pass and five composition levels, each step a few roundings of the magnitude sum R_t / D_t."""
    from oracle import losses as oracle
    reward, mask, value = gae_case(T + N, T, N, exact=False)
    adv0, ret0 = run_gae(reward, mask, value, 0.99, 0.95, use_gae, 0)
    a32, r32 = oracle.gae(reward[:, :, None], mask[:, :, None], value[:, :, None], 0.99, 0.95, use_gae)
    assert_equal(ret0, r32[:, :, 0], "mode 0 returns")
    assert_equal(adv0, a32[:, :, 0], "mode 0 advantages")
    adv64, ret64, R, D = gae_ref64(reward, mask, value, 0.99, 0.95, use_gae)
    C = (T + 31) // 32
    k = 4 * C + 24
    adv1, ret1 = run_gae(reward, mask, value, 0.99, 0.95, use_gae, 1)
    assert_within(ret1, ret64, k * U * R, "mode 1 returns")
    assert_within(adv1, adv64, k * U * (D + (0 if use_gae else R)), "mode 1 advantages")


# ================================================================================================= normalize_advantage
def normalize_contract(x):
    """The kernel's contract: mean and unbiased variance in float64, mean and std rounded once to float32, then
    (x - mean) / std with one rounding each.  Also asserts the premise that float64 summation order cannot change the
    rounded mean / std on this data (x on a 2**-12 grid: the sum is exact; the variance's float32 rounding is decided
    with margin)."""
    xd = x.to(F64)
    M = x.numel()
    s = float(xd.sum())
    assert s * 4096.0 == round(s * 4096.0) and abs(s) * 4096 < 2.0 ** 53, "premise: the float64 sum is exact"
    mean = s / M
    d = xd - mean
    q = math.fsum((d * d).tolist())
    slack = M * 2.0 ** -52 * q
    lo, hi = np.float32(math.sqrt(max(q - slack, 0.0) / (M - 1))), np.float32(math.sqrt((q + slack) / (M - 1)))
    assert lo == hi, "premise: the std's float32 rounding does not depend on the float64 summation order"
    meanf, stdf = f32(mean), f32(float(lo))
    return (x - meanf) / stdf


@gpu
@pytest.mark.parametrize("M", [2, 3, 1023, 1024, 1025, 2 ** 20])
def test_normalize_advantage(rl, M):
    """b2rl_normalize_advantage bit-exact against its contract, and within a bound of oracle.normalize_advantage in
    float32 (whose mean and std carry float32 summation error)."""
    from oracle import losses as oracle
    L = rl_lib()
    x = torch.round(torch.randn(M, generator=_gen(M)) * 4096.0 * 2) / 4096.0
    x[0] += 3.0                                        # keep M = 2 / 3 from degenerate values
    want = normalize_contract(x)
    d = dev(x)
    L.call("b2rl_normalize_advantage", L.ptr(d), M, L.stream())
    torch.cuda.synchronize()
    got = d.cpu()
    assert_equal(got, want, "normalized advantages")
    o32 = oracle.normalize_advantage(x)
    lg = math.log2(M) + 4
    mean_abs = float(x.to(F64).abs().mean())
    std = float(x.to(F64).std())
    bound = lg * U * (mean_abs / std + 2 * want.to(F64).abs()) + 4 * U * want.to(F64).abs()
    assert_within(got, o32, bound, "against oracle.normalize_advantage in float32")


# ================================================================================================= PPO / A2C
def ppo_ref(logp, ent, v, old, adv, ret, clip, ew, ratio=None):
    """float64 PPO_agent.py:77-86 and the gradient of policy_loss + value_loss: torch.min splits a tie evenly, clamp passes
    the gradient on the closed interval [1 - clip, 1 + clip]."""
    logp, ent, v, old, adv, ret = [t.to(F64) for t in (logp, ent, v, old, adv, ret)]
    M = logp.numel()
    ratio = (logp - old).exp() if ratio is None else ratio.to(F64)
    lo, hi = float(f32(1.0) - f32(clip)), float(f32(1.0) + f32(clip))
    obj, rc = ratio * adv, ratio.clamp(lo, hi)
    objc = rc * adv
    inside = ((ratio >= lo) & (ratio <= hi)).to(F64)
    g = torch.where(obj < objc, adv * ratio, torch.where(obj > objc, inside * adv * ratio, 0.5 * adv * ratio * (1 + inside)))
    e = ret - v
    out = torch.stack([-torch.minimum(obj, objc).mean() - ew * ent.mean(), 0.5 * (e * e).mean(), (old - logp).mean()])
    return out, -g / M, torch.full((M,), -ew / M, dtype=F64), -e / M, torch.minimum(obj, objc)


def ppo_case(seed, M, kind):
    """Integer data.  kind "one": d = 0 everywhere (ratio exactly 1); "clip": d in {0, +-2} (clamp active for |d| = 2);
    adv = 0 on some rows in both."""
    g = _gen(seed)
    old = ints(g, (M,), -6, -1)
    d = torch.zeros(M) if kind == "one" else 2.0 * ints(g, (M,), -1, 1)
    logp = old + d
    adv = ints(g, (M,), -3, 3)
    adv[::5] = 0.0
    ent, v, ret = ints(g, (M,), 0, 3), ints(g, (M,), -3, 3), ints(g, (M,), -3, 3)
    return logp, ent, v, old, adv, ret


def run_ppo(args, clip, ew):
    L = rl_lib()
    M = args[0].numel()
    out, dl, de, dv = nan_like((4,)), nan_like((M,)), nan_like((M,)), nan_like((M,))
    d = [dev(t) for t in args]                                                             # alive until the kernel is done
    L.call("b2rl_ppo_loss", *[L.ptr(t) for t in d], float(clip), float(ew), M, L.ptr(out), L.ptr(dl), L.ptr(de),
           L.ptr(dv), L.stream())
    torch.cuda.synchronize()
    return out.cpu()[:3], dl.cpu(), de.cpu(), dv.cpu()


PPO_M = [1, 64, 1000, 1024, 1025, 4096]


@gpu
@pytest.mark.parametrize("M", PPO_M)
@pytest.mark.parametrize("clip", [0.2, 0.0])
def test_ppo_loss_ratio_one_exact(rl, M, clip):
    """ratio exactly 1 (d = 0): obj == objc on every row, so the tie rule decides the gradient (half through each branch;
    with clip = 0 the ratio sits on both clamp bounds, and the closed interval passes the second half).  Losses and all
    three gradients exact; 1/M rounds for ragged M and is emulated in float32."""
    args = ppo_case(M + int(clip * 10), M, "one")
    ew = 0.5
    got = run_ppo(args, clip, ew)
    out, dl, de, dv, terms = ppo_ref(*args, clip, ew)
    logp, ent, v, old, adv, ret = args
    invM = f32(1.0) / f32(float(M))
    for t in (terms, ent, (ret - v) ** 2, old - logp):
        assert_exact_premise(t, "ppo sums")
    s_obj, s_ent, s_v, s_kl = [f32(float(t.to(F64).sum())) for t in (terms, ent, (ret - v) ** 2, old - logp)]
    want = torch.stack([(-(s_obj * invM)) - f32(ew) * (s_ent * invM), f32(0.5) * (s_v * invM), s_kl * invM])
    assert_equal(got[0], want, "policy / value loss, approx_kl")
    assert_equal(got[1], (-adv) * invM, "dlogp (the tie rule)")
    assert_equal(got[2], torch.full((M,), float(-f32(ew) * invM)), "dentropy")
    assert_equal(got[3], (-(ret - v)) * invM, "dv")


@gpu
@pytest.mark.parametrize("M", PPO_M)
def test_ppo_loss_clipped(rl, M):
    """d in {0, +-2} with clip 0.2: rows outside the interval take the clamped objective and a zero gradient (exact),
    rows where the unclipped objective is smaller carry expf's 2 ulp; sums within their bound."""
    args = ppo_case(2000 + M, M, "clip")
    clip, ew = 0.2, 0.5
    got = run_ppo(args, clip, ew)
    out, dl, de, dv, terms = ppo_ref(*args, clip, ew)
    logp, ent, v, old, adv, ret = args
    d = (logp - old).to(F64)
    rel = 2 * ULP_EXPF * U + 2 * U
    assert_within(got[1], dl, rel * dl.abs(), "dlogp")
    zero = (d.abs() == 2) & (dl == 0)
    assert bool((got[1][zero] == 0).all()), "no gradient through the clamp outside the interval"
    if M >= 64:
        assert bool(zero.any()) and bool(((d.abs() == 2) & (dl != 0)).any()), "premise: both branches occur"
    invM = 1.0 / M
    assert_within(got[0][0], out[0], (rel + (M + 3) * U) * (terms.abs().sum() + ew * ent.abs().sum()) * invM, "policy loss")
    assert_within(got[0][1:], out[1:], 2 * U * out[1:].abs(), "value loss, approx_kl (1/M rounds once, the product once)")
    assert_within(got[3], dv, 2 * U * dv.abs(), "dv")


def run_a2c(args, ew, vw):
    L = rl_lib()
    M = args[0].numel()
    out, dl, de, dv = nan_like((4,)), nan_like((M,)), nan_like((M,)), nan_like((M,))
    d = [dev(t) for t in args]                                                             # alive until the kernel is done
    L.call("b2rl_a2c_loss", *[L.ptr(t) for t in d], float(ew), float(vw), M, L.ptr(out), L.ptr(dl), L.ptr(de),
           L.ptr(dv), L.stream())
    torch.cuda.synchronize()
    return out.cpu(), dl.cpu(), de.cpu(), dv.cpu()


@gpu
@pytest.mark.parametrize("M", PPO_M)
def test_a2c_loss_exact(rl, M):
    """A2C on integers with dyadic weights (entropy 1/2, value 1/4: a dv without the value weight is off by 4x): the four
    outputs and three gradients exact, 1/M emulated in float32 for ragged M."""
    g = _gen(3000 + M)
    logp, ent, v, adv, ret = ints(g, (M,), -6, 0), ints(g, (M,), 0, 3), ints(g, (M,), -3, 3), ints(g, (M,), -3, 3), \
        ints(g, (M,), -3, 3)
    ew, vw = 0.5, 0.25
    got = run_a2c((logp, ent, v, adv, ret), ew, vw)
    invM = f32(1.0) / f32(float(M))
    e = ret - v
    for t in (logp * adv, ent, e * e):
        assert_exact_premise(t, "a2c sums")
    s_p, s_e, s_v = [f32(float(t.to(F64).sum())) for t in (logp * adv, ent, e * e)]
    pl, el, vl = -(s_p * invM), s_e * invM, f32(0.5) * (s_v * invM)
    assert_equal(got[0], torch.stack([(pl - f32(ew) * el) + f32(vw) * vl, pl, vl, el]), "objective, policy, value, entropy")
    assert_equal(got[1], (-adv) * invM, "dlogp")
    assert_equal(got[2], torch.full((M,), float(-f32(ew) * invM)), "dentropy")
    assert_equal(got[3], ((-f32(vw)) * e) * invM, "dv")


# ================================================================================================= CPU: the references
def test_c51_reference_matches_oracle_cpu():
    """c51_ref64's KL is oracle.c51_kl in float64 (production shape, double-Q on and off), and on exact data the float32
    emulation is the float64 projection bit for bit."""
    from oracle import losses as oracle
    for dq in (False, True):
        c = c51_case(11 + int(dq), 37, 6, 51, -10.0, 10.0, 0.99, dq, exact=False)
        m, kl = c51_ref64(c.lp, c.pt, c.po, c.action, c.reward, c.mask, 0.99, -10.0, 10.0)
        want = oracle.c51_kl(c.lp.to(F64), c.pt.to(F64), None if c.po is None else c.po.to(F64), c.action,
                             c.reward.to(F64), c.mask.to(F64), c51_atoms(-10.0, 10.0, 51).to(F64), -10.0, 10.0, 0.99)
        assert torch.allclose(kl, want, rtol=1e-9, atol=1e-9)          # (the kernel's 1e-5 is float32)
        assert torch.allclose(m.sum(-1), torch.ones(37, dtype=F64))
        m32, _, _ = c51_emulate(c.lp, c.pt, c.po, c.action, c.reward, c.mask, 0.99, -10.0, 10.0)
        assert_within(m32, m, (51 + 4) * U * m.abs() + 51 * U * m.abs().max(), "float32 emulation vs float64")
    for B, A, N in C51_EXACT:
        for dq in (False, True):
            gamma_n = 0.5 if (B + N) % 2 else 1.0
            c = c51_case(B * 7 + N + int(dq), B, A, N, -8.0, 8.0, gamma_n, dq)
            m32, _, _ = c51_emulate(c.lp, c.pt, c.po, c.action, c.reward, c.mask, gamma_n, -8.0, 8.0)
            m64, _ = c51_ref64(c.lp, c.pt, c.po, c.action, c.reward, c.mask, gamma_n, -8.0, 8.0)
            assert torch.equal(m32.to(F64), m64), (B, A, N, dq)
            assert grid(c.pt) <= 64 and grid(m64) <= 256


def test_c51_projection_edges_cpu():
    """The clamp and the on-atom cases on one hand-made sample: r = 2, gamma = 1 pushes z >= 6 past v_max = 8, all that mass
    lands on the last atom; r = 0.5, gamma = 1/2 with delta_z = 1 puts z / 2 + 1/2 halfway between atoms for even z."""
    N, A = 17, 1
    pt = torch.full((1, A, N), 1.0 / 16)
    pt[0, 0, 0] = 0.0
    lp = torch.log(torch.full((1, A, N), 1.0 / N))
    for r, gm, expect_last in ((2.0, 1.0, 3.0 / 16), (0.5, 0.5, None)):
        c = (lp, pt, None, torch.zeros(1, dtype=torch.int64), torch.tensor([r]), torch.ones(1))
        m32, _, z = c51_emulate(*c, gm, -8.0, 8.0)
        m64, _ = c51_ref64(*c, gm, -8.0, 8.0)
        assert torch.equal(m32.to(F64), m64)
        if expect_last is not None:
            assert math.isclose(float(m64[0, -1]), expect_last, rel_tol=1e-12)
        else:
            assert bool((m64 * 32 == (m64 * 32).round()).all()) and not bool((m64 * 16 == (m64 * 16).round()).all())
        assert math.isclose(float(m64.sum()), 1.0, rel_tol=1e-12)


def test_qr_reference_matches_oracle_and_autograd_cpu():
    """qr_ref64's vec is oracle.qr_loss in float64 and its dquant is autograd of mean(vec) and of sum(gw * vec * B)."""
    from oracle import losses as oracle
    for B, A, N, exact in ((9, 4, 8, True), (37, 6, 200, False)):
        c = qr_case(B + N, B, A, N, 1.0 if exact else 0.99, exact=exact)
        vec, loss, dq, _, _, _ = qr_ref64(c.quant, c.qn, c.action, c.reward, c.mask, c.gamma_n, 1.0)
        q = c.quant.to(F64).requires_grad_(True)
        want = oracle.qr_loss(q, c.qn.to(F64), c.action, c.reward.to(F64), c.mask.to(F64), c.gamma_n)
        assert torch.allclose(vec, want.detach(), rtol=1e-6, atol=1e-6)      # the oracle rounds tau and T in float32
        want.mean().backward()
        assert torch.allclose(dq, q.grad, rtol=1e-6, atol=1e-9)
        gw = ints(_gen(B), (N,), -3, 3) / 64.0
        _, _, dqw, _, _, _ = qr_ref64(c.quant, c.qn, c.action, c.reward, c.mask, c.gamma_n, 1.0, gw=gw)
        q.grad = None
        oracle.qr_loss(q, c.qn.to(F64), c.action, c.reward.to(F64), c.mask.to(F64), c.gamma_n).mul(gw.to(F64) * B).sum() \
            .backward()
        assert torch.allclose(dqw, q.grad, rtol=1e-6, atol=1e-6)       # (the oracle's targets are float64)


def test_gae_reference_matches_oracle_cpu():
    from oracle import losses as oracle
    for T, N, use_gae in ((33, 5, True), (65, 3, False)):
        r, m, v = gae_case(T, T, N, exact=False)
        a, rt, _, _ = gae_ref64(r, m, v, 0.99, 0.95, use_gae)
        wa, wr = oracle.gae(r.to(F64)[:, :, None], m.to(F64)[:, :, None], v.to(F64)[:, :, None], 0.99, 0.95, use_gae)
        assert torch.allclose(a, wa[:, :, 0], rtol=1e-12, atol=1e-12) and torch.allclose(rt, wr[:, :, 0], rtol=1e-12, atol=1e-12)
    for T in GAE_T:                                   # premise of the exact cases
        for N in GAE_N:
            r, m, v = gae_case(T * 131 + N, T, N)
            C = (T + 31) // 32
            if T > 32:
                assert bool((m[C - 1, ::2] == 0).all()) and bool((m[C, ::2] == 0).all()), "zero masks on a chunk boundary"
            a, rt, R, D = gae_ref64(r, m, v, 1.0, 1.0, True)
            assert float(D.max()) * grid(a) < EXACT and float(R.max()) * grid(rt) < EXACT


def test_normalize_contract_matches_oracle_cpu():
    from oracle import losses as oracle
    for M in (2, 3, 1023, 1025):
        x = torch.round(torch.randn(M, generator=_gen(M)) * 4096.0 * 2) / 4096.0
        x[0] += 3.0
        got = normalize_contract(x)
        want = oracle.normalize_advantage(x.to(F64))
        assert_within(got, want, 4 * U * (want.abs() + 1), "contract vs float64 oracle")


def test_ppo_a2c_reference_gradients_match_autograd_cpu():
    """ppo_ref's gradients are autograd of oracle.ppo_losses in float64 -- including the ties of torch.min (adv = 0, ratio
    exactly 1) and the closed clamp interval at clip = 0 -- and the A2C gradients are autograd of oracle.a2c_loss."""
    from oracle import losses as oracle
    for kind, clip in (("one", 0.2), ("one", 0.0), ("clip", 0.2)):
        args = ppo_case(5, 64, kind)
        logp, ent, v, old, adv, ret = [t.to(F64).requires_grad_(i in (0, 1, 2)) for i, t in enumerate(args)]
        out, dl, de, dv, _ = ppo_ref(*args, clip, 0.5)
        pl, vl, kl = oracle.ppo_losses(logp, ent, v, old, adv, ret, clip, 0.5)
        (pl + vl).backward()
        assert torch.allclose(out, torch.stack([pl, vl, kl]).detach(), rtol=1e-6)
        assert torch.allclose(dl, logp.grad, rtol=1e-6, atol=1e-12), kind
        assert torch.allclose(de, ent.grad) and torch.allclose(dv, v.grad)
    M = 37
    g = _gen(6)
    logp, ent, v, adv, ret = [ints(g, (M,), -3, 3).to(F64).requires_grad_(True) for _ in range(5)]
    oracle.a2c_loss(logp, v, ret, adv.detach(), ent, 0.5, 0.25).backward()
    assert torch.allclose(logp.grad, -adv.detach() / M) and torch.allclose(ent.grad, torch.full((M,), -0.5 / M, dtype=F64))
    assert torch.allclose(v.grad, -0.25 * (ret - v).detach() / M)


def test_exact_premises_cpu():
    """The data of the exact DQN / QR / PPO cases is what the GPU tests claim."""
    for B in (1, 37, 4096):
        c = dqn_case(B, B, 6, True, 0.5)
        d = dqn_emulate(c.q, c.qt, c.qo, c.action, c.reward, c.mask, 0.5)
        assert_exact_premise((d * d) * 0.5, "dqn loss")
    for B, A, N in QR_EXACT:
        c = qr_case(B * 3 + N + 1, B, A, N, 1.0)
        _, _, _, terms, gt, _ = qr_ref64(c.quant, c.qn, c.action, c.reward, c.mask, 1.0, 1.0)
        assert_exact_premise(terms.permute(1, 0, 2).reshape(N, -1), "qr vec")
        assert grid(qr_tau32(N)) <= 2 * N
    for M in PPO_M:
        args = ppo_case(M, M, "one")
        assert torch.equal(args[0], args[3]), "d = 0: ratio exactly 1"
        assert bool((args[4] == 0).any()) or M < 5
