"""The fully-connected heads between fc4 and the losses compared EXACTLY with a float64 reference: the narrow value heads of
csrc/head.cu (head_fwd_kernel, head_bwd_kernel, the DQN head in one launch, dqn_head_fused_kernel, and in two,
dqn_head_loss_kernel + head_bwd_kernel), the distributional head of network/fused.py (wgmma GEMMs + csrc/disthead.cu) in
both backward branches, the first-maximum rule of every argmax, and the address-keyed fc4-ReLU registries of
network/nature_tc.py.

Exactness by choice of data: features are bf16 integers 0..3 (zeros included, so the ReLU mask matters), fp32 weights
integers in -2..2, biases integers, rewards in {-1, 0, 1}, gamma_n in {0.5, 1}, and B a power of two, so every gradient
g = -delta / B is dyadic.  While the magnitudes of a sum's terms, scaled to integers, add up to less than 2**24, fp32
accumulation is exact in ANY order (lane split, warp shuffles, row groups, atomics), so each output has exactly one correct
value and the checks are ``torch.equal``.  Every case asserts that premise on its own data.  Where a step rounds -- the
dueling mean divides by A, ragged B makes 1/B inexact -- the reference takes that step in float32 in the kernel's order
(bit-exact), and sums over rounded terms are held to a bound derived from the data, n * 2**-24 * sum|terms| (first order),
instead of a fudge factor.  One Gaussian-operand case per kernel keeps a precision regression from hiding behind integers.

Outputs are pre-filled with sentinels (bf16 -12345 for gradients and GEMM operands, NaN for q / delta / logits /
probabilities) and every accumulated gradient (head weights and biases, fc4's column sums, the distributional head's
.grad) with nonzero integers, so that stray or missing stores and overwrite-instead-of-accumulate fail.

The CPU tests at the end pin the reference against F.linear, autograd and oracle/losses.py in float64."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

gpu = pytest.mark.gpu

F64, F32, BF = torch.float64, torch.float32, torch.bfloat16
EXACT = 2.0 ** 24           # sum |terms| (scaled to integers) below this: fp32 accumulation is exact in any order
U = 2.0 ** -24              # unit roundoff of fp32
SENT = -12345.0             # bf16 sentinel of gradient / operand buffers (-12352 after rounding)
GEFF_LD = 33                # row stride of the effective-gradient scratch of b2rl_dqn_head_two (HEAD_MAX_OUT + 1)


def _pow2(n):
    return n > 0 and n & (n - 1) == 0


# ================================================================================================= float64 reference
def head_dots(phi, Wa, ba, Wv=None, bv=None):
    """[B, n_out] float64: phi Wa^T + ba, with phi Wv^T + bv as the last column for a dueling head."""
    W = Wa if Wv is None else torch.cat([Wa, Wv])
    b = ba if bv is None else torch.cat([ba, bv])
    return phi.to(F64) @ W.to(F64).t() + b.to(F64)


def dueling_combine(d, A):
    """q = v + (adv - mean(adv)) from the dot products d [B, A + 1] in d's dtype, in the kernel's order (head_combine:
    sequential sum over the A advantages, one division, then v + (adv - mean)).  float32 on exact dot products is
    bit-exact with the kernel; float64 is the plain reference."""
    s = torch.zeros(d.shape[0], dtype=d.dtype, device=d.device)
    for a in range(A):
        s = s + d[:, a]
    mean = s / float(A)
    return d[:, A:A + 1] + (d[:, :A] - mean[:, None])


def head_q(d, A, dueling):
    return dueling_combine(d, A) if dueling else d[:, :A]


def dqn_delta(q, qt, qo, action, reward, mask, gamma_n):
    """DQN target and delta in q's dtype, in the kernel's order: target = r + (gamma_n * q_next) * mask, delta =
    target - q[a].  q_next = max_a qt, or qt at the FIRST maximum of qo (double-Q)."""
    if qo is not None:
        qnext = qt.gather(1, torch.argmax(qo, 1, keepdim=True))[:, 0]
    else:
        qnext = qt.max(1).values
    target = reward.to(q.dtype) + (gamma_n * qnext) * mask.to(q.dtype)
    return target - q.gather(1, action.long()[:, None])[:, 0]


def inv(B, dtype):
    return torch.ones((), dtype=dtype) / float(B)


def dqn_geff(delta, action, A, dueling, B, w=None):
    """Effective output gradient [B, n_out] of mean(0.5 * (w * delta)^2) with respect to the head's dot products, in
    delta's dtype and the kernel's order: g_a = -(delta * w) * w * (1/B) at the taken action, spread by the dueling
    combine as g_n - g_a / A for the advantages and g_a for the value."""
    w = torch.ones_like(delta) if w is None else w.to(delta.dtype)
    g_ab = (-(delta * w) * w) * inv(B, delta.dtype)
    onehot = F.one_hot(action.long(), A).to(delta.dtype) * g_ab[:, None]
    if not dueling:
        return onehot
    return torch.cat([onehot - (g_ab / float(A))[:, None], g_ab[:, None]], 1)


def head_geff(gq, A, dueling):
    """Effective output gradient of head_bwd_kernel from dL/dq [B, A] (head_geff: sequential sum, one division)."""
    if not dueling:
        return gq.clone()
    s = torch.zeros(gq.shape[0], dtype=gq.dtype, device=gq.device)
    for a in range(A):
        s = s + gq[:, a]
    return torch.cat([gq - (s / float(A))[:, None], s[:, None]], 1)


def head_bwd(geff, phi, Wa, Wv=None, relu=False):
    """float64 head backward: dphi = geff W (masked by phi > 0 for a ReLU feature), dW = geff^T phi, db = sum_b geff.
    Returns (dphi, dW [n_out, K], db [n_out])."""
    W = (Wa if Wv is None else torch.cat([Wa, Wv])).to(F64)
    g = geff.to(F64)
    x = phi.to(F64)
    dphi = g @ W
    if relu:
        dphi = dphi * (x > 0)
    return dphi, g.t() @ x, g.sum(0)


def dphi_kernel_order(geff32, phi, Wa, Wv=None, relu=False):
    """bf16 dphi as head_bwd_body computes it: g = fma(geff_n, W_n, g) for n = 0 .. n_out-1 in float32 (the products are
    exact for integer W, so each step is one rounding like fmaf), masked, rounded once to bf16."""
    W = (Wa if Wv is None else torch.cat([Wa, Wv])).float()
    g = torch.zeros((geff32.shape[0], W.shape[1]), dtype=F32, device=geff32.device)
    for n in range(W.shape[0]):
        g = g + geff32[:, n:n + 1] * W[n]
    if relu:
        g = torch.where(phi.float() > 0, g, torch.zeros_like(g))
    return g.to(BF)


def log_softmax_fwd(x):
    """(log_prob, prob) over the last dimension, float64: x - max - log(sum exp(x - max))."""
    x = x.to(F64)
    z = x - x.max(-1, keepdim=True).values
    lp = z - torch.log(torch.exp(z).sum(-1, keepdim=True))
    return lp, torch.exp(lp)


def log_softmax_bwd(dlogp, prob):
    """dlogits = dlogp - prob * sum_n dlogp (float64)."""
    d = dlogp.to(F64)
    return d - prob.to(F64) * d.sum(-1, keepdim=True)


def dist_bwd_prep(dout, prob, ld):
    """b2rl_dist_head_bwd_prep: (bf16 operand [B, ld] with zero padding columns [A*N, ld), bias gradient [A*N] (float64))
    from dout [B, A, N] and prob (None: QR-DQN, the operand is dout itself)."""
    B = dout.shape[0]
    v = dout.to(F64) if prob is None else log_softmax_bwd(dout, prob)
    v = v.reshape(B, -1)
    g = torch.zeros((B, ld), dtype=BF, device=dout.device)
    g[:, :v.shape[1]] = v.float().to(BF)
    return g, v, v.sum(0)


# ================================================================================================= checks
def assert_exact_premise(abs_sum, scale, what):
    """Every term of the sums behind ``what`` is a multiple of 1/scale and their magnitudes add up to abs_sum."""
    worst = float(abs_sum.max()) * scale
    assert worst < EXACT, "%s: sum |terms| * %g = %g is not below 2**24, fp32 accumulation could round" % (what, scale, worst)


def grid(x):
    """The smallest power of two 2**s such that every element of x is a multiple of 2**-s (x dyadic)."""
    y, s = x.to(F64), 1.0
    while not torch.equal(y * s, (y * s).round()):
        s *= 2.0
        assert s < 2.0 ** 60, "not a dyadic rational"
    return s


def assert_within(got, ref, bound, what):
    err = (got.to(F64).cpu() - ref.to(F64).cpu()).abs()
    bad = err > bound.cpu()
    assert not bool(bad.any()), "%s: %d of %d elements beyond the bound (worst err %.3g, its bound %.3g)" % (
        what, int(bad.sum()), bad.numel(), float(err.max()), float(bound.cpu().reshape(-1)[int(err.argmax())]))


def check_sum(got, init, ref, abs_terms, n, exact, scale, what):
    """got = init + ref accumulated by the kernel: equal when ``exact`` (premise asserted), else within n * U * sum|terms|."""
    want = init.to(F64).cpu() + ref.cpu()
    if exact:
        assert_exact_premise(abs_terms + init.to(F64).abs().cpu(), scale, what)
        assert torch.equal(got.to(F64).cpu(), want), what
    else:
        assert_within(got, want, n * U * (abs_terms.cpu() + init.to(F64).abs().cpu()), what)


def assert_softmax_within(logp, prob, x, N):
    """dist_softmax_kernel against float64.  With xm = |x - max|: x - max rounds once (U xm), each expf is within 2 ulp,
    the sum of N of them adds N roundings, logf one ulp of |log s|, the last subtraction one rounding of |log_prob|; prob
    = expf(x - max) / s adds the division's rounding (denormal results: an absolute 2**-126)."""
    lp64, p64 = log_softmax_fwd(x)
    x64 = x.to(F64)
    xm = x64.max(-1, keepdim=True).values - x64
    ls = -(lp64 + xm)
    assert_within(logp, lp64, U * (xm + 2 * ls.abs() + lp64.abs() + 2 * N + 8), "log_prob")
    assert_within(prob, p64, U * (xm + 2 * N + 10) * p64 + 2.0 ** -126, "prob")


def bf16_representable(x):
    return torch.equal(x.float().to(BF).to(F64), x.to(F64))


# ================================================================================================= data
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def ints(g, shape, lo, hi, dtype=F32):
    return torch.randint(lo, hi + 1, shape, generator=g).to(dtype)


def features(g, B, K, gaussian=False):
    if gaussian:
        return torch.relu(torch.randn(B, K, generator=g)).to(BF)
    return ints(g, (B, K), 0, 3, BF)


def head_params(g, K, A, dueling, gaussian=False):
    if gaussian:
        p = [torch.randn(A, K, generator=g) * 0.05, torch.randn(A, generator=g)]
        p += [torch.randn(1, K, generator=g) * 0.05, torch.randn(1, generator=g)] if dueling else [None, None]
    else:
        p = [ints(g, (A, K), -2, 2), ints(g, (A,), -3, 3)]
        p += [ints(g, (1, K), -2, 2), ints(g, (1,), -3, 3)] if dueling else [None, None]
    return p


def dev(t):
    return None if t is None else t.cuda()


def nan_like(shape, dtype=F32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def sentinel(shape):
    return torch.full(shape, SENT, dtype=BF, device="cuda")


def prefilled(g, shape):
    """Nonzero integers: the kernels must add to them."""
    v = ints(g, shape, 1, 4) * (1 - 2 * ints(g, shape, 0, 1))
    return v


# ================================================================================================= GPU fixture
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


def _lib():
    from deeprl_b200 import _lib
    return _lib


# ================================================================================================= narrow head kernels
# (B, K, A, dueling, relu): n_out = A + dueling reaches 1, 2, 8, 9, 19, 20 and 32 (NB = 8, 19, 32), K = 72 and 264 leave a
# partial 64-column block of the backward grid and a partial 256-feature chunk of head_row_dots
HEAD_CASES = [
    (1, 64, 1, False, False), (4, 72, 1, True, True), (16, 264, 8, False, True), (16, 264, 8, True, False),
    (512, 512, 19, False, True), (512, 512, 19, True, False), (2048, 512, 31, True, True), (37, 72, 31, False, False),
    (37, 512, 7, True, True), (4, 264, 16, True, True),
]


@gpu
@pytest.mark.parametrize("B,K,A,dueling,relu", HEAD_CASES)
def test_head_fwd_bwd_exact(rl, B, K, A, dueling, relu):
    """b2rl_head_fwd and b2rl_head_bwd(_relu) (csrc/head.cu) on integer data: q, gphi, the weight / bias gradients and the
    column sums against the float64 reference."""
    L = _lib()
    g = _gen(B * 1000 + K + A)
    phi = features(g, B, K)
    Wa, ba, Wv, bv = head_params(g, K, A, dueling)
    gq = ints(g, (B, A), -2, 2)
    n_out = A + int(dueling)
    # ---- forward
    d = head_dots(phi, Wa, ba, Wv, bv)
    assert_exact_premise((phi.to(F64) @ torch.cat([Wa] + ([Wv] if dueling else [])).to(F64).abs().t()), 1, "dot products")
    q_ref = head_q(d.float(), A, dueling)
    q = nan_like((B, A))
    D = [dev(t) for t in (phi, Wa, ba, Wv, bv, gq)]          # held until the kernels ran
    L.call("b2rl_head_fwd", *[L.ptr(t) for t in D[:5]], B, K, A, L.ptr(q), L.stream())
    # ---- backward, into pre-filled accumulators
    gphi = sentinel((B, K))
    inits = [prefilled(g, t.shape) for t in (Wa, ba)] + ([prefilled(g, t.shape) for t in (Wv, bv)] if dueling else [None, None])
    gWa, gba, gWv, gbv = [dev(t.clone()) if t is not None else None for t in inits]
    colsum0 = prefilled(g, (K,))
    colsum = dev(colsum0.clone())
    args = [L.ptr(D[5]), L.ptr(D[0]), L.ptr(D[1]), L.ptr(D[3]), B, K, A, L.ptr(gphi), L.ptr(gWa), L.ptr(gba),
            L.ptr(gWv), L.ptr(gbv)]
    if relu:
        L.call("b2rl_head_bwd_relu", *args, L.ptr(colsum), L.stream())
    else:
        L.call("b2rl_head_bwd", *args, L.stream())
    torch.cuda.synchronize()
    assert torch.equal(q.cpu(), q_ref), "q"
    if not dueling:
        assert torch.equal(q.cpu().to(F64), d), "plain head: q equals the float64 dot products"
    geff = head_geff(gq, A, dueling)                          # float32, kernel order
    exact = not dueling or _pow2(A)
    scale = grid(geff) if exact else 1.0
    if exact:
        assert torch.equal(geff.to(F64), head_geff(gq.to(F64), A, dueling)), "geff is exact"
    dphi, dW, db = head_bwd(geff, phi, Wa, Wv, relu)
    Wall = torch.cat([Wa] + ([Wv] if dueling else [])).to(F64)
    gphi_ref = dphi_kernel_order(geff, phi, Wa, Wv, relu)
    if exact:
        assert_exact_premise(geff.to(F64).abs() @ Wall.abs(), scale, "dphi")
        assert torch.equal(gphi_ref.to(F64), dphi.float().to(BF).to(F64)), "kernel-order dphi equals the float64 one"
    assert torch.equal(gphi.cpu(), gphi_ref), "gphi"
    x = phi.to(F64)
    abs_dW = geff.to(F64).abs().t() @ x
    n = B + 8
    check_sum(gWa, inits[0], dW[:A], abs_dW[:A], n, exact, scale, "dW_a")
    check_sum(gba, inits[1], db[:A], geff[:, :A].to(F64).abs().sum(0), n, exact, scale, "db_a")
    if dueling:
        check_sum(gWv, inits[2], dW[A:], abs_dW[A:], n, exact, scale, "dW_v")
        check_sum(gbv, inits[3], db[A:], geff[:, A:].to(F64).abs().sum(0), n, exact, scale, "db_v")
    if relu:
        # the column sums are those of the stored bf16 values (as the separate mask / bias-gradient pass computes them)
        gs = gphi_ref.to(F64)
        check_sum(colsum, colsum0, gs.sum(0), gs.abs().sum(0), n, exact, scale, "relu column sums")
    else:
        assert torch.equal(colsum.cpu(), colsum0), "relu_colsum untouched without the ReLU branch"
    assert n_out <= 32


@gpu
@pytest.mark.parametrize("B,K,A,dueling,relu", [(512, 512, 6, True, True), (37, 264, 18, False, False), (64, 512, 31, True, True)])
def test_head_fwd_bwd_gaussian(rl, B, K, A, dueling, relu):
    """Gaussian operands: every output within its first-order fp32 error bound of float64."""
    L = _lib()
    g = _gen(B + K + A + 7)
    phi = features(g, B, K, gaussian=True)
    Wa, ba, Wv, bv = head_params(g, K, A, dueling, gaussian=True)
    gq = torch.randn(B, A, generator=g) / B
    q = nan_like((B, A))
    D = [dev(t) for t in (phi, Wa, ba, Wv, bv, gq)]          # held until the kernels ran
    L.call("b2rl_head_fwd", *[L.ptr(t) for t in D[:5]], B, K, A, L.ptr(q), L.stream())
    gphi = sentinel((B, K))
    z = lambda t: None if t is None else torch.zeros_like(t, device="cuda")
    gWa, gba, gWv, gbv = z(Wa), z(ba), z(Wv), z(bv)
    colsum = torch.zeros(K, device="cuda")
    args = [L.ptr(D[5]), L.ptr(D[0]), L.ptr(D[1]), L.ptr(D[3]), B, K, A, L.ptr(gphi), L.ptr(gWa), L.ptr(gba),
            L.ptr(gWv), L.ptr(gbv)]
    if relu:
        L.call("b2rl_head_bwd_relu", *args, L.ptr(colsum), L.stream())
    else:
        L.call("b2rl_head_bwd", *args, L.stream())
    torch.cuda.synchronize()
    # forward: a lane's chain of K/32 fmas, 5 shuffle levels, the bias; the dueling combine adds A + 3 roundings of
    # quantities bounded by the largest |dot| of the row
    Wall = torch.cat([Wa] + ([Wv] if dueling else [])).to(F64)
    d = head_dots(phi, Wa, ba, Wv, bv)
    S = phi.to(F64) @ Wall.abs().t() + torch.cat([ba] + ([bv] if dueling else [])).to(F64).abs()
    if dueling:
        bound = (K // 32 + 8 + A + 3) * U * 3 * S.max(1, keepdim=True).values.expand(B, A)
    else:
        bound = (K // 32 + 8) * U * S
    assert_within(q, head_q(d, A, dueling), bound, "q")
    geff = head_geff(gq, A, dueling)                              # float32 as the kernel forms it
    dphi, dW, db = head_bwd(geff, phi, Wa, Wv, relu)
    absd = geff.to(F64).abs() @ Wall.abs()
    assert_within(gphi, dphi, 2.0 ** -8 * dphi.abs() + (A + 3) * U * absd, "gphi (fp32 chain + one bf16 rounding)")
    n = B + 8
    abs_dW = geff.to(F64).abs().t() @ phi.to(F64)
    assert_within(gWa, dW[:A], n * U * abs_dW[:A], "dW_a")
    assert_within(gba, db[:A], n * U * geff[:, :A].to(F64).abs().sum(0), "db_a")
    if dueling:
        assert_within(gWv, dW[A:], n * U * abs_dW[A:], "dW_v")
        assert_within(gbv, db[A:], n * U * geff[:, A:].to(F64).abs().sum(0), "db_v")
    if relu:
        gs = gphi.cpu().to(F64)
        assert_within(colsum, gs.sum(0), n * U * gs.abs().sum(0), "relu column sums")


# ================================================================================================= the DQN head in one / two launches
def _dqn_case(seed, B, K, A, dueling, double_q, gamma_n=0.5, per=False, gaussian=False, ties=None):
    g = _gen(seed)
    c = SimpleNamespace(B=B, K=K, A=A, dueling=dueling, gamma_n=gamma_n)
    c.phi, c.phi_t = features(g, B, K, gaussian), features(g, B, K, gaussian)
    c.phi_o = features(g, B, K, gaussian) if double_q else None
    c.Wa, c.ba, c.Wv, c.bv = head_params(g, K, A, dueling, gaussian)
    c.Wa_t, c.ba_t, c.Wv_t, c.bv_t = head_params(g, K, A, dueling, gaussian)
    if ties == "all":                       # every online advantage row identical: each q row is a tie of all actions
        c.Wa[:] = c.Wa[0]
        c.ba[:] = c.ba[0]
    elif ties == "pair":                    # actions 2 and 4 identical and dominant: the first maximum is 2
        c.Wa[4] = c.Wa[2]
        c.ba[2] = c.ba[4] = 1000.0
    c.action = torch.randint(0, A, (B,), generator=g)
    c.action[0] = A - 1
    c.reward = ints(g, (B,), -1, 1)
    c.mask = (torch.rand(B, generator=g) > 0.2).float()
    c.is_prob = (torch.rand(B, generator=g) * 1e-3 + 1e-6) if per else None
    return c


def _dqn_reference(c):
    """q, delta, geff of the case in float32 in the kernel's order (bit-exact on exact dot products), with the float64 dots."""
    ddots = lambda x, W, b, Wv, bv: head_dots(x, W, b, Wv, bv)
    q32 = lambda dd: head_q(dd.float(), c.A, c.dueling)
    d = ddots(c.phi, c.Wa, c.ba, c.Wv, c.bv)
    dt = ddots(c.phi_t, c.Wa_t, c.ba_t, c.Wv_t, c.bv_t)
    do = ddots(c.phi_o, c.Wa, c.ba, c.Wv, c.bv) if c.phi_o is not None else None
    r = SimpleNamespace(d=d, dt=dt, do=do, q=q32(d), qt=q32(dt), qo=None if do is None else q32(do))
    r.delta = dqn_delta(r.q, r.qt, r.qo, c.action, c.reward, c.mask, c.gamma_n)
    return r


def _run_dqn_head(c, two, g, scratch=None, init=None):
    """b2rl_dqn_head_two / b2rl_dqn_head_fused through the C ABI on sentinel-filled outputs and pre-filled accumulators."""
    L = _lib()
    B, K, A = c.B, c.K, c.A
    o = SimpleNamespace()
    o.gphi, o.q, o.delta = sentinel((B, K)), nan_like((B, A)), nan_like((B,))
    o.prio = nan_like((B,)) if c.is_prob is not None else None
    o.loss = nan_like((1,))
    if init is None:
        init = [prefilled(g, t.shape) if t is not None else None for t in (c.Wa, c.ba, c.Wv, c.bv)] + [prefilled(g, (K,))]
    o.init = init
    o.gWa, o.gba, o.gWv, o.gbv, o.colsum = [dev(t.clone()) if t is not None else None for t in init]
    o.scratch = scratch if scratch is not None else torch.zeros(B + 64, device="cuda")
    o.geff = nan_like((B, GEFF_LD))
    o.dev = {}                                           # device copies, held until the kernels ran

    def P(t):
        if t is None:
            return None
        o.dev[len(o.dev)] = dev(t)
        return L.ptr(o.dev[len(o.dev) - 1])
    args = [P(c.phi), P(c.phi_t), P(c.phi_o), P(c.Wa), P(c.ba), P(c.Wv), P(c.bv), P(c.Wa_t), P(c.ba_t), P(c.Wv_t), P(c.bv_t),
            P(c.action), P(c.reward), P(c.mask), float(c.gamma_n), B, K, A, P(c.is_prob), 0.4, None, 0.01, 0.5,
            L.ptr(o.gphi), L.ptr(o.gWa), L.ptr(o.gba), L.ptr(o.gWv), L.ptr(o.gbv), L.ptr(o.colsum), L.ptr(o.q),
            L.ptr(o.delta), L.ptr(o.prio), L.ptr(o.loss), L.ptr(o.scratch)]
    if two:
        L.call("b2rl_dqn_head_two", *args, L.ptr(o.geff), L.stream())
    else:
        L.call("b2rl_dqn_head_fused", *args, L.stream())
    torch.cuda.synchronize()
    return o


def _check_dqn_head(c, r, o, two, exact_data=True):
    """Every output of one b2rl_dqn_head_* call against the reference r."""
    B, K, A, dueling = c.B, c.K, c.A, c.dueling
    n_out = A + int(dueling)
    assert torch.equal(o.q.cpu(), r.q), "q"
    assert torch.equal(o.delta.cpu(), r.delta), "delta"
    w64 = None
    if c.is_prob is not None:
        from deeprl_b200 import ops
        ref = ops.dqn_loss_fused(dev(r.q), dev(r.qt), dev(r.qo), dev(c.action), dev(c.reward), dev(c.mask), c.gamma_n,
                                 is_prob=dev(c.is_prob), beta=0.4, eps=0.01, alpha=0.5)
        torch.cuda.synchronize()
        assert torch.equal(o.prio, ref["priority"]), "priorities bit-equal to dqn_loss_fused"
        p64 = (r.delta.to(F64).abs() + 0.01) ** 0.5
        assert_within(o.prio, p64, 2 * 2.0 ** -23 * p64, "priorities within 2 ulp of float64")
        # IS weights: dL/dq of the taken action is dqn_loss_fused's bit for bit (checked through geff below), and
        # -delta w^2 / B within the roundings of powf, of the division by the largest weight and of three products
        dq = ref["dq"].cpu()
        w64 = (c.is_prob.to(F64) * B + 1e-6) ** -0.4
        w64 = w64 / w64.max()
        g64 = -r.delta.to(F64) * w64 ** 2 / B
        assert_within(dq.gather(1, c.action[:, None])[:, 0], g64, 16 * U * g64.abs(), "IS-weighted gradient vs float64")
        geff = head_geff(dq, A, dueling)
    else:
        geff = dqn_geff(r.delta, c.action, A, dueling, B)
    exact = exact_data and _pow2(B) and (not dueling or _pow2(A)) and c.is_prob is None
    scale = grid(geff) if exact else 1.0                 # geff * scale are integers; W and phi are integers
    if exact:
        g64 = dqn_geff(r.delta.to(F64), c.action, A, dueling, B)
        assert torch.equal(geff.to(F64), g64), "geff is exact"
    if two:
        got = o.geff.cpu()
        assert torch.equal(got[:, :n_out], geff), "geff of the row kernel"
        assert bool(got[:, n_out:].isnan().all()), "no geff store past n_out"
    dphi, dW, db = head_bwd(geff, c.phi, c.Wa, c.Wv, relu=True)
    gphi_ref = dphi_kernel_order(geff, c.phi, c.Wa, c.Wv, relu=True)
    Wall = torch.cat([c.Wa] + ([c.Wv] if dueling else [])).to(F64)
    if exact:
        assert_exact_premise(geff.to(F64).abs() @ Wall.abs(), scale, "dphi")
        assert torch.equal(gphi_ref.to(F64), dphi.float().to(BF).to(F64))
    assert torch.equal(o.gphi.cpu(), gphi_ref), "gphi"
    abs_dW = geff.to(F64).abs().t() @ c.phi.to(F64)
    n = B + 8
    check_sum(o.gWa, o.init[0], dW[:A], abs_dW[:A], n, exact, scale, "dW_a")
    check_sum(o.gba, o.init[1], db[:A], geff[:, :A].to(F64).abs().sum(0), n, exact, scale, "db_a")
    if dueling:
        check_sum(o.gWv, o.init[2], dW[A:], abs_dW[A:], n, exact, scale, "dW_v")
        check_sum(o.gbv, o.init[3], db[A:], geff[:, A:].to(F64).abs().sum(0), n, exact, scale, "db_v")
    gs = gphi_ref.to(F64)
    check_sum(o.colsum, o.init[4], gs.sum(0), gs.abs().sum(0), n, exact, scale, "fc4 column sums")
    # loss = mean(0.5 (w delta)^2): B positive terms, each rounded twice, a reduction tree and the product with 1/B
    wl = r.delta.to(F64) * (1.0 if w64 is None else w64)
    l64 = (0.5 * wl ** 2).mean()
    n_loss = B + 8 if w64 is None else B + 40          # + the relative error of w^2
    assert_within(o.loss.cpu()[0], l64, torch.tensor(n_loss * U * float(l64) + 1e-30, dtype=F64), "loss")


# (B, K, A, dueling, double_q, two, gamma_n): every n_out boundary, each with the one- and the two-launch form somewhere
DQN_CASES = [
    (4, 64, 1, True, False, True, 1.0), (16, 64, 1, False, True, False, 0.5), (16, 72, 8, False, True, True, 0.5),
    (16, 72, 8, True, True, False, 1.0), (512, 512, 19, False, False, True, 0.5), (64, 264, 16, True, True, False, 0.5),
    (2048, 512, 20, False, True, True, 1.0), (1, 512, 31, False, False, False, 0.5), (512, 512, 31, True, True, True, 0.5),
    (512, 512, 31, True, False, False, 1.0), (37, 264, 18, True, False, False, 0.5), (37, 512, 6, False, True, True, 1.0),
    (2048, 512, 4, True, True, False, 0.5), (1, 72, 2, True, True, True, 0.5), (4, 512, 7, True, False, True, 0.5),
]


@gpu
@pytest.mark.parametrize("B,K,A,dueling,double_q,two,gamma_n", DQN_CASES)
def test_dqn_head_exact(rl, B, K, A, dueling, double_q, two, gamma_n):
    c = _dqn_case(B * 7 + K + A, B, K, A, dueling, double_q, gamma_n)
    r = _dqn_reference(c)
    o = _run_dqn_head(c, two, _gen(B + A))
    _check_dqn_head(c, r, o, two)


@gpu
@pytest.mark.parametrize("B,A,dueling,double_q,two", [(512, 6, True, True, True), (37, 18, False, False, False),
                                                      (64, 31, True, False, False)])
def test_dqn_head_per(rl, B, A, dueling, double_q, two):
    """PER block: priorities bit-equal to dqn_loss_fused and within 2 ulp of float64, IS-weighted gradients."""
    c = _dqn_case(B + A + 99, B, 512, A, dueling, double_q, 0.5, per=True)
    r = _dqn_reference(c)
    o = _run_dqn_head(c, two, _gen(B))
    _check_dqn_head(c, r, o, two)


@gpu
@pytest.mark.parametrize("two", [True, False])
def test_dqn_head_gaussian(rl, two):
    """Gaussian operands (plain head, max target): q and delta within the dot products' error bound of float64, the
    gradients within the accumulation bound of float64 sums of the kernel's own geff."""
    B, K, A = 256, 512, 6
    c = _dqn_case(5, B, K, A, False, False, 0.99, gaussian=True)
    o = _run_dqn_head(c, two, _gen(6))
    d = head_dots(c.phi, c.Wa, c.ba)
    dt = head_dots(c.phi_t, c.Wa_t, c.ba_t)
    S = lambda x, W, b: x.to(F64) @ W.to(F64).abs().t() + b.to(F64).abs()
    bq = (K // 32 + 8) * U * S(c.phi, c.Wa, c.ba)
    assert_within(o.q, d, bq, "q")
    delta64 = dqn_delta(d, dt, None, c.action, c.reward, c.mask, 0.99)
    bt = (K // 32 + 8) * U * S(c.phi_t, c.Wa_t, c.ba_t).max(1).values
    bd = bq.gather(1, c.action[:, None])[:, 0] + bt + 3 * U * (delta64.abs() + c.reward.abs().to(F64) + dt.abs().max(1).values)
    assert_within(o.delta, delta64, bd, "delta")
    geff = dqn_geff(o.delta.cpu(), c.action, A, False, B)      # float32 from the kernel's delta, in its order
    dphi, dW, db = head_bwd(geff, c.phi, c.Wa, None, relu=True)
    absd = geff.to(F64).abs() @ c.Wa.to(F64).abs()
    assert_within(o.gphi, dphi, 2.0 ** -8 * dphi.abs() + (A + 3) * U * absd, "gphi")
    n = B + 8
    assert_within(o.gWa, o.init[0].to(F64) + dW, n * U * (geff.to(F64).abs().t() @ c.phi.to(F64) + o.init[0].abs()), "dW")
    assert_within(o.gba, o.init[1].to(F64) + db, n * U * (geff.to(F64).abs().sum(0) + o.init[1].abs()), "db")


@gpu
@pytest.mark.parametrize("two", [True, False])
def test_dqn_head_loss_counter_two_batch_sizes(rl, two):
    """Consecutive calls with different B on the same scratch: the last-CTA counter re-arms itself and the second
    loss is that of the second batch (a stale partial or counter would give a wrong sum)."""
    scratch = torch.zeros(2048 + 64, device="cuda")
    for i, (B, A, dueling) in enumerate(((512, 6, True), (37, 4, False), (2048, 18, False), (16, 31, True))):
        c = _dqn_case(300 + i, B, 512, A, dueling, i % 2 == 0, 0.5)
        r = _dqn_reference(c)
        o = _run_dqn_head(c, two, _gen(i), scratch=scratch)
        _check_dqn_head(c, r, o, two)
        assert int(scratch[:1].view(torch.int32)) == 0, "the loss counter is re-armed"


@gpu
@pytest.mark.parametrize("ties", ["all", "pair"])
@pytest.mark.parametrize("dueling", [False, True])
@pytest.mark.parametrize("two", [True, False])
def test_dqn_head_double_q_ties(rl, ties, dueling, two):
    """Double-Q with tied online values on s': the head kernels take the FIRST maximum, as torch.argmax does (a later
    maximum picks another target value, so delta differs)."""
    B, K, A = 64, 264, 6
    c = _dqn_case(41 + int(dueling), B, K, A, dueling, True, 1.0, ties=ties)
    r = _dqn_reference(c)
    first = torch.argmax(r.qo, 1)
    assert bool((first == (0 if ties == "all" else 2)).all()), "the data has the intended ties"
    if ties == "pair":
        assert torch.equal(r.qo[:, 2], r.qo[:, 4])
    assert not torch.equal(r.qt.gather(1, first[:, None]), r.qt[:, 4 if ties == "pair" else A - 1:][:, :1]), \
        "a different choice would change the target"
    o = _run_dqn_head(c, two, _gen(3))
    _check_dqn_head(c, r, o, two)


@gpu
def test_dqn_loss_double_q_ties_vs_oracle(rl):
    """b2rl_dqn_loss on tied online values against oracle/losses.py (torch.argmax: the first maximum)."""
    from deeprl_b200 import ops
    from oracle import losses as oracle
    g = _gen(11)
    B, A = 300, 5
    q, qt = ints(g, (B, A), -4, 4), ints(g, (B, A), -4, 4)
    qo = ints(g, (B, A), -1, 1)                     # 3 values over 5 actions: most rows hold a tie at the maximum
    assert int((qo == qo.max(1, keepdim=True).values).sum(1).gt(1).sum()) > B // 2
    action, reward, mask = torch.randint(0, A, (B,), generator=g), ints(g, (B,), -1, 1), ints(g, (B,), 0, 1)
    want = oracle.dqn_delta(q.to(F64), qt.to(F64), qo.to(F64), action, reward.to(F64), mask.to(F64), 0.5)
    got = ops.dqn_loss_fused(dev(q), dev(qt), dev(qo), dev(action), dev(reward), dev(mask), 0.5)["delta"]
    assert torch.equal(got.cpu().to(F64), want)


@gpu
@pytest.mark.parametrize("double_q", [False, True])
def test_c51_ties_vs_oracle(rl, double_q):
    """C51 with identical expected values for different next-state distributions: the kernel takes the first maximum,
    as the oracle (torch.argmax) does, and gives its KL."""
    from deeprl_b200 import ops
    from oracle import losses as oracle
    g = _gen(12 + int(double_q))
    B, A, N, vmin, vmax = 64, 4, 51, -10.0, 10.0
    atoms = torch.tensor(np.linspace(vmin, vmax, N), dtype=F32)
    pn = torch.zeros(B, A, N)
    pn[:, :, 10] = 1.0                               # E = z_10 < 0 for every action ...
    lo, hi = torch.randint(0, 2, (B,), generator=g), torch.randint(2, 4, (B,), generator=g)
    rows = torch.arange(B)
    pn[rows, lo] = 0.0
    pn[rows, lo, 25] = 1.0                           # ... but E = z_25 = 0 for action lo
    pn[rows, hi] = 0.0
    pn[rows, hi, 0] = 0.5                            # ... and E = 0.5 v_min + 0.5 v_max = 0 for action hi > lo
    pn[rows, hi, N - 1] = 0.5
    e = (pn * atoms).sum(-1)
    assert torch.equal(e[rows, lo], e[rows, hi]) and torch.equal(torch.argmax(e, 1), lo), "tied expected values"
    lp = torch.log_softmax(torch.randn(B, A, N, generator=g), -1)
    action, reward, mask = torch.randint(0, A, (B,), generator=g), ints(g, (B,), -1, 1), ints(g, (B,), 0, 1)
    po = pn if double_q else None
    want = oracle.c51_kl(lp.to(F64), pn.to(F64), None if po is None else po.to(F64), action, reward.to(F64), mask.to(F64),
                         atoms.to(F64), vmin, vmax, 0.99)
    got = ops.c51_loss_fused(dev(lp), dev(pn), dev(po), dev(action), dev(reward), dev(mask), 0.99, vmin, vmax)["kl"]
    torch.cuda.synchronize()
    np.testing.assert_allclose(got.cpu().numpy(), want.numpy(), rtol=1e-5, atol=1e-5)


@gpu
def test_qr_ties_vs_oracle(rl):
    """QR-DQN with identical quantile sums for different next-state quantile vectors: first maximum, oracle loss."""
    from deeprl_b200 import ops
    from oracle import losses as oracle
    g = _gen(13)
    B, A, N = 32, 4, 200
    qn = ints(g, (B, A, N), -3, -1)                  # negative sums ...
    rows = torch.arange(B)
    lo, hi = torch.randint(0, 2, (B,), generator=g), torch.randint(2, 4, (B,), generator=g)
    qn[rows, lo] = 0.0                               # ... except two actions with sum 0 and different quantiles
    qn[rows, hi] = torch.tensor([-2.0, 2.0]).repeat(N // 2)
    s = qn.sum(-1)
    assert torch.equal(s[rows, lo], s[rows, hi]) and torch.equal(torch.argmax(s, 1), lo), "tied quantile sums"
    quant = torch.randn(B, A, N, generator=g)
    action, reward, mask = torch.randint(0, A, (B,), generator=g), ints(g, (B,), -1, 1), ints(g, (B,), 0, 1)
    want = oracle.qr_loss(quant.to(F64), qn.to(F64), action, reward.to(F64), mask.to(F64), 0.99)
    r = ops.qr_loss_fused(dev(quant), dev(qn), dev(action), dev(reward), dev(mask), 0.99)
    torch.cuda.synchronize()
    np.testing.assert_allclose(r["vec"].cpu().numpy(), want.numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(float(r["loss"]), float(want.mean()), rtol=1e-5)


# ================================================================================================= distributional head
@gpu
@pytest.mark.parametrize("rows,N", [(1, 51), (37 * 3, 51), (37 * 18, 200), (512 * 4, 51)])
def test_dist_softmax(rl, rows, N):
    """dist_softmax_kernel (rows not a multiple of its 8 rows per CTA included) within the fp32 bound of float64:
    log_prob = (x - m) - log(s) with s a sum of N expf values, prob = expf(x - m) / s."""
    L = _lib()
    g = _gen(rows + N)
    x = torch.randn(rows, N, generator=g) * 3
    prob, logp = nan_like((rows + 1, N)), nan_like((rows + 1, N))
    xd = dev(x)
    L.call("b2rl_dist_softmax", L.ptr(xd), rows, N, L.ptr(prob), L.ptr(logp), L.stream())
    torch.cuda.synchronize()
    lp64, p64 = log_softmax_fwd(x)
    assert_softmax_within(logp[:rows], prob[:rows], x, N)
    assert bool(prob[rows:].isnan().all() and logp[rows:].isnan().all()), "no store past the last row"


def _zero_sum_ints(g, shape):
    """Integers in {-1, 0, 1} whose sum over the last dimension is zero: the log_softmax backward d - p * sum(d) is then d,
    exactly, whatever p."""
    x = (torch.rand(shape, generator=g) < 0.125).float()
    perm = torch.argsort(torch.rand(shape, generator=g), -1)
    return x - x.gather(-1, perm)


@gpu
@pytest.mark.parametrize("B,A,N,softmax", [(1, 4, 51, True), (37, 4, 51, False), (37, 6, 51, True), (13, 18, 200, False),
                                           (512, 18, 51, True)])
def test_dist_bwd_prep_exact(rl, B, A, N, softmax):
    """b2rl_dist_head_bwd_prep: the bf16 operand (its padding columns [A*N, ld) zero), the bias gradient accumulated into
    pre-filled integers, B % 8 != 0 included (the tile rows past B are zero)."""
    L = _lib()
    g = _gen(B * A + N)
    AN = A * N
    ld = (AN + 7) // 8 * 8
    dout = _zero_sum_ints(g, (B, A, N)) if softmax else ints(g, (B, A, N), -2, 2)
    prob = torch.softmax(torch.randn(B, A, N, generator=g), -1) if softmax else None
    op = sentinel((B, ld))
    db0 = prefilled(g, (AN,))
    db = dev(db0.clone())
    dd, pd = dev(dout), dev(prob)
    L.call("b2rl_dist_head_bwd_prep", L.ptr(dd), L.ptr(pd), B, A, N, L.ptr(op), ld, L.ptr(db), L.stream())
    torch.cuda.synchronize()
    g_ref, v, dbias = dist_bwd_prep(dout, prob, ld)
    assert torch.equal(v, dout.to(F64).reshape(B, -1)), "integer operand"
    assert torch.equal(op.cpu(), g_ref), "bf16 operand and zero padding"
    if ld > AN:
        assert not bool(op[:, AN:].float().abs().gt(0).any())
    check_sum(db, db0, dbias, v.abs().sum(0), B + 8, True, 1, "bias gradient")


@gpu
@pytest.mark.parametrize("B,A,N", [(37, 4, 51), (512, 6, 51)])
def test_dist_bwd_prep_gaussian(rl, B, A, N):
    L = _lib()
    g = _gen(B + A + N + 1)
    AN = A * N
    ld = (AN + 7) // 8 * 8
    dout = torch.randn(B, A, N, generator=g) / B
    prob = torch.softmax(torch.randn(B, A, N, generator=g), -1)
    op = sentinel((B, ld))
    db = torch.zeros(AN, device="cuda")
    dd, pd = dev(dout), dev(prob)
    L.call("b2rl_dist_head_bwd_prep", L.ptr(dd), L.ptr(pd), B, A, N, L.ptr(op), ld, L.ptr(db), L.stream())
    torch.cuda.synchronize()
    _, v, dbias = dist_bwd_prep(dout, prob, ld)
    d64, p64 = dout.to(F64), prob.to(F64)
    tv = ((N + 3) * U * (d64.abs() + p64 * d64.abs().sum(-1, keepdim=True))).reshape(B, -1)
    assert_within(op[:, :AN], v, 2.0 ** -8 * v.abs() + tv, "operand (fp32 + one bf16 rounding)")
    assert not bool(op[:, AN:].float().abs().gt(0).any())
    assert_within(db, dbias, (B + 8) * U * v.abs().sum(0) + tv.sum(0), "bias gradient")


# (kind, A, N, B, relu): A*N = 204 / 306 / 918 (C51), 800 / 3600 (QR), never a multiple of 64; both backward branches
DIST_CASES = [
    ("c51", 4, 51, 1, True), ("c51", 4, 51, 37, False), ("c51", 6, 51, 512, True), ("c51", 18, 51, 37, True),
    ("c51", 18, 51, 512, False), ("qr", 4, 200, 37, True), ("qr", 18, 200, 1, False), ("qr", 18, 200, 512, True),
    ("qr", 4, 200, 512, False), ("c51", 6, 51, 37, True),
]


@gpu
@pytest.mark.parametrize("kind,A,N,B,relu", DIST_CASES)
def test_dist_head_exact(rl, kind, A, N, B, relu):
    """fused.dist_head (wgmma GEMMs + csrc/disthead.cu) on integer data.  ReLU branch: phi registered as fc4's ReLU output
    and a sink with db4, so dphi = relu_mask(g W) and fc4's column sums come from b2rl_gemm_bwd_bf16's epilogue."""
    from deeprl_b200.network import fused, nature_tc
    g = _gen(A * N + B + int(relu))
    K, AN = 512, A * N
    softmax = kind == "c51"
    fc = torch.nn.Linear(K, AN).cuda()
    with torch.no_grad():
        fc.weight.copy_(ints(g, (AN, K), -2, 2))
        fc.bias.copy_(ints(g, (AN,), -4, 4))
    fc._w16 = fc.weight.detach().to(BF)
    w0, b0 = prefilled(g, (AN, K)), prefilled(g, (AN,))
    fc.weight.grad, fc.bias.grad = dev(w0.clone()), dev(b0.clone())
    phi = dev(features(g, B, K)).requires_grad_(True)
    gout = _zero_sum_ints(g, (B, A, N))              # sparse, so that dphi stays exact in bf16
    db40 = prefilled(g, (K,))
    sink = SimpleNamespace(db4=dev(db40.clone()))
    before = set(nature_tc.PREMASKED)
    if relu:
        nature_tc.mark_relu_features(phi)
    try:
        with nature_tc.grad_sink(sink):
            out, prob = fused.dist_head(phi, fc, A, N, softmax)
            out.backward(dev(gout))
        torch.cuda.synchronize()
        new = [k for k in nature_tc.PREMASKED if k not in before]
        if relu:
            assert len(new) == 1 and nature_tc.PREMASKED[new[0]][1] is sink.db4, "the masked gradient is recorded with db4"
        else:
            assert not new
    finally:
        for k in [k for k in nature_tc.PREMASKED if k not in before]:
            del nature_tc.PREMASKED[k]
        nature_tc.RELU_FEATURES.pop(phi.data_ptr(), None)
    W, x = fc.weight.detach().cpu().to(F64), phi.detach().cpu().to(F64)
    logits = x @ W.t() + fc.bias.detach().cpu().to(F64)
    assert_exact_premise(x @ W.abs().t(), 1, "logits")
    if softmax:
        assert_softmax_within(out.detach().reshape(B * A, N), prob.reshape(B * A, N), logits.view(B * A, N), N)
    else:
        assert torch.equal(out.detach().cpu().to(F64), logits.view(B, A, N)), "quantiles"
    gv = gout.to(F64).reshape(B, AN)                  # the log_softmax backward of a zero-sum gradient is the gradient
    dphi = gv @ W
    if relu:
        dphi = dphi * (x > 0)
    assert_exact_premise(gv.abs() @ W.abs(), 1, "dphi")
    assert bf16_representable(dphi), "premise: dphi is exact in bf16"
    assert torch.equal(phi.grad.cpu().to(F64), dphi), "dphi"
    check_sum(fc.weight.grad, w0, gv.t() @ x, gv.abs().t() @ x, 0, True, 1, "dW")
    check_sum(fc.bias.grad, b0, gv.sum(0), gv.abs().sum(0), 0, True, 1, "db")
    if relu:
        check_sum(sink.db4, db40, dphi.sum(0), dphi.abs().sum(0), 0, True, 1, "fc4 column sums")
    else:
        assert torch.equal(sink.db4.cpu(), db40), "db4 untouched by the plain branch"


@gpu
@pytest.mark.parametrize("relu", [False, True])
def test_dist_head_gaussian(rl, relu):
    """C51 head on Gaussian operands: every gradient within the accumulation bound of float64."""
    from deeprl_b200.network import fused, nature_tc
    g = _gen(77 + int(relu))
    B, K, A, N = 37, 512, 4, 51
    AN = A * N
    fc = torch.nn.Linear(K, AN).cuda()
    fc._w16 = fc.weight.detach().to(BF)
    phi = dev(features(g, B, K, gaussian=True)).requires_grad_(True)
    gout = dev(torch.randn(B, A, N, generator=g) / B)
    sink = SimpleNamespace(db4=torch.zeros(K, device="cuda"))
    before = set(nature_tc.PREMASKED)
    if relu:
        nature_tc.mark_relu_features(phi)
    try:
        with nature_tc.grad_sink(sink):
            out, prob = fused.dist_head(phi, fc, A, N, True)
            out.backward(gout)
        torch.cuda.synchronize()
    finally:
        for k in [k for k in nature_tc.PREMASKED if k not in before]:
            del nature_tc.PREMASKED[k]
        nature_tc.RELU_FEATURES.pop(phi.data_ptr(), None)
    # reference from the kernel's own probabilities (checked against float64 by test_dist_softmax) and bf16 operand
    v = log_softmax_bwd(gout.cpu(), prob.detach().cpu()).reshape(B, AN)
    W, x = fc._w16.cpu().to(F64), phi.detach().cpu().to(F64)
    tv = (N + 3) * U * (gout.cpu().to(F64).abs() + prob.detach().cpu().to(F64) * gout.cpu().to(F64).abs().sum(-1, keepdim=True))
    tv = 2.0 ** -8 * v.abs() + tv.reshape(B, AN)           # the bf16 operand: fp32 error + one bf16 rounding
    dW = v.t() @ x
    assert_within(fc.weight.grad, dW, (B + 8) * U * (v.abs().t() @ x) + tv.t() @ x, "dW")
    assert_within(fc.bias.grad, v.sum(0), (B + 8) * U * v.abs().sum(0) + tv.sum(0), "db")
    dphi = v @ W
    m = (x > 0) if relu else torch.ones_like(x, dtype=torch.bool)
    tphi = (AN + 8) * U * (v.abs() @ W.abs()) + tv @ W.abs()
    assert_within(phi.grad, dphi * m, (2.0 ** -8 * dphi.abs() + tphi) * m, "dphi")
    if relu:
        assert_within(sink.db4, (dphi * m).sum(0), ((B + 8) * U * dphi.abs() + tphi).mul(m).sum(0), "fc4 column sums")


# ================================================================================================= address-keyed registries
@gpu
def test_relu_registry_survives_address_reuse(rl):
    """A bf16 NatureConvBody output (registered as relu(fc4) features) is freed and the allocator hands its address to a
    tanh FCBody feature tensor: the narrow head must NOT treat that tensor as ReLU features (which zeroes its gradient
    where it is negative), and its backward must leave no pre-masked entry behind for a later body backward to pick up."""
    from deeprl_b200.network import fused, nature_tc
    B, K, A = 4096, 512, 6
    torch.manual_seed(0)
    body = rl.NatureConvBody(in_channels=4).cuda()
    fcb = rl.FCBody(16, hidden_units=(K,), gate=torch.tanh_).cuda().to(BF)
    fa, fv = torch.nn.Linear(K, A).cuda(), torch.nn.Linear(K, 1).cuda()
    x0 = torch.randint(0, 256, (B, 64, 21, 21), device="cuda").to(BF).contiguous(memory_format=torch.channels_last)
    s = torch.randn(B, 16, device="cuda").to(BF)
    with torch.no_grad():
        body(x0)                                      # warm-up: packed weights and library workspaces exist outside the pool
    fcb(s).float().sum().backward()
    fcb.zero_grad()
    before = set(nature_tc.PREMASKED)
    # A private pool holding only the body's blocks: y4 (4 MB) is the first block of its own 20 MB segment, the freed
    # convolution outputs (26 MB and more) are larger, so the 4 MB feature tensor -- the first allocation of the FCBody
    # forward, its tanh works in place -- best fits y4's freed segment and starts at y4's address.
    pool = torch.cuda.MemPool()
    with torch.cuda.use_mem_pool(pool), torch.no_grad():
        y4 = body(x0)
    addr = y4.data_ptr()
    assert addr in nature_tc.RELU_FEATURES
    del y4
    with torch.cuda.use_mem_pool(pool):
        phi = fcb(s)
    assert phi.data_ptr() == addr, "precondition: the allocator did not hand the freed y4 address to the FCBody features"
    assert bool((phi < 0).any()), "the tanh features have negative entries"
    gq = torch.randn(B, A, device="cuda")
    q = fused.narrow_head(phi, fa, fv)
    q.backward(gq)
    # torch reference on the same bf16 features
    xr = phi.detach().float().requires_grad_(True)
    wa, ba_, wv, bv_ = [t.detach().clone().requires_grad_(True) for t in (fa.weight, fa.bias, fv.weight, fv.bias)]
    adv = xr @ wa.t() + ba_
    qr = (xr @ wv.t() + bv_) + (adv - adv.mean(1, keepdim=True))
    qr.backward(gq)
    torch.cuda.synchronize()
    np.testing.assert_allclose(q.detach().cpu().numpy(), qr.detach().cpu().numpy(), rtol=1e-5, atol=1e-4)
    gx = fcb.layers[0].weight.grad
    assert gx is not None
    for got, want in ((fa.weight.grad, wa.grad), (fa.bias.grad, ba_.grad), (fv.weight.grad, wv.grad), (fv.bias.grad, bv_.grad)):
        np.testing.assert_allclose(got.cpu().numpy(), want.cpu().numpy(), rtol=1e-4, atol=1e-5)
    # the gradient reaching the tanh features: through tanh_'s backward, compare the pre-activation's input gradient
    gphi = torch.autograd.grad(fused.narrow_head(phi, fa, fv), phi, gq)[0]
    np.testing.assert_allclose(gphi.float().cpu().numpy(), xr.grad.cpu().numpy(), rtol=1e-2, atol=1e-3)
    assert set(nature_tc.PREMASKED) == before, "no pre-masked gradient left behind"
    del q, gphi, phi
    torch.cuda.synchronize()


# ================================================================================================= CPU: pin the reference
def test_reference_head_forward_vs_linear():
    g = _gen(1)
    B, K, A = 9, 40, 5
    phi = torch.randn(B, K, generator=g, dtype=F64)
    Wa, ba, Wv, bv = [torch.randn(*s, generator=g, dtype=F64) for s in ((A, K), (A,), (1, K), (1,))]
    assert torch.allclose(head_dots(phi, Wa, ba)[:, :A], F.linear(phi, Wa, ba), rtol=1e-13, atol=1e-12)
    d = head_dots(phi, Wa, ba, Wv, bv)
    adv, v = F.linear(phi, Wa, ba), F.linear(phi, Wv, bv)
    want = v.expand_as(adv) + (adv - adv.mean(1, keepdim=True))          # network_heads.py DuelingNet
    assert torch.allclose(head_q(d, A, True), want, rtol=1e-13, atol=1e-12)


def test_reference_dueling_combine_float32_order():
    """The float32 combine is one sequential sum, one division and two subtractions / additions, each rounded once."""
    d = torch.tensor([[1.0, 2.0, 4.0, 10.0]], dtype=F32)
    q = dueling_combine(d, 3)
    mean = torch.tensor(7.0, dtype=F32) / 3.0
    assert torch.equal(q, 10.0 + (d[:, :3] - mean))


def test_reference_head_backward_vs_autograd():
    g = _gen(2)
    B, K, A = 7, 24, 5
    phi = torch.randn(B, K, generator=g, dtype=F64)
    Wa, ba, Wv, bv = [torch.randn(*s, generator=g, dtype=F64, requires_grad=True) for s in ((A, K), (A,), (1, K), (1,))]
    gq = torch.randn(B, A, generator=g, dtype=F64)
    for dueling in (False, True):
        for relu in (False, True):
            x = phi.clone().requires_grad_(True)
            xin = torch.relu(x) if relu else x
            d = head_dots(xin, Wa, ba, Wv if dueling else None, bv if dueling else None)
            q = head_q(d, A, dueling)
            grads = torch.autograd.grad((q * gq).sum(), [x, Wa, ba] + ([Wv, bv] if dueling else []))
            geff = head_geff(gq, A, dueling)
            dphi, dW, db = head_bwd(geff, torch.relu(phi) if relu else phi, Wa.detach(), Wv.detach() if dueling else None, relu)
            if relu:                                  # the kernel masks with phi > 0 where phi is the ReLU's output
                dphi = dphi * (phi > 0)
            assert torch.allclose(dphi, grads[0], rtol=1e-12, atol=1e-12)
            assert torch.allclose(dW[:A], grads[1], rtol=1e-12, atol=1e-12)
            assert torch.allclose(db[:A], grads[2], rtol=1e-12, atol=1e-12)
            if dueling:
                assert torch.allclose(dW[A:], grads[3], rtol=1e-12, atol=1e-12)
                assert torch.allclose(db[A:], grads[4], rtol=1e-12, atol=1e-12)


def test_reference_dqn_delta_and_geff_vs_oracle_and_autograd():
    """dqn_delta against oracle/losses.py, dqn_geff against autograd of mean(0.5 (w delta)^2) through the dueling combine."""
    from oracle import losses as oracle
    g = _gen(3)
    B, A = 16, 6
    for dueling in (False, True):
        d = torch.randn(B, A + int(dueling), generator=g, dtype=F64, requires_grad=True)
        qt, qo = torch.randn(B, A, generator=g, dtype=F64), torch.randn(B, A, generator=g, dtype=F64)
        action, reward, mask = torch.randint(0, A, (B,), generator=g), ints(g, (B,), -1, 1, F64), ints(g, (B,), 0, 1, F64)
        w = torch.rand(B, generator=g, dtype=F64) + 0.5
        for qn_o in (None, qo):
            q = head_q(d, A, dueling)
            delta = dqn_delta(q, qt, qn_o, action, reward, mask, 0.99)
            assert torch.allclose(delta, oracle.dqn_delta(q, qt, qn_o, action, reward, mask, 0.99), rtol=1e-14, atol=1e-14)
            loss = (0.5 * (w * delta) ** 2).mean()
            (gd,) = torch.autograd.grad(loss, d)
            assert torch.allclose(dqn_geff(delta.detach(), action, A, dueling, B, w), gd, rtol=1e-12, atol=1e-14)


def test_reference_log_softmax_and_dist_bwd_prep_vs_autograd():
    g = _gen(4)
    B, A, N, K = 3, 4, 51, 16
    x = torch.randn(B, A, N, generator=g, dtype=F64, requires_grad=True)
    lp, p = log_softmax_fwd(x)
    assert torch.allclose(lp, torch.log_softmax(x, -1), rtol=1e-13, atol=1e-13)
    assert torch.allclose(p, torch.softmax(x, -1), rtol=1e-13, atol=1e-15)
    dl = torch.randn(B, A, N, generator=g, dtype=F64)
    (gx,) = torch.autograd.grad((torch.log_softmax(x, -1) * dl).sum(), x)
    assert torch.allclose(log_softmax_bwd(dl, p.detach()), gx, rtol=1e-12, atol=1e-14)
    # operand and bias gradient of a linear layer under the log_softmax
    phi = torch.randn(B, K, generator=g, dtype=F64)
    W = torch.randn(A * N, K, generator=g, dtype=F64, requires_grad=True)
    b = torch.zeros(A * N, dtype=F64, requires_grad=True)
    out = torch.log_softmax(F.linear(phi, W, b).view(B, A, N), -1)
    gW, gb = torch.autograd.grad((out * dl).sum(), (W, b))
    op, v, dbias = dist_bwd_prep(dl, torch.softmax(F.linear(phi, W, b).view(B, A, N), -1).detach(), 208)
    assert op.shape == (B, 208) and not bool(op[:, A * N:].float().abs().gt(0).any()), "zero padding columns"
    assert torch.allclose(dbias, gb, rtol=1e-12, atol=1e-13)
    assert torch.allclose(v.t() @ phi, gW, rtol=1e-12, atol=1e-13)
    # QR: no softmax, the operand is the gradient itself
    _, v2, db2 = dist_bwd_prep(dl, None, 208)
    assert torch.equal(v2, dl.reshape(B, -1)) and torch.equal(db2, dl.reshape(B, -1).sum(0))


def test_reference_zero_sum_gradient_passes_log_softmax_backward_unchanged():
    g = _gen(5)
    d = _zero_sum_ints(g, (6, 4, 51))
    assert torch.equal(d.sum(-1), torch.zeros(6, 4)) and set(d.unique().tolist()) <= {-1.0, 0.0, 1.0}
    p = torch.softmax(torch.randn(6, 4, 51, generator=g, dtype=F64), -1)
    assert torch.equal(log_softmax_bwd(d, p), d.to(F64))


def test_reference_argmax_takes_the_first_maximum():
    """torch.argmax, which the reference and the oracle use, returns the first of tied maxima (the kernels' rule)."""
    x = torch.tensor([[1.0, 3.0, 3.0, 0.0], [2.0, 2.0, 2.0, 2.0], [0.0, -1.0, 5.0, 5.0]])
    assert torch.argmax(x, 1).tolist() == [1, 0, 2]
    assert torch.argmax(x.to(F64), 1).tolist() == [1, 0, 2]


@pytest.mark.parametrize("B,K,A,dueling,double_q,two,gamma_n", DQN_CASES)
def test_dqn_cases_meet_their_premise(B, K, A, dueling, double_q, two, gamma_n):
    """The data of every exact DQN head case keeps its sums below 2**24 (checked on the CPU, where the data is made)."""
    c = _dqn_case(B * 7 + K + A, B, K, A, dueling, double_q, gamma_n)
    r = _dqn_reference(c)
    Wall = torch.cat([c.Wa] + ([c.Wv] if dueling else [])).to(F64)
    assert_exact_premise(c.phi.to(F64) @ Wall.abs().t(), 1, "dot products")
    assert torch.equal(r.q.to(F64), head_q(r.d, A, dueling)) or (dueling and not _pow2(A))
    if _pow2(B) and (not dueling or _pow2(A)):
        geff = dqn_geff(r.delta, c.action, A, dueling, B)
        assert torch.equal(geff.to(F64), dqn_geff(r.delta.to(F64), c.action, A, dueling, B))
        scale = grid(geff)
        assert_exact_premise(geff.to(F64).abs() @ Wall.abs(), scale, "dphi")
        assert_exact_premise(geff.to(F64).abs().t() @ c.phi.to(F64) + 4, scale, "dW")
