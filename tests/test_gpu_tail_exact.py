"""The tail of the DQN update compared EXACTLY with a float64 reference: csrc/tail.cu (kernel A nature_grad_reduce_kernel:
split-K gradient reduce, layout map, bias gradients, per-unit sums of squares and clip_grad_norm_'s coefficient; kernel B
nature_fused_opt_kernel: RMSprop / centered RMSprop / Adam, gradient re-zeroing, bf16 shadow and packed GEMM operands) and
the optimizer entry points of csrc/optim.cu behind FlatOptimizer (b2rl_clip_rmsprop, b2rl_clip_adam, b2rl_clip_adam_gated,
b2rl_grad_norm).

Reference contract.  The C ABI receives lr, alpha, betas and eps as float32, so the reference applies torch's RMSprop,
centered RMSprop and Adam formulas, and clip_grad_norm_'s min(max_norm / (norm + 1e-6), 1), to the float32-rounded
hyperparameters, evaluated in float64.  The CPU tests at the end pin it against torch.optim and clip_grad_norm_.

Exactness by choice of data.  Gradients are integers from {0, +-1, +-3, +-7} (sparse, so that the sum of squares of the
whole 1.7 M-element arena stays below 2**24 and every sum of them is exact in any order).  Split-K partials are integers
that add up to the wanted gradient; partial slots past the count hold 2**20, so a read past the count changes the sum.
The clip is off or inactive and grad_scale is a power of two, so the coefficient is exactly grad_scale.  The optimizer
state before each step is built from the effective gradient gr so that every intermediate of the update is a float32
number (RMSprop: alpha = 1/2, avg = |gr| 2**j, square_avg_old = 2 r**2 - gr**2 with r = avg - eps, so the new square_avg
is r**2 and gr / avg = +-2**-j; Adam: step 1 from zero moments with betas (1/2, 3/4) and eps = grad_scale, so every update
is lr v / (|v| + 1) for the integer v).  Then any FMA contraction gives the same bits and the checks are torch.equal.  Each
case asserts that premise on its own data.  Adam's step 1 is the only exact Adam step: no dyadic beta2 makes
1 - beta2**t a square for t > 1.

Gaussian cases at the production arena (VanillaNet(18) / DuelingNet(18) on NatureConvBody, production hyperparameters)
are teacher-forced: each step's reference starts from the kernel's own state, gradient and coefficient, and every element
is held to a first-order bound of the kernel's operation sequence on that element's data (powf's 4-ulp error in the bias
corrections included).

Outputs are pre-filled with sentinels: the gradient arena's body regions with -12345 before kernel A, the bf16 shadow and
the packed operands with bf16 -12345 before kernel B, so that a missing store fails."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu

F64, F32, BF = torch.float64, torch.float32, torch.bfloat16
U = 2.0 ** -24              # unit roundoff of fp32
EXACT = 2.0 ** 24           # integer sums whose |terms| add up to less than this are exact in fp32, in any order
SENT = -12345.0
BIG = 2.0 ** 20             # partial slots past the partial count
U_PLAIN, U_W1, U_W2, U_W3, U_W4, U_B1, U_B2, U_B3, U_B4 = range(9)
MAX_UNIT = 4 * 256 * 4      # kernel B: MAXV float4 per thread x 256 threads; elements past this are never updated
P_COUNTS = (1, 3, 4, 5, 28, 29, 32, 33, 36)   # both sides of p + 28 < P, the remainder loop, B = 32 / 512 counts
LR_EXACT = 2.0 ** -10


def f32(x):
    """A hyperparameter as the C ABI receives it."""
    return float(np.float32(x))


def hyper(lr, a, b, eps):
    return SimpleNamespace(lr=f32(lr), a=f32(a), b=f32(b), eps=f32(eps))


# ================================================================================================= float64 reference
def clip_coef(norm, max_norm, grad_scale):
    """clip_grad_norm_'s factor min(max_norm / (norm + 1e-6), 1) times grad_scale (max_norm <= 0: no clip).  ``norm`` is
    the norm of grad * grad_scale."""
    c = max_norm / (norm + 1e-6) if max_norm > 0 else 1.0
    return min(c, 1.0) * grad_scale


def coef_f32(norm, max_norm, grad_scale):
    """The same in float32, in the kernels' order."""
    n, one = np.float32(norm), np.float32(1.0)
    c = np.float32(max_norm) / (n + np.float32(1e-6)) if np.float32(max_norm) > 0 else one
    return float(np.float32(min(c, one)) * np.float32(grad_scale))


def rmsprop_ref(p, gr, sq, ga, hp, centered, trace=None):
    """torch.optim.RMSprop (_single_tensor_rmsprop, no momentum / weight decay) in float64 with the float32
    hyperparameters ``hp``; ``gr`` is the gradient after the clip coefficient.  Returns (param, square_avg, grad_avg).
    ``trace``: a list that receives every intermediate value."""
    t = trace if trace is not None else []
    a_sq, w_gr = hp.a * sq, (1 - hp.a) * gr
    s = a_sq + w_gr * gr
    t += [gr, a_sq, w_gr, w_gr * gr, s]
    if centered:
        d = gr - ga
        ga = ga + (1 - hp.a) * d                   # grad_avg.lerp_(grad, 1 - alpha)
        var = s - ga * ga
        t += [d, (1 - hp.a) * d, ga, ga * ga, var]
    else:
        var = s
    root = torch.sqrt(var)
    avg = root + hp.eps
    ratio = gr / avg
    p = p - hp.lr * ratio
    t += [root, avg, ratio, hp.lr * ratio, p]
    return p, s, ga


def adam_ref(p, gr, m, v, step, hp, trace=None):
    """torch.optim.Adam (_single_tensor_adam, foreach=False, no weight decay / amsgrad) in float64 with the float32
    hyperparameters (hp.a = beta1, hp.b = beta2).  Returns (param, exp_avg, exp_avg_sq)."""
    t = trace if trace is not None else []
    d = gr - m
    m = m + (1 - hp.a) * d                          # exp_avg.lerp_(grad, 1 - beta1)
    b_v, w_gr = hp.b * v, (1 - hp.b) * gr
    v = b_v + w_gr * gr
    pw1, pw2 = hp.a ** step, hp.b ** step
    bc1, bc2 = 1 - pw1, 1 - pw2
    step_size, bc2s = hp.lr / bc1, math.sqrt(bc2)
    root = torch.sqrt(v)
    q = root / bc2s
    denom = q + hp.eps
    ratio = m / denom
    p = p - step_size * ratio
    t += [gr, d, (1 - hp.a) * d, m, b_v, w_gr, w_gr * gr, v, root, q, denom, ratio, step_size * ratio, p]
    t += [torch.tensor([pw1, pw2, bc1, bc2, step_size, bc2s], dtype=F64)]
    return p, m, v


def representable(x):
    x = x.to(F64)
    return bool(torch.equal(x.float().to(F64), x))


def assert_premise(trace, what):
    """Every intermediate of the update is a float32 number: each rounding of the kernel is exact, FMA or not."""
    for i, x in enumerate(trace):
        assert bool(torch.isfinite(x).all()), "%s: intermediate %d not finite" % (what, i)
        assert representable(x), "%s: intermediate %d is not a float32 number" % (what, i)


# ------------------------------------------------------------------------------------------------- first-order bounds
def sqrt_err(d, e):
    """|sqrt(d + err) - sqrt(d)| for |err| <= e (float64 tensors)."""
    d = d.clamp_min(0.0)
    lin = torch.where(d > 0, e / torch.sqrt(d), torch.full_like(d, math.inf))
    return torch.minimum(lin, torch.sqrt(e))


def lerp_err(old, gr, new, w):
    """old + w (gr - old) with gr carrying one rounding (g * coef): sub, mul, add."""
    return w * U * (gr.abs() + 2 * (gr - old).abs()) + U * new.abs()


def sq_avg_err(old, gr, new, w):
    """(1 - w) old + w gr gr with old >= 0: two products, gr's own rounding twice, one add."""
    return U * ((1 - w) * old + 4 * w * gr * gr + new)


def rmsprop_bounds(p, gr, sq, ga, hp, centered):
    """Per-element first-order bounds (|param|, |square_avg|, |grad_avg| errors) of the kernel's operation sequence
    against rmsprop_ref on the same inputs.  gr = g * coef exactly (the kernel rounds it once)."""
    w = 1 - hp.a
    p1, s, ga1 = rmsprop_ref(p, gr, sq, ga, hp, centered)
    es = sq_avg_err(sq, gr, s, w)
    if centered:
        ega = lerp_err(ga, gr, ga1, w)
        var = s - ga1 * ga1
        evar = es + 2 * ga1.abs() * ega + U * ga1 * ga1 + U * var.abs()
    else:
        ega, var, evar = torch.zeros_like(gr), s, es
    root = torch.sqrt(var.clamp_min(0.0))
    avg = root + hp.eps
    eavg = sqrt_err(var, evar) + U * root + U * avg
    ratio = (gr / avg).abs()
    eratio = ratio * (2 * U + eavg / avg)
    ep = hp.lr * eratio + U * hp.lr * ratio + U * p1.abs()
    return ep, es, ega


def adam_bounds(p, gr, m, v, step, hp):
    """As rmsprop_bounds for Adam; powf is within 4 ulp (CUDA C Programming Guide, single-precision functions)."""
    p1, m1, v1 = adam_ref(p, gr, m, v, step, hp)
    em = lerp_err(m, gr, m1, 1 - hp.a)
    ev = sq_avg_err(v, gr, v1, 1 - hp.b)
    pw1, pw2 = hp.a ** step, hp.b ** step
    bc1, bc2 = 1 - pw1, 1 - pw2
    ebc1, ebc2 = 8 * U * pw1 + U * bc1, 8 * U * pw2 + U * bc2
    ss, bc2s = hp.lr / bc1, math.sqrt(bc2)
    ess = ss * (ebc1 / bc1 + U)
    ebc2s = ebc2 / (2 * bc2s) + U * bc2s
    root = torch.sqrt(v1)
    q = root / bc2s
    eq = (sqrt_err(v1, ev) + U * root) / bc2s + q * (ebc2s / bc2s + U)
    denom = q + hp.eps
    ed = eq + U * denom
    ratio = (m1 / denom).abs()
    er = em / denom + ratio * (ed / denom + U)
    ep = ess * ratio + ss * er + U * ss * ratio + U * p1.abs()
    return ep, em, ev


def assert_within(got, ref, bound, what):
    err = (got.to(F64).cpu() - ref.to(F64).cpu()).abs()
    bad = ~(err <= bound.cpu())
    assert not bool(bad.any()), "%s: %d of %d elements beyond the bound (worst err %.3g, its bound %.3g)" % (
        what, int(bad.sum()), bad.numel(), float(err.max()), float(bound.cpu().reshape(-1)[int(err.argmax())]))


def ulps(a, b):
    """Distance in float32 ulps of b."""
    return abs(float(a) - float(b)) / float(np.spacing(np.float32(abs(float(b)))))


# ================================================================================================= float32 emulation (CPU pins)
def rmsprop_f32(p, g, coef, sq, ga, hp, centered):
    """The kernel's operation sequence in float32, one rounding per operation (no contraction)."""
    c = lambda x: torch.tensor(x, dtype=F32)
    one, a = c(1.0), c(hp.a)
    gr = g * c(coef)
    s = a * sq + ((one - a) * gr) * gr
    if centered:
        ga = ga + (one - a) * (gr - ga)
        avg = torch.sqrt(s - ga * ga) + c(hp.eps)
    else:
        avg = torch.sqrt(s) + c(hp.eps)
    return p - c(hp.lr) * (gr / avg), s, ga


def adam_f32(p, g, coef, m, v, step, hp):
    c = lambda x: torch.tensor(x, dtype=F32)
    one, b1, b2 = c(1.0), c(hp.a), c(hp.b)
    gr = g * c(coef)
    m = m + (one - b1) * (gr - m)
    v = b2 * v + ((one - b2) * gr) * gr
    t = c(float(step))
    bc1, bc2 = one - torch.pow(b1, t), one - torch.pow(b2, t)
    ss, bc2s = c(hp.lr) / bc1, torch.sqrt(bc2)
    denom = torch.sqrt(v) / bc2s + c(hp.eps)
    return p - ss * (m / denom), m, v


# ================================================================================================= layouts (restated packers)
def pack_w1f(w1):      # [32][(ty, tx, c, dy, dx)]: 8x8 / stride 4 = 2x2 taps over the space-to-depth(4) grid
    n, c = w1.shape[:2]
    return w1.reshape(n, c, 2, 4, 2, 4).permute(0, 2, 4, 1, 3, 5).reshape(n, 4 * c * 16)


def pack_w2f(w2):      # [64][(ty, tx, py, px, c)]
    return w2.reshape(64, 32, 2, 2, 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(64, 512)


def pack_w2d(w2):      # [(py, px, c)][(ty, tx, n)]: conv2's dgrad operand
    return w2.reshape(64, 32, 2, 2, 2, 2).permute(3, 5, 1, 2, 4, 0).reshape(128, 256)


def pack_w3f(w3):      # [64][(dy, dx, c)]
    return w3.permute(0, 2, 3, 1).reshape(64, 576)


def pack_w3d(w3):      # [c][(dy, dx, n)]
    return w3.permute(1, 2, 3, 0).reshape(64, 576)


def pack_w4p(w4):      # fc4 columns in (h, w, c) order
    return w4.reshape(-1, 64, 7, 7).permute(0, 2, 3, 1).reshape(w4.shape[0], 3136)


PACKERS = (pack_w1f, pack_w2f, pack_w3f, pack_w4p)


def unpack(G, packer, shape):
    """Inverse of a packer: the reference-layout tensor whose packed form is G."""
    n = math.prod(shape)
    idx = packer(torch.arange(n).view(shape)).reshape(-1)
    out = torch.empty(n, dtype=G.dtype)
    out[idx] = G.reshape(-1)
    return out.view(shape)


def ref_index(kind, k, c1):
    """Python mirror of tail.cu ref_index: index in the reference layout of a row of GEMM-layout element k."""
    if kind == U_W1:
        per = 16 * c1
        tap = k // per
        c = k - tap * per
        f, dy, dx, ty, tx = c >> 4, (c & 15) >> 2, c & 3, tap >> 1, tap & 1
        return (f * 8 + 4 * ty + dy) * 8 + 4 * tx + dx
    if kind == U_W2:
        tap, r = k >> 7, k & 127
        ty, tx, py, px, c = tap >> 1, tap & 1, r >> 6, (r >> 5) & 1, r & 31
        return (c * 4 + 2 * ty + py) * 4 + 2 * tx + px
    if kind == U_W3:
        return (k & 63) * 9 + (k >> 6)
    return (k & 63) * 49 + (k >> 6)


def packed_ref(body, scale):
    """The six bf16 GEMM operands of the body's current fp32 weights (conv1 pre-multiplied by ``scale`` in float32)."""
    w1, w2, w3, w4 = [m.weight.detach().cpu() for m in (body.conv1, body.conv2, body.conv3, body.fc4)]
    w1 = w1 * torch.tensor(f32(scale), dtype=F32)
    return [t.to(BF) for t in (pack_w1f(w1), pack_w2f(w2), pack_w2d(w2), pack_w3f(w3), pack_w3d(w3), pack_w4p(w4))]


def unit_elements(units, c1):
    """(arena index, unit id) of every element kernel A reads or writes for each unit of a unit table."""
    idx, uid = [], []
    for i, (off, ln, kind, w) in enumerate(units.tolist()):
        if U_W1 <= kind <= U_W3:
            e = off + ref_index(kind, (w >> 16) * 256 + torch.arange(ln), c1)
        else:
            e = off + torch.arange(ln)
        idx.append(e)
        uid.append(torch.full((ln,), i))
    return torch.cat(idx), torch.cat(uid)


# ================================================================================================= data
def _gen(seed):
    return torch.Generator().manual_seed(seed)


VALS = torch.tensor([0.0, 1.0, -1.0, 3.0, -3.0, 7.0, -7.0], dtype=F64)
PROBS = torch.tensor([0.5, 0.2, 0.2, 0.04, 0.04, 0.01, 0.01])


def sparse_ints(g, shape):
    """Integers from {0, +-1, +-3, +-7} (E[v^2] = 2.1): |v| + 1 is a power of two, as the exact Adam step needs."""
    n = math.prod(shape)
    return VALS[torch.multinomial(PROBS, n, replacement=True, generator=g)].view(shape)


def split_partials(g, S, P):
    """[P + 2, *S.shape] float32 integer partials whose first P add up to S (float64 integers); two more slots of 2**20."""
    x = torch.randint(-1, 2, (P + 2,) + tuple(S.shape), generator=g).to(F64)
    x[0] = S - x[1:P].sum(0)
    x[P:] = BIG
    assert float(x[:P].abs().sum(0).max()) < EXACT
    return x.float()


def arena_size(net):
    return sum((p.numel() + 3) // 4 * 4 for p in net.parameters())


# ================================================================================================= GPU fixture + harness
@pytest.fixture(scope="module")
def rl():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import deeprl_b200 as rl
    rl.select_device(0)
    return rl


def _lib():
    from deeprl_b200 import _lib
    return _lib


def exact_hyper(kind, gs):
    """Hyperparameters of the exact cases for grad_scale gs: RMSprop eps = gs / 8, Adam eps = gs."""
    if kind == "adam":
        return hyper(LR_EXACT, 0.5, 0.75, gs)
    return hyper(LR_EXACT, 0.5, 0.0, gs / 8)


PROD = {"rmsprop": hyper(2.5e-4, 0.95, 0.0, 0.01), "centered": hyper(2.5e-4, 0.95, 0.0, 0.01),
        "adam": hyper(2.5e-4, 0.9, 0.999, 0.01 / 32)}


def make_opt(rl, params, kind, hp, shadow):
    o = rl.ops.FlatOptimizer(params, "adam" if kind == "adam" else "rmsprop", hp.lr, alpha=hp.a, eps=hp.eps,
                             centered=kind == "centered", betas=(hp.a, hp.b))
    if shadow:
        o.shadow = torch.full((o.n,), SENT, dtype=BF, device="cuda")
    return o


def set_hyper(o, hp):
    o.lr, o.eps = hp.lr, hp.eps
    if o.kind == "adam":
        o.betas = (hp.a, hp.b)
    else:
        o.alpha = hp.a


class Tail:
    """A NatureConvBody network, its FlatOptimizer arena and NatureTail, with the arena layout on the host."""

    def __init__(self, rl, head, kind, hp, c1=4, scale=2.0 ** -8, A=18, seed=0, shadow=True):
        from deeprl_b200.network.tail import NatureTail
        torch.manual_seed(seed)
        body = rl.NatureConvBody(in_channels=c1)
        self.net = rl.DuelingNet(A, body) if head == "dueling" else rl.VanillaNet(A, body)
        self.body, self.kind, self.c1, self.scale = body, kind, c1, scale
        self.o = make_opt(rl, self.net.parameters(), kind, hp, shadow)
        self.tail = NatureTail(self.o, body, scale)
        o = self.o
        self.n = o.n
        base = o.flat.data_ptr()
        off = lambda p: (p.data_ptr() - base) // 4
        mods = (body.conv1, body.conv2, body.conv3, body.fc4)
        self.w = [(off(m.weight), tuple(m.weight.shape)) for m in mods]
        self.b = [(off(m.bias), m.bias.numel()) for m in mods]
        self.real = torch.zeros(self.n, dtype=torch.bool)            # parameter elements (False: padding)
        self.body_mask = torch.zeros(self.n, dtype=torch.bool)
        for name, p in self.net.named_parameters():
            self.real[off(p):off(p) + p.numel()] = True
            if name.startswith("body."):
                self.body_mask[off(p):off(p) + p.numel()] = True
        self.head_mask = self.real & ~self.body_mask
        self.a_units = self.tail.a_units.cpu()
        self.a_idx, self.a_uid = unit_elements(self.a_units, c1)

    def gemm_sums(self, ref):
        """The four weight gradients in reference layout -> GEMM layout (packers)."""
        return [pk(r) for pk, r in zip(PACKERS, ref)]

    def arena_of(self, wref, bias, head):
        """Flat float64 arena holding the four reference-layout weight gradients, the biases and the head values."""
        a = torch.zeros(self.n, dtype=F64)
        for (o_, shp), r in zip(self.w, wref):
            a[o_:o_ + math.prod(shp)] = r.reshape(-1)
        for (o_, k), r in zip(self.b, bias):
            a[o_:o_ + k] = r
        a[self.head_mask] = head
        return a

    def exact_grads(self, g, scale_mode_exact=True):
        """Integer gradients of every parameter.  Returns (arena float64 the tail must write, kernel inputs)."""
        shapes = [s for _, s in self.w]
        v = [sparse_ints(g, s) for s in shapes]
        if scale_mode_exact:                 # conv1: sums 2**8 v, times scale 2**-8 = v exactly
            T1 = v[0] * (1.0 / self.scale)
            a1 = v[0]
        else:                                 # conv1: integer sums times scale, one float32 rounding
            T1 = sparse_ints(g, shapes[0]) * torch.randint(1, 40, shapes[0], generator=g).to(F64)
            a1 = (T1.float() * torch.tensor(f32(self.scale), dtype=F32)).to(F64)
        bias = [sparse_ints(g, (k,)) for _, k in self.b]
        head = sparse_ints(g, (int(self.head_mask.sum()),))
        sums = self.gemm_sums([T1] + v[1:])
        return self.arena_of([a1] + v[1:], bias, head), SimpleNamespace(sums=sums, bias=bias, head=head)

    def gaussian_grads(self, g):
        shapes = [s for _, s in self.w]
        sums = [None] * 4
        f32_ = lambda t: t.float().to(F64)               # the float32 values the kernels receive
        bias = [f32_(torch.randn(k, generator=g, dtype=F64) * 0.05) for _, k in self.b]
        head = f32_(torch.randn(int(self.head_mask.sum()), generator=g, dtype=F64) * 0.05)
        return SimpleNamespace(sums=sums, bias=bias, head=head, shapes=shapes)

    def load(self, inp, P, g, gaussian=False):
        """Kernel A's inputs on the device: split-K partials, fc4's GEMM-layout gradient, bias accumulators, the head's
        gradient in the arena, the body's arena regions set to the sentinel.  Returns the partial tensors (float32 CPU)."""
        parts = []
        for layer in range(3):
            if gaussian:
                rows, L = self.w[layer][1][0], math.prod(self.w[layer][1][1:])
                x = torch.randn((P[layer] + 2, rows, L), generator=g) * (0.02 / math.sqrt(P[layer]))
                x[P[layer]:] = BIG
            else:
                x = split_partials(g, inp.sums[layer], P[layer])
            parts.append(x)
        g4 = (torch.randn((self.w[3][1][0], 3136), generator=g) * 0.01) if gaussian else inp.sums[3].float()
        parts.append(g4)
        self.dev_parts = [t.cuda() for t in parts]
        for d, b in zip((self.tail.db1, self.tail.db2, self.tail.db3, self.tail.db4), inp.bias):
            d.copy_(b.float())
        gin = torch.zeros(self.n, dtype=F32)
        gin[self.body_mask] = SENT
        gin[self.head_mask] = inp.head.float()
        self.o.grad.copy_(gin)
        return parts

    def reduce(self, P):
        d = self.dev_parts
        self.tail.reduce(d[0], P[0], d[1], P[1], d[2], P[2], d[3])

    def arena_from_partials(self, parts, P, inp):
        """float64 arena of Gaussian partials (summed in float64, unpacked) and the bound of kernel A's fp32 sums."""
        wref, bnd = [], []
        for layer in range(4):
            shp = self.w[layer][1]
            x = parts[layer].to(F64)
            if layer < 3:
                S, A_ = x[:P[layer]].sum(0), x[:P[layer]].abs().sum(0)
                eb = (P[layer] + 4) * U * A_
            else:
                S, eb = x, torch.zeros_like(x)
            S, eb = unpack(S, PACKERS[layer], shp), unpack(eb, PACKERS[layer], shp)
            if layer == 0:
                S, eb = S * f32(self.scale), eb * f32(self.scale) + U * (S * f32(self.scale)).abs()
            wref.append(S)
            bnd.append(eb)
        return self.arena_of(wref, inp.bias, inp.head), \
            self.arena_of(bnd, [torch.zeros(k, dtype=F64) for _, k in self.b], torch.zeros_like(inp.head))

    def unit_sums(self, arena):
        """float64 sum of squares of the arena over each unit of kernel A's table."""
        return torch.zeros(len(self.a_units), dtype=F64).index_add_(0, self.a_uid, arena[self.a_idx] ** 2)

    def sentinel_outputs(self):
        for t in self.tail.packed().tensors():
            t.fill_(SENT)
        if self.o.shadow is not None:
            self.o.shadow.fill_(SENT)

    def state(self):
        o = self.o
        return SimpleNamespace(p=o.flat.cpu().to(F64), g=o.grad.cpu().to(F64), s1=o.s1.cpu().to(F64),
                               s2=o.s2.cpu().to(F64), step=int(o.step_dev), sc=o.scratch[:3].cpu().clone())

    def check_after_step(self, what):
        """The gradient arena is zero, the shadow is the bf16 parameters, the packed operands are the packers of the new
        fp32 weights."""
        o = self.o
        assert float(o.grad.abs().max()) == 0.0, "%s: kernel B re-zeroes the gradient arena" % what
        if o.shadow is not None:
            assert torch.equal(o.shadow, o.flat.to(BF)), "%s: shadow == bf16(parameters)" % what
        for i, (got, want) in enumerate(zip(self.tail.packed().tensors(), packed_ref(self.body, self.scale))):
            assert torch.equal(got.cpu(), want), "%s: packed operand %d" % (what, i)


def dyadic_state(g, gr, kind, gs, p=None):
    """Optimizer state before an exact step with effective gradient gr (float64, integers times gs).  Returns
    (p, s1, s2) float64; p is kept when given (it stays on the update's grid)."""
    n = gr.numel()
    if kind == "adam":
        if p is None:
            p = torch.randint(-2 ** 12, 2 ** 12, (n,), generator=g).to(F64) * 2.0 ** -13
        return p, torch.zeros(n, dtype=F64), torch.zeros(n, dtype=F64)
    if p is None:
        p = torch.randint(-2 ** 11, 2 ** 11, (n,), generator=g).to(F64) * 2.0 ** -12
    eps = gs / 8
    j = torch.randint(0, 3, (n,), generator=g).to(F64)
    r_free = torch.randint(1, 33, (n,), generator=g).to(F64) * eps
    avg = torch.where(gr != 0, gr.abs() * 2.0 ** j, r_free + eps)
    r = avg - eps
    if kind == "centered":
        ga_new = torch.randint(-16, 17, (n,), generator=g).to(F64) * eps
        return p, 2 * (r * r + ga_new * ga_new) - gr * gr, 2 * ga_new - gr
    return p, 2 * r * r - gr * gr, torch.zeros(n, dtype=F64)


def exact_step_ref(kind, p, gr, s1, s2, hp, what):
    """Reference of one exact step (asserting its premise): (p, s1, s2) float64."""
    tr = []
    assert bool((s1 >= 0).all()), "%s: square averages are non-negative" % what
    if kind == "adam":
        out = adam_ref(p, gr, s1, s2, 1, hp, tr)
    else:
        out = rmsprop_ref(p, gr, s1, s2, hp, kind == "centered", tr)
    assert_premise(tr + [p, s1, s2], what)
    return out


def write_state(o, p, s1, s2):
    o.flat.copy_(p.float())
    o.s1.copy_(s1.float())
    o.s2.copy_(s2.float())


# ================================================================================================= kernel A alone
# (P, c1, head, kind, grad_scale, clip, conv1 scale): every partial count, c1 up to 16 (4 segments per conv1 row), Adam's
# step bump, clip off / inactive / active, grad_scale 1/3, and conv1's production scale 1/255
REDUCE_CASES = [
    (1, 4, "vanilla", "rmsprop", 1.0, "off", 2.0 ** -8), (3, 8, "dueling", "adam", 0.5, "inactive", 1 / 255),
    (4, 4, "dueling", "rmsprop", 0.25, "active", 2.0 ** -8), (5, 12, "vanilla", "adam", 1 / 3, "active", 2.0 ** -8),
    (28, 4, "vanilla", "centered", 1 / 3, "off", 1 / 255), (29, 16, "dueling", "rmsprop", 1.0, "active", 2.0 ** -8),
    (32, 4, "dueling", "adam", 0.5, "off", 2.0 ** -8), (33, 4, "vanilla", "rmsprop", 1.0, "inactive", 1 / 255),
    (36, 8, "vanilla", "adam", 0.25, "active", 2.0 ** -8),
]


@gpu
@pytest.mark.parametrize("P,c1,head,kind,gs,clip,scale", REDUCE_CASES)
def test_grad_reduce_exact(rl, P, c1, head, kind, gs, clip, scale):
    """Kernel A (NatureTail.reduce) on integer data, three consecutive calls: the arena through the inverse of the packers
    (padding zero), the bias accumulators re-zeroed, every unit's sum of squares, norm = sqrtf(t) * grad_scale and the
    coefficient in float32, the counter re-armed, Adam's step bumped once per call."""
    T = Tail(rl, head, kind, exact_hyper(kind, 1.0), c1=c1, scale=scale, seed=P)
    g = _gen(P * 100 + c1)
    o, tail = T.o, T.tail
    exact_scale = scale == 2.0 ** -8
    o.step_dev.fill_(5)
    for call in range(3):
        want, inp = T.exact_grads(g, exact_scale)
        assert float((want ** 2).sum()) < EXACT, "premise: the sum of squares of the arena is an exact fp32 integer"
        T.load(inp, (P, P, P), g)
        u = T.unit_sums(want)
        t = float(u.sum())
        norm = float(np.float32(np.sqrt(np.float32(t))) * np.float32(gs))
        max_norm = {"off": 0.0, "inactive": 1e6, "active": f32(0.5 * norm)}[clip]
        tail.max_norm, tail.grad_scale = max_norm, gs
        T.reduce((P, P, P))
        torch.cuda.synchronize()
        what = "call %d" % call
        assert torch.equal(o.grad.cpu().to(F64), want), "%s: gradient arena" % what
        assert float(o.grad.cpu()[~T.real].abs().max()) == 0.0, "%s: padding stays zero" % what
        assert float(tail.db.abs().max()) == 0.0, "%s: bias accumulators re-zeroed" % what
        got_u = tail.unit_sumsq.cpu().to(F64)
        if exact_scale:
            assert torch.equal(got_u, u), "%s: unit sums of squares" % what
            assert float(o.scratch[0]) == norm, "%s: norm = sqrtf(t) * grad_scale" % what
        else:
            # conv1's values are fl(T / 255): each square rounds once, a unit's 256 of them are added in a tree
            w1 = (T.a_units[:, 2] == U_W1)
            assert torch.equal(got_u[~w1], u[~w1]), "%s: unit sums of squares (integer units)" % what
            assert_within(got_u[w1], u[w1], (256 + 16) * U * u[w1], "%s: conv1 unit sums of squares" % what)
            t64 = float(u.sum())
            et = (len(u) // 256 + 16) * U * t64 + float(((256 + 16) * U * u[w1]).sum())
            n64 = math.sqrt(t64) * gs
            assert abs(float(o.scratch[0]) - n64) <= (et / (2 * math.sqrt(t64)) * gs + 2 * U * n64), "%s: norm" % what
            norm = float(o.scratch[0])
        # coefficient from the kernel's own norm; for grad_scale 1/3 the compiler may contract sqrtf(t) * gs + 1e-6f into
        # one FMA, which can move the coefficient by one ulp
        want_c = coef_f32(norm, max_norm, gs)
        got_c = float(o.scratch[1])
        if clip == "active":
            assert want_c < gs, "premise: the clip is active"
        else:
            assert want_c == f32(gs), "premise: coefficient = grad_scale"
        if gs in (1.0, 0.5, 0.25):
            assert got_c == want_c, "%s: coefficient" % what
        else:
            assert ulps(got_c, want_c) <= 1.0, "%s: coefficient within 1 ulp (FMA contraction)" % what
        assert int(o.scratch[2:3].view(torch.int32)) == 0, "%s: last-CTA counter re-armed" % what
        assert int(o.step_dev) == (5 + call + 1 if kind == "adam" else 5), "%s: Adam step bump" % what
        o.grad.zero_()


# ================================================================================================= reduce + step, exact
GS_SCHEDULE = ((1.0, 0.0), (0.5, 1e6), (0.25, 0.0))          # (grad_scale, max_norm) of consecutive steps
P_SCHEDULE = ((1, 28, 33), (3, 29, 36), (4, 5, 32))


@gpu
@pytest.mark.parametrize("kind", ["rmsprop", "centered", "adam"])
@pytest.mark.parametrize("head", ["vanilla", "dueling"])
def test_tail_step_exact(rl, kind, head):
    """NatureTail.reduce + step, three consecutive updates: parameters, moments, step count exact; gradient re-zeroed;
    shadow and packed operands rewritten from sentinels."""
    T = Tail(rl, head, kind, exact_hyper(kind, 1.0), seed=7)
    g = _gen(11 + len(kind) + len(head))
    o, tail = T.o, T.tail
    p = None
    for step, ((gs, max_norm), P) in enumerate(zip(GS_SCHEDULE, P_SCHEDULE)):
        what = "step %d" % step
        hp = exact_hyper(kind, gs)
        set_hyper(o, hp)
        want, inp = T.exact_grads(g)
        T.load(inp, P, g)
        if kind == "adam":
            o.step_dev.zero_()
        tail.max_norm, tail.grad_scale = max_norm, gs
        T.reduce(P)
        torch.cuda.synchronize()
        assert torch.equal(o.grad.cpu().to(F64), want), "%s: kernel A arena" % what
        assert float(o.scratch[1]) == gs, "%s: coefficient = grad_scale" % what
        gr = want * gs
        p, s1, s2 = dyadic_state(g, gr, kind, gs, p)
        write_state(o, p, s1, s2)
        T.sentinel_outputs()
        ref = exact_step_ref(kind, p, gr, s1, s2, hp, what)
        tail.step(max_norm=max_norm, grad_scale=gs)
        torch.cuda.synchronize()
        assert torch.equal(o.flat.cpu().to(F64), ref[0]), "%s: parameters" % what
        assert torch.equal(o.s1.cpu().to(F64), ref[1]), "%s: square_avg / exp_avg" % what
        if kind != "rmsprop":
            assert torch.equal(o.s2.cpu().to(F64), ref[2]), "%s: grad_avg / exp_avg_sq" % what
        assert int(o.step_dev) == (1 if kind == "adam" else 0)
        T.check_after_step(what)
        p = ref[0]


@gpu
@pytest.mark.parametrize("kind,W", [("rmsprop", 2), ("centered", 3), ("adam", 4), ("adam", 3), ("rmsprop", 4),
                                    ("centered", 2)])
def test_tail_split_reduce_and_reduced_elsewhere(rl, kind, W):
    """Multi-GPU tail on one GPU: reduce_w4 + reduce_rest write the arena reduce writes and bump Adam's step once; then an
    all-reduce of W ranks holding the same gradient is simulated (arena * W) and step(reduced_elsewhere=True,
    grad_scale=1/W) recomputes the norm over the arena (b2rl_grad_norm) and takes the exact step."""
    from deeprl_b200 import _lib
    T = Tail(rl, "dueling" if W % 2 else "vanilla", kind, exact_hyper(kind, 1.0), seed=W)
    g = _gen(W * 10 + len(kind))
    o, tail = T.o, T.tail
    gs = 1.0 / W
    p = None
    for step, P in enumerate(P_SCHEDULE):
        what = "step %d" % step
        hp = exact_hyper(kind, 1.0)                   # the effective gradient is the rank's own: (W g) / W
        set_hyper(o, hp)
        want, inp = T.exact_grads(g)
        T.load(inp, P, g)
        o.step_dev.zero_()
        tail.max_norm, tail.grad_scale = 0.0, 1.0
        T.reduce(P)
        torch.cuda.synchronize()
        full = o.grad.clone()
        assert torch.equal(full.cpu().to(F64), want), "%s: reduce" % what
        # the same sums (split into other partials) through the split tables
        T.load(inp, P, g)
        o.step_dev.zero_()
        tail.reduce_w4(T.dev_parts[3])
        tail.reduce_rest(T.dev_parts[0], P[0], T.dev_parts[1], P[1], T.dev_parts[2], P[2])
        torch.cuda.synchronize()
        assert torch.equal(o.grad, full), "%s: reduce_w4 + reduce_rest write the arena reduce writes" % what
        assert float(tail.db.abs().max()) == 0.0, "%s: bias accumulators re-zeroed" % what
        assert int(o.step_dev) == (1 if kind == "adam" else 0), "%s: Adam's step bumped once" % what
        o.grad.mul_(float(W))                           # all-reduce (sum) of W identical ranks
        summed = o.grad.cpu()
        assert torch.equal(summed * torch.tensor(f32(gs), dtype=F32), want.float()), \
            "premise: (W g) * fl(1/W) rounds back to g"
        gr = want
        p, s1, s2 = dyadic_state(g, gr, kind, 1.0, p)
        write_state(o, p, s1, s2)
        T.sentinel_outputs()
        ref = exact_step_ref(kind, p, gr, s1, s2, hp, what)
        tail.step(max_norm=0.0, grad_scale=gs, reduced_elsewhere=True)
        torch.cuda.synchronize()
        t = float((want ** 2).sum())
        assert t < EXACT
        assert float(o.scratch[0]) == float(np.sqrt(np.float32(t))), "%s: norm over the all-reduced arena" % what
        assert float(o.scratch[1]) == f32(gs), "%s: coefficient 1/W" % what
        assert torch.equal(o.flat.cpu().to(F64), ref[0]), "%s: parameters" % what
        assert torch.equal(o.s1.cpu().to(F64), ref[1]), "%s: first moment" % what
        if kind != "rmsprop":
            assert torch.equal(o.s2.cpu().to(F64), ref[2]), "%s: second moment" % what
        T.check_after_step(what)
        p = ref[0]


@gpu
@pytest.mark.parametrize("kind", ["rmsprop", "centered", "adam"])
def test_fused_opt_unit_partials_branch(rl, kind):
    """Kernel B given the unit partials (every CTA adds them itself) matches the branch NatureTail uses (the coefficient
    from the norm scratch) bit for bit: parameters, moments, gradient, shadow, packed operands, norm and coefficient."""
    L = _lib()
    T = Tail(rl, "dueling", kind, PROD[kind], scale=1 / 255, seed=3)
    g = _gen(5)
    o, tail = T.o, T.tail
    hp = PROD[kind]
    for step in range(3):
        inp = T.gaussian_grads(g)
        T.load(inp, (33, 29, 36), g, gaussian=True)
        tail.max_norm, tail.grad_scale = (0.25, 1 / 3) if step != 1 else (0.0, 1.0)
        T.reduce((33, 29, 36))
        saved = [t.clone() for t in (o.flat, o.grad, o.s1, o.s2, o.step_dev, o.scratch)]
        T.sentinel_outputs()
        tail.step(max_norm=tail.max_norm, grad_scale=tail.grad_scale)
        out_a = [t.clone() for t in (o.flat, o.grad, o.s1, o.s2, o.shadow)] + [t.clone() for t in tail.packed().tensors()]
        sc_a = o.scratch[:2].clone()
        for dst, src in zip((o.flat, o.grad, o.s1, o.s2, o.step_dev, o.scratch), saved):
            dst.copy_(src)
        T.sentinel_outputs()
        o.scratch[:2] = float("nan")
        pk = tail.packed()
        a, b = (hp.a, hp.b) if kind == "adam" else (hp.a, 0.0)
        L.call("b2rl_nature_fused_opt", L.ptr(tail.b_units), tail.n_b, L.ptr(o.flat), L.ptr(o.grad), L.ptr(o.s1),
               L.ptr(o.s2), tail.kind, hp.lr, a, b, hp.eps, float(tail.max_norm), float(tail.grad_scale),
               L.ptr(tail.unit_sumsq), tail.n_a, L.ptr(o.scratch), L.ptr(o.step_dev), tail.c1, tail.n4, tail.scale,
               L.ptr(pk.w1f), L.ptr(pk.w2f), L.ptr(pk.w2d), L.ptr(pk.w3f), L.ptr(pk.w3d), L.ptr(pk.w4p), 1,
               L.ptr(o.shadow), L.stream())
        torch.cuda.synchronize()
        out_b = [o.flat, o.grad, o.s1, o.s2, o.shadow] + list(pk.tensors())
        for i, (x, y) in enumerate(zip(out_a, out_b)):
            assert torch.equal(x, y), "step %d: output %d differs between the two coefficient branches" % (step, i)
        assert torch.equal(sc_a, o.scratch[:2]), "step %d: norm and coefficient" % step


# ================================================================================================= FlatOptimizer entry points
FLAT_SHAPES = [(512, 3136), (18, 512), (37,), (5, 3), (1,)]      # > 296 * 2048 elements: the grid-stride loops run


@gpu
@pytest.mark.parametrize("kind", ["rmsprop", "centered", "adam"])
@pytest.mark.parametrize("shadow", [True, False])
def test_clip_optimizer_exact(rl, kind, shadow):
    """b2rl_clip_rmsprop / b2rl_clip_adam (FlatOptimizer.step), three consecutive steps on exact data: parameters and
    moments exact, the gradient untouched, the norm of grad * grad_scale exact, the coefficient grad_scale."""
    g = _gen(21 + len(kind) + int(shadow))
    params = [torch.nn.Parameter(torch.zeros(s, device="cuda")) for s in FLAT_SHAPES]
    o = make_opt(rl, params, kind, exact_hyper(kind, 1.0), shadow)
    real = torch.zeros(o.n, dtype=torch.bool)
    for off, p in zip(o.offsets, params):
        real[off:off + p.numel()] = True
    p = None
    for step, (gs, max_norm) in enumerate(GS_SCHEDULE):
        what = "step %d" % step
        hp = exact_hyper(kind, gs)
        set_hyper(o, hp)
        v = torch.zeros(o.n, dtype=F64)
        v[real] = sparse_ints(g, (int(real.sum()),))
        gr = v * gs
        p, s1, s2 = dyadic_state(g, gr, kind, gs, p)
        write_state(o, p, s1, s2)
        o.grad.copy_(v.float())
        if kind == "adam":
            o.step_dev.zero_()
        if shadow:
            o.shadow.fill_(SENT)
        ref = exact_step_ref(kind, p, gr, s1, s2, hp, what)
        o.step(max_norm=max_norm, grad_scale=gs)
        torch.cuda.synchronize()
        t = float((gr ** 2).sum())
        assert t * (1 / gs) ** 2 < EXACT, "premise: exact sum of squares"
        assert float(o.scratch[0]) == float(np.sqrt(np.float32(t))), "%s: norm" % what
        assert float(o.scratch[1]) == gs, "%s: coefficient" % what
        assert int(o.scratch[2:3].view(torch.int32)) == 0, "%s: counter re-armed" % what
        assert torch.equal(o.flat.cpu().to(F64), ref[0]), "%s: parameters" % what
        assert torch.equal(o.s1.cpu().to(F64), ref[1]), "%s: first moment" % what
        if kind != "rmsprop":
            assert torch.equal(o.s2.cpu().to(F64), ref[2]), "%s: second moment" % what
        assert torch.equal(o.grad.cpu().to(F64), v), "%s: FlatOptimizer.step leaves the gradient alone" % what
        if shadow:
            assert torch.equal(o.shadow, o.flat.to(BF)), "%s: shadow" % what
        if kind == "adam":
            assert int(o.step_dev) == 1
        p = ref[0]


@gpu
def test_clip_adam_gated(rl):
    """b2rl_clip_adam_gated: open (gate < max, gate == max) steps exactly; closed (gate > max, gate NaN) changes neither
    parameters, moments, step count nor shadow."""
    g = _gen(31)
    params = [torch.nn.Parameter(torch.zeros(s, device="cuda")) for s in FLAT_SHAPES[1:]]
    o = make_opt(rl, params, "adam", exact_hyper("adam", 1.0), True)
    real = torch.zeros(o.n, dtype=torch.bool)
    for off, prm in zip(o.offsets, params):
        real[off:off + prm.numel()] = True
    gate = torch.zeros(1, device="cuda")
    p = None
    for i, (gval, gmax, is_open) in enumerate([(0.5, 1.0, True), (2.0, 1.0, False), (float("nan"), 1.0, False),
                                                (1.0, 1.0, True), (float("nan"), 1.0, False), (1.5, 1.25, False),
                                                (-3.0, -2.0, True)]):
        what = "call %d (gate %r, max %r)" % (i, gval, gmax)
        gate.fill_(gval)
        v = torch.zeros(o.n, dtype=F64)
        v[real] = sparse_ints(g, (int(real.sum()),))
        o.grad.copy_(v.float())
        if is_open:
            p, s1, s2 = dyadic_state(g, v, "adam", 1.0, p)
            write_state(o, p, s1, s2)
            o.step_dev.zero_()
            ref = exact_step_ref("adam", p, v, s1, s2, exact_hyper("adam", 1.0), what)
        before = [t.clone() for t in (o.flat, o.s1, o.s2, o.step_dev, o.shadow)]
        o.step(max_norm=0.0, gate=gate, gate_max=gmax)
        torch.cuda.synchronize()
        if is_open:
            assert torch.equal(o.flat.cpu().to(F64), ref[0]), "%s: parameters" % what
            assert torch.equal(o.s1.cpu().to(F64), ref[1]) and torch.equal(o.s2.cpu().to(F64), ref[2]), what
            assert int(o.step_dev) == 1, "%s: step bumped" % what
            assert torch.equal(o.shadow, o.flat.to(BF)), "%s: shadow" % what
            p = ref[0]
        else:
            for j, (x, y) in enumerate(zip(before, (o.flat, o.s1, o.s2, o.step_dev, o.shadow))):
                assert torch.equal(x, y), "%s: state %d changed by a closed gate" % (what, j)
        assert torch.equal(o.grad.cpu().to(F64), v)


@gpu
def test_adam_powf_calibration(rl):
    """Premise of the exact Adam cases: on the device, 1 - powf(beta, 1) is 1 - beta and every other operation of step 1 is
    exact for dyadic betas whose 1 - beta2 is a square, so the update is exactly lr v / (|v| + 1) (g = v eps) for every
    beta1 in {1/2, 3/4, 7/8} and beta2 in {3/4, 15/16, 63/64}.  A powf(beta, 1) one ulp off would move step_size or
    sqrt(bc2) and every nonzero update with it."""
    g = _gen(41)
    params = [torch.nn.Parameter(torch.zeros(4096, device="cuda"))]
    o = make_opt(rl, params, "adam", exact_hyper("adam", 1.0), False)
    for b1 in (0.5, 0.75, 0.875):
        for b2 in (0.75, 0.9375, 63 / 64):
            for eps in (1.0, 2.0 ** -7):
                hp = hyper(LR_EXACT, b1, b2, eps)
                set_hyper(o, hp)
                v = sparse_ints(g, (o.n,))
                o.grad.copy_((v * eps).float())
                o.flat.zero_()
                o.s1.zero_()
                o.s2.zero_()
                o.step_dev.zero_()
                o.step()
                torch.cuda.synchronize()
                want = -LR_EXACT * v / (v.abs() + 1)
                tr = []
                ref = adam_ref(torch.zeros(o.n, dtype=F64), v * eps, torch.zeros(o.n, dtype=F64),
                               torch.zeros(o.n, dtype=F64), 1, hp, tr)
                assert_premise(tr, "betas (%g, %g)" % (b1, b2))
                assert torch.equal(ref[0], want)
                assert torch.equal(o.flat.cpu().to(F64), want), "betas (%g, %g) eps %g" % (b1, b2, eps)


GRAD_NORM_N = [1, 5, 4099, 296 * 2048, 296 * 2048 + 4, None]     # None: the VanillaNet(18) NatureConvBody arena


@gpu
@pytest.mark.parametrize("n", GRAD_NORM_N)
def test_grad_norm_exact(rl, n):
    """b2rl_grad_norm: scalar tail (n % 4 != 0), exactly one full grid, the grid-stride loop and the production arena;
    three consecutive calls on one scratch (clip off, active, inactive) with elements past n at 1e4."""
    L = _lib()
    if n is None:
        n = arena_size(rl.VanillaNet(18, rl.NatureConvBody(in_channels=4)))
    g = _gen(n % 1000 + 3)
    buf = torch.full((n + 64,), 1e4, dtype=F32)
    v = sparse_ints(g, (n,))
    v[-1] = 7.0                                     # the last element counts
    buf[:n] = v.float()
    d = buf.cuda()
    scratch = torch.zeros(512, device="cuda")
    for call, (gs, mode) in enumerate(((1.0, "off"), (0.25, "active"), (0.5, "inactive"))):
        t = float(((v * gs) ** 2).sum())
        assert t / gs ** 2 < EXACT, "premise: exact sum of squares"
        norm = float(np.sqrt(np.float32(t)))
        max_norm = {"off": 0.0, "active": f32(norm / 3), "inactive": 1e6}[mode]
        scratch[:2] = float("nan")
        L.call("b2rl_grad_norm", L.ptr(d), n, gs, max_norm, L.ptr(scratch), L.stream())
        torch.cuda.synchronize()
        assert float(scratch[0]) == norm, "call %d: norm" % call
        want_c = coef_f32(norm, max_norm, gs)
        assert (want_c < gs) == (mode == "active")
        assert float(scratch[1]) == want_c, "call %d: coefficient" % call
        assert int(scratch[2:3].view(torch.int32)) == 0, "call %d: counter re-armed" % call


# ================================================================================================= Gaussian, production arena
@gpu
@pytest.mark.parametrize("kind", ["rmsprop", "centered", "adam"])
@pytest.mark.parametrize("head", ["vanilla", "dueling"])
@pytest.mark.parametrize("clip", ["active", "inactive"])
def test_tail_gaussian_teacher_forced(rl, kind, head, clip):
    """Production arena and hyperparameters, Gaussian gradients, three updates.  Kernel A's arena within the bound of its
    fp32 partial sums, its unit sums and norm within n 2**-24 sum g**2 of the kernel's own arena, the coefficient from its
    norm; kernel B's parameters and moments within the first-order bound of its operation sequence, teacher-forced from
    the kernel's state, gradient and coefficient."""
    hp = PROD[kind]
    T = Tail(rl, head, kind, hp, scale=1 / 255, seed=17)
    g = _gen(19 + len(kind) + len(head) + len(clip))
    o, tail = T.o, T.tail
    max_norm = 5.0 if clip == "active" else 1e4
    P = (29, 33, 4)
    for step in range(3):
        what = "step %d" % step
        inp = T.gaussian_grads(g)
        parts = T.load(inp, P, g, gaussian=True)
        tail.max_norm, tail.grad_scale = max_norm, 1.0
        T.reduce(P)
        torch.cuda.synchronize()
        st = T.state()
        want, bnd = T.arena_from_partials(parts, P, inp)
        assert_within(st.g, want, bnd, "%s: kernel A arena" % what)
        u = T.unit_sums(st.g)
        depth = 64 + len(u) // 256                  # additions behind one term: thread loop, block trees, unit sum
        assert_within(tail.unit_sumsq.cpu(), u, depth * U * u, "%s: unit sums of squares" % what)
        t64 = float((st.g ** 2).sum())
        n64 = math.sqrt(t64)
        assert abs(float(st.sc[0]) - n64) <= depth * U * t64 / (2 * n64) + 2 * U * n64, "%s: norm" % what
        coef = float(st.sc[1])
        assert ulps(coef, coef_f32(float(st.sc[0]), max_norm, 1.0)) <= 1.0, "%s: coefficient" % what
        assert (coef < 1.0) == (clip == "active"), "premise: the clip is %s" % clip
        T.sentinel_outputs()
        tail.step(max_norm=max_norm, grad_scale=1.0)
        torch.cuda.synchronize()
        gr = st.g * coef
        if kind == "adam":
            assert int(o.step_dev) == st.step == step + 1
            ref = adam_ref(st.p, gr, st.s1, st.s2, st.step, hp)
            bounds = adam_bounds(st.p, gr, st.s1, st.s2, st.step, hp)
        else:
            ref = rmsprop_ref(st.p, gr, st.s1, st.s2, hp, kind == "centered")
            bounds = rmsprop_bounds(st.p, gr, st.s1, st.s2, hp, kind == "centered")
        assert_within(o.flat, ref[0], bounds[0], "%s: parameters" % what)
        assert_within(o.s1, ref[1], bounds[1], "%s: first moment" % what)
        if kind != "rmsprop":
            assert_within(o.s2, ref[2], bounds[2], "%s: second moment" % what)
        moved = (o.flat.cpu().to(F64) - st.p).abs()
        assert float(moved.max()) > 0, "the update moved the parameters"
        T.check_after_step(what)


@gpu
@pytest.mark.parametrize("head", ["vanilla", "dueling"])
def test_unit_tables(rl, head):
    """NatureTail's kernel B table tiles [0, n) with 16-byte-aligned units whose lengths are multiples of 4 and at most
    MAXV * 256 * 4 (kernel B skips anything past that); kernel A's table touches every arena element exactly once."""
    T = Tail(rl, head, "rmsprop", PROD["rmsprop"])
    b = T.tail.b_units.cpu()
    off, ln = b[:, 0], b[:, 1]
    assert bool((off % 4 == 0).all()) and bool((ln % 4 == 0).all()), "16-byte-aligned units, lengths multiple of 4"
    assert bool((ln > 0).all()) and bool((ln <= MAX_UNIT).all()), "unit lengths within kernel B's reach"
    order = torch.argsort(off)
    ends = off[order] + ln[order]
    assert int(off[order][0]) == 0 and int(ends[-1]) == T.n and torch.equal(off[order][1:], ends[:-1]), "tiles [0, n)"
    cover = torch.zeros(T.n, dtype=torch.int64).index_add_(0, T.a_idx, torch.ones_like(T.a_idx))
    assert bool((cover[T.real] == 1).all()), "kernel A: every parameter element once"
    assert bool((cover <= 1).all())


# ================================================================================================= CPU: pin the reference
def test_reference_matches_torch_optimizers():
    """Given the same float32-rounded hyperparameters, the float64 reference is torch.optim.RMSprop (plain, centered) and
    torch.optim.Adam (foreach=False) on float64 parameters, over several steps."""
    g = _gen(1)
    n = 257
    for kind in ("rmsprop", "centered", "adam"):
        hp = PROD[kind]
        p0 = torch.randn(n, generator=g, dtype=F64)
        tp = p0.clone().requires_grad_(True)
        if kind == "adam":
            opt = torch.optim.Adam([tp], lr=hp.lr, betas=(hp.a, hp.b), eps=hp.eps, foreach=False)
        else:
            opt = torch.optim.RMSprop([tp], lr=hp.lr, alpha=hp.a, eps=hp.eps, centered=kind == "centered", foreach=False)
        p, s1, s2 = p0.clone(), torch.zeros(n, dtype=F64), torch.zeros(n, dtype=F64)
        for step in range(1, 7):
            gr = torch.randn(n, generator=g, dtype=F64) * (0.01 if step % 2 else 3.0)
            tp.grad = gr.clone()
            opt.step()
            if kind == "adam":
                p, s1, s2 = adam_ref(p, gr, s1, s2, step, hp)
                st = opt.state[tp]
                mine = ((st["exp_avg"], s1), (st["exp_avg_sq"], s2))
            else:
                p, s1, s2 = rmsprop_ref(p, gr, s1, s2, hp, kind == "centered")
                st = opt.state[tp]
                mine = ((st["square_avg"], s1),) + (((st["grad_avg"], s2),) if kind == "centered" else ())
            torch.testing.assert_close(tp.detach(), p, rtol=1e-13, atol=1e-15)
            for x, y in mine:
                torch.testing.assert_close(x, y, rtol=1e-13, atol=1e-18)
    # the float32 rounding of the hyperparameters is visible: 1 - fl(0.999) is 1.3e-5 away from 1 - 0.999, relatively
    assert abs((1 - f32(0.999)) / (1 - 0.999) - 1) > 1e-5


def test_reference_clip_matches_clip_grad_norm():
    g = _gen(2)
    for max_norm in (0.5, 1e6):
        grads = [torch.randn(s, generator=g, dtype=F64) for s in ((7, 3), (11,), (1,))]
        ps = [torch.zeros_like(x, requires_grad=True) for x in grads]
        for p, x in zip(ps, grads):
            p.grad = x.clone()
        total = torch.nn.utils.clip_grad_norm_(ps, max_norm)
        norm = math.sqrt(sum(float((x ** 2).sum()) for x in grads))
        assert abs(float(total) - norm) <= 1e-14 * norm
        c = clip_coef(norm, max_norm, 1.0)
        assert (c < 1.0) == (max_norm == 0.5)
        for p, x in zip(ps, grads):
            torch.testing.assert_close(p.grad, x * c, rtol=1e-14, atol=0.0)
    # grad_scale: the norm of grad * s, and the coefficient multiplies the raw gradient
    assert clip_coef(10.0, 5.0, 0.5) == pytest.approx(0.5 * 5.0 / (10.0 + 1e-6), rel=1e-15)


@pytest.mark.parametrize("kind", ["rmsprop", "centered", "adam"])
def test_float32_emulation_within_bounds(kind):
    """The kernel's operation sequence in float32 stays within the first-order bounds of the Gaussian tests, over steps
    that start from the emulation's own state (teacher forcing), clip active and inactive, production hyperparameters."""
    g = _gen(3 + len(kind))
    hp = PROD[kind]
    n = 20000
    p = torch.randn(n, generator=g) * 0.05
    s1, s2 = torch.zeros(n), torch.zeros(n)
    for step in range(1, 9):
        gv = torch.randn(n, generator=g) * 10.0 ** float(torch.randint(-4, 1, (1,), generator=g))
        coef = f32(0.37 if step % 2 else 1.0)
        P, S1, S2 = p.to(F64), s1.to(F64), s2.to(F64)
        gr = gv.to(F64) * coef
        if kind == "adam":
            p, s1, s2 = adam_f32(p, gv, coef, s1, s2, step, hp)
            ref, bnd = adam_ref(P, gr, S1, S2, step, hp), adam_bounds(P, gr, S1, S2, step, hp)
        else:
            c = kind == "centered"
            p, s1, s2 = rmsprop_f32(p, gv, coef, s1, s2, hp, c)
            ref, bnd = rmsprop_ref(P, gr, S1, S2, hp, c), rmsprop_bounds(P, gr, S1, S2, hp, c)
        assert_within(p, ref[0], bnd[0], "step %d parameters" % step)
        assert_within(s1, ref[1], bnd[1], "step %d first moment" % step)
        if kind != "rmsprop":
            assert_within(s2, ref[2], bnd[2], "step %d second moment" % step)
        # the bound is not vacuous: a few ulps of the parameter (Adam's bias corrections carry powf's error)
        in_ulps = bnd[0] / (ref[0].abs() * 2.0 ** -23)
        assert float(in_ulps.median()) < (16.0 if kind == "adam" else 2.0)


@pytest.mark.parametrize("kind", ["rmsprop", "centered", "adam"])
@pytest.mark.parametrize("gs", [1.0, 0.5, 0.25])
def test_dyadic_cases_meet_their_premise(kind, gs):
    """Every exact case's data: all intermediates are float32 numbers, and the float32 emulation equals the float64
    reference bit for bit, three steps in a row with the parameters carried over."""
    g = _gen(int(4 / gs) + len(kind))
    hp = exact_hyper(kind, gs)
    n = 50000
    p = None
    for step in range(3):
        v = sparse_ints(g, (n,))
        gr = v * gs
        p, s1, s2 = dyadic_state(g, gr, kind, gs, p)
        ref = exact_step_ref(kind, p, gr, s1, s2, hp, "step %d" % step)
        if kind == "adam":
            emu = adam_f32(p.float(), v.float(), gs, s1.float(), s2.float(), 1, hp)
            assert torch.equal(ref[0], p - LR_EXACT * v / (v.abs() + 1)), "Adam step 1: lr v / (|v| + 1)"
        else:
            emu = rmsprop_f32(p.float(), v.float(), gs, s1.float(), s2.float(), hp, kind == "centered")
        for x, y in zip(emu, ref):
            assert torch.equal(x.to(F64), y)
        p = ref[0]
    # the W-rank all-reduce premise of the split test: (W v) * fl(1/W) rounds back to v
    for W in (2, 3, 4):
        v = VALS.float()
        assert torch.equal((v * W) * torch.tensor(f32(1.0 / W), dtype=F32), v)


@pytest.mark.parametrize("c1", [4, 8, 12, 16])
def test_ref_index_inverts_the_packers(c1):
    """The Python mirror of tail.cu's ref_index maps each GEMM-layout element of a row to the reference-layout element the
    packers take it from, for conv1 .. fc4; kernel B's dgrad stores match pack_w2d / pack_w3d."""
    shapes = [(32, c1, 8, 8), (64, 32, 4, 4), (64, 64, 3, 3), (3, 3136)]
    for kind, shp, pk in zip((U_W1, U_W2, U_W3, U_W4), shapes, PACKERS):
        ar = torch.arange(math.prod(shp)).view(shp)
        G = pk(ar)
        rows, L = G.shape
        k = torch.arange(L)
        for r in range(rows):
            assert torch.equal(G[r], r * L + ref_index(kind, k, c1)), "kind %d row %d" % (kind, r)
        assert torch.equal(unpack(G, pk, shp), ar), "unpack inverts the packer"
    # dgrad orientations: w2d[(k & 127) * 256 + (k >> 7) * 64 + row] and w3d[(k & 63) * 576 + (k >> 6) * 64 + row]
    for shp, pf, pd, rl_ in (((64, 32, 4, 4), pack_w2f, pack_w2d, 512), ((64, 64, 3, 3), pack_w3f, pack_w3d, 576)):
        ar = torch.arange(math.prod(shp)).view(shp)
        Gf, Gd = pf(ar), pd(ar).reshape(-1)
        k = torch.arange(rl_)
        for r in range(64):
            dst = (k & 127) * 256 + (k >> 7) * 64 + r if rl_ == 512 else (k & 63) * 576 + (k >> 6) * 64 + r
            assert torch.equal(Gd[dst], Gf[r])


def test_plain_units_tile_the_gaps():
    """network/tail.py _plain_units: the plain units and the covered ranges tile [0, n), each plain unit at most
    PLAIN_CHUNK long, 16-byte aligned when the covered ranges are."""
    from deeprl_b200.network.tail import PLAIN_CHUNK, _plain_units
    g = _gen(9)
    assert PLAIN_CHUNK <= MAX_UNIT and PLAIN_CHUNK % 4 == 0
    for trial in range(50):
        covered, pos = [], 0
        for _ in range(int(torch.randint(0, 8, (1,), generator=g))):
            pos += 4 * int(torch.randint(0, 1500, (1,), generator=g))
            ln = 4 * int(torch.randint(1, 2000, (1,), generator=g))
            covered.append((pos, ln))
            pos += ln
        n = pos + 4 * int(torch.randint(0, 3000, (1,), generator=g))
        if n == 0:
            continue
        perm = torch.randperm(len(covered), generator=g).tolist()
        units = _plain_units([covered[i] for i in perm], n)
        cover = torch.zeros(n, dtype=torch.int64)
        for off, ln, kind, w in units:
            assert kind == U_PLAIN and w == 0 and 0 < ln <= PLAIN_CHUNK and off % 4 == 0 and ln % 4 == 0
            cover[off:off + ln] += 1
        for off, ln in covered:
            cover[off:off + ln] += 1
        assert bool((cover == 1).all()), "trial %d: plain units + covered ranges tile [0, n)" % trial
