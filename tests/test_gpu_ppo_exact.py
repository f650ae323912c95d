"""The persistent PPO minibatch update (csrc/ppo_persistent.cu, arithmetic in csrc/ppo_phases.h, sequences ppo_sequence.inc /
ppo_dp_sequence.inc) checked EXACTLY against a float64 restatement of PPO_agent.py:68-99, in a regime where every kernel
operation is exact or rounds the way IEEE does:

- integer states and weights / biases that are multiples of 16, so every pre-activation is 0 or at least 16 in magnitude:
  tanhf returns exactly 0 or +-1 and 1 - h^2 is 1 or 0 (calibrated on the kernel's own tanhf, not assumed);
- std parameters that are powers of two >= 32: softplus(p) = p, sd^2, sd^3, 1/sd exact, softplus' = 1;
- actions = mean + dyadic offsets, dyadic advantages, returns and entropy weight; old log-probs set from the kernel's own
  float32 log-prob of each offset pattern (calibrated: mb = 4 identical rows and old = 0 make stats[2] = -lp exactly), so the
  ratio is exactly 1 (old = lp; a tie of torch.min, g = adv) or exactly 0 (old = lp + 120);
- Adam with beta1 = beta2 = 1/2, dyadic lr and eps, at step 1 (step_size 2 lr) or a step >= 25 (both bias corrections
  round to 1): every product is exact, so FMA contraction cannot matter, and a float32 emulation of the IEEE sqrtf, division and
  additions reproduces the kernel bit for bit.

Every case asserts its premises on its own data: pre-activations in {0} u [16, 2048], every product and every partial sum of
the forward and backward passes a multiple of a common power of two q with sum |terms| < 2^24 q (hence exact in float32 in
any order, with or without contraction).  Where the regime needs a rounding (1/mb for mb = 12, 1/W for W = 3, the kl and
value-loss means) the reference rounds in float32 in the kernel's order.  The policy-loss statistic contains logf and is held
to a first-order bound.

Backends: "emul" is the host build of the same phases (tests/host_emul, threads run one after another; CPU), "cuda" the
sm_90a kernel through the C ABI (GPU).  On the device further invariants are checked bit for bit: one launch against the same
permutation split over several launches, closed gates, NaN arena padding, and the data-parallel kernel against itself and
against the single-process kernel."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_ppo_data_parallel import dp_region_floats  # noqa: E402
from test_ppo_persistent import A_KEYS, C_KEYS, I32, I64, arena, batches_for, fp, make_problem  # noqa: E402

gpu = pytest.mark.gpu
F32, F64 = np.float32, np.float64
HALF_LOG_2PI = 0.91893853320467274178
ZMAX = 2048                                # pre-activations of the exact cases stay within the calibrated range
BACKENDS = ["emul", pytest.param("cuda", marks=gpu)]
EXACT_HP = dict(a_lr=2.0 ** -6, a_b1=0.5, a_b2=0.5, a_eps=2.0 ** -10, c_lr=2.0 ** -5, c_b1=0.5, c_b2=0.5, c_eps=2.0 ** -12,
                clip=0.25, ent_w=2.0 ** -7, gate=1e30)
HP_KEYS = ("a_lr", "a_b1", "a_b2", "a_eps", "c_lr", "c_b1", "c_b2", "c_eps", "clip", "ent_w", "gate")
GAUSS_HP = dict(a_lr=3e-4, a_b1=0.9, a_b2=0.999, a_eps=1e-8, c_lr=1e-3, c_b1=0.9, c_b2=0.999, c_eps=1e-8, clip=0.2, ent_w=0.01,
                gate=0.015)
ARENAS = ("a_flat", "a_m", "a_v", "c_flat", "c_m", "c_v")


# ------------------------------------------------------------------------------------------------ backends
@pytest.fixture(scope="module")
def emul_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ppo_exact_emul") / "ppo_emul.so")
    d = os.path.join(ROOT, "tests", "host_emul")
    subprocess.run(["g++", "-O2", "-fno-strict-aliasing", "-std=c++17", "-shared", "-fPIC", "-o", out,
                    os.path.join(d, "ppo_emul.cpp"), os.path.join(d, "ppo_dp_emul.cpp")], check=True)
    return ctypes.CDLL(out)


@pytest.fixture(params=BACKENDS)
def be(request):
    if request.param == "cuda":
        if not torch.cuda.is_available():
            pytest.skip("needs a GPU")
        return Backend("cuda")
    return Backend("emul", request.getfixturevalue("emul_lib"))


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return Backend("cuda")


def shapes_of(D, A, H1, H2):
    return {A_KEYS[0]: (H1, D), A_KEYS[1]: (H1,), A_KEYS[2]: (H2, H1), A_KEYS[3]: (H2,), A_KEYS[4]: (A, H2), A_KEYS[5]: (A,),
            A_KEYS[6]: (A,), C_KEYS[0]: (H1, D), C_KEYS[1]: (H1,), C_KEYS[2]: (H2, H1), C_KEYS[3]: (H2,), C_KEYS[4]: (1, H2),
            C_KEYS[5]: (1,)}


def initial_arenas(P):
    tw = {k: torch.from_numpy(np.asarray(v, F32)) for k, v in P["w"].items()}
    a_flat, a_off = arena(tw, A_KEYS)
    c_flat, c_off = arena(tw, C_KEYS)
    ar = dict(a_flat=a_flat, c_flat=c_flat, a_m=np.zeros_like(a_flat), a_v=np.zeros_like(a_flat), c_m=np.zeros_like(c_flat),
              c_v=np.zeros_like(c_flat))
    return ar, a_off, c_off


def padding_mask(n, off, keys, shapes):
    pad = np.ones(n, bool)
    for k, o in zip(keys, off):
        pad[o:o + int(np.prod(shapes[k]))] = False
    return pad


def tensor_of(flat, P, key):
    keys, off = (A_KEYS, P["a_off"]) if key in A_KEYS else (C_KEYS, P["c_off"])
    o = int(off[keys.index(key)])
    shp = P["shapes"][key]
    return flat[o:o + int(np.prod(shp))].reshape(shp)


class Backend:
    def __init__(self, name, lib=None):
        self.name, self.lib = name, lib

    def run(self, P, perm, hp, arenas=None, steps=(0, 0), nb=None):
        """One call of the minibatch kernel: perm [n_batches][mb] rows of P; arenas default to P's weights and zero moments."""
        D, A, H1, H2 = P["dims"]
        ar = {k: v.copy() for k, v in (arenas or initial_arenas(P)[0]).items()}
        perm = np.ascontiguousarray(perm, np.int64)
        nb = perm.shape[0] if nb is None else nb
        mb = perm.shape[1]
        a_step, c_step = np.array([steps[0]], np.int64), np.array([steps[1]], np.int64)
        stats = np.full(4, np.nan, F32)
        rows = [np.ascontiguousarray(P[k], F32) for k in ("st", "ac", "old", "ret", "adv")]
        sc = [float(hp[k]) for k in HP_KEYS]
        if self.name == "emul":
            rc = self.lib.ppo_emul_minibatch_updates(
                *[fp(r) for r in rows], D, A, H1, H2, mb, perm.ctypes.data_as(I64), nb, fp(ar["a_flat"]), fp(ar["a_m"]),
                fp(ar["a_v"]), a_step.ctypes.data_as(I64), P["a_off"].ctypes.data_as(I32), fp(ar["c_flat"]), fp(ar["c_m"]),
                fp(ar["c_v"]), c_step.ctypes.data_as(I64), P["c_off"].ctypes.data_as(I32), *[ctypes.c_float(s) for s in sc],
                fp(stats), 512)
            assert rc == 0
        else:
            from deeprl_b200 import _lib
            cu = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
            t = {k: cu(v) for k, v in ar.items()}
            r = [cu(x) for x in rows]
            tp, ta, tc, ts = cu(perm), cu(a_step), cu(c_step), cu(stats)
            p = _lib.ptr
            _lib.call("b2rl_ppo_minibatch_updates", *[p(x) for x in r], D, A, H1, H2, mb, p(tp), nb, p(t["a_flat"]), p(t["a_m"]),
                      p(t["a_v"]), p(ta), p(torch.from_numpy(P["a_off"])), p(t["c_flat"]), p(t["c_m"]), p(t["c_v"]), p(tc),
                      p(torch.from_numpy(P["c_off"])), *sc, p(ts), _lib.stream())
            torch.cuda.synchronize()
            ar = {k: v.cpu().numpy() for k, v in t.items()}
            a_step, c_step, stats = ta.cpu().numpy(), tc.cpu().numpy(), ts.cpu().numpy()
        return dict(ar, a_step=int(a_step[0]), c_step=int(c_step[0]), stats=stats)

    def run_dp(self, Ps, perms, hp, arenas=None, steps=(0, 0)):
        """The data-parallel kernel with W = len(Ps) ranks in one launch (one device) / in lockstep (host); every rank starts
        from the same arenas.  Returns one result dict per rank."""
        W, P = len(Ps), Ps[0]
        D, A, H1, H2 = P["dims"]
        ar0 = arenas or initial_arenas(P)[0]
        ar = {k: np.tile(v, W) for k, v in ar0.items()}
        a_n, c_n = ar0["a_flat"].size, ar0["c_flat"].size
        R = P["st"].shape[0]
        nb, mb = perms[0].shape
        perm = np.ascontiguousarray(np.concatenate(perms), np.int64)
        a_step, c_step = np.full(W, steps[0], np.int64), np.full(W, steps[1], np.int64)
        stats, status = np.full(4 * W, np.nan, F32), np.zeros(W, np.int64)
        rows = [np.ascontiguousarray(np.concatenate([q[k] for q in Ps]), F32) for k in ("st", "ac", "old", "ret", "adv")]
        sc = [float(hp[k]) for k in HP_KEYS]
        rf = dp_region_floats(a_n, c_n)
        if self.name == "emul":
            regions = np.zeros(W * rf, F32)
            rc = self.lib.ppo_emul_minibatch_updates_dp(
                *[fp(r) for r in rows], D, A, H1, H2, mb, perm.ctypes.data_as(I64), nb, fp(ar["a_flat"]), fp(ar["a_m"]),
                fp(ar["a_v"]), a_step.ctypes.data_as(I64), P["a_off"].ctypes.data_as(I32), fp(ar["c_flat"]), fp(ar["c_m"]),
                fp(ar["c_v"]), c_step.ctypes.data_as(I64), P["c_off"].ctypes.data_as(I32), *[ctypes.c_float(s) for s in sc],
                fp(stats), R, a_n, c_n, W, fp(regions), ctypes.c_int64(rf), ctypes.c_int64(0), status.ctypes.data_as(I64), 512,
                0, 0)
            assert rc == 0
        else:
            from deeprl_b200 import _lib
            cu = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
            t = {k: cu(v) for k, v in ar.items()}
            r = [cu(x) for x in rows]
            tp, ta, tc, ts, tst = cu(perm), cu(a_step), cu(c_step), cu(stats), cu(status)
            regions = torch.zeros(W * rf, dtype=torch.float32, device="cuda")
            table = (ctypes.c_void_p * W)(*[regions.data_ptr() + 4 * q * rf for q in range(W)])
            p = _lib.ptr
            _lib.call("b2rl_ppo_minibatch_updates_dp", *[p(x) for x in r], D, A, H1, H2, mb, p(tp), nb, p(t["a_flat"]),
                      p(t["a_m"]), p(t["a_v"]), p(ta), p(torch.from_numpy(P["a_off"])), p(t["c_flat"]), p(t["c_m"]), p(t["c_v"]),
                      p(tc), p(torch.from_numpy(P["c_off"])), *sc, p(ts), R, a_n, c_n, W, 0, table, 0, int(5e9), p(tst), W,
                      _lib.stream())
            torch.cuda.synchronize()
            ar = {k: v.cpu().numpy() for k, v in t.items()}
            a_step, c_step, stats, status = ta.cpu().numpy(), tc.cpu().numpy(), ts.cpu().numpy(), tst.cpu().numpy()
        assert not status.any(), status
        out = []
        for q in range(W):
            d = {k: ar[k][q * v.size // W:(q + 1) * v.size // W] for k, v in ar.items()}
            out.append(dict(d, a_step=int(a_step[q]), c_step=int(c_step[q]), stats=stats[4 * q:4 * q + 4]))
        return out


# ------------------------------------------------------------------------------------------------ exactness premises
def lowbit(x):
    """The lowest set bit of every element (a power of two; inf for 0): x is a multiple of it."""
    x = np.asarray(x, F64)
    assert np.isfinite(x).all()
    m, e = np.frexp(np.abs(x))
    mi = (m * 2.0 ** 53).astype(np.int64)
    return np.where(x == 0, np.inf, np.ldexp((mi & -mi).astype(F64), e - 53))


def exact(x):
    """x is representable in float32."""
    x = np.asarray(x, F64)
    assert np.array_equal(x.astype(F32).astype(F64), x), "not exact in float32"
    return x


def xsum(t, axis):
    """Sum along `axis`, asserting that every float32 partial sum in any order is exact."""
    q = lowbit(t).min(axis=axis)
    mag = np.abs(t).sum(axis=axis)
    assert (mag < 2.0 ** 24 * q).all() or not mag.any(), "a float32 sum is not exact"
    return np.asarray(t, F64).sum(axis=axis)


def mm(a, wt, bias=None):
    """sum_k a[.., n, k] wt[.., j, k] (+ bias[j]), asserting the premise of xsum for every output: all products are multiples
    of q = lowbit(a) lowbit(wt) (per matrix of a batch) and sum |terms| < 2^24 q."""
    a, wt = np.asarray(a, F64), np.asarray(wt, F64)
    wT = np.swapaxes(wt, -1, -2)
    out, mag = a @ wT, np.abs(a) @ np.abs(wT)
    q = lowbit(a).min(axis=(-2, -1), keepdims=True) * lowbit(wt).min(axis=(-2, -1), keepdims=True)
    if bias is not None:
        out, mag = out + bias, mag + np.abs(bias)
        q = np.minimum(q, lowbit(bias).min())
    assert ((mag < 2.0 ** 24 * q) | (mag == 0)).all(), "a float32 dot product is not exact"
    return out


def tern(z):
    """tanh in the exact regime: the pre-activation is 0 or 16 <= |z| <= ZMAX, where the kernel's tanhf is 0 or +-1."""
    az = np.abs(z)
    assert ((az == 0) | (az >= 16)).all() and az.max() <= ZMAX, "pre-activation outside {0} u [16, %d]" % ZMAX
    return np.sign(z)


def sum4(p):
    """sum_strided4 of ppo_phases.h in float32 along the last axis: four sequential chains, (s0 + s1) + (s2 + s3)."""
    p = np.asarray(p, F32)
    assert p.shape[-1] % 4 == 0
    s = [np.add.accumulate(p[..., i::4], axis=-1, dtype=F32)[..., -1] for i in range(4)]
    return (s[0] + s[1]) + (s[2] + s[3])


def swap(x):
    return np.swapaxes(x, -1, -2)


# ------------------------------------------------------------------------------------------------ float64 reference
def forward(w, x):
    h1 = tern(mm(x, w[A_KEYS[0]], w[A_KEYS[1]]))
    h2 = tern(mm(h1, w[A_KEYS[2]], w[A_KEYS[3]]))
    mu = tern(mm(h2, w[A_KEYS[4]], w[A_KEYS[5]]))
    ch1 = tern(mm(x, w[C_KEYS[0]], w[C_KEYS[1]]))
    ch2 = tern(mm(ch1, w[C_KEYS[2]], w[C_KEYS[3]]))
    v = mm(ch2, w[C_KEYS[4]], w[C_KEYS[5]])[..., 0]
    return h1, h2, mu, ch1, ch2, v


def reference(w, x, act, old, adv, ret, lp, hp):
    """One minibatch update's gradients and statistics (PPO_agent.py:79-99) for a batch of minibatches: x [B][mb][D] etc.;
    lp [B][mb] the kernel's float32 log-probs of the rows.  Gradients in float64 (exact by the asserted premises), the
    means that the regime lets round (1/mb, kl, value loss) in float32 in the kernel's order."""
    mb = x.shape[-2]
    inv = F32(1) / F32(mb)
    h1, h2, mu, ch1, ch2, v = forward(w, x)
    sd = w["std"]
    assert ((sd >= 32) & (np.log2(sd) % 1 == 0)).all(), "std parameters must be powers of two >= 32"
    # critic: value loss 0.5 mean (ret - v)^2 and d / dv
    e = exact(ret - v)
    dv = ((-e.astype(F32)) * inv).astype(F64)
    vl = F32(0.5) * (F32(xsum(exact(e * e), -1)) / F32(mb))
    # actor: ratio exactly 1 or 0, clipped surrogate, torch.min's tie split
    r = np.asarray(lp, F32) - np.asarray(old, F32)
    assert ((r == 0) | (r <= -110)).all(), "log-ratio neither 0 nor below expf's underflow"
    ratio = (r == 0).astype(F64)
    clip = float(F32(hp["clip"]))
    obj, objc = ratio * adv, exact(np.clip(ratio, 1 - clip, 1 + clip) * adv)
    inside = (ratio >= 1 - clip) & (ratio <= 1 + clip)
    g = np.where(obj < objc, adv * ratio, np.where(obj > objc, np.where(inside, adv * ratio, 0.0),
                                                  0.5 * adv * ratio + np.where(inside, 0.5 * adv * ratio, 0.0)))
    gl = ((-exact(g).astype(F32)) * inv).astype(F64)
    kl = sum4(np.asarray(old, F32) - np.asarray(lp, F32)) * inv
    s_pl = xsum(exact(np.minimum(obj, objc)), -1)
    ent_terms = 0.5 + HALF_LOG_2PI + np.log(sd)
    ent_w = float(F32(hp["ent_w"]))
    pl = -(s_pl / mb) - ent_w * ent_terms.sum()
    pl_tol = (sd.size + 4) * 2.0 ** -23 * (np.abs(s_pl / mb) + ent_w * np.abs(ent_terms).sum())
    gate = kl <= F32(hp["gate"])
    # policy head: d / d pre-tanh mean and d / d std parameter (softplus' = 1)
    t = exact(act - mu)
    dmu = exact(gl[..., None] * exact(t / (sd * sd))) * (1 - mu * mu)
    dent = float(F32(-ent_w) / F32(mb))
    dsd = exact(exact(gl[..., None] * exact(exact(t * t / (sd * sd * sd)) - 1 / sd)) + dent / sd)
    ad2 = mm(dmu, swap(w[A_KEYS[4]])) * (1 - h2 * h2)
    ad1 = mm(ad2, swap(w[A_KEYS[2]])) * (1 - h1 * h1)
    grads = {A_KEYS[0]: mm(swap(ad1), swap(x)), A_KEYS[1]: xsum(ad1, -2), A_KEYS[2]: mm(swap(ad2), swap(h1)),
             A_KEYS[3]: xsum(ad2, -2), A_KEYS[4]: mm(swap(dmu), swap(h2)), A_KEYS[5]: xsum(dmu, -2), A_KEYS[6]: xsum(dsd, -2)}
    cd2 = exact(dv[..., None] * w[C_KEYS[4]][0]) * (1 - ch2 * ch2)
    cd1 = mm(cd2, swap(w[C_KEYS[2]])) * (1 - ch1 * ch1)
    grads.update({C_KEYS[0]: mm(swap(cd1), swap(x)), C_KEYS[1]: xsum(cd1, -2), C_KEYS[2]: mm(swap(cd2), swap(ch1)),
                  C_KEYS[3]: xsum(cd2, -2), C_KEYS[4]: mm(dv[..., None, :], swap(ch2)), C_KEYS[5]: xsum(dv, -1)[..., None]})
    for k in grads:
        exact(grads[k])
    return dict(grads=grads, vl=vl, kl=kl, pl=pl, pl_tol=pl_tol, gate=gate, lp=lp)


def adam32(p, g, m, v, t, lr, b1, b2, eps):
    """_single_tensor_adam as adam_elem / wgrad_adam_tile evaluate it, in float32 (numpy rounds every operation as IEEE does).
    beta^t in float64 is exact for beta = 1/2; the calibration test checks the device's powf against it."""
    f = F32
    p, g, m, v = (np.asarray(z, f) for z in (p, g, m, v))
    bc1, bc2 = f(1) - f(b1 ** t), f(1) - f(b2 ** t)
    step_size, bc2s = f(lr) / bc1, np.sqrt(bc2)
    m = m + (f(1) - f(b1)) * (g - m)
    v = f(b2) * v + ((f(1) - f(b2)) * g) * g
    denom = np.sqrt(v) / bc2s + f(eps)
    return p - step_size * (m / denom), m, v


def expected_arenas(P, ar0, grads, gate, hp, steps):
    """The six arenas after one update with these (unbatched) gradients from arenas ar0 at step counts `steps`."""
    ar = {k: v.copy() for k, v in ar0.items()}
    for net, keys, off, t, on in (("a", A_KEYS, P["a_off"], steps[0] + 1, gate), ("c", C_KEYS, P["c_off"], steps[1] + 1, True)):
        if not on:
            continue
        for k, o in zip(keys, off):
            n = int(np.prod(P["shapes"][k]))
            sl = slice(int(o), int(o) + n)
            ar[net + "_flat"][sl], ar[net + "_m"][sl], ar[net + "_v"][sl] = adam32(
                ar[net + "_flat"][sl], np.asarray(grads[k], F64).ravel(), ar[net + "_m"][sl], ar[net + "_v"][sl], t,
                hp[net + "_lr"], hp[net + "_b1"], hp[net + "_b2"], hp[net + "_eps"])
    return ar


def assert_arenas_equal(got, want, what=""):
    for k in ARENAS:
        a, b = got[k], want[k]
        same = (a == b) | (np.isnan(a) & np.isnan(b))
        assert same.all(), "%s %s: %d elements differ, first at %d: %r vs %r" % (
            what, k, int((~same).sum()), int(np.argmax(~same)), a[~same][:3], b[~same][:3])


# ------------------------------------------------------------------------------------------------ exact problems
OFFSET_MULT = np.array([0.0, 0.5, -0.5, 1.0, -1.0, 2.0, -2.0])     # action - mean, in units of sd


def exact_problem(D, A, H1, H2, rows, seed, mb, n_patterns=3, p0=0.6, frac_ratio0=0.25):
    """Integer states, weights and biases in 16 {-1, 0, 1}, std parameters in {32, 64}; actions the mean plus one of a few
    offset patterns; dyadic advantages and returns (multiples of 3 when 3 divides mb, so that 1/mb rounds away).  `kind`
    per row: 0 ratio exactly 1, 1 ratio exactly 0 (old = lp + 120); `old` is filled in by calibrate_old."""
    rng = np.random.default_rng(seed)
    shp = shapes_of(D, A, H1, H2)
    w16 = lambda s: 16.0 * rng.choice([-1.0, 0.0, 1.0], size=s, p=[(1 - p0) / 2, p0, (1 - p0) / 2])
    w = {k: w16(shp[k]) for k in A_KEYS[:6] + C_KEYS[:4]}
    w["std"] = rng.choice([32.0, 64.0], A)
    w[C_KEYS[4]] = rng.integers(-2, 3, (1, H2)).astype(F64)
    w[C_KEYS[5]] = rng.integers(-4, 5, (1,)).astype(F64)
    x = rng.choice([-1.0, 0.0, 1.0], size=(rows, D), p=[0.3, 0.4, 0.3])
    _, _, mu, _, _, v = forward(w, x)
    pats = rng.choice(OFFSET_MULT, size=(n_patterns, A)) * w["std"]
    pat = rng.integers(0, n_patterns, rows)
    pat[:n_patterns] = np.arange(n_patterns)                     # row i < n_patterns represents pattern i
    three = 3.0 if mb % 3 == 0 else 1.0
    adv = three * rng.choice([-2.0, -1.0, -0.5, 0.5, 1.0, 2.0], rows)
    ret = v + three * 0.5 * rng.integers(-4, 5, rows)
    kind = (rng.random(rows) < frac_ratio0).astype(np.int64)
    ent_w = 2.0 ** -7 if mb % 3 else 3 * 2.0 ** -8
    P = dict(dims=(D, A, H1, H2), shapes=shp, w=w, st=x, ac=mu + pats[pat], old=np.zeros(rows), adv=adv, ret=ret, pat=pat,
             pats=pats, kind=kind, ent_w=ent_w)
    _, P["a_off"], P["c_off"] = initial_arenas(P)
    return P


def lp64(P, i):
    """Normal(mean, sd).log_prob summed over actions in float64, and a first-order bound of the kernel's float32 evaluation
    (3A roundings of the sum's size, logf within 1 ulp)."""
    sd, t = P["w"]["std"], P["pats"][i]
    terms = -t * t / (2 * sd * sd) - np.log(sd) - HALF_LOG_2PI
    return terms.sum(), (3 * sd.size + 2) * 2.0 ** -24 * np.abs(terms).sum()


def calibrate_old(be, P, hp):
    """The kernel's own float32 log-prob of every offset pattern: a minibatch of 4 copies of a row with old = 0 gives
    kl = ((-lp - lp) + (-lp - lp)) / 4 = -lp exactly.  Then old = lp (ratio 1) or fl(lp + 120) (ratio 0) per row."""
    lps = []
    for i in range(len(P["pats"])):
        Q = dict(P, old=np.zeros_like(P["old"]))
        out = be.run(Q, np.full((1, 4), i, np.int64), dict(hp, a_lr=0.0, c_lr=0.0))
        lp = -out["stats"][2]
        want, tol = lp64(P, i)
        assert abs(float(lp) - want) <= tol, ("log-prob of pattern", i, float(lp), want, tol)
        lps.append(lp)
    lp_row = np.asarray(lps, F32)[P["pat"]]
    P["lp"] = lp_row
    P["old"] = np.where(P["kind"] == 1, lp_row + F32(120), lp_row).astype(F32)
    return P


def ref_for(P, perm, hp):
    f = lambda k: np.asarray(P[k], F64)[perm]
    return reference(P["w"], f("st"), f("ac"), P["old"][perm], f("adv"), f("ret"), P["lp"][perm], hp)


def unbatch(grads, b):
    return {k: v[b] for k, v in grads.items()}


# ------------------------------------------------------------------------------------------------ calibration
def test_tanh_calibration(be):
    """Premise of the exact regime, on the kernel's own tanhf (ppo_tanh, the one copy every layer calls): tanhf(16 k) is
    exactly sign(k) for every k in [-128, 255], and tanhf(0) = 0.  Read through the critic: D = 1, x = 1, critic layer 1
    weights 16 (k + base), layer 2 zero (h2 = 0), value head 1, ret = -1 on 4 rows: dv = 1/4 and with beta1 = 0 the
    exp_avg of critic layer 2 is exactly its gradient sum_n dv h1[n][k] = tanhf(16 (k + base))."""
    H1, H2 = 128, 4
    for base in (-128, 0, 128):
        P = dict(dims=(1, 1, H1, H2), shapes=shapes_of(1, 1, H1, H2), st=np.ones((4, 1)), ac=np.zeros((4, 1)), old=np.zeros(4),
                 adv=np.ones(4), ret=-np.ones(4))
        w = {k: np.zeros(s) for k, s in P["shapes"].items()}
        w["std"][:] = 32.0
        z = 16.0 * (np.arange(H1) + base)
        w[C_KEYS[0]][:, 0] = z
        w[C_KEYS[4]][:] = 1.0
        P["w"] = w
        _, P["a_off"], P["c_off"] = initial_arenas(P)
        out = be.run(P, np.zeros((1, 4), np.int64), dict(EXACT_HP, a_lr=0.0, c_lr=0.0, c_b1=0.0))
        got = tensor_of(out["c_m"], P, C_KEYS[2])
        assert np.array_equal(got, np.broadcast_to(np.sign(z), (H2, H1))), (base, got[0][got[0] != np.sign(z)])


@pytest.mark.parametrize("t0", [0, 24, 99, 5120])
def test_adam_powf_calibration(be, t0):
    """Premise of adam32: on the device, with beta1 = beta2 = 1/2 at step t0 + 1, 1 - powf(1/2, t) is 1 - 2^-t (and rounds to
    1 from t = 25 on), so a known gradient from zero moments moves every parameter exactly as the float32 emulation says.
    A bias correction with t - 1, or without its square root, changes every element."""
    P = exact_problem(4, 1, 4, 4, 8, seed=5, mb=4)
    calibrate_old(be, P, EXACT_HP)
    perm = np.arange(4)[None]
    out = be.run(P, perm, EXACT_HP, steps=(t0, t0))
    ref = ref_for(P, perm, EXACT_HP)
    assert bool(ref["gate"][0])
    want = expected_arenas(P, initial_arenas(P)[0], unbatch(ref["grads"], 0), True, EXACT_HP, (t0, t0))
    assert_arenas_equal(out, want, "t0 = %d" % t0)
    assert (out["a_step"], out["c_step"]) == (t0 + 1, t0 + 1)


# ------------------------------------------------------------------------------------------------ 1. one minibatch, exactly
# (D, A, H1, H2, mb): scalar K tails (D % 4), ragged J tiles (H, A not multiples of 4), the non-vector Adam path (K % 4 != 0),
# lda padding (A = 5, 6), mb = 12 (1/mb inexact) and the examples' shape
SHAPES = [(17, 6, 64, 30, 64), (1, 1, 4, 12, 4), (3, 5, 12, 4, 12), (4, 32, 30, 64, 64), (1, 6, 128, 4, 12),
          (17, 5, 64, 128, 12), (3, 1, 30, 4, 128), (256, 32, 12, 30, 4), (17, 6, 64, 64, 64)]


def fits(D, A, H1, H2, mb):
    from deeprl_b200 import _lib
    return int(_lib.lib().b2rl_ppo_minibatch_smem_bytes(D, A, H1, H2, mb)) <= 227 * 1024


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "D%d-A%d-H%dx%d-mb%d" % s)
@pytest.mark.parametrize("clip", [0.25, 0.0])
def test_one_minibatch_exact(be, shape, clip):
    """One minibatch with lr != 0: every parameter, exp_avg, exp_avg_sq, both step counts, value loss, kl and the actor step
    counter bit for bit against float64 + the float32 Adam emulation; the policy loss to its first-order bound.  clip = 0
    with ratio exactly 1 tells <= from < in the `inside` test (a strict test halves g)."""
    D, A, H1, H2, mb = shape
    assert fits(*shape)
    hp = dict(EXACT_HP, clip=clip)
    P = exact_problem(D, A, H1, H2, 2 * mb, seed=hash(shape) % 1000 + int(clip * 8), mb=mb)
    hp["ent_w"] = P["ent_w"]
    calibrate_old(be, P, hp)
    perm = np.random.default_rng(3).permutation(2 * mb)[:mb][None]
    ref = ref_for(P, perm, hp)
    steps = (0, 24) if mb % 8 else (24, 0)
    assert bool(ref["gate"][0])
    out = be.run(P, perm, hp, steps=steps)
    want = expected_arenas(P, initial_arenas(P)[0], unbatch(ref["grads"], 0), True, hp, steps)
    assert_arenas_equal(out, want, str(shape))
    assert (out["a_step"], out["c_step"]) == (steps[0] + 1, steps[1] + 1)
    st = out["stats"]
    assert st[1] == ref["vl"][0] and st[2] == ref["kl"][0] and st[3] == 1.0
    assert abs(float(st[0]) - ref["pl"][0]) <= ref["pl_tol"][0], (st[0], ref["pl"][0], ref["pl_tol"][0])
    moved = [k for k in A_KEYS + C_KEYS if np.any(ref["grads"][k][0] != 0)]
    assert set(moved) & set(A_KEYS) and set(moved) & set(C_KEYS)   # the comparison is not between two untouched copies


def test_gate_at_equality_and_closed(be):
    """The gate `kl <= gate_max` with kl == gate_max bit for bit opens it; the next float32 below closes it, and a closed gate
    leaves the actor's parameters, moments and step count untouched while the critic still steps."""
    P = exact_problem(17, 6, 64, 64, 128, seed=11, mb=64, frac_ratio0=0.3)
    calibrate_old(be, P, EXACT_HP)
    perm = np.arange(64)[None]
    kl = ref_for(P, perm, EXACT_HP)["kl"][0]
    assert kl > 0
    for gmax, open_ in ((kl, True), (np.nextafter(kl, F32(0)), False)):
        hp = dict(EXACT_HP, gate=float(gmax))
        ref = ref_for(P, perm, hp)
        assert bool(ref["gate"][0]) == open_
        ar0 = initial_arenas(P)[0]
        out = be.run(P, perm, hp)
        assert_arenas_equal(out, expected_arenas(P, ar0, unbatch(ref["grads"], 0), open_, hp, (0, 0)), "gate %s" % open_)
        assert (out["a_step"], out["c_step"], float(out["stats"][3])) == (int(open_), 1, float(open_))
        assert out["stats"][2] == kl


# ------------------------------------------------------------------------------------------------ 2. a whole iteration, exactly
def iteration_problem(rows, seed):
    P = exact_problem(17, 6, 64, 64, rows, seed=seed, mb=64, p0=0.7, frac_ratio0=0.08)
    return P


def iteration_expectation(P, perm, hp):
    """lr = 0: weights stay fixed, so every minibatch's gradient is computed on its own in float64; the moments follow the
    float32 recurrence of adam_elem (exact to emulate: with beta = 1/2 and g^2 exact, every product is exact)."""
    nb = perm.shape[0]
    ar = initial_arenas(P)[0]
    gates, last = [], None
    grads = {k: [] for k in A_KEYS + C_KEYS}
    for c0 in range(0, nb, 256):
        ref = ref_for(P, perm[c0:c0 + 256], hp)
        gates.append(ref["gate"])
        for k in grads:
            g = ref["grads"][k]
            exact(g * g)
            grads[k].append(g.reshape(g.shape[0], -1).astype(F32))
        last = ref
    gates = np.concatenate(gates)
    grads = {k: np.concatenate(v) for k, v in grads.items()}
    for net, keys, off, on in (("a", A_KEYS, P["a_off"], gates), ("c", C_KEYS, P["c_off"], np.ones(nb, bool))):
        for k, o in zip(keys, off):
            n = int(np.prod(P["shapes"][k]))
            sl = slice(int(o), int(o) + n)
            m, v = ar[net + "_m"][sl], ar[net + "_v"][sl]
            for b in np.nonzero(on)[0]:
                g = grads[k][b]
                m = m + F32(0.5) * (g - m)
                v = F32(0.5) * v + (F32(0.5) * g) * g
            ar[net + "_m"][sl], ar[net + "_v"][sl] = m, v
    return ar, gates, last


@pytest.mark.parametrize("be_rows", [("emul", 2048, 2), pytest.param(("cuda", 32768, 10), marks=gpu)], ids=["emul", "cuda"])
def test_iteration_exact(request, be_rows):
    """The bench-size iteration in one launch (cuda: 32 768 rows, mb 64, 10 epochs = 5 120 minibatches, perm indices up to
    2^15 - 1; host: 64 minibatches), lr = 0 so the weights stay fixed.  Per-row old offsets make the kl gate open for some
    minibatches and close for others, with one kl exactly equal to gate_max.  Final moments, parameters, both step counts and
    the last minibatch's statistics bit for bit.  Catches a prefetch of the wrong row / buffer."""
    name, rows, epochs = be_rows
    be = _cuda() if name == "cuda" else Backend("emul", request.getfixturevalue("emul_lib"))
    P = iteration_problem(rows, seed=rows)
    hp = dict(EXACT_HP, a_lr=0.0, c_lr=0.0, ent_w=P["ent_w"])
    calibrate_old(be, P, hp)
    perm = batches_for(rows, epochs, 64, seed=21)
    nb = perm.shape[0]
    if name == "cuda":
        assert nb == 5120 and perm.max() == 2 ** 15 - 1
    kls = sum4(np.asarray(P["old"], F32)[perm] - np.asarray(P["lp"], F32)[perm]) * (F32(1) / F32(64))
    hp["gate"] = float(np.sort(kls)[nb // 2])                    # a minibatch's kl, bit for bit: about half the gates open
    want, gates, last = iteration_expectation(P, perm, hp)
    assert 0 < gates.sum() < nb and (kls == F32(hp["gate"])).any()
    out = be.run(P, perm, hp)
    assert_arenas_equal(out, want, "iteration")
    assert out["a_step"] == int(gates.sum()) and out["c_step"] == nb
    st = out["stats"]
    assert st[3] == gates.sum() and st[1] == last["vl"][-1] and st[2] == last["kl"][-1]
    assert abs(float(st[0]) - last["pl"][-1]) <= last["pl_tol"][-1]


# ------------------------------------------------------------------------------------------------ 2b. Gaussian data, per element
U, ULP = 2.0 ** -24, 2.0 ** -23          # float32 unit roundoff; an ulp of a normal y is at most 2^-23 |y|


class E:
    """A float64 value and a first-order bound on |its float32 evaluation - value|: every rounded operation adds U |result|
    (with or without FMA contraction: a contracted product only removes a rounding), a CUDA function documented to k ulp
    adds k 2^-23 |result|, and input errors propagate through the derivative."""

    def __init__(self, v, e=0.0):
        self.v = np.asarray(v, F64)
        self.e = np.broadcast_to(np.asarray(e, F64), self.v.shape).copy()

    @staticmethod
    def of(x):
        return x if isinstance(x, E) else E(x)

    def __add__(a, b):
        b = E.of(b)
        v = a.v + b.v
        return E(v, a.e + b.e + U * np.abs(v))

    __radd__ = __add__

    def __sub__(a, b):
        return a + (-E.of(b))

    def __rsub__(a, b):
        return E.of(b) + (-a)

    def __neg__(a):
        return E(-a.v, a.e)

    def __mul__(a, b):
        b = E.of(b)
        v = a.v * b.v
        return E(v, np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e + U * np.abs(v))

    __rmul__ = __mul__

    def __truediv__(a, b):
        b = E.of(b)
        assert (b.e <= 1e-2 * np.abs(b.v)).all()                 # (first order: the factor covers the second)
        v = a.v / b.v
        return E(v, (a.e + np.abs(v) * b.e) / np.abs(b.v) * (1 + 2e-2) + U * np.abs(v))

    def __rtruediv__(a, b):
        return E.of(b) / a

    def __getitem__(a, i):
        return E(a.v[i], a.e[i])

    @property
    def T(a):
        return E(swap(a.v), swap(a.e))


def efn(f, df, ulps, x):
    v = f(x.v)
    return E(v, np.abs(df(x.v)) * x.e + ulps * ULP * np.abs(v))


def ewhere(c, a, b):
    a, b = E.of(a), E.of(b)
    return E(np.where(c, a.v, b.v), np.where(c, a.e, b.e))


def edot(a, wt, bias=None):
    """sum_k a[.., n, k] wt[.., j, k] (+ bias[j]) in any order, with or without FMA: (K + 1) U sum |terms| for the roundings."""
    K = a.v.shape[-1] + (bias is not None)
    wT, weT = swap(wt.v), swap(wt.e)
    v, mag = a.v @ wT, np.abs(a.v) @ np.abs(wT)
    e = np.abs(a.v) @ weT + a.e @ np.abs(wT) + a.e @ weT
    if bias is not None:
        v, mag, e = v + bias.v, mag + np.abs(bias.v), e + bias.e
    return E(v, e + K * U * mag)


def etanh(z):
    return efn(np.tanh, lambda x: 1 - np.tanh(x) ** 2, 2, z)                    # tanhf: 2 ulp


def eexp(z):
    return efn(np.exp, np.exp, 2, z)                                            # expf: 2 ulp


def gauss_reference(w, x, act, old, adv, ret, hp):
    """One minibatch in the kernel's formulas (ppo_phases.h ph1-ph9) on float32 inputs: float64 gradients with a first-order
    bound on the kernel's float32 error, from the magnitudes and CUDA's documented errors (tanhf 2, expf 2, logf 1, log1pf 1
    ulp; IEEE +, *, /, sqrt 1/2 ulp).  Also returns which branch of the clipped surrogate every row took."""
    W = {k: E(np.asarray(v, F32)) for k, v in w.items()}
    X = E(np.asarray(x, F32))
    f32 = lambda z: np.asarray(z, F32).astype(F64)
    act, old, adv, ret = f32(act), f32(old), f32(adv), f32(ret)
    mb = x.shape[-2]
    inv = 1.0 / mb
    assert mb & (mb - 1) == 0                                   # 1/mb exact
    h1 = etanh(edot(X, W[A_KEYS[0]], W[A_KEYS[1]]))
    h2 = etanh(edot(h1, W[A_KEYS[2]], W[A_KEYS[3]]))
    mu = etanh(edot(h2, W[A_KEYS[4]], W[A_KEYS[5]]))
    ch1 = etanh(edot(X, W[C_KEYS[0]], W[C_KEYS[1]]))
    ch2 = etanh(edot(ch1, W[C_KEYS[2]], W[C_KEYS[3]]))
    v = edot(ch2, W[C_KEYS[4]], W[C_KEYS[5]])[..., 0]
    p = W["std"]
    assert (p.v < 20).all()                                     # softplus = log1pf(expf(p)), softplus' = 1 / (1 + expf(-p))
    sd = efn(np.log1p, lambda y: 1 / (1 + y), 1, eexp(p))
    lsd = efn(np.log, lambda y: 1 / y, 1, sd)
    dv = -(E(ret) - v) * inv
    C = E(HALF_LOG_2PI, U * HALF_LOG_2PI)                       # the float32 literal
    t = E(act) - mu
    lp = E(np.zeros(x.shape[:-1]))
    for j in range(act.shape[-1]):
        tj = t[..., j]
        lp = lp + (-(tj * tj) / ((2.0 * sd[j]) * sd[j]) - lsd[j] - C)
    ratio = eexp(lp - E(old))
    lo, hi = float(F32(1) - F32(hp["clip"])), float(F32(1) + F32(hp["clip"]))
    inside = (ratio.v >= lo) & (ratio.v <= hi)
    A_ = E(adv)
    obj = A_ * ratio
    objc = ewhere(inside, obj, E(np.clip(ratio.v, lo, hi)) * A_)
    lt = ~inside & (obj.v < objc.v)                             # outside, the unclipped term is the minimum: g = adv ratio
    gt = ~inside & (obj.v > objc.v)                             # outside, the clipped term is the minimum: g = 0
    half = (0.5 * A_) * ratio
    g = ewhere(inside, half + half, ewhere(lt, A_ * ratio, E(np.zeros_like(ratio.v))))
    # a row whose ratio lies within its bound of 1 -+ clip may take either branch in float32: its g is then anything in
    # [0, adv ratio] (or the tie), so its bound widens by |adv ratio|
    margin = np.minimum(np.abs(ratio.v - lo), np.abs(ratio.v - hi))
    amb = margin <= 2 * ratio.e
    g = E(g.v, g.e + np.where(amb, np.abs(A_.v * ratio.v) * (1 + 2 * ratio.e), 0.0))
    gl = -g * inv
    dent = float(F32(-hp["ent_w"]) / F32(mb))
    sig = 1.0 / (1.0 + eexp(-p))
    dmu = (gl[..., None] * (t / (sd * sd))) * (1.0 - mu * mu)
    dsd = (gl[..., None] * ((t * t) / ((sd * sd) * sd) - 1.0 / sd) + dent * (1.0 / sd)) * sig
    ad2 = edot(dmu, W[A_KEYS[4]].T) * (1.0 - h2 * h2)
    ad1 = edot(ad2, W[A_KEYS[2]].T) * (1.0 - h1 * h1)
    ones = E(np.ones((1, mb)))
    colsum = lambda d: edot(d.T, ones)[..., 0]
    grads = {A_KEYS[0]: edot(ad1.T, X.T), A_KEYS[1]: colsum(ad1), A_KEYS[2]: edot(ad2.T, h1.T), A_KEYS[3]: colsum(ad2),
             A_KEYS[4]: edot(dmu.T, h2.T), A_KEYS[5]: colsum(dmu), A_KEYS[6]: colsum(dsd)}
    cd2 = (dv[..., None] * W[C_KEYS[4]][0]) * (1.0 - ch2 * ch2)
    cd1 = edot(cd2, W[C_KEYS[2]].T) * (1.0 - ch1 * ch1)
    dvm = E(dv.v[..., None, :], dv.e[..., None, :])
    grads.update({C_KEYS[0]: edot(cd1.T, X.T), C_KEYS[1]: colsum(cd1), C_KEYS[2]: edot(cd2.T, ch1.T), C_KEYS[3]: colsum(cd2),
                  C_KEYS[4]: edot(dvm, ch2.T), C_KEYS[5]: edot(dvm, ones)[..., 0]})
    return grads, dict(inside=int(inside.sum()), lt=int(lt.sum()), gt=int(gt.sum()), ambiguous=int(amb.sum()))


def autograd_gradients(w, x, act, old, adv, ret, hp):
    """The same gradients by torch autograd in float64 through the oracle (nets.gaussian_actor_critic, losses.ppo_losses)."""
    from oracle import losses, nets
    t = lambda z: torch.from_numpy(np.asarray(np.asarray(z, F32), F64))
    sd = {k: t(v).requires_grad_() for k, v in w.items()}
    out = nets.gaussian_actor_critic(sd, t(x), t(act))
    col = lambda z: t(z)[:, None]
    pl, vl, _ = losses.ppo_losses(out["log_pi_a"], out["entropy"], out["v"], col(old), col(adv), col(ret),
                                  float(F32(hp["clip"])), float(F32(hp["ent_w"])))
    ga = torch.autograd.grad(pl, [sd[k] for k in A_KEYS])
    gc = torch.autograd.grad(vl, [sd[k] for k in C_KEYS])
    return {k: g.numpy() for k, g in zip(A_KEYS + C_KEYS, list(ga) + list(gc))}


def gauss_bench_problem(rows, seed):
    """Gaussian rows at the bench shape with std parameters in (0, 3) (softplus through log1pf(expf(p)), softplus' < 1) and
    old log-probs 0.4 nats around the new ones, so that rows fall inside the clip interval and outside it on both sides."""
    P = gauss_problem(rows, seed)
    rng = np.random.default_rng(seed)
    P["w"]["std"] = rng.uniform(0, 3, P["w"]["std"].shape).astype(F32).astype(F64)
    from oracle import nets
    with torch.no_grad():
        sd = {k: torch.from_numpy(np.asarray(v, F32)) for k, v in P["w"].items()}
        lp = nets.gaussian_actor_critic(sd, torch.from_numpy(P["st"]), torch.from_numpy(P["ac"]))["log_pi_a"].numpy().ravel()
    P["old"] = (lp + 0.4 * rng.standard_normal(rows)).astype(F32)
    _, P["a_off"], P["c_off"] = initial_arenas(P)
    return P


def gauss_rows(P, perm):
    return [np.asarray(P[k], F64)[perm] for k in ("st", "ac", "old", "adv", "ret")]


def test_gauss_reference_is_the_autograd_gradient():
    """CPU: the kernel-formula reference's values are torch autograd's float64 gradients of the oracle's PPO losses, and its
    bounds mean something: their median is below 1 % of each tensor's largest gradient (the worst-case (K + 1) u per dot
    product and the tanhf / expf errors carried through three layers dominate)."""
    P = gauss_bench_problem(2048, seed=31)
    perm = batches_for(2048, 1, 64, seed=3)[:4]
    for b in range(perm.shape[0]):
        x, act, old, adv, ret = gauss_rows(P, perm[b])
        ref, br = gauss_reference(P["w"], x, act, old, adv, ret, GAUSS_HP)
        ag = autograd_gradients(P["w"], x, act, old, adv, ret, GAUSS_HP)
        assert br["inside"] and br["lt"] and br["gt"], br
        if br["ambiguous"]:
            continue
        for k in A_KEYS + C_KEYS:
            scale = np.abs(ag[k]).max()
            assert np.abs(ref[k].v - ag[k].reshape(ref[k].v.shape)).max() <= 1e-10 * scale, k
            assert np.median(ref[k].e) <= 1e-2 * scale, (k, np.median(ref[k].e), scale)


def gauss_kernel_gradients(be, P, perm_row, steps=(0, 0)):
    """One minibatch from zero moments with beta1 = 1/2 and lr = 0: exp_avg = fl(0.5 g) = 0.5 g exposes the float32 gradient."""
    hp = dict(GAUSS_HP, a_lr=0.0, c_lr=0.0, a_b1=0.5, c_b1=0.5, gate=1e30)
    out = be.run(P, perm_row[None], hp, steps=steps)
    assert out["a_step"] == steps[0] + 1
    return {k: 2.0 * tensor_of(out[("a" if k in A_KEYS else "c") + "_m"], P, k).astype(F64) for k in A_KEYS + C_KEYS}


@pytest.mark.parametrize("be_rows", [("emul", 2048, 3), pytest.param(("cuda", 32768, 12), marks=gpu)], ids=["emul", "cuda"])
def test_gauss_gradients_within_first_order_bound(request, be_rows):
    """Gaussian minibatches at the bench shape (cuda: a sample of the 5 120 minibatches of a 32 768-row iteration, one launch
    each; host: the float32 evaluation of the same phases with glibc's functions): every gradient element within the
    first-order bound.  The data reach softplus' < 1, log1pf(expf(p)) and all three branches of the clipped surrogate."""
    name, rows, n = be_rows
    be = _cuda() if name == "cuda" else Backend("emul", request.getfixturevalue("emul_lib"))
    P = gauss_bench_problem(rows, seed=rows + 5)
    perm = batches_for(rows, 10 if name == "cuda" else 1, 64, seed=17)
    order = np.random.default_rng(1).permutation(perm.shape[0])
    seen, done = dict(inside=0, lt=0, gt=0), 0
    for b in order:
        if done == n:
            break
        ref, br = gauss_reference(P["w"], *gauss_rows(P, perm[b]), GAUSS_HP)
        if br["ambiguous"]:                                     # a row on the clip boundary: the branch is not determined
            continue
        done += 1
        seen = {k: seen[k] + br[k] for k in seen}
        got = gauss_kernel_gradients(be, P, perm[b])
        for k in A_KEYS + C_KEYS:
            err = np.abs(got[k] - ref[k].v.reshape(got[k].shape))
            bound = ref[k].e.reshape(got[k].shape)
            assert (err <= bound).all(), (int(b), k, float((err - bound).max()), float(bound.max()))
    assert done == n and all(seen.values()), seen


@pytest.mark.parametrize("be_rows", [("emul", 2048), pytest.param(("cuda", 32768), marks=gpu)], ids=["emul", "cuda"])
def test_teacher_forced_adam_step_within_bound(request, be_rows):
    """One minibatch with the examples' learning rates and betas from a random Adam state at step 9: parameters and moments
    within the gradient's bound carried through Adam (powf 4 ulp, IEEE sqrtf / division / additions)."""
    name, rows = be_rows
    be = _cuda() if name == "cuda" else Backend("emul", request.getfixturevalue("emul_lib"))
    P = gauss_bench_problem(rows, seed=rows + 9)
    perm = batches_for(rows, 1, 64, seed=19)[:1]
    ref, _ = gauss_reference(P["w"], *gauss_rows(P, perm[0]), GAUSS_HP)
    rng = np.random.default_rng(4)
    ar0 = initial_arenas(P)[0]
    for k in ("a_m", "c_m"):
        ar0[k] = (1e-3 * rng.standard_normal(ar0[k].size)).astype(F32)
    for k in ("a_v", "c_v"):
        ar0[k] = rng.uniform(1e-7, 1e-5, ar0[k].size).astype(F32)
    t0 = 9
    hp = dict(GAUSS_HP, gate=1e30)
    out = be.run(P, perm, hp, arenas=ar0, steps=(t0, t0))
    assert (out["a_step"], out["c_step"]) == (t0 + 1, t0 + 1)
    f = lambda z: float(F32(z))
    for net, keys in (("a", A_KEYS), ("c", C_KEYS)):
        lr, b1, b2, eps = (f(hp[net + s]) for s in ("_lr", "_b1", "_b2", "_eps"))
        pw1, pw2 = b1 ** (t0 + 1), b2 ** (t0 + 1)
        bc1 = 1.0 - E(pw1, 4 * ULP * pw1)
        bc2s = efn(np.sqrt, lambda y: 0.5 / np.sqrt(y), 0.5, 1.0 - E(pw2, 4 * ULP * pw2))
        step = lr / bc1
        for k in keys:
            shp = P["shapes"][k]
            g = E(ref[k].v.reshape(-1), ref[k].e.reshape(-1))
            sl = slice(int(P[net + "_off"][keys.index(k)]), int(P[net + "_off"][keys.index(k)]) + int(np.prod(shp)))
            p0, m0, v0 = (E(ar0[net + s][sl]) for s in ("_flat", "_m", "_v"))
            m = m0 + (1.0 - b1) * (g - m0)
            v = b2 * v0 + ((1.0 - b2) * g) * g
            denom = efn(np.sqrt, lambda y: 0.5 / np.sqrt(y), 0.5, v) / bc2s + eps
            p = p0 - step * (m / denom)
            for name_, want, got in (("param", p, out[net + "_flat"][sl]), ("exp_avg", m, out[net + "_m"][sl]),
                                     ("exp_avg_sq", v, out[net + "_v"][sl])):
                err = np.abs(got - want.v)
                assert (err <= want.e).all(), (k, name_, float((err - want.e).max()))
            assert np.abs(p.v - p0.v).max() > 100 * p.e.max(), k      # the step is resolved, not lost in the bound


# ------------------------------------------------------------------------------------------------ 3. device invariants
def gauss_problem(rows, seed, D=17, A=6, H1=64, H2=64):
    sd0, states, actions, log_pi_old, ret, adv = make_problem(D, A, H1, H2, rows, seed)
    adv_n = (adv - adv.mean()) / adv.std()
    w = {k: v.numpy().astype(F64) for k, v in sd0.items()}
    P = dict(dims=(D, A, H1, H2), shapes=shapes_of(D, A, H1, H2), w=w, st=states.numpy(), ac=actions.numpy(),
             old=log_pi_old.numpy().ravel(), ret=ret.numpy().ravel(), adv=adv_n.numpy().ravel())
    _, P["a_off"], P["c_off"] = initial_arenas(P)
    return P


def chain(be, P, perm, hp, splits):
    state, total, out = initial_arenas(P)[0], 0.0, None
    steps, b0 = (0, 0), 0
    for n in splits:
        out = be.run(P, perm[b0:b0 + n], hp, arenas=state, steps=steps)
        state = {k: out[k] for k in ARENAS}
        steps, b0, total = (out["a_step"], out["c_step"]), b0 + n, total + float(out["stats"][3])
    assert b0 == perm.shape[0]
    return out, total


@pytest.mark.parametrize("be_rows", [("emul", 1024, 2), pytest.param(("cuda", 32768, 10), marks=gpu)], ids=["emul", "cuda"])
def test_launch_splitting(request, be_rows):
    """One launch of a Gaussian iteration (real lr, default betas) equals the same permutation split into launches of 1, 7,
    512 (host: 16) and the rest: parameters, moments and step counts bit for bit, the last minibatch's statistics equal and
    the actor steps of the parts adding up.  n_batches = 0 leaves the arenas unchanged."""
    name, rows, epochs = be_rows
    be = _cuda() if name == "cuda" else Backend("emul", request.getfixturevalue("emul_lib"))
    P = gauss_problem(rows, seed=4)
    perm = batches_for(rows, epochs, 64, seed=8)
    nb = perm.shape[0]
    whole = be.run(P, perm, GAUSS_HP)
    mid = 512 if name == "cuda" else 16
    parts, total = chain(be, P, perm, GAUSS_HP, [1, 7, mid, nb - 8 - mid])
    assert_arenas_equal(parts, whole, "split")
    assert (parts["a_step"], parts["c_step"]) == (whole["a_step"], whole["c_step"]) and whole["c_step"] == nb
    assert 0 < whole["a_step"] and total == whole["stats"][3] == whole["a_step"]
    assert np.array_equal(parts["stats"][:3], whole["stats"][:3])
    none = be.run(P, perm, GAUSS_HP, arenas={k: whole[k] for k in ARENAS}, steps=(whole["a_step"], nb), nb=0)
    assert_arenas_equal(none, whole, "n_batches = 0")
    assert (none["a_step"], none["c_step"]) == (whole["a_step"], nb) and np.array_equal(none["stats"], np.zeros(4, F32))


def test_closed_gate_leaves_the_actor_untouched(be):
    """gate_max below every kl: after a whole Gaussian iteration the actor's parameters, moments and step count are the
    input's bit for bit (from a nonzero Adam state), the critic stepped once per minibatch, and no actor step is counted."""
    P = gauss_problem(512, seed=6)
    perm = batches_for(512, 2, 64, seed=2)
    warm = be.run(P, perm[:3], GAUSS_HP)                         # a nonzero Adam state to start from
    ar0 = {k: warm[k] for k in ARENAS}
    out = be.run(P, perm, dict(GAUSS_HP, gate=-np.inf), arenas=ar0, steps=(warm["a_step"], 3))
    for k in ("a_flat", "a_m", "a_v"):
        assert np.array_equal(out[k], ar0[k]), k
    assert out["a_step"] == warm["a_step"] > 0 and out["c_step"] == 3 + perm.shape[0] and out["stats"][3] == 0
    assert not np.array_equal(out["c_flat"], ar0["c_flat"])


@pytest.mark.parametrize("shape", [(3, 5, 30, 12, 12), (17, 6, 64, 64, 64)], ids=["ragged", "bench"])
def test_arena_padding_stays_nan(be, shape):
    """The padding between tensors of all six arenas (FlatOptimizer aligns every tensor to 4 elements) is NaN before and after
    a Gaussian run, and the tensors themselves come out as from zero padding."""
    D, A, H1, H2, mb = shape
    P = gauss_problem(4 * mb, seed=9, D=D, A=A, H1=H1, H2=H2)
    perm = batches_for(4 * mb, 2, mb, seed=5)
    ar0 = initial_arenas(P)[0]
    pads = {k: padding_mask(ar0[k].size, P[k[0] + "_off"], A_KEYS if k[0] == "a" else C_KEYS, P["shapes"]) for k in ARENAS}
    assert all(m.any() for m in pads.values())
    nanned = {k: np.where(pads[k], np.nan, v).astype(F32) for k, v in ar0.items()}
    clean = be.run(P, perm, GAUSS_HP)
    out = be.run(P, perm, GAUSS_HP, arenas=nanned)
    for k in ARENAS:
        assert np.isnan(out[k][pads[k]]).all(), k
        assert np.array_equal(out[k][~pads[k]], clean[k][~pads[k]]), k


# ------------------------------------------------------------------------------------------------ 4. data-parallel form
def dp_problems(W, seed, straddle=False):
    """W ranks with the same weights and their own exact-regime rows (bench shape, one minibatch of 64 each)."""
    base = exact_problem(17, 6, 64, 64, 64, seed=seed, mb=64)
    Ps = [base]
    for r in range(1, W):
        Q = exact_problem(17, 6, 64, 64, 64, seed=seed, mb=64)       # same weights and patterns (same seed) ...
        rng = np.random.default_rng(seed * 31 + r)
        Q["st"] = rng.choice([-1.0, 0.0, 1.0], size=Q["st"].shape, p=[0.3, 0.4, 0.3])   # ... own states, actions, rows
        _, _, mu, _, _, v = forward(Q["w"], Q["st"])
        Q["pat"] = rng.integers(0, len(Q["pats"]), 64)
        Q["pat"][:len(Q["pats"])] = np.arange(len(Q["pats"]))     # row i < n_patterns represents pattern i
        Q["ac"] = mu + Q["pats"][Q["pat"]]
        Q["adv"] = rng.choice([-2.0, -1.0, -0.5, 0.5, 1.0, 2.0], 64)
        Q["ret"] = v + 0.5 * rng.integers(-4, 5, 64)
        Q["kind"] = (rng.random(64) < 0.25).astype(np.int64)
        Ps.append(Q)
    if straddle:
        Ps[0]["kind"][:] = 0                                         # rank 0: kl 0; rank 1: every fourth row at ratio 0
        Ps[1]["kind"][:] = (np.arange(64) % 4 == 0)
    return Ps


def dp_expectation(Ps, hp, perm):
    """The union minibatch: every rank's gradient and loss values (float64, exact), summed over ranks 0..W-1 in float32 and
    scaled by fl(1/W) (exact for W a power of two; for W = 3 the one rounding the kernel makes, emulated)."""
    W = len(Ps)
    refs = [ref_for(P, perm, hp) for P in Ps]
    invW = F32(1) / F32(W)
    grads = {}
    for k in A_KEYS + C_KEYS:
        s = F32(xsum(np.stack([r["grads"][k][0] for r in refs]), 0))
        grads[k] = (s * invW).astype(F64)
    mean = lambda key: np.add.accumulate(np.array([r[key][0] for r in refs], F32), dtype=F32)[-1] * invW
    kl, vl = mean("kl"), mean("vl")
    pl = np.mean([r["pl"][0] for r in refs])
    tol = max(r["pl_tol"][0] for r in refs) + W * 2.0 ** -23 * max(abs(r["pl"][0]) for r in refs)
    return grads, kl, vl, pl, tol, [bool(r["gate"][0]) for r in refs]


@pytest.mark.parametrize("W", [2, 3, 4, 8])
def test_dp_union_exact(be, W):
    """W ranks with distinct rows, one update: parameters, moments, step counts and the mean kl / value loss bit for bit
    against the float64 union (W = 3: with the kernel's one rounding of fl(1/3) per element emulated), identical on every
    rank."""
    Ps = dp_problems(W, seed=40 + W)
    hp = dict(EXACT_HP, ent_w=Ps[0]["ent_w"])
    for P in Ps:
        calibrate_old(be, P, hp)
    perm = np.arange(64)[None]
    grads, kl, vl, pl, tol, _ = dp_expectation(Ps, hp, perm)
    outs = be.run_dp(Ps, [perm] * W, hp)
    want = expected_arenas(Ps[0], initial_arenas(Ps[0])[0], grads, True, hp, (0, 0))
    for r, out in enumerate(outs):
        assert_arenas_equal(out, want, "rank %d" % r)
        assert (out["a_step"], out["c_step"]) == (1, 1)
        assert out["stats"][2] == kl and out["stats"][1] == vl and out["stats"][3] == 1
        assert abs(float(out["stats"][0]) - pl) <= tol


def test_dp_gate_decided_by_the_mean_kl(be):
    """Two ranks whose own kls straddle gate_max (rank 0: 0, rank 1: above it) with the mean exactly gate_max: the union's
    gate opens on every rank.  A kl sum without the 1/W would close it."""
    Ps = dp_problems(2, seed=77, straddle=True)
    hp = dict(EXACT_HP, ent_w=Ps[0]["ent_w"])
    for P in Ps:
        calibrate_old(be, P, hp)
    perm = np.arange(64)[None]
    _, kl, _, _, _, _ = dp_expectation(Ps, hp, perm)
    hp["gate"] = float(kl)
    grads, kl, vl, _, _, own = dp_expectation(Ps, hp, perm)
    assert own == [True, False]
    outs = be.run_dp(Ps, [perm] * 2, hp)
    want = expected_arenas(Ps[0], initial_arenas(Ps[0])[0], grads, True, hp, (0, 0))
    for out in outs:
        assert_arenas_equal(out, want, "straddle")
        assert out["a_step"] == 1 and out["stats"][3] == 1 and out["stats"][2] == kl


@pytest.mark.parametrize("be_rows", [("emul", 1024, 2), pytest.param(("cuda", 32768, 10), marks=gpu)], ids=["emul", "cuda"])
def test_dp_one_rank_is_the_single_process_kernel_exactly(request, be_rows):
    """In the exact regime (lr = 0, beta = 1/2: contraction cannot matter) the data-parallel kernel with one rank equals the
    single-process kernel bit for bit over a whole iteration, gates opening and closing."""
    name, rows, epochs = be_rows
    be = _cuda() if name == "cuda" else Backend("emul", request.getfixturevalue("emul_lib"))
    P = iteration_problem(rows, seed=rows + 1)
    hp = dict(EXACT_HP, a_lr=0.0, c_lr=0.0, ent_w=P["ent_w"])
    calibrate_old(be, P, hp)
    perm = batches_for(rows, epochs, 64, seed=23)
    kls = sum4(np.asarray(P["old"], F32)[perm] - np.asarray(P["lp"], F32)[perm]) * (F32(1) / F32(64))
    hp["gate"] = float(np.sort(kls)[perm.shape[0] // 2])
    single = be.run(P, perm, hp)
    (dp,) = be.run_dp([P], [perm], hp)
    assert_arenas_equal(dp, single, "W = 1")
    assert (dp["a_step"], dp["c_step"]) == (single["a_step"], single["c_step"]) and 0 < dp["a_step"] < perm.shape[0]
    assert np.array_equal(dp["stats"], single["stats"])


@pytest.mark.parametrize("be_rows", [("emul", 1024, 2), pytest.param(("cuda", 32768, 10), marks=gpu)], ids=["emul", "cuda"])
def test_dp_two_identical_ranks_equal_one(request, be_rows):
    """Gaussian bench iteration, real lr and default betas: two ranks with identical rows and permutations equal one rank bit
    for bit (both go through the same adam_elem site; g + g, * 1/2 and the kl mean are exact)."""
    name, rows, epochs = be_rows
    be = _cuda() if name == "cuda" else Backend("emul", request.getfixturevalue("emul_lib"))
    P = gauss_problem(rows, seed=12)
    perm = batches_for(rows, epochs, 64, seed=13)
    (one,) = be.run_dp([P], [perm], GAUSS_HP)
    for out in be.run_dp([P, P], [perm, perm], GAUSS_HP):
        assert_arenas_equal(out, one, "W = 2")
        assert (out["a_step"], out["c_step"]) == (one["a_step"], one["c_step"])
        assert np.array_equal(out["stats"], one["stats"])
    assert 0 < one["a_step"] < perm.shape[0]
