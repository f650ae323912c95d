"""TEST INFRASTRUCTURE -- host restatement of the device random draws (``Philox`` in deeprl_b200/csrc/common.cuh), numpy-vectorised
over counters, so that every draw a kernel makes can be reproduced bit for bit.

Philox4x32-10 (Salmon, Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC'11): a 128-bit counter
(c0, c1, c2, c3) and a 64-bit key (k0, k1), ten rounds of two 32x32 -> 64-bit multiplies, the key bumped by the Weyl constants
between rounds.  The kernels use key = ``seed`` (k0 low word), counter = (``ctr`` low word, ``ctr`` high word, ``stream`` low
word, ``stream`` high word).  On top of one 128-bit block:

* ``u24``    float32 (x >> 8) / 2^24 in [0, 1)
* ``u53``    float64 ((x >> 5) 2^26 + (y >> 6)) / 2^53 in [0, 1)
* ``below``  the high 64 bits of ((x << 32) | y) * n, an integer in [0, n)
* ``normal`` Box-Muller on u1 = ((x >> 8) + 1) / 2^24 in (0, 1] and u2 = (y >> 8) / 2^24, here in float64 (the device's
  logf / cospif are within a few float32 ulp of it)

and the two picks the actor kernels make from them, in float32 operation for operation (``epsilon_greedy``,
``categorical_inverse_cdf``).
"""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)
_32 = np.uint64(32)


def _u64(x):
    return np.asarray(x, dtype=np.uint64) if not isinstance(x, int) else np.asarray(x & 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)


def gen(seed, ctr, stream=0):
    """Philox4x32-10 of key ``seed`` (uint64) at counter (``ctr`` uint64, ``stream`` uint64): four uint32 arrays shaped like
    ``ctr`` broadcast against ``seed`` and ``stream``."""
    seed, ctr, stream = np.broadcast_arrays(_u64(seed), _u64(ctr), _u64(stream))
    k0, k1 = (seed & _LO).astype(np.uint32), (seed >> _32).astype(np.uint32)
    c0, c1 = (ctr & _LO).astype(np.uint32), (ctr >> _32).astype(np.uint32)
    c2, c3 = (stream & _LO).astype(np.uint32), (stream >> _32).astype(np.uint32)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = M0 * c0.astype(np.uint64)
            p1 = M1 * c2.astype(np.uint64)
            hi0, lo0 = (p0 >> _32).astype(np.uint32), (p0 & _LO).astype(np.uint32)
            hi1, lo1 = (p1 >> _32).astype(np.uint32), (p1 & _LO).astype(np.uint32)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
            k0, k1 = k0 + W0, k1 + W1
    return c0, c1, c2, c3


def u24(seed, ctr, stream):
    return ((gen(seed, ctr, stream)[0] >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)).astype(np.float32)


def u53(seed, ctr, stream):
    x, y = gen(seed, ctr, stream)[:2]
    a, b = (x >> np.uint32(5)).astype(np.uint64), (y >> np.uint32(6)).astype(np.uint64)
    return (a * np.uint64(67108864) + b).astype(np.float64) * (1.0 / 9007199254740992.0)


def below(seed, ctr, stream, n):
    """Integer in [0, n): the high word of the 128-bit product of the 64-bit draw ((x << 32) | y) and ``n`` (n < 2^32)."""
    x, y = gen(seed, ctr, stream)[:2]
    n = np.broadcast_to(_u64(n), x.shape)
    assert np.all(n < np.uint64(1 << 32)), "below: n must stay below 2^32"
    # (xh 2^32 + xl) n / 2^64 = (xh n + (xl n >> 32)) >> 32, every term below 2^64
    return (x.astype(np.uint64) * n + ((y.astype(np.uint64) * n) >> _32)) >> _32


def normal(seed, ctr, stream):
    """Box-Muller in float64 on the two 24-bit uniforms of one block."""
    x, y = gen(seed, ctr, stream)[:2]
    u1 = ((x >> np.uint32(8)).astype(np.float64) + 1.0) / 16777216.0
    u2 = (y >> np.uint32(8)).astype(np.float64) / 16777216.0
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def epsilon_greedy(seed, ctr0, stream, N, A, epsilon, greedy):
    """The epsilon-greedy actor kernels' pick for rows n < N: random when u24(ctr0 + 2n) < epsilon, then
    min(int(u24(ctr0 + 2n + 1) * A), A - 1) (float32 product); otherwise ``greedy[n]``.  Returns (actions, explored)."""
    c = _u64(ctr0) + np.uint64(2) * np.arange(N, dtype=np.uint64)
    explore = u24(seed, c, stream) < np.float32(epsilon)
    rand = np.minimum((u24(seed, c + np.uint64(1), stream) * np.float32(A)).astype(np.int64), A - 1)
    return np.where(explore, rand, np.asarray(greedy, np.int64)), explore


def categorical_inverse_cdf(u, logits, dtype=np.float32):
    """The categorical actor's pick per row: target = u * sum_j exp(z_j - max z), the first j whose running sum of
    exp(z_j - max z) exceeds the target, A - 1 if none does; sums left to right in ``dtype``.  Returns (actions, the
    distance of each target to its nearest partial-sum boundary relative to the row's total)."""
    z = np.asarray(logits, dtype)
    e = np.exp(z - z.max(axis=1, keepdims=True)).astype(dtype)
    s = np.zeros(z.shape[0], dtype)
    for j in range(z.shape[1]):
        s = (s + e[:, j]).astype(dtype)
    target = (np.asarray(u, dtype) * s).astype(dtype)
    pick = np.full(z.shape[0], z.shape[1] - 1, np.int64)
    done = np.zeros(z.shape[0], bool)
    c = np.zeros(z.shape[0], dtype)
    gap = np.full(z.shape[0], np.inf)
    for j in range(z.shape[1]):
        c = (c + e[:, j]).astype(dtype)
        gap = np.minimum(gap, np.abs(c.astype(np.float64) - target.astype(np.float64)))
        hit = ~done & (target < c)
        pick[hit] = j
        done |= hit
    return pick, gap / s.astype(np.float64)
