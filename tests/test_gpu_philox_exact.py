"""Every device random draw against the host Philox4x32-10 mirror (oracle/philox.py), draw for draw.

The statistical tests beside each kernel check the distributions (frequencies, moments, Kolmogorov-Smirnov); these check that
each kernel takes exactly its draws: its key, stream and counter layout, and the advance of its counter.  A row reading
another row's counter, a 64-bit key or counter cut to 32 bits, overlapping counters of consecutive launches, another stream
or a wrong integer reduction all change the draws here, whatever their distribution.

Keys and counters are chosen so that the high words carry data: the key is above 2^32 with both halves nonzero, the counters
start just below a multiple of 2^32 above 2^33, so that the draws of one launch carry into the counter's high word.

Bars: bit-exact for integers, uniforms and every quantity the kernel computes in a fully specified order; for normals
|z - z_mirror| <= 2^-18 max(1, |z|) (the device's logf / cospif against float64 Box-Muller: a few float32 ulp; any wrong draw is
an O(1) difference)."""
import ctypes
import importlib
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)
from oracle import philox  # noqa: E402

KEY = 0x9E3779B97F4A7C15                    # both 32-bit halves nonzero
C0 = (3 << 32) - 100                        # the first launch's draws run across the carry into the high word
TANH, RELU = 0, 1
NORMAL_TOL = 2.0 ** -18


def _normal_close(got, want, scale=1.0):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    err = np.abs(got - scale * want) / (scale * np.maximum(1.0, np.abs(want)))
    assert err.max() <= NORMAL_TOL, (float(err.max()), int(err.argmax()))


# ------------------------------------------------------------------------------------------------ CPU: the mirror itself
def _block(key, c):
    return [int(w) for w in philox.gen(key, c[0] | (c[1] << 32), c[2] | (c[3] << 32))]


def test_mirror_reproduces_the_random123_known_answers():
    """The three Philox4x32-10 known-answer vectors of Random123 (kat_vectors)."""
    assert _block(0, (0, 0, 0, 0)) == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    assert _block(0xFFFFFFFFFFFFFFFF, (0xFFFFFFFF,) * 4) == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    assert _block(0x299F31D0A4093822, (0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344)) == \
        [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


def test_mirror_derived_draws():
    """u24 / u53 / below / normal from one block, and the vectorised form equals the scalar one."""
    ctr = np.uint64(C0) + np.arange(64, dtype=np.uint64)
    x, y = (np.asarray(w, np.uint64) for w in philox.gen(KEY, ctr, 5)[:2])
    assert np.array_equal(philox.u24(KEY, ctr, 5), (x >> np.uint64(8)).astype(np.float32) / np.float32(2 ** 24))
    want53 = np.array([((int(a) >> 5) * 2 ** 26 + (int(b) >> 6)) / 2.0 ** 53 for a, b in zip(x, y)])
    assert np.array_equal(philox.u53(KEY, ctr, 5), want53)
    for n in (1, 7, 1000, 100_003, 2 ** 32 - 1):
        want = np.array([((int(a) << 32 | int(b)) * n) >> 64 for a, b in zip(x, y)], np.uint64)
        assert np.array_equal(philox.below(KEY, ctr, 5, n), want)
    u1, u2 = ((x >> np.uint64(8)) + np.uint64(1)) / 2.0 ** 24, (y >> np.uint64(8)) / 2.0 ** 24
    assert np.array_equal(philox.normal(KEY, ctr, 5), np.sqrt(-2 * np.log(u1)) * np.cos(2 * np.pi * u2))
    for k in (0, 17, 63):
        assert [int(w[k]) for w in philox.gen(KEY, ctr, 5)] == [int(w) for w in philox.gen(KEY, int(ctr[k]), 5)]


def _curand():
    for name in ("libcurand.so.10", "libcurand.so"):
        try:
            return ctypes.CDLL(name)
        except OSError:
            pass
    return None


def test_mirror_matches_curand_host_generator():
    """cuRAND's host CURAND_RNG_PSEUDO_PHILOX4_32_10 generator: its k-th block of four words is the block at counter
    (0, 0, k, 0) of the seed; checked for the first four blocks of three seeds with both key halves nonzero."""
    lib = _curand()
    if lib is None:
        pytest.skip("no libcurand could be loaded: the optional cross-check against cuRAND's host generator is skipped")
    for seed in (0x0123456789ABCDEF, KEY, 0xDEADBEEF00C0FFEE):
        gen = ctypes.c_void_p()
        assert lib.curandCreateGeneratorHost(ctypes.byref(gen), 161) == 0           # CURAND_RNG_PSEUDO_PHILOX4_32_10
        try:
            assert lib.curandSetPseudoRandomGeneratorSeed(gen, ctypes.c_ulonglong(seed)) == 0
            out = np.zeros(16, np.uint32)
            assert lib.curandGenerate(gen, out.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(16)) == 0
        finally:
            lib.curandDestroyGenerator(gen)
        want = np.concatenate([np.array([int(w) for w in philox.gen(seed, 0, k)], np.uint32) for k in range(4)])
        assert np.array_equal(out, want), hex(seed)


def test_mirror_picks():
    """epsilon-greedy and the categorical inverse CDF on hand-made draws."""
    acts, explored = philox.epsilon_greedy(KEY, C0, 17, 512, 5, 0.3, np.arange(512) % 5)
    u = philox.u24(KEY, np.uint64(C0) + np.uint64(2) * np.arange(512, dtype=np.uint64), 17)
    assert np.array_equal(explored, u < np.float32(0.3)) and 0 < explored.sum() < 512
    assert np.array_equal(acts[~explored], (np.arange(512) % 5)[~explored])
    pick, gap = philox.categorical_inverse_cdf([0.0, 0.2, 0.5, 0.999], np.zeros((4, 4)))
    assert pick.tolist() == [0, 0, 2, 3] and np.allclose(gap, [0.25, 0.05, 0.0, 0.001], atol=1e-6)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def rl():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import deeprl_b200 as rl
    rl.select_device(0)
    rl.Config.COMPUTE_DTYPE = torch.float32
    torch.backends.cuda.matmul.allow_tf32 = False
    return rl


def _harness(name):
    """Another device test module's kernel harness (the same launch code its own tests use)."""
    return importlib.import_module(name)


def _counter(v=C0):
    return torch.full((1,), v, dtype=torch.int64, device="cuda")


# ---- replay rings whose frame payload is the ring index
def _payload_ring(rl, cls, cap, B, hl, n, pos, seed_rows, priorities=None):
    g = torch.Generator(device="cuda").manual_seed(seed_rows)
    rp = cls(cap, B, n, 0.9, hl, seed=KEY)
    frames = torch.arange(cap, dtype=torch.int64, device="cuda").view(cap, 1).view(torch.uint8)
    act = torch.randint(0, 7, (cap,), device="cuda", generator=g).int()
    rew = torch.randn(cap, dtype=torch.float64, device="cuda", generator=g)
    msk = (torch.rand(cap, device="cuda", generator=g) > 0.15).int()
    rp.item_shape, rp.item_dtype = (1,), np.dtype(np.int64)
    if priorities is None:
        rp.load_synthetic(frames, act, rew, msk, pos)
    else:
        rp.load_synthetic(frames, act, rew, msk, pos, priorities=priorities)
    return rp, act.cpu().numpy(), rew.cpu().numpy(), msk.cpu().numpy()


def _oracle_ring(ocls, cap, B, hl, n, pos, size, act, rew, msk):
    o = ocls(cap, B, n, 0.9, hl)
    o.data = dict(state=[np.array([i], np.int64) for i in range(cap)], action=list(act), reward=list(rew), mask=list(msk))
    o.pos, o._size = pos, size
    return o


def _check_scalars(bufs, tr):
    assert np.array_equal(bufs["action"].cpu().numpy(), np.asarray(tr.action, np.int64))
    assert np.array_equal(bufs["reward"].cpu().numpy(), np.asarray(tr.reward, np.float64).astype(np.float32))
    assert np.array_equal(bufs["mask"].cpu().numpy(), np.asarray(tr.mask).astype(np.float32))


def _sentinel(bufs):
    for k in ("idx", "action", "tree_idx"):
        bufs[k].fill_(-7)
    for k in ("reward", "mask", "prob64", "prob"):
        bufs[k].fill_(float("nan"))


@pytest.mark.gpu
@pytest.mark.parametrize("cap,B", [(64, 1), (64, 37), (64, 512), (100_003, 512)])
def test_uniform_replay_philox_candidates(rl, cap, B):
    """select_uniform_kernel's candidate g is below(size) at ring_state[4] + g on stream 1: the mirror's candidates through
    oracle/replay.py's valid-index filter give the indices, the candidates consumed, action / n-step reward / mask (both through
    the fused scalars and through the gather) and the frames; the counter advances by the stream length.  The ring is full,
    with the cursor seam, the first history - 1 slots and the last n_step slots invalid."""
    from oracle.replay import UniformReplay as OU
    hl, n, pos = 4, 3, 20 if cap == 64 else 54_321
    rp, act, rew, msk = _payload_ring(rl, rl.UniformReplay, cap, B, hl, n, pos, seed_rows=cap + B)
    ora = _oracle_ring(OU, cap, B, hl, n, pos, cap, act, rew, msk)
    n_cand = min(8192, max(2 * B, B + 256))
    cand = philox.below(KEY, np.uint64(C0) + np.arange(n_cand, dtype=np.uint64), 1, cap).astype(np.int64)
    tr, taken, used = ora.sample(B, candidates=cand)
    bufs = rp._buffers(B, torch.uint8, "nchw")
    _sentinel(bufs)
    rp.ring_state[4] = C0
    rp.select(B, bufs["idx"], scalars=bufs)
    assert np.array_equal(bufs["idx"].cpu().numpy(), taken)
    assert rp._status.tolist() == [B, used] and int(rp.ring_state[4]) == C0 + n_cand
    _check_scalars(bufs, tr)
    _sentinel(bufs)
    rp.ring_state[4] = C0
    got = rp.sample(B)
    assert np.array_equal(bufs["idx"].cpu().numpy(), taken) and int(rp.ring_state[4]) == C0 + n_cand
    assert np.array_equal(got.state.cpu().numpy(), tr.state) and np.array_equal(got.next_state.cpu().numpy(), tr.next_state)
    _check_scalars(bufs, tr)


@pytest.mark.gpu
def test_uniform_replay_philox_dry_stream(rl):
    """A ring too sparse for the candidate stream (8 of 4096 slots filled, 2 valid): the accepted mirror candidates in stream
    order, then the tail cycled j -> accepted[j % accepted]; status = (accepted, every candidate); scalars and frames of the
    cycled indices."""
    from oracle.replay import UniformReplay as OU
    cap, B, hl, n, size = 4096, 512, 4, 3, 8
    rp, act, rew, msk = _payload_ring(rl, rl.UniformReplay, cap, B, hl, n, size, seed_rows=5)
    rp.ring_state[0], rp.ring_state[1] = size, size
    rp.pos, rp._size = size, size
    ora = _oracle_ring(OU, cap, B, hl, n, size, size, act, rew, msk)
    n_cand = 2 * B
    cand = philox.below(KEY, np.uint64(C0) + np.arange(n_cand, dtype=np.uint64), 1, size).astype(np.int64)
    acc = np.asarray([c for c in cand if ora.valid_index(int(c))], np.int64)
    assert 0 < len(acc) < B
    want = acc[np.arange(B) % len(acc)]
    rows = [ora.construct_transition(int(i)) for i in want]
    tr = OU._stack(rows, type(rows[0]))
    bufs = rp._buffers(B, torch.uint8, "nchw")
    _sentinel(bufs)
    rp.ring_state[4] = C0
    rp.select(B, bufs["idx"], scalars=bufs)
    assert np.array_equal(bufs["idx"].cpu().numpy(), want)
    assert rp._status.tolist() == [len(acc), n_cand] and int(rp.ring_state[4]) == C0 + n_cand
    _check_scalars(bufs, tr)
    _sentinel(bufs)
    rp.ring_state[4] = C0
    got = rp.sample(B, check=False)
    assert np.array_equal(bufs["idx"].cpu().numpy(), want)
    assert np.array_equal(got.state.cpu().numpy(), tr.state) and np.array_equal(got.next_state.cpu().numpy(), tr.next_state)
    _check_scalars(bufs, tr)


def _per_priorities(cap, hl, n, pos, share, seed):
    """Leaves in [0.5, 1.5), the invalid slots (first hl - 1, the seam, the last n) heavy enough to hold ``share`` of the mass."""
    rng = np.random.RandomState(seed)
    p = rng.uniform(0.5, 1.5, cap)
    bad = np.r_[np.arange(hl - 1), np.arange(pos - n, pos + hl - 1), np.arange(cap - n, cap)]
    p[bad] = share / (1 - share) * p.sum() / len(bad)
    return torch.from_numpy(p).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("cap,B", [(1000, 64), (100_003, 512)])
def test_prioritized_replay_philox_draws(rl, cap, B):
    """sumtree_sample_kernel without given draws: the stratified u_i are u53 at ring_state[4] + i on stream 2, the back-fill
    picks below(len) at ring_state[4] + B + k on stream 3.  The mirror's draws through oracle/replay.py's PrioritizedReplay
    give, bit for bit and over rounds of update_priorities: tree and data indices, float64 sampling probabilities, frames and
    scalars, the tree after each round's updates and max_priority; status[0] is the valid count; the counter advances by 2B."""
    from oracle.replay import PrioritizedReplay as OP
    hl, n, pos = 4, 3, cap // 3 + 7
    prio0 = _per_priorities(cap, hl, n, pos, 0.3, cap)
    rp, act, rew, msk = _payload_ring(rl, rl.PrioritizedReplay, cap, B, hl, n, pos, seed_rows=cap, priorities=prio0)
    ora = _oracle_ring(OP, cap, B, hl, n, pos, cap, act, rew, msk)
    ora.tree.tree[:] = rp.tree.tree.cpu().numpy()
    ora.tree.write, ora.tree.n_entries = pos, cap
    rp.ring_state[4] = C0
    rng = np.random.RandomState(7)
    bufs = rp._buffers(B, torch.uint8, "nchw")
    for rd in range(3):
        ctr = C0 + 2 * B * rd
        u = philox.u53(KEY, np.uint64(ctr) + np.arange(B, dtype=np.uint64), 2)
        seg = ora.tree.total() / B
        n_valid = sum(ora.valid_index(int(ora.tree.get(seg * i + (seg * (i + 1) - seg * i) * u[i])[2])) for i in range(B))
        assert 0 < n_valid < B, n_valid                 # back-fills happen
        k = np.arange(B - n_valid, dtype=np.uint64)
        fills = philox.below(KEY, np.uint64(ctr + B) + k, 3, np.uint64(n_valid) + k).astype(np.int64)
        want = ora.sample(uniforms=u, fills=fills)
        _sentinel(bufs)
        got = rp.sample()
        assert int(rp.ring_state[4]) == ctr + 2 * B and int(rp._status[0]) == n_valid
        assert np.array_equal(got.idx.cpu().numpy(), want.idx)
        assert np.array_equal(bufs["idx"].cpu().numpy(), want.idx - cap + 1)
        assert np.array_equal(bufs["prob64"].cpu().numpy(), want.sampling_prob)
        assert np.array_equal(got.state.cpu().numpy(), want.state) and np.array_equal(got.next_state.cpu().numpy(), want.next_state)
        _check_scalars(bufs, want)
        p = (np.abs(rng.randn(B)) * 3 + 0.05).astype(np.float32)
        rp.update_priorities((got.idx, torch.from_numpy(p).cuda()))
        ora.update_priorities(zip(want.idx, p))
        assert np.array_equal(rp.tree.tree.cpu().numpy(), ora.tree.tree), rd
        assert rp.max_priority == float(ora.max_priority)


@pytest.mark.gpu
def test_prioritized_sample_without_a_valid_draw(rl):
    """Every stratified draw lands on an invalid slot: status[0] = 0 and, instead of whatever the output buffers held, every
    row holds data index history - 1, its leaf and that leaf's probability, as select_uniform_kernel does; the host check
    still raises.  Only the index outputs are read (nothing is gathered from such a batch)."""
    cap, B, hl, n, pos = 16, 8, 4, 1, 8
    prio = torch.zeros(cap, dtype=torch.float64, device="cuda")
    prio[[0, 1, 2, 7, 8, 9, 10, 15]] = 1.0                  # the invalid slots: first hl - 1, the seam, the last n
    rp, *_ = _payload_ring(rl, rl.PrioritizedReplay, cap, B, hl, n, pos, seed_rows=1, priorities=prio)
    bufs = rp._buffers(B, torch.uint8, "nchw")
    _sentinel(bufs)
    u, fills = np.full(B, 0.5), np.zeros(B, np.int64)
    rp._select_per(B, bufs, uniforms=u, fills=fills, check=False)
    assert int(rp._status[0]) == 0
    leaf = hl - 1 + cap - 1
    assert bufs["tree_idx"].tolist() == [leaf] * B and bufs["idx"].tolist() == [hl - 1] * B
    want = float(rp.tree.tree[leaf]) / float(rp.tree.tree[0])
    assert bufs["prob64"].tolist() == [want] * B
    with pytest.raises(IndexError):
        rp.sample(uniforms=u, fills=fills)


# ---- epsilon-greedy actor steps (stream 17)
EPS_KERNELS = ["nstep", "dueling", "c51", "qr", "rainbow"]


def _eps_actor(rl, kernel, N, D, H, A):
    """(q_values(obs) on the eager network, step(obs, counter, seed, eps) -> actions) for one kernel.  The distributional
    heads get K = 64 // (A + 1) atoms or quantiles (at least 2), so that N rows of (A + 1) K logits fit in shared memory."""
    K = max(2, 64 // (A + 1))
    if kernel == "nstep":
        net, step = _harness("test_nstep_dqn_device")._actor(rl, RELU, N, D, H, A)

        def q(x):
            with torch.no_grad():
                return net(x.float())["q"]
        return q, lambda obs, c, s, e: step(obs, c, s, e)[1]
    if kernel == "dueling":
        net, step = _harness("test_dqn_device")._dueling_actor(rl, TANH, N, D, H, A)

        def q(x):
            with torch.no_grad():
                return net(x.float())["q"]
        return q, step
    if kernel in ("c51", "qr"):
        kind = 0 if kernel == "c51" else 1
        return _harness("test_dist_dqn_device")._dist_actor(rl, kind, RELU if kind == 0 else TANH, N, D, H, A, K)
    _, q, step = _harness("test_rainbow_device")._actor(rl, False, RELU, N, D, H, A, K)
    ncounter = _counter(0)

    def rstep(obs, c, s, e):
        act = step(obs, c, ncounter, s, e)[0]
        assert int(ncounter) == 0
        return act
    return q, rstep


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", EPS_KERNELS)
@pytest.mark.parametrize("A", [2, 5, 18])
@pytest.mark.parametrize("eps", [1.0, 0.3])
def test_epsilon_greedy_draws(rl, kernel, A, eps):
    """Two consecutive steps of 256 rows: row n explores iff u24(ctr0 + 2n) < epsilon and then takes
    min(int(u24(ctr0 + 2n + 1) A), A - 1), else the eager network's argmax (every row's top-2 margin above 1e-3); the second
    step starts at ctr0 + 2N; the counter ends at ctr0 + 4N."""
    N, D, H = 256, 6, 32
    q_values, step = _eps_actor(rl, kernel, N, D, H, A)
    cand = torch.randn(8192, D, dtype=torch.float64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(A))
    top = q_values(cand).topk(2, dim=1).values
    obs = cand[(top[:, 0] - top[:, 1]) > 1e-3][:N].contiguous()
    assert obs.shape[0] == N
    greedy = q_values(obs).argmax(1).cpu().numpy()
    counter = _counter()
    for s in range(2):
        want, explored = philox.epsilon_greedy(KEY, C0 + 2 * N * s, 17, N, A, eps, greedy)
        got = step(obs, counter, KEY, eps).cpu().numpy()
        assert np.array_equal(got, want), (s, np.nonzero(got != want)[0][:8])
        assert int(counter) == C0 + 2 * N * (s + 1)
        if eps < 1:
            assert 0 < explored.sum() < N and (want[explored] != greedy[explored]).any()


# ---- A2C categorical actor (stream 13)
@pytest.mark.gpu
@pytest.mark.parametrize("A", [2, 5, 18])
def test_a2c_categorical_draws(rl, A):
    """Zero logits: expf(0) = 1 and the partial sums are exact integers, so every row's pick is the mirror's float32 inverse
    CDF of u24 at ctr0 + n, bit for bit, over two consecutive steps (the counter advances by N)."""
    h = _harness("test_a2c_device")
    N, D, H = 256, 6, 32
    net, step = h._actor(rl, h.CAT, TANH, N, D, H, A)
    with torch.no_grad():
        net.fc_action.weight.zero_(), net.fc_action.bias.zero_()
    obs = torch.randn(N, D, dtype=torch.float64, device="cuda")
    counter = _counter()
    for s in range(2):
        u = philox.u24(KEY, np.uint64(C0 + N * s) + np.arange(N, dtype=np.uint64), 13)
        want, _ = philox.categorical_inverse_cdf(u, np.zeros((N, A), np.float32))
        got = step(obs, counter, KEY)[1].cpu().numpy()[:, 0].astype(np.int64)
        assert np.array_equal(got, want) and int(counter) == C0 + N * (s + 1)


@pytest.mark.gpu
def test_a2c_categorical_draws_general_logits(rl):
    """Logits of a trained-looking head: the picks equal a float64 inverse CDF on the float64 logits of the same network, for
    every row whose target is further than 1e-5 (relative) from a partial-sum boundary; fewer than 1 % are excluded.  Four
    steps of 256 rows."""
    import copy
    h = _harness("test_a2c_device")
    N, D, H, A, steps = 256, 6, 32, 6, 4
    net, step = h._actor(rl, h.CAT, TANH, N, D, H, A)
    n64 = copy.deepcopy(net).double().cpu()
    counter = _counter()
    got, want, gap = [], [], []
    for s in range(steps):
        obs = torch.randn(N, D, dtype=torch.float64, device="cuda")
        got.append(step(obs, counter, KEY)[1].cpu().numpy()[:, 0].astype(np.int64))
        with torch.no_grad():
            logits = n64.fc_action(n64.phi_body(obs.float().double().cpu())).numpy()
        u = philox.u24(KEY, np.uint64(C0 + N * s) + np.arange(N, dtype=np.uint64), 13)
        w, g = philox.categorical_inverse_cdf(u, logits, np.float64)
        want.append(w), gap.append(g)
    got, want, keep = np.concatenate(got), np.concatenate(want), np.concatenate(gap) > 1e-5
    assert keep.mean() > 0.99, keep.mean()
    assert np.array_equal(got[keep], want[keep]) and int(counter) == C0 + N * steps
    assert len(set(want[keep].tolist())) == A


# ---- Gaussian actor steps (A2C stream 13, PPO stream 7)
@pytest.mark.gpu
def test_a2c_gaussian_draws(rl):
    """Mean head zeroed (tanh(0) = 0): action = softplus(std) z with z the normal at ctr0 + n A + j, distinct observations per
    row, two consecutive steps (the counter advances by N A)."""
    import torch.nn.functional as F
    h = _harness("test_a2c_device")
    N, D, H, A = 128, 17, 32, 8
    net, step = h._actor(rl, h.GAUSS, RELU, N, D, H, A)
    with torch.no_grad():
        net.fc_action.weight.zero_(), net.fc_action.bias.zero_()
        net.std.copy_(torch.linspace(-1.0, 1.0, A))
    sd = F.softplus(net.std.detach()).cpu().numpy().astype(np.float64)
    obs = torch.randn(N, D, dtype=torch.float64, device="cuda")
    counter = _counter()
    for s in range(2):
        z = philox.normal(KEY, np.uint64(C0 + N * A * s) + np.arange(N * A, dtype=np.uint64), 13).reshape(N, A)
        act = step(obs, counter, KEY)[1].cpu().numpy().astype(np.float64)
        _normal_close(act / sd, z)
        assert int(counter) == C0 + N * A * (s + 1)


@pytest.mark.gpu
def test_ppo_gaussian_draws(rl):
    """gaussian_actor_step_kernel: the same with the normal at ctr0 + n A + j of stream 7, 64 rows x 16 dimensions."""
    import torch.nn.functional as F
    from deeprl_b200.component.actor import DeviceGaussianActor
    N, D, A = 64, 17, 16
    torch.manual_seed(0)
    net = rl.GaussianActorCriticNet(D, A, actor_body=rl.FCBody(D, gate=torch.tanh), critic_body=rl.FCBody(D, gate=torch.tanh))
    with torch.no_grad():
        net.fc_action.weight.zero_(), net.fc_action.bias.zero_()
        net.std.copy_(torch.linspace(-0.5, 0.7, A))
    sd = F.softplus(net.std.detach()).cpu().numpy().astype(np.float64)
    actor = DeviceGaussianActor(net, rl.MeanStdNormalizer(), N, seed=KEY)
    actor.counter.fill_(C0)
    raw = np.random.RandomState(0).randn(N, D).astype(np.float32)
    for s in range(2):
        out = actor.step(raw, update=False)
        z = philox.normal(KEY, np.uint64(C0 + N * A * s) + np.arange(N * A, dtype=np.uint64), 7).reshape(N, A)
        assert float(out["mean"].abs().max()) == 0.0
        _normal_close(out["action"].cpu().numpy().astype(np.float64) / sd, z)
        assert int(actor.counter) == C0 + N * A * (s + 1)


# ---- NoisyLinear noise (stream 29)
@pytest.mark.gpu
def test_rainbow_actor_noise_draws(rl):
    """The actor step's noise vector is noise_std x the normal at noise_counter + i, consecutive steps back to back; the
    epsilon counter stays."""
    rb = _harness("test_rainbow_device")
    N, D, H, A, K, std = 4, 6, 32, 5, 51, 0.5
    nz = rb.noise_len(D, H, H, A, K)
    _, _, step = rb._actor(rl, True, RELU, N, D, H, A, K)
    obs = torch.randn(N, D, dtype=torch.float64, device="cuda")
    counter, ncounter = _counter(77), _counter()
    for s in range(2):
        _, used = step(obs, counter, ncounter, KEY, 1.0)
        z = philox.normal(KEY, np.uint64(C0 + nz * s) + np.arange(nz, dtype=np.uint64), 29)
        _normal_close(used.cpu().numpy(), z, std)
        assert int(ncounter) == C0 + nz * (s + 1) and int(counter) == 77


@pytest.mark.gpu
def test_rainbow_update_noise_draws(rl):
    """The update draws the target network's vector at counter + i and the online one at counter + noise_len + i (std x normal,
    written to the arenas test_drawn_noise reads); the counter advances by 2 noise_len per update, two updates back to back."""
    rb = _harness("test_rainbow_device")
    noisy, gate, dims, cfg, sd0, tgt0, batch, _ = rb.case_setup(0)
    nz, std = rb.noise_len(*dims), 0.5
    counter = _counter()
    for s in range(2):
        st = rb.EmulState(noisy, sd0, tgt0)
        _, _, written = rb.cabi_update(st, noisy, gate, batch, dims[1], dims[2], cfg, None, seed=KEY, counter=counter, std=std)
        base = np.uint64(C0 + 2 * nz * s)
        _normal_close(st.target_noise, philox.normal(KEY, base + np.arange(nz, dtype=np.uint64), 29), std)
        _normal_close(written[:nz], philox.normal(KEY, base + np.uint64(nz) + np.arange(nz, dtype=np.uint64), 29), std)
        rb.check_noise_arena(written, written[:nz], dims)
        assert int(counter) == C0 + 2 * nz * (s + 1)
