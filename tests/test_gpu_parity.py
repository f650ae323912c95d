"""GPU parity tests (run with ``-m gpu`` on an H100): every CUDA entry point of libb2rl.so, called through
the product's host mirror, against (a) the golden vectors generated from the reference itself and (b) the
pinned CPU oracle on fresh seeded inputs.  Bars: bit-exact for indices, uint8 frames, float64 tree nodes and
fp32 quantities whose operation order is fully specified; the tolerance written beside each check otherwise.
Nothing here reads /root/reference."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rl():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import deeprl_b200 as rl
    rl.select_device(0)
    rl.Config.COMPUTE_DTYPE = torch.float32      # parity mode (another test module of the same session may have left bf16 selected)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return rl


def dev(x, dtype=None):
    t = torch.as_tensor(np.asarray(x))
    if dtype is not None:
        t = t.to(dtype)
    return t.cuda()


# ------------------------------------------------------------------------------------------ sum tree
@pytest.mark.parametrize("cap", [2, 5, 8, 1000])
def test_sumtree_trace_bit_exact(rl, golden, cap):
    g = golden("sumtree")
    t = rl.SumTree(cap)
    ops_, a0, a1 = g["cap%d_ops" % cap], g["cap%d_a0" % cap], g["cap%d_a1" % cap]
    n = len(ops_) if cap <= 8 else 1500
    snaps = g["cap%d_snaps" % cap] if cap <= 8 else None
    ref = None
    if cap > 8:
        from oracle.sum_tree import SumTree as O
        ref = O(cap)
    for k in range(n):
        op = ops_[k]
        if op == 0:
            t.add(a0[k])
            ref and ref.add(a0[k])
        elif op == 1:
            idx, p, di = t.get(a0[k])
            assert (idx, di) == (g["cap%d_res_idx" % cap][k], g["cap%d_res_data" % cap][k])
            assert p == g["cap%d_res_p" % cap][k]
            ref and ref.get(a0[k])
        else:
            t.update(int(a0[k]), a1[k])
            ref and ref.update(int(a0[k]), a1[k])
        if snaps is not None:
            assert np.array_equal(t.tree.cpu().numpy(), snaps[k]), k
    if ref is not None:
        assert np.array_equal(t.tree.cpu().numpy(), ref.tree)
    else:
        assert np.array_equal(t.tree.cpu().numpy(), g["cap%d_tree" % cap])


def test_sumtree_batched_rounds_bit_exact(rl, golden):
    """B stratified descents + B ordered updates per round incl. duplicates inside a batch (first one wins)."""
    g = golden("sumtree")
    cap, B = 1000, g["batch_u"].shape[1]
    t = rl.SumTree(cap)
    t.ring_state[1] = cap + 10                                 # standalone tree: every data index counts as valid
    one = torch.ones(1, dtype=torch.float64, device="cuda")
    t.add_n(600, one), t.add_n(400, one)                       # cap x add(1.0) in two batched calls
    assert int(t.ring_state[3]) == 0 and float(t.tree[0]) == 1000.0
    ti, di = (torch.empty(B, dtype=torch.int64, device="cuda") for _ in range(2))
    pr = torch.empty(B, dtype=torch.float64, device="cuda")
    st = torch.zeros(2, dtype=torch.int32, device="cuda")
    maxp = torch.ones(1, dtype=torch.float64, device="cuda")
    for it in range(g["batch_u"].shape[0]):
        t.sample_batch(B, 1, 1, ti, di, pr, st, uniforms=dev(g["batch_u"][it]), fills=dev(np.zeros(B, np.int64)))
        assert int(st[0]) == B
        np.testing.assert_allclose((pr * t.tree[0]).cpu().numpy(), g["batch_p"][it], rtol=1e-15)
        t.update_batch(dev(g["batch_idx"][it]), dev(g["batch_prio"][it]), maxp)
        assert np.array_equal(t.tree.cpu().numpy(), g["batch_trees"][it]), it
    assert float(maxp) == float(max(1.0, g["batch_prio"].max()))


def test_sumtree_million_leaves_vs_oracle(rl):
    """BASELINE capacity (1M leaves, not a power of two -> leaves on two depths): bit-exact against the oracle
    over rounds of 512 stratified draws + 512 float32 priority updates, then structural invariants."""
    from oracle.sum_tree import SumTree as O
    cap, B = 1_000_000, 512
    rng = np.random.RandomState(3)
    rp = rl.PrioritizedReplay(cap, B, history_length=4)
    frames = torch.zeros((cap, 16), dtype=torch.uint8, device="cuda")
    z = torch.zeros(cap, device="cuda")
    rp.load_synthetic(frames, z.int(), z.double(), torch.ones(cap, dtype=torch.int32, device="cuda"), pos=123457)
    ora = O(cap)
    ora.tree[:] = rp.tree.tree.cpu().numpy()
    ora.write = 123457
    bufs = rp._buffers(B, torch.uint8, "nchw")
    for it in range(6):
        u = rng.rand(B)
        rp._select_per(B, bufs, uniforms=u, fills=np.zeros(B, np.int64))
        seg = ora.total() / B
        got = [ora.get(seg * i + (seg * (i + 1) - seg * i) * u[i]) for i in range(B)]
        o_idx = np.asarray([x[0] for x in got])
        valid = np.asarray([(x[2] - 3 >= 0 and x[2] + 1 < 123457) or (x[2] - 3 >= 123457 and x[2] + 1 < cap) for x in got])
        assert valid.all()                                       # (no back-fill needed at this density)
        assert np.array_equal(bufs["tree_idx"].cpu().numpy(), o_idx)
        prio = ((np.abs(rng.randn(B)) + 0.01) ** 0.5).astype(np.float32)
        rp.update_priorities((bufs["tree_idx"], dev(prio)))
        for i, p in zip(o_idx, prio):
            ora.update(int(i), p)
        assert np.array_equal(rp.tree.tree.cpu().numpy(), ora.tree), it
    t = rp.tree.tree
    leaves = t[cap - 1:]
    assert abs(float(t[0]) - float(leaves.sum())) < 1e-6 * float(t[0])      # root == sum of leaves (fp64 drift only)


# ------------------------------------------------------------------------------------------ uniform replay
def _feed_all(rp, g, pre):
    fr, ac, rw, mk = g[pre + "frames"], g[pre + "actions"], g[pre + "rewards"], g[pre + "masks"]
    for i in range(len(fr)):
        rp.feed(dict(state=[fr[i]], action=[ac[i]], reward=[rw[i]], mask=[mk[i]]))


def test_uniform_replay_matches_reference(rl, golden):
    g = golden("replay_uniform")
    for c in range(int(g["n_cases"])):
        pre = "u%d_" % c
        M, hl, n, feeds, B = (int(x) for x in g[pre + "cfg"])
        rp = rl.UniformReplay(M, B, n, float(g[pre + "discount"]), hl)
        _feed_all(rp, g, pre)
        assert (rp.pos, rp.size()) == (g[pre + "pos"], g[pre + "size"])
        assert rp.ring_state[:2].tolist() == [rp.pos, rp.size()]
        assert np.array_equal([rp.valid_index(i) for i in range(rp.size())], g[pre + "valid"])
        assert np.array_equal(rp.compute_valid_indices(), g[pre + "compute_valid_indices"])
        for k, i in enumerate(g[pre + "valid_idx"]):
            tr = rp.construct_transition(int(i))
            assert np.array_equal(tr.state.cpu().numpy(), g[pre + "tr_state"][k])
            assert np.array_equal(tr.next_state.cpu().numpy(), g[pre + "tr_next"][k])
            assert int(tr.action) == g[pre + "tr_action"][k] and float(tr.mask) == g[pre + "tr_mask"][k]
            assert float(tr.reward) == np.float32(g[pre + "tr_reward"][k])
        assert rp.construct_transition(int(np.nonzero(~g[pre + "valid"])[0][0])) is None
        smp = rp.sample(candidates=g[pre + "cand"])
        assert np.array_equal(smp.state.cpu().numpy(), g[pre + "s_state"])
        assert np.array_equal(smp.next_state.cpu().numpy(), g[pre + "s_next"])
        assert np.array_equal(smp.action.cpu().numpy(), g[pre + "s_action"])
        assert np.array_equal(smp.reward.cpu().numpy(), g[pre + "s_reward"].astype(np.float32))
        assert np.array_equal(smp.mask.cpu().numpy(), g[pre + "s_mask"].astype(np.float32))


def test_uniform_feed_quirk_and_errors(rl, golden):
    g = golden("replay_uniform")
    rp = rl.UniformReplay(4, 1)
    one = lambda v: [np.asarray([x], np.int64) for x in v]
    rp.feed(dict(state=one([0, 1, 2, 3]), action=[0, 1, 2, 3], reward=[0, 1, 2, 3], mask=[1, 1, 1, 1]))
    rp.feed(dict(state=one([10, 11]), action=[10, 11], reward=[10, 11], mask=[1, 1]))
    assert np.array_equal(rp.frames.view(torch.int64).view(-1).cpu().numpy(), g["quirk_state"])
    assert (rp.pos, rp.size()) == (g["quirk_pos"], g["quirk_size"])
    with pytest.raises(RuntimeError, match="Undefined key"):
        rp.feed(dict(bogus=[1]))
    with pytest.raises(NotImplementedError):
        rp.update_priorities([])
    with pytest.raises(rl._lib.B2RLError):
        rl.UniformReplay(4, 1, device="cpu")
    empty = rl.UniformReplay(8, 2)
    with pytest.raises(ValueError):
        empty.sample()
    rp2 = rl.UniformReplay(8, 4, history_length=4)
    for i in range(3):                                           # too few items for any valid index
        rp2.feed(dict(state=[np.zeros(16, np.uint8)], action=[0], reward=[0.0], mask=[1]))
    with pytest.raises(RuntimeError, match="exhausted"):
        rp2.sample()


def test_uniform_philox_sampling_is_valid_and_uniform(rl):
    M, B, hl = 4096, 512, 4
    rp = rl.UniformReplay(M, B, 1, 0.99, hl, seed=7)
    fr = torch.arange(M, device="cuda", dtype=torch.int64).view(M, 1).expand(M, 2).contiguous().view(torch.uint8)
    z = torch.zeros(M, device="cuda")
    rp.item_shape, rp.item_dtype = (2,), np.dtype(np.int64)
    rp.load_synthetic(fr, z.int(), z.double(), torch.ones(M, dtype=torch.int32, device="cuda"), pos=1000)
    seen = []
    for _ in range(40):
        t = rp.sample()
        i = t.state[:, -1, 0].cpu().numpy()                      # the frame payload IS its ring index
        assert all(rp.valid_index(int(x)) for x in i)
        assert np.array_equal(t.state[:, :, 0].cpu().numpy(), i[:, None] + np.arange(-3, 1))
        assert np.array_equal(t.next_state[:, :, 0].cpu().numpy(), i[:, None] + np.arange(-2, 2))
        seen.append(i)
    seen = np.concatenate(seen)
    assert len(np.unique(seen)) > 0.9 * M * (1 - np.exp(-len(seen) / M)) and abs(seen.mean() - M / 2) < 0.05 * M
    assert int(rp.ring_state[4]) > 0                             # the device counter advanced: batches differ
    a, b = rp.sample().state.clone(), rp.sample().state
    assert not torch.equal(a, b)


# ------------------------------------------------------------------------------------------ prioritized replay
def test_prioritized_replay_matches_reference(rl, golden):
    g = golden("replay_per")
    for c in range(int(g["n_cases"])):
        pre = "p%d_" % c
        M, hl, n, feeds, B, rounds = (int(x) for x in g[pre + "cfg"])
        fr, ac, rw, mk = g[pre + "frames"], g[pre + "actions"], g[pre + "rewards"], g[pre + "masks"]
        rp = rl.PrioritizedReplay(M, B, n, float(g[pre + "discount"]), hl)
        _feed_all(rp, g, pre)
        for rd in range(rounds):
            assert rp.tree.total() == g[pre + "total"][rd]
            smp = rp.sample(uniforms=g[pre + "u"][rd], fills=g[pre + "fills"][rd])
            for k in ("state", "next_state", "action", "idx"):
                assert np.array_equal(getattr(smp, k).cpu().numpy(), g[pre + "s_" + k][rd]), (c, rd, k)
            assert np.array_equal(smp.reward.cpu().numpy(), g[pre + "s_reward"][rd].astype(np.float32))
            assert np.array_equal(smp.mask.cpu().numpy(), g[pre + "s_mask"][rd].astype(np.float32))
            assert np.array_equal(smp.sampling_prob.cpu().numpy(), g[pre + "s_sampling_prob"][rd].astype(np.float32))
            assert np.array_equal(rp._buffers(B, torch.uint8, "nchw")["prob64"].cpu().numpy(), g[pre + "s_sampling_prob"][rd])
            idx = np.asarray(g[pre + "s_idx"][rd], np.float32).astype(np.int64)      # tensor(idx).long() round trip
            rp.update_priorities(zip(idx, g[pre + "prio"][rd]))
            base = feeds + rd * 2
            for j in range(2):
                k2 = (base + j) % feeds
                rp.feed(dict(state=[fr[k2]], action=[ac[k2]], reward=[rw[k2]], mask=[mk[k2]]))
            assert np.array_equal(rp.tree.tree.cpu().numpy(), g[pre + "tree"][rd]), (c, rd)
            assert rp.max_priority == g[pre + "max_priority"][rd]


# ------------------------------------------------------------------------------------------ gather at full size
def test_gather_full_size_properties(rl):
    """BASELINE sizes: 1M x 84x84 uint8 ring (7.06 GB), batch 512.  Checks the TMA gather against an independent
    torch indexing expression, the fused normalize variants against the float64 LUT definition, and that
    state / next_state overlap by history-1 frames."""
    cap, B, hl = 1_000_000, 512, 4
    g = torch.Generator(device="cuda").manual_seed(0)
    frames = torch.empty((cap, 7056), dtype=torch.uint8, device="cuda")
    for s in range(0, cap, 100_000):
        frames[s:s + 100_000] = torch.randint(0, 256, (100_000, 7056), dtype=torch.uint8, device="cuda", generator=g)
    act = torch.randint(0, 4, (cap,), device="cuda", generator=g).int()
    rew = (torch.randint(0, 3, (cap,), device="cuda", generator=g) - 1).double()
    msk = (torch.rand(cap, device="cuda", generator=g) > 1e-3).int()
    rp = rl.UniformReplay(cap, B, 1, 0.99, hl, seed=1)
    rp.item_shape, rp.item_dtype = (84, 84), np.dtype(np.uint8)
    rp.load_synthetic(frames, act, rew, msk, pos=123457)
    t = rp.sample()
    idx = rp._buffers(B, torch.uint8, "nchw")["idx"]
    assert t.state.shape == (B, 4, 84, 84) and t.state.dtype == torch.uint8
    rows = idx[:, None] + torch.arange(-3, 1, device="cuda")[None]
    assert torch.equal(t.state.view(B, 4, 7056), frames[rows])
    assert torch.equal(t.next_state.view(B, 4, 7056), frames[rows + 1])
    assert torch.equal(t.state[:, 1:], t.next_state[:, :-1])
    assert torch.equal(t.action, act[idx].long()) and torch.equal(t.reward, rew[idx].float()) and torch.equal(t.mask, msk[idx].float())
    cand = idx.clone()
    lut64 = torch.from_numpy((np.arange(256, dtype=np.float64) * (1.0 / 255)).astype(np.float32)).cuda()
    f32 = rp.sample_normalized(out_dtype=torch.float32, candidates=cand)
    assert torch.equal(f32.state, lut64[t.state.long()]) and torch.equal(f32.next_state, lut64[t.next_state.long()])
    for dt in (torch.bfloat16, torch.float16):
        for cl in (False, True):
            x = rp.sample_normalized(out_dtype=dt, channels_last=cl, candidates=cand)
            assert x.state.shape == (B, 4, 84, 84)
            assert cl == x.state.is_contiguous(memory_format=torch.channels_last) or not cl
            assert torch.equal(x.state, lut64[t.state.long()].to(dt)) and torch.equal(x.next_state, lut64[t.next_state.long()].to(dt))
    # space-to-depth(4) layout with exact integer conversion: [B, 64, 21, 21], channel = f*16 + dy*4 + dx
    x = rp.sample_normalized(out_dtype=torch.bfloat16, scale=None, layout="s2d", candidates=cand)
    assert x.state.shape == (B, 64, 21, 21) and x.state.is_contiguous(memory_format=torch.channels_last)
    ref = t.state.view(B, 4, 21, 4, 21, 4).permute(0, 1, 3, 5, 2, 4).reshape(B, 64, 21, 21).to(torch.bfloat16)
    assert torch.equal(x.state, ref)
    refn = t.next_state.view(B, 4, 21, 4, 21, 4).permute(0, 1, 3, 5, 2, 4).reshape(B, 64, 21, 21).to(torch.bfloat16)
    assert torch.equal(x.next_state, refn)
    xf = rp.sample_normalized(out_dtype=torch.float32, scale=1.0 / 255, layout="s2d", candidates=cand)
    assert torch.equal(xf.state, lut64[t.state.long()].view(B, 4, 21, 4, 21, 4).permute(0, 1, 3, 5, 2, 4).reshape(B, 64, 21, 21))
    xi = rp.sample_normalized(out_dtype=torch.float16, scale=None, layout="nhwc", candidates=cand)
    assert torch.equal(xi.state, t.state.to(torch.float16))
    # n-step returns (n=3) against the float64 recurrence of replay.py:137-139
    rp3 = rl.UniformReplay(cap, B, 3, 0.9, hl, seed=2)
    rp3.item_shape, rp3.item_dtype = (84, 84), np.dtype(np.uint8)
    rp3.load_synthetic(frames, act, rew, msk, pos=123457)
    t3 = rp3.sample()
    i3 = rp3._buffers(B, torch.uint8, "nchw")["idx"]
    r, m = rew.cpu().numpy(), msk.cpu().numpy()
    exp_r, exp_m = [], []
    for i in i3.cpu().numpy():
        cr, cm = 0, 1
        for k in (2, 1, 0):
            cr = r[i + k] + m[i + k] * 0.9 * cr
            cm = cm and m[i + k]
        exp_r.append(np.float32(cr)), exp_m.append(np.float32(cm))
    assert np.array_equal(t3.reward.cpu().numpy(), np.asarray(exp_r)) and np.array_equal(t3.mask.cpu().numpy(), np.asarray(exp_m))
    assert torch.equal(t3.next_state.view(B, 4, 7056), frames[i3[:, None] + torch.arange(0, 4, device="cuda")[None]])


# ------------------------------------------------------------------------------------------ loss kernels
def test_loss_boundary_matches_reference(rl, golden):
    """Identical head outputs in -> the reference's loss tensors out.  DQN delta is bit-exact (operation order fully
    specified); C51 / QR within 2e-6 abs / 1e-5 rel (logf, summation order)."""
    g = golden("losses")
    a, r, m = dev(g["action"]), dev(g["reward"], torch.float32), dev(g["mask"], torch.float32)
    q, qt, qo = dev(g["dqn_q"]), dev(g["dqn_qn_t"]), dev(g["dqn_qn_o"])
    for double in (0, 1):
        for n in (1, 3):
            out = rl.ops.dqn_loss_fused(q, qt, qo if double else None, a, r, m, 0.99 ** n)
            assert np.array_equal(out["delta"].cpu().numpy(), g["dqn_d%d_n%d_delta" % (double, n)])
            np.testing.assert_allclose(out["loss"].cpu().numpy()[0], g["dqn_d%d_n%d_loss" % (double, n)], rtol=1e-6)
    lp, pt, po = dev(g["c51_logp"]), dev(g["c51_pn_t"]), dev(g["c51_pn_o"])
    for double in (0, 1):
        out = rl.ops.c51_loss_fused(lp, pt, po if double else None, a, r, m, 0.99, -10, 10)
        np.testing.assert_allclose(out["kl"].cpu().numpy(), g["c51_d%d_kl" % double], rtol=1e-5, atol=2e-6)
        np.testing.assert_allclose(out["loss"].cpu().numpy()[0], g["c51_d%d_loss" % double], rtol=1e-5)
    out = rl.ops.qr_loss_fused(dev(g["qr_quant"]), dev(g["qr_qn"]), a, r, m, 0.99)
    np.testing.assert_allclose(out["vec"].cpu().numpy(), g["qr_vec"], rtol=1e-5, atol=2e-6)
    np.testing.assert_allclose(out["loss"].cpu().numpy()[0], g["qr_loss"], rtol=1e-5)


def _oracle_grads(fn, leaf):
    leaf = leaf.clone().requires_grad_(True)
    out = fn(leaf)
    out.backward()
    return out.detach(), leaf.grad


@pytest.mark.parametrize("B,A", [(512, 4), (512, 18), (37, 6), (1, 3), (2048, 6)])
def test_dqn_loss_and_gradient_vs_oracle(rl, B, A):
    from oracle import losses as L
    gen = torch.Generator().manual_seed(B * 31 + A)
    q, qt, qo = (torch.randn(B, A, generator=gen) for _ in range(3))
    a = torch.randint(0, A, (B,), generator=gen)
    r = torch.randint(-1, 2, (B,), generator=gen).float()
    m = (torch.rand(B, generator=gen) > 0.1).float()
    prob = torch.rand(B, generator=gen).double().div(B * 0.7).float()
    for double in (False, True):
        for per in (False, True):
            def f(qq):
                d = L.dqn_delta(qq, qt, qo if double else None, a, r, m, 0.99)
                if per:
                    _, _, d = L.per_block(d, prob, 0.4, 0.01, 0.5)
                return L.dqn_reduce(d)
            loss, grad = _oracle_grads(f, q)
            kw = dict(is_prob=prob.cuda(), beta=0.4, eps=0.01, alpha=0.5) if per else {}
            out = rl.ops.dqn_loss_fused(q.cuda(), qt.cuda(), qo.cuda() if double else None, a.cuda(), r.cuda(), m.cuda(), 0.99, **kw)
            d_ref = L.dqn_delta(q, qt, qo if double else None, a, r, m, 0.99)
            assert np.array_equal(out["delta"].cpu().numpy(), d_ref.numpy())
            np.testing.assert_allclose(out["loss"].cpu().numpy()[0], loss.numpy(), rtol=1e-5)
            np.testing.assert_allclose(out["dq"].cpu().numpy(), grad.numpy(), rtol=1e-5, atol=1e-9)
            if per:
                prio = L.per_block(d_ref, prob, 0.4, 0.01, 0.5)[0]
                # torch-CPU's pow(x, 0.5) is not the correctly rounded sqrt: 1 ulp differences (1.2e-7 relative)
                np.testing.assert_allclose(out["priority"].cpu().numpy(), prio.numpy(), rtol=3e-7, atol=0)
    # autograd wrapper (compute_loss contract)
    qg = q.cuda().requires_grad_(True)
    d = rl.ops.dqn_delta(qg, qt.cuda(), None, a.cuda(), r.cuda(), m.cuda(), 0.99)
    d.pow(2).mul(0.5).mean().backward()
    _, grad = _oracle_grads(lambda qq: L.dqn_reduce(L.dqn_delta(qq, qt, None, a, r, m, 0.99)), q)
    np.testing.assert_allclose(qg.grad.cpu().numpy(), grad.numpy(), rtol=1e-5, atol=1e-9)


@pytest.mark.parametrize("B,A,N", [(512, 4, 51), (64, 6, 51), (5, 3, 11), (512, 18, 51)])
def test_c51_loss_and_gradient_vs_oracle(rl, B, A, N):
    from oracle import losses as L
    gen = torch.Generator().manual_seed(N + B)
    lg, lt, lo = (torch.randn(B, A, N, generator=gen) * 2 for _ in range(3))
    pt, po = torch.softmax(lt, -1), torch.softmax(lo, -1)
    a = torch.randint(0, A, (B,), generator=gen)
    r = torch.randint(-1, 2, (B,), generator=gen).float()
    m = (torch.rand(B, generator=gen) > 0.1).float()
    atoms = torch.from_numpy(np.linspace(-10, 10, N)).float()
    prob = torch.rand(B, generator=gen).div(B * 0.7)
    for double in (False, True):
        for per in (False, True):
            def f(x):
                kl = L.c51_kl(torch.log_softmax(x, -1), pt, po if double else None, a, r, m, atoms, -10, 10, 0.99)
                if per:
                    kl = L.per_block(kl, prob, 0.5, 0.01, 0.5)[2]
                return kl.mean()
            lp = torch.log_softmax(lg, -1)
            kl_ref = L.c51_kl(lp, pt, po if double else None, a, r, m, atoms, -10, 10, 0.99)
            lpl = lp.clone().requires_grad_(True)
            klg = L.c51_kl(lpl, pt, po if double else None, a, r, m, atoms, -10, 10, 0.99)
            (L.per_block(klg, prob, 0.5, 0.01, 0.5)[2] if per else klg).mean().backward()
            kw = dict(is_prob=prob.cuda(), beta=0.5, eps=0.01, alpha=0.5) if per else {}
            out = rl.ops.c51_loss_fused(lp.cuda(), pt.cuda(), po.cuda() if double else None, a.cuda(), r.cuda(), m.cuda(),
                                        0.99, -10, 10, **kw)
            np.testing.assert_allclose(out["kl"].cpu().numpy(), kl_ref.numpy(), rtol=1e-5, atol=2e-6)
            np.testing.assert_allclose(out["dlogp"].cpu().numpy(), lpl.grad.numpy(), rtol=1e-5, atol=1e-8)
            ref_loss = (L.per_block(kl_ref, prob, 0.5, 0.01, 0.5)[2] if per else kl_ref).mean()
            np.testing.assert_allclose(out["loss"].cpu().numpy()[0], ref_loss.numpy(), rtol=1e-5)
    lpg = torch.log_softmax(lg, -1).cuda().requires_grad_(True)
    rl.ops.c51_kl(lpg, pt.cuda(), None, a.cuda(), r.cuda(), m.cuda(), 0.99, -10, 10).mean().backward()
    lpl = torch.log_softmax(lg, -1).requires_grad_(True)
    L.c51_kl(lpl, pt, None, a, r, m, atoms, -10, 10, 0.99).mean().backward()
    np.testing.assert_allclose(lpg.grad.cpu().numpy(), lpl.grad.numpy(), rtol=1e-5, atol=1e-8)


@pytest.mark.parametrize("B,A,N", [(512, 4, 200), (32, 6, 200), (7, 3, 5), (64, 18, 32)])
def test_qr_loss_and_gradient_vs_oracle(rl, B, A, N):
    from oracle import losses as L
    gen = torch.Generator().manual_seed(N * 7 + B)
    qv, qn = torch.randn(B, A, N, generator=gen), torch.randn(B, A, N, generator=gen)
    a = torch.randint(0, A, (B,), generator=gen)
    r = torch.randint(-1, 2, (B,), generator=gen).float()
    m = (torch.rand(B, generator=gen) > 0.1).float()
    ql = qv.clone().requires_grad_(True)
    vec = L.qr_loss(ql, qn, a, r, m, 0.99)
    vec.mean().backward()
    out = rl.ops.qr_loss_fused(qv.cuda(), qn.cuda(), a.cuda(), r.cuda(), m.cuda(), 0.99)
    np.testing.assert_allclose(out["vec"].cpu().numpy(), vec.detach().numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(out["loss"].cpu().numpy()[0], vec.mean().item(), rtol=1e-5)
    np.testing.assert_allclose(out["dquant"].cpu().numpy(), ql.grad.numpy(), rtol=1e-4, atol=1e-8)
    # autograd wrapper with a non-uniform upstream gradient
    w = torch.rand(N, generator=gen)
    ql2 = qv.clone().requires_grad_(True)
    (L.qr_loss(ql2, qn, a, r, m, 0.99) * w).sum().backward()
    qg = qv.cuda().requires_grad_(True)
    (rl.ops.qr_vector(qg, qn.cuda(), a.cuda(), r.cuda(), m.cuda(), 0.99) * w.cuda()).sum().backward()
    np.testing.assert_allclose(qg.grad.cpu().numpy(), ql2.grad.numpy(), rtol=1e-4, atol=1e-8)


# ------------------------------------------------------------------------------------------ on-policy kernels
def test_gae_matches_reference(rl, golden):
    g = golden("onpolicy")
    for (T, N) in ((128, 8), (2048, 16)):
        k = "gae_%d_%d_" % (T, N)
        adv, ret = rl.ops.gae(dev(g[k + "reward"]), dev(g[k + "mask"]), dev(g[k + "v"]), 0.99, 0.95, exact=True)
        assert np.array_equal(adv.cpu().numpy(), g[k + "adv"]) and np.array_equal(ret.cpu().numpy(), g[k + "ret"])
        adv2, ret2 = rl.ops.gae(dev(g[k + "reward"]), dev(g[k + "mask"]), dev(g[k + "v"]), 0.99, 0.95, exact=False)
        scale = np.abs(g[k + "adv"]).max()
        np.testing.assert_allclose(adv2.cpu().numpy(), g[k + "adv"], rtol=1e-5, atol=1e-5 * scale)   # scan re-associates
        np.testing.assert_allclose(ret2.cpu().numpy(), g[k + "ret"], rtol=1e-5, atol=1e-5 * np.abs(g[k + "ret"]).max())
    for it in range(g["a2c_gae_reward"].shape[0]):
        adv, ret = rl.ops.gae(dev(g["a2c_gae_reward"][it]), dev(g["a2c_gae_mask"][it]), dev(g["a2c_gae_v"][it]), 0.99, 0.95)
        assert np.array_equal(adv.cpu().numpy(), g["a2c_gae_advantage"][it]) and np.array_equal(ret.cpu().numpy(), g["a2c_gae_ret"][it])
    # no-GAE branch (A2C_agent.py:46-47) and ragged shapes
    from oracle import losses as L
    gen = torch.Generator().manual_seed(5)
    for (T, N) in ((1, 1), (7, 3), (33, 130), (100, 5)):
        r, m, v = torch.randn(T, N, 1, generator=gen), (torch.rand(T, N, 1, generator=gen) > 0.1).float(), torch.randn(T + 1, N, 1, generator=gen)
        for use in (True, False):
            a_ref, r_ref = L.gae(r, m, v, 0.99, 0.95, use)
            a_dev, r_dev = rl.ops.gae(r.cuda(), m.cuda(), v.cuda(), 0.99, 0.95, use, exact=True)
            assert np.array_equal(a_dev.cpu().numpy(), a_ref.numpy()) and np.array_equal(r_dev.cpu().numpy(), r_ref.numpy())
            a_s, r_s = rl.ops.gae(r.cuda(), m.cuda(), v.cuda(), 0.99, 0.95, use, exact=False)
            np.testing.assert_allclose(a_s.cpu().numpy(), a_ref.numpy(), rtol=1e-4, atol=1e-4)


def test_ppo_a2c_losses_vs_oracle(rl):
    from oracle import losses as L
    gen = torch.Generator().manual_seed(2)
    for M in (64, 24, 1, 2000):
        lp, ent, v, old, adv, ret = (torch.randn(M, 1, generator=gen) * 0.3 for _ in range(6))
        lp1, ent1, v1 = (x.clone().requires_grad_(True) for x in (lp, ent, v))
        pl, vl, kl = L.ppo_losses(lp1, ent1, v1, old, adv, ret, 0.2, 0.01)
        pl.backward(), vl.backward()
        out = rl.ops.ppo_loss_fused(lp.cuda(), ent.cuda(), v.cuda(), old.cuda(), adv.cuda(), ret.cuda(), 0.2, 0.01)
        np.testing.assert_allclose(out["out"][:3].cpu().numpy(), [pl.item(), vl.item(), kl.item()], rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(out["dlogp"].cpu().numpy(), lp1.grad.numpy().ravel(), rtol=1e-5, atol=1e-9)
        np.testing.assert_allclose(out["dent"].cpu().numpy(), ent1.grad.numpy().ravel(), rtol=1e-5, atol=1e-9)
        np.testing.assert_allclose(out["dv"].cpu().numpy(), v1.grad.numpy().ravel(), rtol=1e-5, atol=1e-9)
        lp2, ent2, v2 = (x.clone().requires_grad_(True) for x in (lp, ent, v))
        obj = L.a2c_loss(lp2, v2, ret, adv, ent2, 0.01, 0.5)
        obj.backward()
        o2 = rl.ops.a2c_loss_fused(lp.cuda(), ent.cuda(), v.cuda(), adv.cuda(), ret.cuda(), 0.01, 0.5)
        np.testing.assert_allclose(o2["out"][0].item(), obj.item(), rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(o2["dlogp"].cpu().numpy(), lp2.grad.numpy().ravel(), rtol=1e-5, atol=1e-9)
        np.testing.assert_allclose(o2["dv"].cpu().numpy(), v2.grad.numpy().ravel(), rtol=1e-5, atol=1e-9)
    x = torch.randn(32768, 1, generator=gen) * 3 + 1
    ref = L.normalize_advantage(x)
    got = rl.ops.normalize_advantage_(x.cuda().clone())
    np.testing.assert_allclose(got.cpu().numpy(), ref.numpy(), rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------ optimizer kernels
@pytest.mark.parametrize("kind", ["rmsprop", "rmsprop_plain", "adam"])
def test_fused_clip_optimizer_vs_torch(rl, kind):
    gen = torch.Generator().manual_seed(4)
    shapes = [(32, 4, 8, 8), (32,), (64, 32, 4, 4), (64,), (512, 3136), (512,), (6, 512), (6,), (3,)]
    ps = [torch.randn(s, generator=gen) * 0.1 for s in shapes]
    ref = [p.clone().requires_grad_(True) for p in ps]
    mine = [torch.nn.Parameter(p.clone().cuda()) for p in ps]
    if kind == "adam":
        topt = torch.optim.Adam(ref, lr=2.5e-4, eps=0.01 / 32)
        mopt = rl.ops.FlatOptimizer.from_torch(torch.optim.Adam(mine, lr=2.5e-4, eps=0.01 / 32))
    else:
        c = kind == "rmsprop"
        topt = torch.optim.RMSprop(ref, lr=2.5e-4, alpha=0.95, eps=0.01, centered=c)
        mopt = rl.ops.FlatOptimizer.from_torch(torch.optim.RMSprop(mine, lr=2.5e-4, alpha=0.95, eps=0.01, centered=c))
    for it in range(5):
        gs = [torch.randn(s, generator=gen) * (3.0 if it % 2 else 0.01) for s in shapes]      # clipped / unclipped steps
        for p, g_ in zip(ref, gs):
            p.grad = g_.clone()
        norm = torch.nn.utils.clip_grad_norm_(ref, 5.0)
        topt.step()
        mopt.zero_grad()
        for p, g_ in zip(mine, gs):
            p.grad.add_(g_.cuda())
        mopt.step(max_norm=5.0)
        exact = float(torch.cat([g_.double().reshape(-1) for g_ in gs]).norm())
        assert abs(mopt.total_norm.item() - exact) <= 2e-6 * exact           # our fp32 tree sum vs the float64 norm
        np.testing.assert_allclose(mopt.total_norm.item(), norm.item(), rtol=1e-4)   # torch-CPU's fp32 running sum drifts
        for p, q_ in zip(ref, mine):
            np.testing.assert_allclose(q_.detach().cpu().numpy(), p.detach().numpy(), rtol=2e-5, atol=2e-7)


# ------------------------------------------------------------------------------------------ dense path (fused layers)
def test_fused_layers_and_space_to_depth_conv1(rl):
    """csrc/dense.cu epilogues + network/fused.py against plain torch: bias+ReLU forward, ReLU-mask + bias-grad backward,
    and the space-to-depth formulation of conv1 (8x8 stride 4 over 4 frames == 2x2 stride 1 over 64 channels)."""
    from deeprl_b200.network import fused
    gen = torch.Generator(device="cuda").manual_seed(0)
    for rows, C in ((204800, 32), (41472, 64), (512, 512), (100, 8), (7, 2048)):
        y = torch.randn(rows, C, device="cuda", generator=gen).to(torch.bfloat16)
        b = torch.randn(C, device="cuda", generator=gen)
        ref = torch.relu(y.float() + b).to(torch.bfloat16)
        got = fused.bias_act_(y.clone(), b, True)
        assert torch.equal(got, ref)
        gy = torch.randn(rows, C, device="cuda", generator=gen).to(torch.bfloat16)
        g, db = fused.act_bwd_bias_grad(gy, ref, True)
        gref = torch.where(ref > 0, gy, torch.zeros_like(gy))
        assert torch.equal(g, gref)
        torch.testing.assert_close(db, gref.float().sum(0), rtol=1e-4, atol=1e-3 * max(1.0, rows ** 0.5))
    # space-to-depth conv1 == direct conv1 (fp32, exact same products; summation order differs)
    w = torch.randn(32, 4, 8, 8, device="cuda", generator=gen) * 0.05
    x = torch.randint(0, 256, (16, 4, 84, 84), device="cuda", generator=gen).float()
    xs = x.view(16, 4, 21, 4, 21, 4).permute(0, 1, 3, 5, 2, 4).reshape(16, 64, 21, 21)
    ref = torch.nn.functional.conv2d(x, w, stride=4)
    got = torch.nn.functional.conv2d(xs, fused.space_to_depth_weight(w, 4), stride=1)
    torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-3)
    # whole NatureConvBody: fused bf16 path (s2d integer frames, 1/255 folded) vs plain fp32 path on normalized frames
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    try:
        torch.manual_seed(0)
        net = rl.VanillaNet(6, rl.NatureConvBody(in_channels=4))
        frames = torch.randint(0, 256, (32, 4, 84, 84), device="cuda", generator=gen)
        xs16 = frames.view(32, 4, 21, 4, 21, 4).permute(0, 1, 3, 5, 2, 4).reshape(32, 64, 21, 21).to(torch.bfloat16) \
            .contiguous(memory_format=torch.channels_last)
        with rl.frame_scale(1.0 / 255):
            q_fused = net(xs16)["q"]
        gq = torch.randn(32, 6, device="cuda", generator=gen)
        net.zero_grad()
        q_fused.backward(gq)
        g_fused = {k: p.grad.clone() for k, p in net.named_parameters()}
        rl.Config.COMPUTE_DTYPE = torch.float32
        net.zero_grad()
        q_ref = net(frames.float() / 255)["q"]
        q_ref.backward(gq)
        scale = q_ref.abs().max().item()
        assert (q_fused - q_ref).abs().max().item() < 0.03 * scale          # bf16 operands: ~1e-2 relative
        for k, p in net.named_parameters():
            rel = (g_fused[k] - p.grad).norm() / (p.grad.norm() + 1e-12)
            assert rel < 0.2, (k, float(rel))          # bf16 activations + gradients through 5 layers at batch 32
    finally:
        rl.Config.COMPUTE_DTYPE = torch.float32


def test_tcgen05_gemm_vs_torch(rl):
    """csrc/gemm.cu against torch.mm on the layer shapes of the path (fc4, heads, conv2/conv3 as implicit GEMMs) and on
    ragged shapes; K-major and MN-major operands, fused bias / ReLU, bf16 / fp32 / split-K outputs.
    bf16 products are exact in fp32, so the only difference is the accumulation order: rtol 2e-3 on bf16 outputs
    (1 ulp of bf16 is 4e-3), 1e-4 on fp32 outputs."""
    gen = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: (torch.randn(*s, device="cuda", generator=gen) * 0.5).to(torch.bfloat16)
    shapes = [(512, 512, 3136), (512, 4, 512), (512, 204, 512), (41472, 64, 512), (25088, 64, 576), (204800, 32, 256),
              (130, 40, 72), (1, 8, 64), (127, 129, 200)]
    for (M, N, K) in shapes:
        a, b = rnd(M, K), rnd(N, K)
        bias = torch.randn(N, device="cuda", generator=gen)
        ref = a.float() @ b.float().t()
        for bn in ((32, 64, 128) if N > 8 else (32,)):
            got = rl.ops.gemm_bf16(a, b, out_dtype=torch.float32, block_n=bn)
            torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-3 * K ** 0.5)
        got = rl.ops.gemm_bf16(a, b, bias=bias, relu=True)
        torch.testing.assert_close(got.float(), torch.relu(ref + bias), rtol=1e-2, atol=2e-2 * K ** 0.5 * 0.1)
        got = rl.ops.gemm_bf16(a, b, out_dtype=torch.float32, splits=4)
        torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-3 * K ** 0.5)
    # MN-major operands: dW[N_out, K_in] = g^T x with g [rows, N_out], x [rows, K_in] read as stored
    for (rows, n_out, k_in) in [(512, 512, 3136), (41472, 64, 512), (25088, 64, 576), (204800, 32 + 32, 256), (300, 64, 128),
                                (5000, 32, 64)]:
        g, x = rnd(rows, n_out), rnd(rows, k_in)
        ref = g.float().t() @ x.float()
        got = rl.ops.gemm_bf16(g, x, a_major="mn", b_major="mn", out_dtype=torch.float32, splits=1)
        torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-3 * rows ** 0.5)
        got = rl.ops.gemm_bf16(g, x, a_major="mn", b_major="mn", splits=16)
        torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-3 * rows ** 0.5)
    # mixed: dX[rows, K_in] = g [rows, N_out] (K-major) x W [N_out, K_in] (MN-major as the B operand)
    g, w = rnd(512, 512), rnd(512, 3136)
    got = rl.ops.gemm_bf16(g, w, a_major="k", b_major="mn", out_dtype=torch.float32)
    torch.testing.assert_close(got, g.float() @ w.float(), rtol=1e-4, atol=1e-3 * 512 ** 0.5)


@pytest.mark.parametrize("slab", [0, 2])
def test_conv_grid_gemm_vs_torch(rl, slab):
    rl._lib.set_conv_slab(slab)
    try:
        _conv_grid_gemm_vs_torch(rl)
    finally:
        rl._lib.set_conv_slab(2)


def _conv_grid_gemm_vs_torch(rl):
    """Shifted-row wgmma GEMMs of network/nature_tc.py against torch convolutions in fp32 on the same bf16 operands:
    each layer's forward (with the space-to-depth / compaction epilogues), dgrad and wgrad, then the whole body."""
    import torch.nn.functional as F
    from deeprl_b200.network import nature_tc as tc
    from deeprl_b200.network.fused import act_bwd_bias_grad
    gen = torch.Generator(device="cuda").manual_seed(1)
    B = 6
    bf = torch.bfloat16
    rnd = lambda *s, sc=1.0: (torch.randn(*s, device="cuda", generator=gen) * sc)
    w1, w2, w3, w4 = rnd(32, 4, 8, 8, sc=0.05), rnd(64, 32, 4, 4, sc=0.05), rnd(64, 64, 3, 3, sc=0.05), rnd(512, 3136, sc=0.02)
    b1, b2, b3, b4 = rnd(32, sc=0.1), rnd(64, sc=0.1), rnd(64, sc=0.1), rnd(512, sc=0.1)
    frames = torch.randint(0, 256, (B, 4, 84, 84), device="cuda", generator=gen)
    scale = 1.0 / 255
    packed = tc.pack_weights(w1, w2, w3, w4, scale)
    w1f, w2f, w2d, w3f, w3d, w4p = packed
    x0 = frames.view(B, 4, 21, 4, 21, 4).permute(0, 1, 3, 5, 2, 4).reshape(B, 64, 21, 21).to(bf).contiguous(memory_format=torch.channels_last)
    y4, (x0m, x1, y2, y3) = tc.forward_only(x0, packed, b1, b2, b3, b4)
    # fp32 reference on the SAME rounded operands, layer by layer
    deq = lambda w: w.float()
    w1r = tc.unpack_grads(deq(w1f), deq(w2f), deq(w3f), deq(w4p), 1.0, 4)       # bf16-rounded weights back in NCHW layouts
    r1 = torch.relu(F.conv2d(frames.float(), w1r[0], b1, stride=4))            # (scale already folded into w1f)
    x1_ref = r1.view(B, 32, 10, 2, 10, 2).permute(0, 2, 4, 3, 5, 1).reshape(B * 100, 128)
    torch.testing.assert_close(x1.float(), x1_ref, rtol=1e-2, atol=5e-2)
    x1n = x1.float().view(B, 10, 10, 2, 2, 32).permute(0, 5, 1, 3, 2, 4).reshape(B, 32, 20, 20)       # NCHW view of OUR x1
    r2 = torch.relu(F.conv2d(x1n, w1r[1], b2, stride=2))                      # [B,64,9,9]
    y2v = y2.float().view(B, 10, 10, 64)[:, :9, :9].permute(0, 3, 1, 2)
    torch.testing.assert_close(y2v, r2, rtol=1e-2, atol=2e-2)
    r3 = torch.relu(F.conv2d(y2v.contiguous(), w1r[2], b3))                   # [B,64,7,7]
    torch.testing.assert_close(y3.float().view(B, 7, 7, 64).permute(0, 3, 1, 2), r3, rtol=1e-2, atol=2e-2)
    r4 = torch.relu(y3.float().view(B, 3136) @ w4p.float().t() + b4)
    torch.testing.assert_close(y4.float(), r4, rtol=1e-2, atol=2e-2)
    # backward pieces against autograd of the fp32 reference on OUR activations
    gy3c = rnd(B, 3136, sc=0.1).to(bf)
    g3, db3 = act_bwd_bias_grad(gy3c.view(B * 49, 64), y3, True, row_map=1, G=10, V=7, out_rows=B * 100)
    g3n = (gy3c.float().view(B, 7, 7, 64) * (y3.float().view(B, 7, 7, 64) > 0)).permute(0, 3, 1, 2)
    assert torch.equal(g3.view(B, 10, 10, 64)[:, :7, :7].permute(0, 3, 1, 2).float(), g3n.to(bf).float())
    assert float(g3.view(B, 10, 10, 64)[:, 7:].abs().sum()) == 0 and float(g3.view(B, 10, 10, 64)[:, :, 7:].abs().sum()) == 0
    y2l = y2v.contiguous().requires_grad_(True)
    w3l = w1r[2].clone().requires_grad_(True)
    F.conv2d(y2l, w3l).backward(g3n.to(bf).float())
    gw3f = torch.zeros((64, 576), device="cuda")
    tc.conv_gemm(1, y2, g3, 64, 9, 3, 10, 1, gw3f, splits=16, block_n=64)
    torch.testing.assert_close(gw3f.view(64, 3, 3, 64).permute(0, 3, 1, 2), w3l.grad, rtol=1e-3, atol=1e-2)
    gy2 = torch.empty((B * 100, 64), dtype=bf, device="cuda")
    tc.conv_gemm(0, g3, w3d, 64, 9, 3, 10, -1, gy2, block_n=64)
    torch.testing.assert_close(gy2.float().view(B, 10, 10, 64)[:, :9, :9].permute(0, 3, 1, 2), y2l.grad, rtol=1e-2, atol=1e-2)
    assert float(gy2.view(B, 10, 10, 64)[:, 9].abs().sum()) == 0 and float(gy2.view(B, 10, 10, 64)[:, :, 9].abs().sum()) == 0
    g2, db2 = act_bwd_bias_grad(gy2, y2, True)
    g2n = g2.float().view(B, 10, 10, 64)[:, :9, :9].permute(0, 3, 1, 2).contiguous()
    x1l = x1n.clone().requires_grad_(True)
    w2l = w1r[1].clone().requires_grad_(True)
    F.conv2d(x1l, w2l, stride=2).backward(g2n)
    gw2f = torch.zeros((64, 512), device="cuda")
    tc.conv_gemm(1, x1, g2, 64, 4, 2, 10, 1, gw2f, splits=16, block_n=128)
    g_un = tc.unpack_grads(torch.zeros(32, 256, device="cuda"), gw2f, gw3f, torch.zeros(512, 3136, device="cuda"), 1.0, 4)
    torch.testing.assert_close(g_un[1], w2l.grad, rtol=1e-3, atol=1e-2)
    gy1 = torch.empty((B * 100, 128), dtype=bf, device="cuda")
    tc.conv_gemm(0, g2, w2d, 128, 4, 2, 10, -1, gy1, block_n=128)
    gy1n = gy1.float().view(B, 10, 10, 2, 2, 32).permute(0, 5, 1, 3, 2, 4).reshape(B, 32, 20, 20)
    torch.testing.assert_close(gy1n, x1l.grad, rtol=1e-2, atol=1e-2)
    g1, db1 = act_bwd_bias_grad(gy1, x1, True, row_map=2, G=21, V=20, out_rows=B * 441)
    g1n = (gy1n * (x1n > 0)).to(bf).float()
    assert torch.equal(g1.float().view(B, 21, 21, 32)[:, :20, :20].permute(0, 3, 1, 2), g1n)
    torch.testing.assert_close(db1, g1n.sum((0, 2, 3)), rtol=1e-3, atol=1e-2)
    w1l = w1r[0].clone().requires_grad_(True)
    F.conv2d(frames.float(), w1l, stride=4).backward(g1n)
    gw1f = torch.zeros((32, 256), device="cuda")
    tc.conv_gemm(1, x0m, g1, 32, 4, 2, 21, 1, gw1f, splits=32, block_n=64)
    g_un = tc.unpack_grads(gw1f, gw2f, gw3f, torch.zeros(512, 3136, device="cuda"), 1.0, 4)
    torch.testing.assert_close(g_un[0], w1l.grad, rtol=1e-3, atol=0.5)       # sums of 2400 products of magnitude ~100
    # whole body through autograd: wgmma backend vs library backend (both bf16) on a NatureConvBody
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    try:
        torch.manual_seed(0)
        net = rl.VanillaNet(6, rl.NatureConvBody(in_channels=4))
        xs = torch.randint(0, 256, (64, 4, 84, 84), device="cuda", generator=gen)
        xs16 = xs.view(64, 4, 21, 4, 21, 4).permute(0, 1, 3, 5, 2, 4).reshape(64, 64, 21, 21).to(bf).contiguous(memory_format=torch.channels_last)
        gq = torch.randn(64, 6, device="cuda", generator=gen)
        outs = {}
        for backend in ("tcgen05", "library"):
            rl.Config.DENSE_BACKEND = backend
            net.zero_grad()
            with rl.frame_scale(1.0 / 255):
                q = net(xs16)["q"]
            q.backward(gq)
            outs[backend] = (q.detach().clone(), {k: p.grad.clone() for k, p in net.named_parameters()})
        # the training step's path: gradients accumulated straight into the .grad arena by b2rl_nature_unpack_grads
        rl.Config.DENSE_BACKEND = "tcgen05"
        opt = rl.ops.FlatOptimizer.from_torch(torch.optim.RMSprop(net.parameters(), lr=1e-4))
        opt.zero_grad()
        net.body.auto_repack = False
        net.body.repack(1.0 / 255)
        with rl.frame_scale(1.0 / 255):
            net(xs16)["q"].backward(gq)
        net.body.auto_repack = True
        for k, p in net.named_parameters():
            torch.testing.assert_close(p.grad, outs["tcgen05"][1][k], rtol=1e-3, atol=1e-5 * float(outs["tcgen05"][1][k].abs().max() + 1))
        qa, qb = outs["tcgen05"][0], outs["library"][0]
        assert (qa - qb).abs().max() < 0.02 * qb.abs().max()
        for k in outs["library"][1]:
            ga, gb = outs["tcgen05"][1][k], outs["library"][1][k]
            assert (ga - gb).norm() / (gb.norm() + 1e-12) < 0.05, k
    finally:
        rl.Config.COMPUTE_DTYPE = torch.float32
        rl.Config.DENSE_BACKEND = "tcgen05"


def test_narrow_head_kernels_vs_torch(rl):
    """csrc/head.cu (VanillaNet / DuelingNet heads on bf16 features) against the torch expressions of network_heads.py."""
    from deeprl_b200.network import fused
    gen = torch.Generator(device="cuda").manual_seed(3)
    for (B, K, A) in ((512, 512, 4), (512, 512, 18), (37, 64, 6), (1, 512, 2)):
        phi = torch.randn(B, K, device="cuda", generator=gen).to(torch.bfloat16)
        fa, fv = torch.nn.Linear(K, A).cuda(), torch.nn.Linear(K, 1).cuda()
        gq = torch.randn(B, A, device="cuda", generator=gen)
        for dueling in (False, True):
            x = phi.float().requires_grad_(True)
            adv = fa(x)
            q_ref = (fv(x).expand_as(adv) + (adv - adv.mean(1, keepdim=True))) if dueling else adv
            for m in (fa, fv):
                m.zero_grad()
            q_ref.backward(gq)
            ref = [p.grad.clone() for p in (list(fa.parameters()) + (list(fv.parameters()) if dueling else []))]
            for m in (fa, fv):
                m.zero_grad()
            xp = phi.clone().requires_grad_(True)
            q = fused.narrow_head(xp, fa, fv if dueling else None)
            torch.testing.assert_close(q, q_ref.detach(), rtol=1e-5, atol=1e-5)
            q.backward(gq)
            got = [p.grad for p in (list(fa.parameters()) + (list(fv.parameters()) if dueling else []))]
            for a, b in zip(got, ref):
                torch.testing.assert_close(a.reshape(b.shape), b, rtol=1e-4, atol=1e-4)
            torch.testing.assert_close(xp.grad.float(), x.grad, rtol=1e-2, atol=1e-3)       # bf16 output


# ------------------------------------------------------------------------------------------ agents (product code path)
class _Batch:
    pass


def _mk_cfg(rl, name, g, pre):
    c = rl.Config()
    c.merge(dict(tag=None, n_step=1))
    c.task_fn = lambda: rl.Task("CartPole-v0", seed=3)
    c.eval_env = c.task_fn()
    c.history_length, c.batch_size, c.discount = 1, 16, 0.99
    body = lambda: rl.FCBody(c.state_dim, hidden_units=(32, 32))
    if name.startswith("dqn"):
        c.optimizer_fn = lambda p: torch.optim.RMSprop(p, lr=0.00025, alpha=0.95, eps=0.01, centered=True)
        c.network_fn = (lambda: rl.DuelingNet(c.action_dim, body())) if name == "dqn_per" else (lambda: rl.VanillaNet(c.action_dim, body()))
    elif name == "c51":
        c.optimizer_fn = lambda p: torch.optim.Adam(p, lr=0.00025, eps=0.01 / 32)
        c.categorical_v_min, c.categorical_v_max, c.categorical_n_atoms = -100, 100, 50
        c.network_fn = lambda: rl.CategoricalNet(c.action_dim, c.categorical_n_atoms, body())
    else:
        c.optimizer_fn = lambda p: torch.optim.Adam(p, lr=0.00005, eps=0.01 / 32)
        c.num_quantiles = 20
        c.network_fn = lambda: rl.QuantileNet(c.action_dim, c.num_quantiles, body())
    cls = rl.PrioritizedReplay if name == "dqn_per" else rl.UniformReplay
    rk = dict(memory_size=256, batch_size=16, n_step=1, discount=0.99, history_length=1)
    c.replay_fn = lambda: rl.ReplayWrapper(cls, rk, False)
    c.replay_eps, c.replay_alpha = 0.01, 0.5
    c.replay_beta = rl.LinearSchedule(0.4, 1.0, 200)
    c.random_action_prob = rl.LinearSchedule(1.0, 0.1, 100)
    c.target_network_update_freq, c.exploration_steps = 5, 40
    c.sgd_update_frequency, c.gradient_clip, c.async_actor = 4, 5, False
    c.double_q = name == "dqn_per"
    return c


@pytest.mark.parametrize("name", ["dqn_per", "dqn_uni", "c51", "qr"])
def test_agent_update_trajectory_matches_reference(rl, golden, name):
    """The product agents' fused update (networks on the GPU in fp32, fused loss kernel, fused clip+optimizer kernels),
    fed the batches the REFERENCE sampled, reproduces the reference's per-sample loss tensor and parameter trajectory.
    Tolerance: delta 1e-5 rel / 5e-6 abs, parameters 1e-5 abs after ~25 optimizer steps (GPU vs CPU fp32 matmul order)."""
    g = golden("agent_steps")
    pre = name + "_"
    cls = dict(dqn_per=rl.DQNAgent, dqn_uni=rl.DQNAgent, c51=rl.CategoricalDQNAgent, qr=rl.QuantileRegressionDQNAgent)[name]
    ag = cls(_mk_cfg(rl, name, g, pre))
    keys = [str(k) for k in g[pre + "keys"]]
    sd = {k: dev(g[pre + "init." + k]) for k in keys}
    ag.network.load_state_dict(sd)
    ag.target_network.load_state_dict(sd)
    names = [n for n, _ in ag.network.named_parameters()]
    assert names == keys
    fields = ["state", "action", "reward", "next_state", "mask"] + (["sampling_prob", "idx"] if name == "dqn_per" else [])
    TCls = rl.PrioritizedTransition if name == "dqn_per" else rl.Transition
    nb = g[pre + "delta"].shape[0]
    for i in range(nb):
        vals = []
        for f in fields:
            x = g[pre + "b_" + f][i]
            dt = torch.int64 if f in ("action", "idx") else torch.float32
            vals.append(dev(x, dt))
        tr = TCls(*vals)
        with torch.no_grad():
            d = ag.compute_loss(tr)
        np.testing.assert_allclose(d.cpu().numpy(), g[pre + "delta"][i], rtol=1e-5, atol=5e-6)
        if name == "dqn_per":
            ag.replay.update_priorities = lambda info: None                # the recorded batches carry foreign tree indices
        ag._fused_update(tr)
        flat = np.concatenate([p.detach().cpu().numpy().ravel() for p in ag.network.parameters()])
        np.testing.assert_allclose(flat, g[pre + "params"][i], rtol=0, atol=1e-5)
        tflat = np.concatenate([p.detach().cpu().numpy().ravel() for p in ag.target_network.parameters()])
        if not np.allclose(tflat, g[pre + "target"][i], atol=1e-5):
            ag.target_network.load_state_dict(ag.network.state_dict())
            tflat = np.concatenate([p.detach().cpu().numpy().ravel() for p in ag.target_network.parameters()])
            np.testing.assert_allclose(tflat, g[pre + "target"][i], rtol=0, atol=1e-5)
    ag.close()


def test_dqn_agent_runs_end_to_end(rl):
    """DQNAgent.step() on the synthetic Atari-shaped task with PER + double + dueling, sync and async replay."""
    for async_replay in (False, True):
        c = rl.Config()
        c.merge(dict(tag=None, n_step=1))
        c.task_fn = lambda: rl.Task("SyntheticAtari-v0", seed=1)
        c.eval_env = c.task_fn()
        c.history_length, c.batch_size, c.discount = 4, 32, 0.99
        c.optimizer_fn = lambda p: torch.optim.RMSprop(p, lr=0.00025, alpha=0.95, eps=0.01, centered=True)
        c.network_fn = lambda: rl.DuelingNet(c.action_dim, rl.NatureConvBody(in_channels=4))
        rk = dict(memory_size=2000, batch_size=32, n_step=1, discount=0.99, history_length=4)
        c.replay_fn = lambda: rl.ReplayWrapper(rl.PrioritizedReplay, rk, async_replay)
        c.replay_eps, c.replay_alpha, c.replay_beta = 0.01, 0.5, rl.LinearSchedule(0.4, 1.0, 1000)
        c.random_action_prob = rl.LinearSchedule(1.0, 0.1, 100)
        c.state_normalizer, c.reward_normalizer = rl.ImageNormalizer(), rl.SignNormalizer()
        c.target_network_update_freq, c.exploration_steps = 10, 64
        c.sgd_update_frequency, c.gradient_clip, c.async_actor, c.double_q = 4, 5, False, True
        ag = rl.DQNAgent(c)
        p0 = [p.detach().clone() for p in ag.network.parameters()]
        for _ in range(40):
            ag.step()
        torch.cuda.synchronize()
        assert ag.total_steps == 160 and ag.last_loss is not None and torch.isfinite(ag.last_loss).all()
        assert any(not torch.equal(a, b) for a, b in zip(p0, ag.network.parameters()))
        assert abs(ag.replay.replay.tree.total() - float(ag.replay.replay.tree.tree[ag.replay.replay.memory_size - 1:].sum())) < 1e-6
        ag.close()


def test_ppo_agent_minibatch_loop_matches_reference(rl, golden):
    """PPOAgent (product) on the reference's recorded rollouts and minibatch permutations: same parameters after each
    PPO iteration (3 epochs x ragged minibatches, KL-gated actor step), atol 1e-5."""
    g = golden("onpolicy")
    pre = "ppo_small_"
    T, N, mb, epochs, its = (int(x) for x in g[pre + "cfg"])
    c = rl.Config()
    c.merge(dict(tag=None))
    c.num_workers = N
    c.task_fn = lambda: rl.Task("SyntheticCheetah-v0", num_envs=N, seed=6)
    c.eval_env = rl.Task("SyntheticCheetah-v0", seed=6)
    c.network_fn = lambda: rl.GaussianActorCriticNet(
        c.state_dim, c.action_dim, actor_body=rl.FCBody(c.state_dim, gate=torch.tanh),
        critic_body=rl.FCBody(c.state_dim, gate=torch.tanh))
    c.actor_opt_fn = lambda p: torch.optim.Adam(p, 3e-4)
    c.critic_opt_fn = lambda p: torch.optim.Adam(p, 1e-3)
    c.discount, c.use_gae, c.gae_tau, c.gradient_clip = 0.99, True, 0.95, 0.5
    c.rollout_length, c.optimization_epochs, c.mini_batch_size = T, epochs, mb
    c.ppo_ratio_clip, c.target_kl = 0.2, 0.01
    c.state_normalizer = rl.MeanStdNormalizer()
    ag = rl.PPOAgent(c)
    keys = [str(k) for k in g[pre + "keys"]]
    ag.network.load_state_dict({k: dev(g[pre + "init." + k]) for k in keys})
    names = [str(k) for k in g[pre + "param_names"]]
    assert [n for n, _ in ag.network.named_parameters()] == names
    from collections import namedtuple
    Entry = namedtuple("Entry", ["state", "action", "log_pi_a", "ret", "advantage"])
    for it in range(its):
        adv, ret = rl.ops.gae(dev(g[pre + "reward"][it]), dev(g[pre + "mask"][it]), dev(g[pre + "v"][it]), 0.99, 0.95)
        assert np.array_equal(adv.cpu().numpy(), g[pre + "advantage"][it])
        f = lambda k: dev(g[pre + k][it]).reshape(T * N, -1).contiguous()
        entries = Entry(f("state"), f("action"), f("log_pi_a"), ret.reshape(-1, 1).contiguous(), adv.reshape(-1, 1).contiguous())
        ag._normalize(entries)
        for perm in g[pre + "perms"][it]:
            full = len(perm) // mb * mb
            for row in perm[:full].reshape(-1, mb):
                ag._minibatch(entries, row)
            if len(perm) % mb:
                ag._minibatch(entries, perm[full:])
        flat = np.concatenate([p.detach().cpu().numpy().ravel() for p in ag.network.parameters()])
        np.testing.assert_allclose(flat, g[pre + "params"][it], rtol=0, atol=1e-5)
    ag.step()                                                         # and one real iteration end to end
    torch.cuda.synchronize()
    ag.close()


def test_a2c_agent_runs_on_gpu(rl):
    c = rl.Config()
    c.merge(dict(tag=None))
    c.num_workers = 8
    c.task_fn = lambda: rl.Task("CartPole-v0", num_envs=8, seed=4)
    c.eval_env = rl.Task("CartPole-v0", seed=4)
    c.optimizer_fn = lambda p: torch.optim.RMSprop(p, 0.001)
    c.network_fn = lambda: rl.CategoricalActorCriticNet(c.state_dim, c.action_dim, rl.FCBody(c.state_dim, gate=torch.tanh))
    c.discount, c.use_gae, c.gae_tau, c.entropy_weight, c.rollout_length, c.gradient_clip = 0.99, True, 0.95, 0.01, 5, 0.5
    ag = rl.A2CAgent(c)
    for _ in range(10):
        ag.step()
    assert ag.total_steps == 400 and torch.isfinite(ag.last_loss)
    ag.close()
