"""csrc/tail.cu (gradient reduce + fused clip / optimizer / operand pack) and csrc/head.cu dqn_head_fused_kernel against the
separate kernels they replace (which are themselves pinned against torch / the oracle in test_gpu_parity.py), through the
C ABI.  Reference semantics: DQN_agent.py:78-99,120-134 (loss, PER block, clip_grad_norm_, optimizer.step)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


@pytest.fixture(scope="module")
def rl():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import deeprl_b200 as rl
    rl.select_device(0)
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    return rl


def _net(rl, head, A, seed):
    torch.manual_seed(seed)
    body = rl.NatureConvBody(in_channels=4)
    return rl.DuelingNet(A, body) if head == "dueling" else rl.VanillaNet(A, body)


def _opt(rl, net, kind):
    if kind == "adam":
        t = torch.optim.Adam(net.parameters(), lr=2.5e-4, eps=0.01 / 32)
    else:
        t = torch.optim.RMSprop(net.parameters(), lr=2.5e-4, alpha=0.95, eps=0.01, centered=(kind == "rmsprop"))
    return rl.ops.FlatOptimizer.from_torch(t)


@pytest.mark.parametrize("kind", ["rmsprop", "rmsprop_plain", "adam"])
@pytest.mark.parametrize("head", ["vanilla", "dueling"])
def test_tail_matches_unpack_clip_optimizer_pack(rl, kind, head):
    from deeprl_b200 import _lib
    from deeprl_b200.network import nature_tc
    from deeprl_b200.network.tail import NatureTail
    dev = torch.device("cuda", 0)
    scale = 1.0 / 255
    na, nb = _net(rl, head, 6, 0), _net(rl, head, 6, 0)
    oa, ob = _opt(rl, na, kind), _opt(rl, nb, kind)
    assert torch.equal(oa.flat, ob.flat)
    tail = NatureTail(oa, na.body, scale)
    tail.max_norm = 5.0
    g = torch.Generator(device=dev).manual_seed(1)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    p1, p2, p3 = 134, 134, 147
    gw1p, gw2p, gw3p = rnd(148, 32, 256) * 0.1, rnd(148, 64, 512) * 0.1, rnd(148, 64, 576) * 0.1
    gw4p = rnd(512, 3136) * 0.05
    db = [rnd(32), rnd(64), rnd(64), rnd(512)]
    for step in range(3):
        # head gradients: both arenas get the same values where the body does not live
        hg = rnd(oa.n) * 0.3
        for net, o in ((na, oa), (nb, ob)):
            o.grad.zero_()
            for name, p in net.named_parameters():
                if not name.startswith("body."):
                    off = (p.data_ptr() - o.flat.data_ptr()) // 4
                    o.grad[off:off + p.numel()] = hg[off:off + p.numel()]
        for d, t in zip(db, (tail.db1, tail.db2, tail.db3, tail.db4)):
            t.copy_(d)
        # ---- reference: unpack (accumulates into the zeroed arena) + clip / optimizer + pack
        b = nb.body
        _lib.call("b2rl_nature_unpack_grads", _lib.ptr(gw1p), _lib.ptr(gw2p), _lib.ptr(gw3p), _lib.ptr(gw4p), _lib.ptr(db[0]),
                  _lib.ptr(db[1]), _lib.ptr(db[2]), _lib.ptr(db[3]), 4, 512, scale, _lib.ptr(b.conv1.weight.grad),
                  _lib.ptr(b.conv2.weight.grad), _lib.ptr(b.conv3.weight.grad), _lib.ptr(b.fc4.weight.grad),
                  _lib.ptr(b.conv1.bias.grad), _lib.ptr(b.conv2.bias.grad), _lib.ptr(b.conv3.bias.grad), _lib.ptr(b.fc4.bias.grad),
                  p1, p2, p3, _lib.stream())
        # ---- kernel A
        tail.reduce(gw1p, p1, gw2p, p2, gw3p, p3, gw4p)
        torch.cuda.synchronize()
        ga, gb = oa.grad.cpu().numpy(), ob.grad.cpu().numpy()
        np.testing.assert_allclose(ga, gb, rtol=2e-5, atol=1e-6)
        assert float(tail.db.abs().max()) == 0.0, "bias-gradient accumulators must be re-zeroed"
        np.testing.assert_allclose(float(tail.unit_sumsq.double().sum()), float((ob.grad.double() ** 2).sum()), rtol=1e-5)
        # ---- kernel B vs sumsq + optimizer kernels
        ob.step(max_norm=5.0)
        tail.step(max_norm=5.0)
        torch.cuda.synchronize()
        np.testing.assert_allclose(float(oa.scratch[0]), float(ob.scratch[0]), rtol=1e-5)           # total norm
        for x, y in ((oa.flat, ob.flat), (oa.s1, ob.s1), (oa.s2, ob.s2)):
            np.testing.assert_allclose(x.cpu().numpy(), y.cpu().numpy(), rtol=1e-5, atol=1e-7)
        assert float(oa.grad.abs().max()) == 0.0, "the fused optimizer re-zeroes the gradient arena"
        if kind == "adam":
            assert int(oa.step_dev) == int(ob.step_dev) == step + 1
        # the packed bf16 operands are exactly pack(updated fp32 parameters)
        a = na.body
        want = nature_tc.pack_weights(a.conv1.weight.detach(), a.conv2.weight.detach(), a.conv3.weight.detach(),
                                      a.fc4.weight.detach(), scale)
        for got, w in zip(tail.packed().tensors(), want):
            assert torch.equal(got, w)
        gw4p = gw4p * 0.5 + rnd(512, 3136) * 0.02          # vary the gradients between steps


@pytest.mark.parametrize("head,A", [("vanilla", 4), ("dueling", 6), ("vanilla", 18), ("dueling", 18)])
@pytest.mark.parametrize("per", [False, True])
@pytest.mark.parametrize("double_q", [False, True])
@pytest.mark.parametrize("B", [512, 37])
@pytest.mark.parametrize("two", [True, False])
def test_dqn_head_fused_matches_separate_kernels(rl, head, A, per, double_q, B, two):
    from deeprl_b200 import _lib, ops
    dev = torch.device("cuda", 0)
    K = 512
    g = torch.Generator(device=dev).manual_seed(B + A)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    net, net2, tgt = _net(rl, head, A, 3), _net(rl, head, A, 3), _net(rl, head, A, 4)
    phi = torch.relu(rnd(B, K)).to(torch.bfloat16)
    phi_t = torch.relu(rnd(B, K)).to(torch.bfloat16)
    phi_o = torch.relu(rnd(B, K)).to(torch.bfloat16) if double_q else None
    action = torch.randint(0, A, (B,), device=dev, generator=g)
    reward = torch.randint(-1, 2, (B,), device=dev, generator=g).float()
    mask = (torch.rand(B, device=dev, generator=g) > 0.1).float()
    prob = (torch.rand(B, device=dev, generator=g) * 1e-3 + 1e-6) if per else None
    pa = dict(is_prob=prob, beta=0.4, eps=0.01, alpha=0.5) if per else {}
    heads = lambda n: (n.fc_advantage, n.fc_value) if head == "dueling" else (n.fc_head, None)
    for n in (net, net2):
        for p in n.parameters():
            p.grad = torch.zeros_like(p)
    # ---- separate kernels: head_fwd x 2-3, dqn_loss, head_bwd_relu
    def q_of(n, x):
        fa, fv = heads(n)
        q = torch.empty(B, A, device=dev)
        _lib.call("b2rl_head_fwd", _lib.ptr(x), _lib.ptr(fa.weight.detach()), _lib.ptr(fa.bias.detach()),
                  _lib.ptr(None if fv is None else fv.weight.detach()), _lib.ptr(None if fv is None else fv.bias.detach()),
                  B, K, A, _lib.ptr(q), _lib.stream())
        return q
    q, qt = q_of(net2, phi), q_of(tgt, phi_t)
    qo = q_of(net2, phi_o) if double_q else None
    ref = ops.dqn_loss_fused(q, qt, qo, action, reward, mask, 0.99, **pa)
    fa, fv = heads(net2)
    gphi_ref, colsum_ref = torch.empty_like(phi), torch.zeros(K, device=dev)
    _lib.call("b2rl_head_bwd_relu", _lib.ptr(ref["dq"]), _lib.ptr(phi), _lib.ptr(fa.weight.detach()),
              _lib.ptr(None if fv is None else fv.weight.detach()), B, K, A, _lib.ptr(gphi_ref), _lib.ptr(fa.weight.grad),
              _lib.ptr(fa.bias.grad), _lib.ptr(None if fv is None else fv.weight.grad),
              _lib.ptr(None if fv is None else fv.bias.grad), _lib.ptr(colsum_ref), _lib.stream())
    # ---- one launch
    colsum = torch.zeros(K, device=dev)
    r = ops.dqn_head_fused(phi, phi_t, phi_o, heads(net), heads(tgt), action, reward, mask, 0.99, colsum, want_q=True, two=two, **pa)
    torch.cuda.synchronize()
    assert torch.equal(r["q"], q), "same dot-product order as head_fwd: bit-identical q"
    assert torch.equal(r["delta"], ref["delta"])
    if per:
        assert torch.equal(r["priority"], ref["priority"])
    np.testing.assert_allclose(float(r["loss"]), float(ref["loss"]), rtol=1e-5)
    assert torch.equal(r["gphi"], gphi_ref), "masked feature gradient"
    np.testing.assert_allclose(colsum.cpu().numpy(), colsum_ref.cpu().numpy(), rtol=1e-4, atol=1e-6)
    for pa_, pb_ in zip(net.parameters(), net2.parameters()):
        np.testing.assert_allclose(pa_.grad.cpu().numpy(), pb_.grad.cpu().numpy(), rtol=1e-4, atol=1e-6)
    # a second launch re-uses the self-resetting loss counter
    r2 = ops.dqn_head_fused(phi, phi_t, phi_o, heads(net), heads(tgt), action, reward, mask, 0.99, colsum, two=two, **pa)
    torch.cuda.synchronize()
    assert float(r2["loss"]) == float(r["loss"])


@pytest.mark.parametrize("M,N,K,splits,block_n", [(512, 512, 3136, 4, 64), (512, 512, 3136, 2, 32), (37, 200, 3136, 4, 64),
                                                  (256, 512, 512, 1, 128), (512, 512, 3136, 4, 128)])
def test_splitk_fixup_gemm_vs_torch(rl, M, N, K, splits, block_n):
    """b2rl_gemm_splitk_bf16 (one launch: split-K partials + last-arriver fix-up with bias / ReLU) against fp32 torch on the
    same bf16 operands, twice (the tile counters re-arm themselves) and bit-identical between runs (fixed summation order)."""
    from deeprl_b200 import ops
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(M + N + splits)
    a = (torch.randn(M, K, device=dev, generator=g) * 0.5).to(torch.bfloat16)
    b = (torch.randn(N, K, device=dev, generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(N, device=dev, generator=g)
    want = torch.relu(a.float() @ b.float().t() + bias)
    got = ops.gemm_splitk_bf16(a, b, bias=bias, relu=True, splits=splits, block_n=block_n)
    got2 = ops.gemm_splitk_bf16(a, b, bias=bias, relu=True, splits=splits, block_n=block_n)
    torch.cuda.synchronize()
    assert torch.equal(got, got2)
    np.testing.assert_allclose(got.float().cpu().numpy(), want.cpu().numpy(), rtol=1e-2, atol=2e-2)
    # and without bias / activation
    got3 = ops.gemm_splitk_bf16(a, b, splits=splits, block_n=block_n)
    np.testing.assert_allclose(got3.float().cpu().numpy(), (a.float() @ b.float().t()).cpu().numpy(), rtol=1e-2, atol=2e-2)


@pytest.mark.parametrize("kind,A,N", [("c51", 4, 51), ("qr", 4, 200), ("c51", 6, 51), ("qr", 18, 32)])
def test_dist_head_vs_torch(rl, kind, A, N):
    """Distributional head on the wgmma GEMM + csrc/disthead.cu (network/fused.py _DistHead) against fp32 torch on the same bf16
    operands: prob / log_prob (C51) or quantiles (QR-DQN), and the gradients w.r.t. the features, weight and bias."""
    from deeprl_b200.network import fused
    dev = torch.device("cuda", 0)
    B, K = 512, 512
    g = torch.Generator(device=dev).manual_seed(A * N)
    fc = torch.nn.Linear(K, A * N).to(dev)
    fc._w16 = fc.weight.detach().to(torch.bfloat16)
    phi = torch.relu(torch.randn(B, K, device=dev, generator=g)).to(torch.bfloat16).requires_grad_(True)
    softmax = kind == "c51"
    out, prob = fused.dist_head(phi, fc, A, N, softmax)
    # reference: fp32 on the bf16 operands
    phi_r = phi.detach().float().requires_grad_(True)
    w_r = fc._w16.float().requires_grad_(True)
    b_r = fc.bias.detach().clone().requires_grad_(True)
    logits = (phi_r @ w_r.t() + b_r).view(B, A, N)
    ref = torch.log_softmax(logits, -1) if softmax else logits
    np.testing.assert_allclose(out.detach().cpu().numpy(), ref.detach().cpu().numpy(), rtol=2e-3, atol=2e-3)
    if softmax:
        np.testing.assert_allclose(prob.cpu().numpy(), torch.softmax(logits, -1).detach().cpu().numpy(), rtol=2e-3, atol=1e-5)
    grad = torch.randn(B, A, N, device=dev, generator=g) / B
    out.backward(grad)
    ref.backward(grad)
    torch.cuda.synchronize()
    sc = lambda t: float(t.abs().max()) + 1e-12
    assert float((phi.grad.float() - phi_r.grad).abs().max()) <= 2e-2 * sc(phi_r.grad)
    assert float((fc.weight.grad - w_r.grad).abs().max()) <= 2e-2 * sc(w_r.grad)
    assert float((fc.bias.grad - b_r.grad).abs().max()) <= 2e-2 * sc(b_r.grad)
