"""K1 -- conv1 straight from the uint8 replay ring (csrc/gemm.cu fill_slab_u8, b2rl_conv1_u8_fwd / _wgrad_partials) against
the materialising path it replaces (gather -> bf16 space-to-depth matrix -> TMA slab), which is itself pinned against the
reference's frame-stack gather (replay.py:124-134) and torch's conv2d in test_gpu_parity.py.  The operands of every MMA are
the same bits, so the results must be BIT-IDENTICAL."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import bench
    import deeprl_b200 as rl
    rl.select_device(0)
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    bench.CAP = 20_000
    return bench, rl


@pytest.mark.parametrize("B", [512, 37, 1])
@pytest.mark.parametrize("n_step", [1, 3])
def test_conv1_from_ring_is_bit_identical(env, B, n_step):
    bench, rl = env
    from deeprl_b200 import _lib
    from deeprl_b200.network import nature_tc
    dev = torch.device("cuda", 0)
    rp = bench.synthetic_ring(rl, rl.UniformReplay, dev, seed=3)
    rp.n_step = n_step
    cand = torch.randint(8, bench.CAP - 8, (2 * B + 256,), device=dev)
    mat = rp.sample_normalized(batch_size=B, out_dtype=torch.bfloat16, scale=None, layout="s2d", candidates=cand, tag=1)
    ring = rp.sample_normalized(batch_size=B, out_dtype=torch.bfloat16, scale=None, layout="ring", candidates=cand, tag=2)
    for a, b in ((mat.action, ring.action), (mat.reward, ring.reward), (mat.mask, ring.mask)):
        assert torch.equal(a, b)
    torch.manual_seed(0)
    body = rl.NatureConvBody(in_channels=4).to(dev)
    pk = nature_tc.repack(body, 1.0 / 255)
    b1 = body.conv1.bias.detach()
    for which, (m, r) in enumerate(((mat.state, ring.state), (mat.next_state, ring.next_state))):
        assert isinstance(r, nature_tc.RingFrames) and r.first == which * n_step - 3
        assert torch.equal(r.materialize(), m), "RingFrames.materialize() == the gather's space-to-depth output"
        x0m = m.permute(0, 2, 3, 1).reshape(B * 441, 64)
        want = torch.zeros((B * 100, 128), dtype=torch.bfloat16, device=dev)
        got = torch.zeros_like(want)
        nature_tc.conv_gemm(0, x0m, pk.w1f, 32, 4, 2, 21, 1, want, bias=b1, relu=True, out_map=1, G=21, V=20, block_n=32)
        _lib.call("b2rl_conv1_u8_fwd", *r.args(), _lib.ptr(pk.w1f), 32, _lib.ptr(got), got.stride(0), _lib.ptr(b1), 1, 1, 20,
                  _lib.stream())
        torch.cuda.synchronize()
        assert torch.equal(got, want), "conv1 forward from the ring"
        # weight gradient: same split-K partition, same operands -> identical partials
        g1 = (torch.randn(B * 441, 32, device=dev) * 0.1).to(torch.bfloat16)
        pw, nw = nature_tc.wgrad_partials(x0m, g1, 32, 4, 2, 21)
        pg, ng = nature_tc.wgrad_partials_ring(r, g1, 32)
        torch.cuda.synchronize()
        assert nw == ng
        assert torch.equal(pg[:ng], pw[:nw]), "conv1 weight-gradient partials from the ring"


def test_body_forward_backward_from_ring(env):
    """NatureConvBody on RingFrames == on the materialised batch: features and every parameter gradient bit-identical."""
    bench, rl = env
    from deeprl_b200.network.fused import frame_scale
    dev = torch.device("cuda", 0)
    rp = bench.synthetic_ring(rl, rl.UniformReplay, dev, seed=5)
    B = 64
    cand = torch.randint(8, bench.CAP - 8, (2 * B + 256,), device=dev)
    mat = rp.sample_normalized(batch_size=B, out_dtype=torch.bfloat16, scale=None, layout="s2d", candidates=cand, tag=1)
    ring = rp.sample_normalized(batch_size=B, out_dtype=torch.bfloat16, scale=None, layout="ring", candidates=cand, tag=2)
    torch.manual_seed(1)
    net = rl.VanillaNet(4, rl.NatureConvBody(in_channels=4))
    grads = []
    for x in (mat.state, ring.state):
        net.zero_grad()
        with frame_scale(1.0 / 255):
            phi = net.body(x)
        phi.backward(torch.ones_like(phi) * 0.01)
        torch.cuda.synchronize()
        grads.append((phi.detach().clone(), [p.grad.detach().clone() for p in net.body.parameters()]))
    # (fc4's split-K accumulates with fp32 atomics: the features are equal up to their summation order)
    np.testing.assert_allclose(grads[1][0].float().cpu().numpy(), grads[0][0].float().cpu().numpy(), rtol=2e-2, atol=1e-3)
    for a, b in zip(grads[0][1], grads[1][1]):
        np.testing.assert_allclose(b.float().cpu().numpy(), a.float().cpu().numpy(), rtol=2e-2, atol=1e-4)   # fp32 atomics in fc4 / bias sums
