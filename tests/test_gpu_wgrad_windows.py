"""Weight-gradient convolution GEMM with an odd number of 64-channel tap windows: with more than 64 output channels there
is no M-stacking, so a 3x3 convolution has 9 windows -- four CTA groups of two n64 windows and the last window in a launch
of its own (the one-window instantiation of conv_wgrad_wgmma_kernel)."""
import pytest
import torch

from deeprl_b200.network import nature_tc as tc


@pytest.mark.gpu
@pytest.mark.parametrize("n_out", [128, 96])
def test_conv_wgrad_odd_window_count(n_out):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    gen = torch.Generator(device="cuda").manual_seed(5)
    B, G, C, taps_x = 6, 10, 64, 3
    rows = B * G * G
    X = torch.randn(rows, C, device="cuda", generator=gen).to(torch.bfloat16)
    Gr = torch.randn(rows, n_out, device="cuda", generator=gen).to(torch.bfloat16)
    D = torch.zeros((n_out, 9 * C), device="cuda")
    tc.conv_gemm(1, X, Gr, n_out, 9, taps_x, G, 1, D, splits=16, block_n=64)
    ref = torch.empty_like(D)
    for t in range(9):
        s = (t // taps_x) * G + t % taps_x
        xs = torch.zeros(rows, C, device="cuda")
        xs[:rows - s] = X[s:].float()
        ref[:, t * C:(t + 1) * C] = Gr.float().t() @ xs
    torch.testing.assert_close(D, ref, rtol=1e-4, atol=1e-2)
