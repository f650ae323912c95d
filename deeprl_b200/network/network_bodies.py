"""Feature extractors with the reference's module / parameter names
(``deep_rl/network/network_bodies.py``: ``NatureConvBody``:10, ``FCBody``:50, ``DummyBody``:76), so that
reference ``state_dict``s load unchanged (``body.conv1.weight`` ... ``body.fc4.bias``, ``layers.<i>``).

``Config.COMPUTE_DTYPE`` selects the arithmetic of the dense contractions: ``torch.float32`` is the parity
mode (TF32 off, results comparable with the reference at 1e-5), ``torch.bfloat16`` the throughput mode
(bf16 operands, fp32 accumulation, fp32 master weights; inputs may arrive as channels_last bf16 straight from
the fused replay gather).  The contractions themselves are plain library calls (cuDNN / cuBLAS) in this round.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ..utils import Config
from . import fused
from .network_utils import NoisyLinear, layer_init


def _autocast():
    on = Config.DEVICE.type == "cuda" and Config.COMPUTE_DTYPE == torch.bfloat16
    return torch.autocast("cuda", dtype=torch.bfloat16, enabled=on)


class NatureConvBody(nn.Module):
    """conv(in,32,k8,s4) -> conv(32,64,k4,s2) -> conv(64,64,k3,s1) -> fc(3136,512), ReLU after each
    (Mnih et al. 2015; network_bodies.py:10-33)."""

    def __init__(self, in_channels=4, noisy_linear=False):
        super().__init__()
        self.feature_dim = 512
        self.conv1 = layer_init(nn.Conv2d(in_channels, 32, kernel_size=8, stride=4))
        self.conv2 = layer_init(nn.Conv2d(32, 64, kernel_size=4, stride=2))
        self.conv3 = layer_init(nn.Conv2d(64, 64, kernel_size=3, stride=1))
        self.fc4 = NoisyLinear(7 * 7 * 64, 512) if noisy_linear else layer_init(nn.Linear(7 * 7 * 64, 512))
        self.noisy_linear = noisy_linear

    def reset_noise(self):
        if self.noisy_linear:
            self.fc4.reset_noise()

    auto_repack = True        # wgmma backend: refresh the packed bf16 operands at every forward (safe default)

    def repack(self, scale=None):
        """Refresh the packed bf16 GEMM operands from the fp32 parameters (owners that set ``auto_repack = False``
        call this after every parameter change: optimizer step, load_state_dict)."""
        from . import nature_tc
        return nature_tc.repack(self, fused.current_frame_scale() if scale is None else scale)

    def forward(self, x):
        """``x``: [B, C, 84, 84] images, or the space-to-depth(4) tensor [B, 16*C, 21, 21] the fused replay gather
        emits (conv1 then runs as a 2x2 / stride-1 convolution over 16*C channels: same arithmetic, tensor-core
        friendly).  bf16 CUDA inputs take the fused path (``network/fused.py``)."""
        if type(x).__name__ == "RingFrames":              # frame stacks still in the uint8 replay ring (K1)
            if Config.DENSE_BACKEND == "tcgen05" and Config.COMPUTE_DTYPE == torch.bfloat16 and not self.noisy_linear:
                from . import nature_tc
                return nature_tc.nature_body(self, x, fused.current_frame_scale())
            x = x.materialize()
        if x.is_cuda and x.dtype == torch.bfloat16 and Config.COMPUTE_DTYPE == torch.bfloat16 and not self.noisy_linear:
            return self._forward_fused(x)
        if x.dim() == 4 and x.shape[1] == 16 * self.conv1.in_channels and x.shape[-1] * 4 == 84:
            x = F.pixel_shuffle(x.view(x.shape[0], self.conv1.in_channels, 16, x.shape[2], x.shape[3]).flatten(0, 1), 4) \
                .view(x.shape[0], self.conv1.in_channels, 84, 84)
        scale = fused.current_frame_scale()
        with _autocast():
            y = F.relu(self.conv1(x * scale if scale != 1.0 else x))
            y = F.relu(self.conv2(y))
            y = F.relu(self.conv3(y))
            y = y.reshape(y.size(0), -1)          # NCHW flatten order whatever the memory format
            return F.relu(self.fc4(y))

    def _forward_fused(self, x):
        scale = fused.current_frame_scale()
        if (Config.DENSE_BACKEND == "tcgen05" and x.shape[1] == 16 * self.conv1.in_channels and x.shape[1] % 64 == 0
                and tuple(x.shape[2:]) == (21, 21)):
            from . import nature_tc                          # whole body on the wgmma GEMM (csrc/gemm.cu)
            return nature_tc.nature_body(self, x, scale)
        w1 = self.conv1.weight
        if x.shape[1] == 16 * self.conv1.in_channels:                    # space-to-depth input
            w1, stride1 = fused.space_to_depth_weight(w1, 4), 1
        else:
            stride1 = 4
        if scale != 1.0:
            w1 = w1 * scale
        if not x.is_contiguous(memory_format=torch.channels_last):
            x = x.contiguous(memory_format=torch.channels_last)
        y = fused.conv_bias_relu(x, w1, self.conv1.bias, stride1, need_input_grad=False)
        y = fused.conv_bias_relu(y, self.conv2.weight, self.conv2.bias, 2)
        y = fused.conv_bias_relu(y, self.conv3.weight, self.conv3.bias, 1)
        # fc4 over the NHWC-flattened features: permute the (C,H,W)-ordered weight columns instead of the activations
        B, C, H, W = y.shape
        w4 = self.fc4.weight.view(-1, C, H, W).permute(0, 2, 3, 1).reshape(self.fc4.weight.shape[0], -1)
        return fused.linear_bias_relu(y.permute(0, 2, 3, 1).reshape(B, -1), w4, self.fc4.bias, True)


class FCBody(nn.Module):
    def __init__(self, state_dim, hidden_units=(64, 64), gate=F.relu, noisy_linear=False):
        super().__init__()
        dims = (state_dim,) + tuple(hidden_units)
        make = (lambda i, o: NoisyLinear(i, o)) if noisy_linear else (lambda i, o: layer_init(nn.Linear(i, o)))
        self.layers = nn.ModuleList([make(i, o) for i, o in zip(dims[:-1], dims[1:])])
        self.gate = gate
        self.feature_dim = dims[-1]
        self.noisy_linear = noisy_linear

    def reset_noise(self):
        if self.noisy_linear:
            for layer in self.layers:
                layer.reset_noise()

    def forward(self, x):
        for layer in self.layers:
            x = self.gate(layer(x))
        return x


class DummyBody(nn.Module):
    def __init__(self, state_dim):
        super().__init__()
        self.feature_dim = state_dim

    def forward(self, x):
        return x
