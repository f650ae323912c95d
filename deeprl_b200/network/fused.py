"""Fused dense layers for the throughput mode (bf16 operands, fp32 accumulation, fp32 master weights).

``y = relu(conv(x, W) + b)`` and ``y = relu(x W^T + b)`` (network_bodies.py:27-33,70-73) as autograd Functions:
the contraction is a library call this round (cuDNN / cuBLAS implicit-GEMM on bf16 NHWC operands), the bias + ReLU
epilogue and the ReLU-mask + bias-gradient reduction of the backward pass are ``csrc/dense.cu`` kernels
(one streaming pass each instead of ~6 eager elementwise / reduce launches per layer).
"""
import contextlib
import threading

import torch

from .. import _lib
from ..ops import _Scratch

_bf16 = torch.bfloat16
_tls = threading.local()


@contextlib.contextmanager
def frame_scale(scale):
    """Declare that image inputs inside the block are raw integers 0..255 scaled by ``scale`` (the fused replay
    gather emits exact integers in bf16; NatureConvBody folds ``scale`` -- ImageNormalizer's 1/255 -- into conv1)."""
    prev = getattr(_tls, "scale", 1.0)
    _tls.scale = float(scale)
    try:
        yield
    finally:
        _tls.scale = prev


def current_frame_scale():
    return getattr(_tls, "scale", 1.0)


def _rows_c(y):
    """(rows, C) of a bf16 activation stored NHWC (4-d channels_last) or [rows, C] (2-d contiguous)."""
    if y.dim() == 4:
        assert y.is_contiguous(memory_format=torch.channels_last), "activations must be channels_last"
        return y.shape[0] * y.shape[2] * y.shape[3], y.shape[1]
    assert y.is_contiguous()
    return y.shape[0], y.shape[1]


def bias_act_(y, bias, relu=True):
    rows, C = _rows_c(y)
    _lib.call("b2rl_bias_act_bf16", _lib.ptr(y), _lib.ptr(bias), rows, C, int(relu), _lib.stream())
    return y


def act_bwd_bias_grad(gy, y, relu=True, row_map=0, G=0, V=0, out_rows=None):
    """-> (g = gy * (y > 0) in bf16, dbias fp32 [C]).  ``row_map`` re-lays ``g`` out on a G x G grid (csrc/dense.cu)."""
    if row_map:
        C = gy.shape[1] // 4 if row_map == 2 else gy.shape[1]
        rows = out_rows                                  # the kernel walks destination rows and zero-fills padding rows
        assert gy.is_contiguous() and y.is_contiguous() and gy.dtype == _bf16
        g = torch.empty((out_rows, C), dtype=_bf16, device=gy.device)
        db = torch.empty(C, dtype=torch.float32, device=gy.device)
        partial = _Scratch.get(y.device, "act_bwd_partial", 592 * 2048, torch.float32)
        counter = _Scratch.get(y.device, "act_bwd_counter", 1, torch.int32)
        _lib.call("b2rl_act_bwd_bias_grad_bf16", _lib.ptr(gy), _lib.ptr(y), rows, C, int(relu), _lib.ptr(g), _lib.ptr(db),
                  _lib.ptr(partial), _lib.ptr(counter), int(row_map), int(G), int(V), _lib.stream())
        return g, db
    rows, C = _rows_c(y)
    if gy.dim() == 4 and not gy.is_contiguous(memory_format=torch.channels_last):
        gy = gy.contiguous(memory_format=torch.channels_last)
    elif gy.dim() == 2 and not gy.is_contiguous():
        gy = gy.contiguous()
    if gy.dtype != _bf16:
        gy = gy.to(_bf16)
    g = torch.empty_like(gy)
    db = torch.empty(C, dtype=torch.float32, device=y.device)
    partial = _Scratch.get(y.device, "act_bwd_partial", 592 * 2048, torch.float32)
    counter = _Scratch.get(y.device, "act_bwd_counter", 1, torch.int32)
    _lib.call("b2rl_act_bwd_bias_grad_bf16", _lib.ptr(gy), _lib.ptr(y), rows, C, int(relu), _lib.ptr(g), _lib.ptr(db),
              _lib.ptr(partial), _lib.ptr(counter), 0, 0, 0, _lib.stream())
    return g, db


class _ConvBiasReLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, stride, need_input_grad):
        w16 = weight.detach().to(_bf16).contiguous(memory_format=torch.channels_last)
        y = torch.ops.aten.convolution(x, w16, None, [stride, stride], [0, 0], [1, 1], False, [0, 0], 1)
        if not y.is_contiguous(memory_format=torch.channels_last):
            y = y.contiguous(memory_format=torch.channels_last)
        bias_act_(y, bias.detach(), True)
        ctx.save_for_backward(x, w16, y)
        ctx.stride, ctx.need_input_grad = stride, need_input_grad
        return y

    @staticmethod
    def backward(ctx, gy):
        x, w16, y = ctx.saved_tensors
        g, db = act_bwd_bias_grad(gy, y, True)
        s = ctx.stride
        gx, gw, _ = torch.ops.aten.convolution_backward(g, x, w16, None, [s, s], [0, 0], [1, 1], False, [0, 0], 1,
                                                        [ctx.need_input_grad, True, False])
        return gx, gw.float(), db, None, None


def conv_bias_relu(x, weight, bias, stride, need_input_grad=True):
    """``relu(conv2d(x, weight, bias, stride))`` on bf16 channels_last ``x``; ``weight`` / ``bias`` are fp32 (master)."""
    return _ConvBiasReLU.apply(x, weight, bias, stride, need_input_grad)


class _LinearBiasReLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, relu):
        w16 = weight.detach().to(_bf16)
        y = torch.mm(x, w16.t())
        bias_act_(y, bias.detach(), relu)
        ctx.save_for_backward(x, w16, y)
        ctx.relu = relu
        return y

    @staticmethod
    def backward(ctx, gy):
        x, w16, y = ctx.saved_tensors
        g, db = act_bwd_bias_grad(gy, y, ctx.relu)
        gx = torch.mm(g, w16) if ctx.needs_input_grad[0] else None
        gw = torch.mm(g.t(), x).float()
        return gx, gw, db, None


def linear_bias_relu(x, weight, bias, relu=True):
    """``relu(x @ weight.T + bias)`` on bf16 ``x`` [rows, K]; fp32 master ``weight`` [N, K] and ``bias``."""
    return _LinearBiasReLU.apply(x, weight, bias, relu)


def space_to_depth_weight(weight, block=4):
    """[Cout, Cin, k, k] with k = 2*block, stride = block  ->  [Cout, Cin*block*block, 2, 2]: the kernel that, applied
    with stride 1 to the space-to-depth(block) input (channel = cin*block^2 + dy*block + dx), equals the original
    stride-``block`` convolution."""
    co, ci, kh, kw = weight.shape
    assert kh == kw == 2 * block
    w = weight.view(co, ci, 2, block, 2, block)          # (n, f, ky2, dy, kx2, dx)
    return w.permute(0, 1, 3, 5, 2, 4).reshape(co, ci * block * block, 2, 2)


def _fc4_relu_features(phi):
    """True if ``phi`` is the live output of a wgmma NatureConvBody's fc4 ReLU (network/nature_tc.py): the head's backward
    then applies that ReLU's mask and bias gradient itself.  Decided in the forward pass, while the features are alive."""
    from . import nature_tc
    return nature_tc.FUSED_BWD and nature_tc.is_relu_features(phi)


class _NarrowHead(torch.autograd.Function):
    """VanillaNet / DuelingNet head on bf16 features (csrc/head.cu): 2 launches per update instead of ~12."""

    @staticmethod
    def forward(ctx, phi, wa, ba, wv, bv):
        B, K = phi.shape
        A = wa.shape[0]
        q = torch.empty((B, A), dtype=torch.float32, device=phi.device)
        _lib.call("b2rl_head_fwd", _lib.ptr(phi), _lib.ptr(wa.detach()), _lib.ptr(ba.detach()),
                  _lib.ptr(None if wv is None else wv.detach()), _lib.ptr(None if bv is None else bv.detach()), B, K, A,
                  _lib.ptr(q), _lib.stream())
        ctx.save_for_backward(phi)
        ctx.params = (wa, ba, wv, bv)
        ctx.relu = _fc4_relu_features(phi)
        return q

    @staticmethod
    def backward(ctx, gq):
        (phi,) = ctx.saved_tensors
        wa, ba, wv, bv = ctx.params
        B, K = phi.shape
        A = wa.shape[0]
        gq = gq.contiguous().float()
        gphi = torch.empty_like(phi)
        params = [p for p in (wa, ba, wv, bv) if p is not None]
        inplace = all(p.grad is not None and p.grad.dtype == torch.float32 and p.grad.is_contiguous() for p in params)
        if inplace:
            gwa, gba = wa.grad, ba.grad
            gwv, gbv = (wv.grad, bv.grad) if wv is not None else (None, None)
        else:
            z = lambda p: None if p is None else torch.zeros_like(p, dtype=torch.float32)
            gwa, gba, gwv, gbv = z(wa), z(ba), z(wv), z(bv)
        from . import nature_tc
        if ctx.relu:
            # phi = relu(fc4(.)) of a wgmma NatureConvBody: its ReLU backward and bias gradient ride along (the body's
            # backward finds the column sums under the gradient's address and skips its own pass)
            sink = nature_tc.SINK               # persistent accumulator (re-zeroed by the tail's kernel A) or a fresh one
            colsum = sink.db4 if (sink is not None and sink.db4.numel() == K) else torch.zeros(K, dtype=torch.float32, device=phi.device)
            _lib.call("b2rl_head_bwd_relu", _lib.ptr(gq), _lib.ptr(phi), _lib.ptr(wa.detach()),
                      _lib.ptr(None if wv is None else wv.detach()), B, K, A, _lib.ptr(gphi), _lib.ptr(gwa), _lib.ptr(gba),
                      _lib.ptr(gwv), _lib.ptr(gbv), _lib.ptr(colsum), _lib.stream())
            nature_tc.premask(gphi, colsum)
            nature_tc.mark("head_bwd")
        else:
            _lib.call("b2rl_head_bwd", _lib.ptr(gq), _lib.ptr(phi), _lib.ptr(wa.detach()),
                      _lib.ptr(None if wv is None else wv.detach()), B, K, A, _lib.ptr(gphi), _lib.ptr(gwa), _lib.ptr(gba),
                      _lib.ptr(gwv), _lib.ptr(gbv), _lib.stream())
        if inplace:
            return gphi, None, None, None, None
        return gphi, gwa, gba, gwv, gbv


def narrow_head(phi, fc_action, fc_value=None):
    """``q = fc_action(phi)`` or the dueling combine ``v + adv - mean(adv)`` (network_heads.py:18-21, 32-37)."""
    return _NarrowHead.apply(phi.contiguous(), fc_action.weight, fc_action.bias,
                             None if fc_value is None else fc_value.weight, None if fc_value is None else fc_value.bias)


def narrow_head_ok(phi, fc_action, fc_value=None):
    aligned = all(m is None or m.weight.data_ptr() % 16 == 0 for m in (fc_action, fc_value))
    return (phi.is_cuda and phi.dtype == _bf16 and phi.dim() == 2 and phi.shape[1] % 8 == 0 and aligned
            and isinstance(fc_action, torch.nn.Linear) and fc_action.out_features < 32)


def ac_head(phi, fc_action, fc_critic, out=None, draw=None):
    """CategoricalActorCriticNet's head on bf16 features (DummyBody actor / critic bodies, network_heads.py:184-188) in one
    launch (``b2rl_ac_head_fwd``): returns ``out`` [B, A+1] fp32 = (logits, v), no autograd.  ``draw``: (seed, counter int64
    [1], action_out int64 [B], ticket int32 [1]) -- the action of each row is also drawn from softmax(logits) on the device's
    Philox stream into ``action_out``, and the device counter advances by B."""
    B, K = phi.shape
    A = fc_action.out_features
    if out is None:
        out = torch.empty((B, A + 1), dtype=torch.float32, device=phi.device)
    seed, counter, action, ticket = draw if draw is not None else (0, None, None, None)
    _lib.call("b2rl_ac_head_fwd", _lib.ptr(phi), _lib.ptr(fc_action.weight.detach()), _lib.ptr(fc_action.bias.detach()),
              _lib.ptr(fc_critic.weight.detach()), _lib.ptr(fc_critic.bias.detach()), B, K, A, _lib.ptr(out), int(seed),
              _lib.ptr(counter), _lib.ptr(action), _lib.ptr(ticket), _lib.stream())
    return out


def ac_head_backward(phi, geff, fc_action, fc_critic):
    """The backward of ``ac_head`` from the effective output gradients ``geff`` [B, 33] (``ops.a2c_rollout_loss``) on features
    ``phi`` = relu(fc4(.)) of a wgmma NatureConvBody (``b2rl_head_bwd_geff_relu``): the head's weight and bias gradients are
    accumulated into their ``.grad`` (the optimizer arena), fc4's ReLU mask and bias gradient ride along as in
    ``_NarrowHead.backward``.  Returns the bf16 feature gradient, for ``phi.backward``."""
    from . import nature_tc
    if not _fc4_relu_features(phi):
        raise _lib.B2RLError("ac_head_backward: phi must be the live fc4 output of a wgmma NatureConvBody with the fused "
                             "backward epilogues")
    params = (fc_action.weight, fc_action.bias, fc_critic.weight, fc_critic.bias)
    if not all(p.grad is not None and p.grad.dtype == torch.float32 and p.grad.is_contiguous() for p in params):
        raise _lib.B2RLError("ac_head_backward: the head's gradients must be fp32 buffers (a FlatOptimizer arena)")
    B, K = phi.shape
    gphi = torch.empty_like(phi)
    sink = nature_tc.SINK
    colsum = sink.db4 if (sink is not None and sink.db4.numel() == K) else torch.zeros(K, dtype=torch.float32, device=phi.device)
    _lib.call("b2rl_head_bwd_geff_relu", _lib.ptr(geff), _lib.ptr(phi), _lib.ptr(fc_action.weight.detach()),
              _lib.ptr(fc_critic.weight.detach()), B, K, fc_action.out_features, _lib.ptr(gphi),
              *[_lib.ptr(p.grad) for p in params], _lib.ptr(colsum), _lib.stream())
    nature_tc.premask(gphi, colsum)
    nature_tc.mark("head_bwd")
    return gphi


class _DistHead(torch.autograd.Function):
    """Distributional head (CategoricalNet / QuantileNet, network_heads.py:40-55, 89-102) on bf16 features with no cuBLAS / ATen
    kernel: logits = phi W^T + b on the wgmma GEMM, softmax + log_softmax in one launch (csrc/disthead.cu), and in the backward
    pass the log_softmax gradient, the bf16 operand and the bias gradient in one launch followed by the two GEMMs
    (dW = g^T phi, dphi = relu_mask(g W) with fc4's bias gradient from the same epilogue)."""

    @staticmethod
    def forward(ctx, phi, weight, bias, w16, A, N, softmax):
        from ..ops import gemm_bf16
        B, K = phi.shape
        AN = A * N
        logits = gemm_bf16(phi, w16, bias=bias.detach(), out_dtype=torch.float32, block_n=64)
        ctx.dims = (A, N, bool(softmax))
        ctx.params = (weight, bias)
        ctx.relu = _fc4_relu_features(phi)
        if softmax:
            prob = torch.empty((B, A, N), dtype=torch.float32, device=phi.device)
            logp = torch.empty((B, A, N), dtype=torch.float32, device=phi.device)
            _lib.call("b2rl_dist_softmax", _lib.ptr(logits), B * A, N, _lib.ptr(prob), _lib.ptr(logp), _lib.stream())
            ctx.save_for_backward(phi, w16, prob)
            ctx.mark_non_differentiable(prob)
            return logp, prob
        ctx.save_for_backward(phi, w16)
        none = torch.empty(0, device=phi.device)
        ctx.mark_non_differentiable(none)
        return logits.view(B, A, N), none

    @staticmethod
    def backward(ctx, gout, _unused):
        import ctypes
        from . import nature_tc
        from ..ops import gemm_bf16
        A, N, softmax = ctx.dims
        weight, bias = ctx.params
        saved = ctx.saved_tensors
        phi, w16 = saved[0], saved[1]
        prob = saved[2] if softmax else None
        B, K = phi.shape
        AN = A * N
        ld = (AN + 7) // 8 * 8
        gout = gout.contiguous().float()
        g = torch.empty((B, ld), dtype=_bf16, device=phi.device)
        inplace = all(p.grad is not None and p.grad.dtype == torch.float32 and p.grad.is_contiguous() for p in (weight, bias))
        gb = bias.grad if inplace else torch.zeros_like(bias, dtype=torch.float32)
        _lib.call("b2rl_dist_head_bwd_prep", _lib.ptr(gout), _lib.ptr(prob), B, A, N, _lib.ptr(g), ld, _lib.ptr(gb), _lib.stream())
        gv = g[:, :AN]
        # dW [A*N, K] = g^T phi (both operands MN-major: nothing is transposed in memory), accumulated into .grad when it exists
        gw = gemm_bf16(gv, phi, a_major="mn", b_major="mn", out_dtype=torch.float32, block_n=128,
                       out=weight.grad if inplace else None, accumulate=inplace)
        # dphi = (g W) masked by relu(fc4) with fc4's bias gradient from the same epilogue
        gphi = torch.empty_like(phi)
        sink = nature_tc.SINK
        if ctx.relu:
            colsum = sink.db4 if (sink is not None and sink.db4.numel() == K) else torch.zeros(K, dtype=torch.float32, device=phi.device)
            e = _lib.bwd_epilogue(phi, colsum, 0, 0)               # dbias_mod 0: one bias gradient per feature column
            _lib.call("b2rl_gemm_bwd_bf16", _lib.ptr(gv), gv.stride(0), _lib.ptr(w16), 1, w16.stride(0), _lib.ptr(gphi), gphi.stride(0),
                      B, K, AN, 0, 0, 0, ctypes.byref(e), 128, _lib.stream())
            nature_tc.premask(gphi, colsum)
        else:
            gemm_bf16(gv, w16, a_major="k", b_major="mn", out=gphi, block_n=128)
        if inplace:
            return gphi, None, None, None, None, None, None
        return gphi, gw, gb, None, None, None, None


def dist_head(phi, fc, A, N, softmax):
    """``fc`` = the head's nn.Linear with a bf16 copy of its weight in ``fc._w16`` (kept current by the owner: the fused
    optimizer's shadow for the online network, refreshed at target sync for the target network).  Returns (log_prob, prob)
    [B, A, N] for C51 (``softmax``), (quantile, quantile) for QR-DQN."""
    return _DistHead.apply(phi.contiguous(), fc.weight, fc.bias, fc._w16, A, N, softmax)


def dist_head_ok(phi, fc):
    w16 = getattr(fc, "_w16", None)
    return (w16 is not None and phi.is_cuda and phi.dtype == _bf16 and phi.dim() == 2 and phi.shape[1] % 64 == 0
            and isinstance(fc, torch.nn.Linear) and w16.dtype == _bf16 and tuple(w16.shape) == tuple(fc.weight.shape))
