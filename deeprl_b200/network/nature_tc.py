"""NatureConvBody forward + backward entirely on the wgmma GEMM of ``csrc/gemm.cu`` (no cuDNN / cuBLAS).

Reference layer stack: ``network_bodies.py:10-33`` -- conv(4->32,k8,s4), conv(32->64,k4,s2), conv(64->64,k3,s1), fc(3136->512),
ReLU after each.  Every layer is a GEMM over activations stored as [batch * G * G][C] grid matrices:

    x0  [B*21*21][ 64]   frames, space-to-depth(4): written by the replay gather           (conv1 = 2x2 taps, K = 256)
    x1  [B*10*10][128]   relu(conv1), space-to-depth(2): written by conv1's GEMM epilogue   (conv2 = 2x2 taps, K = 512)
    y2  [B*10*10][ 64]   relu(conv2) on the 10-grid (row/col 9 are never read)               (conv3 = 3x3 taps, K = 576)
    y3  [B* 7* 7][ 64]   relu(conv3), compacted by conv3's epilogue == fc4's input in (h, w, c) order
    y4  [B][512]         relu(fc4)

Backward: ReLU mask + bias gradient + re-layout in one pass (``csrc/dense.cu``), then dgrad = the same shifted-row GEMM
with negative shifts and wgrad = MN-major GEMMs with split-K.  Weights are re-laid out from the reference's parameter
layout ([Cout, Cin, kh, kw], (c, h, w)-ordered fc4 columns) to the tap-major bf16 layouts by ONE kernel
(``csrc/pack.cu``) and the weight gradients are mapped back and accumulated into ``.grad`` by ONE kernel, so
``state_dict``s and optimizers see the reference layout only.
"""
import contextlib
import ctypes
import os
import weakref

import torch

from .. import _lib
from ..ops import gemm_bf16, gemm_splitk_bf16
from .fused import act_bwd_bias_grad

_bf16 = torch.bfloat16
_f32 = torch.float32
# fc4 forward, one launch with the bias / ReLU / bf16 epilogue: K split over the FC4_SPLITS CTAs (2, 4 or 8) of a
# thread-block cluster per output tile, the partials summed in distributed shared memory in a fixed order; 0 = the cluster
# size the launcher picks from the shape and the SMs of the device; 1 = one CTA per output tile over all of K
FC4_SPLITS = int(os.environ.get("B2RL_FC4_SPLITS", "0"))
# backward: ReLU mask + bias gradient + re-layout fused into the dgrad GEMM epilogues (b2rl_*_bwd_bf16) instead of three
# b2rl_act_bwd_bias_grad_bf16 passes (B2RL_FUSED_BWD=0 restores them).
FUSED_BWD = os.environ.get("B2RL_FUSED_BWD", "1") == "1"
_ZEROED = {}
TRACE = None               # learner.StepTrace while a traced capture is running: mark(name) records a timing event in the graph


def mark(name, stream=None):
    if TRACE is not None:
        TRACE.mark(name, stream)


AFTER_DGRAD = None         # callable run once, on the current stream, right after the last dgrad GEMM of the backward pass was
                           # launched (the learner forks its late prefetch branch there: beside the weight-gradient tail)
AFTER_RING_READ = None     # callable(stream) run on the current stream right after conv1's weight gradient was launched from the
                           # uint8 ring (K1) on ``stream`` (None: the current stream); that launch is the batch's last ring read,
                           # so the learner forks the next update's ring feeds there
SINK = None                # network/tail.py NatureTail while ``grad_sink`` is active: backward hands it the GEMM-layout gradients
RELU_FEATURES = {}         # data_ptr -> weak reference to the feature tensor y4 = relu(fc4(.)) nature_body produced there
PREMASKED = {}             # data_ptr of a feature gradient already masked by head_bwd_relu -> (that gradient, its column sums = db4)


def mark_relu_features(y4):
    """Record ``y4`` as the output of fc4's ReLU, so that a head on it may fold the ReLU backward into its own."""
    if len(RELU_FEATURES) > 256:
        for k in [k for k, r in RELU_FEATURES.items() if r() is None]:
            del RELU_FEATURES[k]
    RELU_FEATURES[y4.data_ptr()] = weakref.ref(y4)


def is_relu_features(phi):
    """True if ``phi`` lies at the address of a y4 that is still alive.  A live y4 keeps its memory, so ``phi`` is that
    y4 (or a view of it); once y4 is freed, the allocator may hand its address to any other tensor."""
    r = RELU_FEATURES.get(phi.data_ptr())
    return r is not None and r() is not None


def premask(gphi, db4):
    """Record that ``gphi`` is already masked by relu(fc4) with its column sums in ``db4``: the body's backward then skips
    its own mask / bias-gradient pass.  The entry holds ``gphi`` itself, so its address cannot be reused by another
    gradient, and autograd cannot accumulate into it in place, before the body's backward takes the entry."""
    if len(PREMASKED) >= 16:                    # entries nobody took (e.g. the gradient was summed with another one)
        PREMASKED.pop(next(iter(PREMASKED)))
    PREMASKED[gphi.data_ptr()] = (gphi, db4)


def take_premasked(gy4):
    """The column sums recorded by ``premask`` for this very gradient, or None (the entry is removed)."""
    if gy4.dtype != _bf16 or not gy4.is_contiguous():
        return None
    e = PREMASKED.pop(gy4.data_ptr(), None)
    return e[1] if e is not None and e[0].shape == gy4.shape else None


class RingFrames:
    """A batch of frame stacks that is NOT materialised: (uint8 replay ring, sampled indices, offset of the oldest stacked
    frame).  ``UniformReplay.sample_normalized(layout="ring")`` returns these as ``state`` / ``next_state``; conv1's forward
    and weight-gradient kernels read the ring themselves (K1: csrc/gemm.cu ``fill_slab_u8``)."""

    def __init__(self, frames, idx, first, row_bytes, frame_w, history):
        self.frames, self.idx, self.first = frames, idx, int(first)
        self.row_bytes, self.frame_w, self.history = int(row_bytes), int(frame_w), int(history)
        self.batch = idx.shape[0]
        self.grid = self.frame_w // 4
        self.device = frames.device

    is_cuda = True
    dtype = torch.uint8

    @property
    def shape(self):
        return (self.batch, 16 * self.history, self.grid, self.grid)

    def materialize(self):
        """The bf16 space-to-depth tensor [B, 16*history, G, G] (channels_last) this object stands for (tests, fallbacks)."""
        rows = (self.idx + self.first).view(-1, 1) + torch.arange(self.history, device=self.device).view(1, -1)
        x = self.frames.view(-1, self.frame_w, self.frame_w)[rows.view(-1)].view(self.batch, self.history, self.frame_w, self.frame_w)
        g = self.grid
        x = x.view(self.batch, self.history, g, 4, g, 4).permute(0, 2, 4, 1, 3, 5).reshape(self.batch, g, g, 16 * self.history)
        return x.to(_bf16).permute(0, 3, 1, 2)

    # inspection (tests, debugging): a RingFrames reads as the batch it stands for, as the ring holds it now
    def data_ptr(self):
        """Address of the index buffer: batches drawn into different buffer sets differ here."""
        return self.idx.data_ptr()

    def clone(self):
        return self.materialize()

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        m = lambda x: x.materialize() if isinstance(x, RingFrames) else x
        return func(*[m(a) for a in args], **{k: m(v) for k, v in (kwargs or {}).items()})

    def args(self):
        return (_lib.ptr(self.frames), int(self.frames.shape[0]), _lib.ptr(self.idx), self.first, self.row_bytes, self.frame_w,
                self.batch, self.history)


def _zero_grid(key, shape, device):
    """Persistent zero-initialised destination of a scatter epilogue: the tiles overwrite exactly the same rows every time
    and never touch the padding rows, so the buffer is zeroed once."""
    k = (key, tuple(shape), str(device))
    if k not in _ZEROED:
        _ZEROED[k] = torch.zeros(shape, dtype=_bf16, device=device)
    return _ZEROED[k]


@contextlib.contextmanager
def grad_sink(tail):
    """Inside this context the backward pass of ``tail.body`` does not touch ``.grad`` itself: it hands the GEMM-layout
    weight gradients (split-K partials) to ``tail.reduce`` (csrc/tail.cu kernel A) and accumulates the bias gradients in
    the tail's persistent buffers."""
    global SINK
    old, SINK = SINK, tail
    try:
        yield tail
    finally:
        SINK = old


def _sink_for(params):
    t = SINK
    return t if (t is not None and params[0] is t.body.conv1.weight) else None


def _backward_fused(ctx, gy4):
    x0m, x1, y2, y3, y4, w2d, w3d, w4p = ctx.saved_tensors
    B, dev = y4.shape[0], y4.device
    sink = _sink_for(ctx.params)
    db4 = take_premasked(gy4)
    if db4 is not None:
        g4 = gy4                                                                        # masked + summed by b2rl_head_bwd_relu
    else:
        g4, db4 = act_bwd_bias_grad(gy4, y4, True)                                      # fc4's own ReLU / bias gradient
    y3c = y3.view(B, 3136)
    main, side = _budgets(dev)                                  # CTAs of the dgrad chain and of the weight gradients beside it
    with _cta_budget(side):
        gw4p = gemm_bf16(g4, y3c, a_major="mn", b_major="mn", out_dtype=_f32, block_n=128, stream=_fork())
    mark("w_fc4", _WGRAD["stream"])
    if sink is not None and sink.split:
        # multi-GPU: fc4's gradient (95 % of the bytes) goes to the arena NOW, and its all-reduce (sink.early) runs beside the
        # convolution backward instead of after it
        if db4 is not sink.db4:
            sink.db4.copy_(db4)
        side = _WGRAD["stream"]
        with torch.cuda.stream(side) if side is not None else contextlib.nullcontext():
            sink.reduce_w4(gw4p)
            if sink.early is not None:
                sink.early()
    if sink is not None:                   # persistent accumulators, re-zeroed by the tail's kernel A
        db1, db2, db3 = sink.db1, sink.db2, sink.db3
    else:
        db = torch.zeros(32 + 64 + 64, dtype=_f32, device=dev)
        db1, db2, db3 = db[:32], db[32:96], db[96:160]
    # fc4 dgrad -> conv3's output grid (10 x 10 per image), masked by relu(conv3) and summed into db3
    g3 = _zero_grid("g3", (B * 100, 64), dev)
    e3 = _lib.bwd_epilogue(y3c, db3, 64, 64)
    with _cta_budget(main):
        _lib.call("b2rl_gemm_bwd_bf16", _lib.ptr(g4), g4.stride(0), _lib.ptr(w4p), 1, w4p.stride(0), _lib.ptr(g3), 64, B, 3136,
                  g4.shape[1], 4, 10, 7, ctypes.byref(e3), 128, _lib.stream())
    mark("d_fc4")
    with _cta_budget(side):
        gw3p, p3 = wgrad_partials(y2, g3, 64, 9, 3, 10, stream=_fork())
    mark("w_conv3", _WGRAD["stream"])
    # conv3 dgrad on the 10-grid, masked by relu(conv2)
    g2 = torch.empty((B * 100, 64), dtype=_bf16, device=dev)
    e2 = _lib.bwd_epilogue(y2, db2, 64, 0)
    with _cta_budget(main):
        _lib.call("b2rl_conv_gemm_bwd_bf16", _lib.ptr(g3), B * 100, 64, _lib.ptr(w3d), 64, 9, 3, 10, _lib.ptr(g2), 64, 0, 0, 0,
                  ctypes.byref(e2), 64, _lib.stream())
    mark("d_conv3")
    with _cta_budget(side):
        gw2p, p2 = wgrad_partials(x1, g2, 64, 4, 2, 10, stream=_fork())
    mark("w_conv2", _WGRAD["stream"])
    # conv2 dgrad: space-to-depth(2) rows -> conv1's 21-grid, masked by relu(conv1)
    g1 = _zero_grid("g1", (B * 441, 32), dev)
    e1 = _lib.bwd_epilogue(x1, db1, 32, 32)
    with _cta_budget(main):
        _lib.call("b2rl_conv_gemm_bwd_bf16", _lib.ptr(g2), B * 100, 64, _lib.ptr(w2d), 128, 4, 2, 10, _lib.ptr(g1), 32, 3, 21,
                  20, ctypes.byref(e1), 128, _lib.stream())
    mark("d_conv2")
    if AFTER_DGRAD is not None:
        AFTER_DGRAD()
    if ctx.ring is not None:
        gw1p, p1 = wgrad_partials_ring(ctx.ring, g1, 32, stream=_fork())
        if AFTER_RING_READ is not None:
            AFTER_RING_READ(_WGRAD["stream"])
    else:
        gw1p, p1 = wgrad_partials(x0m, g1, 32, 4, 2, 21, stream=_fork())
    mark("w_conv1", _WGRAD["stream"])
    _join()
    return (gw1p, p1, gw2p, p2, gw3p, p3, gw4p), (db1, db2, db3, db4)


_WGRAD = {"stream": None, "ctas": 0}
# CTAs the weight gradients of fc4, conv3 and conv2 hold on the side branch; the dgrad chain gets the other SMs.  Each of these
# kernels takes a whole SM, so with full grids on both branches the block scheduler interleaves them and the dgrads on the
# critical path wait for side CTAs to retire.  32 leaves 100 CTAs of the 132 SMs of an H100 SXM: fc4's dgrad is 100 tiles,
# and the 400-tile convolution dgrads take 4 tiles per CTA on 100 CTAs, as their slowest CTAs already do on 132, so they
# are as fast alone as on full grids; fewer side CTAs leave the weight gradients too slow to finish beside the chain
# (scripts/bwd_sm_budget.py, DESIGN section 7).
SIDE_CTAS = 32


@contextlib.contextmanager
def wgrad_stream(stream, side_ctas=None):
    """Inside this context the backward pass launches its weight-gradient GEMMs on ``stream`` (a second branch of the
    captured graph): they only feed the final gradient unpack, so they overlap the dgrad / ReLU-mask chain, which is
    latency-bound with one CTA per SM.  Buffers are allocated on the current stream and the branch is joined before
    ``backward`` returns, so no allocator bookkeeping is needed.  With a side stream, the weight gradients of fc4, conv3 and
    conv2 run on ``side_ctas`` CTAs (default ``SIDE_CTAS``; 0: full grids) and the dgrads beside them on the remaining
    SMs (``b2rl_set_cta_budget``); conv1's weight gradient, which has nothing beside it, keeps its grid."""
    old = dict(_WGRAD)
    _WGRAD["stream"] = stream
    _WGRAD["ctas"] = 0 if stream is None else (SIDE_CTAS if side_ctas is None else int(side_ctas))
    try:
        yield
    finally:
        _WGRAD.update(old)


@contextlib.contextmanager
def _cta_budget(ctas):
    """Launches inside this context size their grids to at most ``ctas`` CTAs (0: the whole device)."""
    if not ctas:
        yield
        return
    _lib.call("b2rl_set_cta_budget", int(ctas))
    try:
        yield
    finally:
        _lib.call("b2rl_set_cta_budget", 0)


def _budgets(device):
    """(dgrad chain, side branch) CTA budgets of the backward pass: (0, 0) without a side-branch budget."""
    side = _WGRAD["ctas"]
    if not side:
        return 0, 0
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    if not 0 < side < sms:
        raise ValueError("side_ctas must leave SMs for the dgrad chain: 0 < %d < %d" % (side, sms))
    return sms - side, side


def _fork():
    """Stream handle for the next weight-gradient launch (ordered after everything queued on the current stream)."""
    side = _WGRAD["stream"]
    if side is None:
        return None
    side.wait_stream(torch.cuda.current_stream())
    return side.cuda_stream


def _join():
    side = _WGRAD["stream"]
    if side is not None:
        torch.cuda.current_stream().wait_stream(side)


def _max_partials(device):
    """The weight-gradient kernels write at most one split-K partial per SM."""
    return torch.cuda.get_device_properties(device).multi_processor_count


def wgrad_partials(X, G_rows, n_out, taps, taps_x, grid_w, stream=None):
    """Split-K partial weight gradients (one per CTA, no atomics): returns (partials [P_max, n_out, taps*C] fp32, P)."""
    rows, C = X.shape
    if not _lib.CONV_SLAB:                       # tap-addressing mode (tests): atomic accumulation into one "partial"
        out = torch.zeros((1, n_out, taps * C), dtype=_f32, device=X.device)
        conv_gemm(1, X, G_rows, n_out, taps, taps_x, grid_w, 1, out[0], splits=16, block_n=128 if C == 128 else 64)
        return out, 1
    buf = torch.empty((_max_partials(X.device), n_out, taps * C), dtype=_f32, device=X.device)
    n = ctypes.c_int32(0)
    if (C, n_out, taps, taps_x) == (64, 32, 4, 2):   # conv1: the taps-in-M kernel, the same bits as wgrad_partials_ring
        _lib.call("b2rl_conv1_wgrad_partials", _lib.ptr(X), int(rows), int(grid_w), _lib.ptr(G_rows), int(n_out), _lib.ptr(buf),
                  ctypes.byref(n), stream if stream is not None else _lib.stream())
        return buf, int(n.value)
    if n_out == 64 and (C, taps, taps_x) in ((64, 9, 3), (128, 4, 2)):   # conv3 / conv2: every tap of a k-block in one CTA
        _lib.call("b2rl_conv_taps_wgrad_partials", _lib.ptr(X), int(rows), int(C), _lib.ptr(G_rows), int(n_out), int(taps),
                  int(taps_x), int(grid_w), _lib.ptr(buf), ctypes.byref(n), stream if stream is not None else _lib.stream())
        return buf, int(n.value)
    _lib.call("b2rl_conv_wgrad_partials", _lib.ptr(X), int(rows), int(C), _lib.ptr(G_rows), int(n_out), int(taps), int(taps_x),
              int(grid_w), _lib.ptr(buf), ctypes.byref(n), stream if stream is not None else _lib.stream())
    return buf, int(n.value)


def wgrad_partials_ring(ring, G_rows, n_out, stream=None):
    """conv1's split-K partial weight gradients with the activations read from the uint8 ring (K1)."""
    buf = torch.empty((_max_partials(G_rows.device), n_out, 4 * 16 * ring.history), dtype=_f32, device=G_rows.device)
    n = ctypes.c_int32(0)
    _lib.call("b2rl_conv1_u8_wgrad_partials", *ring.args(), _lib.ptr(G_rows), int(n_out), _lib.ptr(buf), ctypes.byref(n),
              stream if stream is not None else _lib.stream())
    return buf, int(n.value)


def conv_gemm(mode, X, W_or_G, n_out, taps, taps_x, grid_w, sign, out, bias=None, relu=False, out_map=0, G=0, V=0, splits=1,
              block_n=64):
    rows, C = X.shape
    out_mode = 2 if mode == 1 else (0 if out.dtype == _bf16 else 1)
    _lib.call("b2rl_conv_gemm_bf16", int(mode), _lib.ptr(X), int(rows), int(C), _lib.ptr(W_or_G), int(n_out), int(taps),
              int(taps_x), int(grid_w), int(sign), _lib.ptr(out), out.stride(0), _lib.ptr(bias), int(relu), out_mode,
              int(out_map), int(G), int(V), int(splits), int(block_n), _lib.stream())
    return out


# ------------------------------------------------------------------------------------------------- weight layouts
class PackedWeights:
    """Persistent bf16 GEMM operands of one NatureConvBody (fixed addresses: CUDA-graph friendly)."""

    def __init__(self, c1, n4, device):
        e = lambda *s: torch.empty(s, dtype=_bf16, device=device)
        self.c1, self.n4 = c1, n4
        self.w1f, self.w2f, self.w2d = e(32, 64 * c1), e(64, 512), e(128, 256)
        self.w3f, self.w3d, self.w4p = e(64, 576), e(64, 576), e(n4, 3136)
        self.scale = None

    def pack(self, w1, w2, w3, w4, scale):
        _lib.call("b2rl_nature_pack_weights", _lib.ptr(w1), _lib.ptr(w2), _lib.ptr(w3), _lib.ptr(w4), self.c1, self.n4,
                  float(scale), _lib.ptr(self.w1f), _lib.ptr(self.w2f), _lib.ptr(self.w2d), _lib.ptr(self.w3f),
                  _lib.ptr(self.w3d), _lib.ptr(self.w4p), _lib.stream())
        self.scale = float(scale)
        return self

    def tensors(self):
        return self.w1f, self.w2f, self.w2d, self.w3f, self.w3d, self.w4p


def pack_weights(w1, w2, w3, w4, scale):
    """Reference layouts -> tap-major bf16 GEMM operands (forward ``f`` and dgrad ``d`` orientations)."""
    ok = all(t.is_contiguous() and t.dtype == _f32 for t in (w1, w2, w3, w4))
    assert ok and tuple(w2.shape) == (64, 32, 4, 4) and tuple(w3.shape) == (64, 64, 3, 3) and w4.shape[1] == 3136
    return PackedWeights(w1.shape[1], w4.shape[0], w1.device).pack(w1, w2, w3, w4, scale).tensors()


def unpack_grads(g1f, g2f, g3f, g4p, scale, c1):
    """fp32 gradients in GEMM layout -> the reference's parameter layouts (torch expressions; tests and the generic
    autograd path -- the training step accumulates with ``b2rl_nature_unpack_grads`` instead)."""
    n1 = g1f.shape[0]
    g1 = (g1f.view(n1, 2, 2, c1, 4, 4).permute(0, 3, 1, 4, 2, 5) * scale).reshape(n1, c1, 8, 8)
    g2 = g2f.view(64, 2, 2, 2, 2, 32).permute(0, 5, 1, 3, 2, 4).reshape(64, 32, 4, 4)
    g3 = g3f.view(64, 3, 3, 64).permute(0, 3, 1, 2).contiguous()
    g4 = g4p.view(-1, 7, 7, 64).permute(0, 3, 1, 2).reshape(g4p.shape[0], 3136)
    return g1, g2, g3, g4


def forward_only(x0, packed, b1, b2, b3, b4):
    """x0: [B, 64, 21, 21] channels_last bf16 (space-to-depth frames).  Returns (y4, saved activations)."""
    w1f, w2f, _, w3f, _, w4p = packed
    B = x0.shape[0]
    dev = x0.device
    x1 = paired_conv1.take(x0, w1f) if paired_conv1.current is not None else None
    if x1 is not None:                                                         # computed by the paired conv1 launch
        x0m = x0
    elif isinstance(x0, RingFrames):                                           # K1: conv1 reads the uint8 ring itself
        x0m = x0
        x1 = torch.empty((B * 100, 128), dtype=_bf16, device=dev)
        _lib.call("b2rl_conv1_u8_fwd", *x0.args(), _lib.ptr(w1f), 32, _lib.ptr(x1), x1.stride(0), _lib.ptr(b1), 1, 1, 20,
                  _lib.stream())
    else:
        x0m = x0.permute(0, 2, 3, 1).reshape(B * 441, x0.shape[1])            # free view of the NHWC memory
        x1 = torch.empty((B * 100, 128), dtype=_bf16, device=dev)
        conv_gemm(0, x0m, w1f, 32, 4, 2, 21, 1, x1, bias=b1, relu=True, out_map=1, G=21, V=20, block_n=32)
    mark("f_conv1")
    y2 = torch.empty((B * 100, 64), dtype=_bf16, device=dev)
    conv_gemm(0, x1, w2f, 64, 4, 2, 10, 1, y2, bias=b2, relu=True, block_n=64)
    mark("f_conv2")
    y3 = torch.empty((B * 49, 64), dtype=_bf16, device=dev)
    conv_gemm(0, y2, w3f, 64, 9, 3, 10, 1, y3, bias=b3, relu=True, out_map=2, G=10, V=7, block_n=64)
    mark("f_conv3")
    # BN 64: at batch 512 the launcher's clusters of 2 make 64 CTAs, so the online and the target network's fc4 (two graph
    # branches) fit the SMs side by side; BN 32 is faster alone (128 CTAs) but not beside the other branch (DESIGN section 7)
    y4 = gemm_splitk_bf16(y3.view(B, 3136), w4p, bias=b4, relu=True, splits=FC4_SPLITS, block_n=64)
    mark("f_fc4")
    return y4, (x0m, x1, y2, y3)


def conv_gemm_dual(X, X2, W, W2, n_out, taps, taps_x, grid_w, out, out2, bias, bias2, out_map=0, G=0, V=0, block_n=64):
    rows, C = X.shape
    _lib.call("b2rl_conv_gemm_dual_bf16", _lib.ptr(X), _lib.ptr(X2), int(rows), int(C), _lib.ptr(W), _lib.ptr(W2), int(n_out),
              int(taps), int(taps_x), int(grid_w), 1, _lib.ptr(out), _lib.ptr(out2), out.stride(0), _lib.ptr(bias),
              _lib.ptr(bias2), 1, 0, int(out_map), int(G), int(V), int(block_n), _lib.stream())


def forward_dual(x0, packed, biases, x0_b, packed_b, biases_b):
    """``forward_only`` for TWO networks of the same shape (online on the states, target on the next states --
    DQN_agent.py:84-99) with ONE launch per layer: every kernel's grid is split between the two operand sets, so the
    per-launch fixed cost (launch, prologue, weight load, pipeline fill and drain -- most of the time of these
    3-tiles-per-CTA kernels) is paid once.  Returns (y4, saved activations of the first network, y4 of the second)."""
    w1f, w2f, _, w3f, _, w4p = packed
    v1f, v2f, _, v3f, _, v4p = packed_b
    b1, b2, b3, b4 = biases
    c1, c2, c3, c4 = biases_b
    B, dev = x0.shape[0], x0.device
    e = lambda *shape: torch.empty(shape, dtype=_bf16, device=dev)
    x0m = x0.permute(0, 2, 3, 1).reshape(B * 441, x0.shape[1])
    x0n = x0_b.permute(0, 2, 3, 1).reshape(B * 441, x0_b.shape[1])
    x1, z1 = e(B * 100, 128), e(B * 100, 128)
    conv_gemm_dual(x0m, x0n, w1f, v1f, 32, 4, 2, 21, x1, z1, b1, c1, out_map=1, G=21, V=20, block_n=32)
    y2, z2 = e(B * 100, 64), e(B * 100, 64)
    conv_gemm_dual(x1, z1, w2f, v2f, 64, 4, 2, 10, y2, z2, b2, c2, block_n=64)
    y3, z3 = e(B * 49, 64), e(B * 49, 64)
    conv_gemm_dual(y2, z2, w3f, v3f, 64, 9, 3, 10, y3, z3, b3, c3, out_map=2, G=10, V=7, block_n=64)
    n4 = w4p.shape[0]
    y4, z4 = e(B, n4), e(B, n4)
    _lib.call("b2rl_gemm_dual_bf16", _lib.ptr(y3), _lib.ptr(z3), 3136, _lib.ptr(w4p), _lib.ptr(v4p), 3136, _lib.ptr(y4),
              _lib.ptr(z4), n4, B, n4, 3136, _lib.ptr(b4), _lib.ptr(c4), 1, 0, 64, _lib.stream())
    return y4, (x0m, x1, y2, y3), z4


def _backward_unfused(ctx, gy4):
    x0m, x1, y2, y3, y4, w2d, w3d, w4p = ctx.saved_tensors
    B = y4.shape[0]
    dev = y4.device
    # ---- fc4
    g4, db4 = act_bwd_bias_grad(gy4, y4, True)                                        # [B, 512]
    y3c = y3.view(B, 3136)
    gw4p = gemm_bf16(g4, y3c, a_major="mn", b_major="mn", out_dtype=_f32, block_n=128, stream=_fork())  # [512, 3136]
    gy3c = gemm_bf16(g4, w4p, a_major="k", b_major="mn", block_n=128)                  # [B, 3136] bf16
    # ---- conv3: mask + bias grad, re-laid out from the compact 7x7 rows to the 10-grid
    g3, db3 = act_bwd_bias_grad(gy3c.view(B * 49, 64), y3, True, row_map=1, G=10, V=7, out_rows=B * 100)
    gw3p, p3 = wgrad_partials(y2, g3, 64, 9, 3, 10, stream=_fork())
    gy2 = torch.empty((B * 100, 64), dtype=_bf16, device=dev)
    conv_gemm(0, g3, w3d, 64, 9, 3, 10, -1, gy2, block_n=64)
    # ---- conv2
    g2, db2 = act_bwd_bias_grad(gy2, y2, True)                                        # rows 9 / cols 9 of gy2 are exact zeros
    gw2p, p2 = wgrad_partials(x1, g2, 64, 4, 2, 10, stream=_fork())
    gy1 = torch.empty((B * 100, 128), dtype=_bf16, device=dev)
    conv_gemm(0, g2, w2d, 128, 4, 2, 10, -1, gy1, block_n=128)
    # ---- conv1: mask + bias grad, re-laid out from space-to-depth(2) rows to the 21-grid of conv1's output positions
    g1, db1 = act_bwd_bias_grad(gy1, x1, True, row_map=2, G=21, V=20, out_rows=B * 441)
    if ctx.ring is not None:
        gw1p, p1 = wgrad_partials_ring(ctx.ring, g1, 32, stream=_fork())
        if AFTER_RING_READ is not None:
            AFTER_RING_READ(_WGRAD["stream"])
    else:
        gw1p, p1 = wgrad_partials(x0m, g1, 32, 4, 2, 21, stream=_fork())
    _join()
    return (gw1p, p1, gw2p, p2, gw3p, p3, gw4p), (db1, db2, db3, db4)


class _NatureBody(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x0, w1, b1, w2, b2, w3, b3, w4, b4, scale, packed, companion=None):
        pk = packed.tensors()
        biases = (b1.detach(), b2.detach(), b3.detach(), b4.detach())
        if companion is None:
            y4, (x0m, x1, y2, y3) = forward_only(x0, pk, *biases)
        else:                                   # (x0 of the other network, its packed weights, its biases): one launch per layer
            x0_b, packed_b, biases_b, _ = companion
            y4, (x0m, x1, y2, y3), z4 = forward_dual(x0, pk, biases, x0_b, packed_b.tensors(), biases_b)
            companion[3].append(z4)
        ctx.ring = x0m if isinstance(x0m, RingFrames) else None
        ctx.save_for_backward(y4 if ctx.ring is not None else x0m, x1, y2, y3, y4, pk[2], pk[4], pk[5])
        ctx.scale, ctx.c1 = scale, w1.shape[1]
        ctx.params = (w1, b1, w2, b2, w3, b3, w4, b4)
        return y4

    @staticmethod
    def backward(ctx, gy4):
        if FUSED_BWD and _lib.CONV_SLAB:
            (gw1p, p1, gw2p, p2, gw3p, p3, gw4p), (db1, db2, db3, db4) = _backward_fused(ctx, gy4)
        else:
            (gw1p, p1, gw2p, p2, gw3p, p3, gw4p), (db1, db2, db3, db4) = _backward_unfused(ctx, gy4)
        params = ctx.params
        sink = _sink_for(params)
        if sink is not None and FUSED_BWD and _lib.CONV_SLAB:
            if sink.split:
                sink.reduce_rest(gw1p, p1, gw2p, p2, gw3p, p3)
            else:
                if db4 is not sink.db4:
                    sink.db4.copy_(db4)
                sink.reduce(gw1p, p1, gw2p, p2, gw3p, p3, gw4p)
            mark("reduce")
            return (None,) * 12
        if all(p.grad is not None and p.grad.dtype == _f32 and p.grad.is_contiguous() for p in params):
            # accumulate straight into the .grad arena (reference layouts), one launch
            w1, b1, w2, b2, w3, b3, w4, b4 = params
            # (the kernel also sums the split-K partials of the three convolution weight gradients)
            _lib.call("b2rl_nature_unpack_grads", _lib.ptr(gw1p), _lib.ptr(gw2p), _lib.ptr(gw3p), _lib.ptr(gw4p), _lib.ptr(db1),
                      _lib.ptr(db2), _lib.ptr(db3), _lib.ptr(db4), ctx.c1, w4.shape[0], float(ctx.scale), _lib.ptr(w1.grad),
                      _lib.ptr(w2.grad), _lib.ptr(w3.grad), _lib.ptr(w4.grad), _lib.ptr(b1.grad), _lib.ptr(b2.grad),
                      _lib.ptr(b3.grad), _lib.ptr(b4.grad), p1, p2, p3, _lib.stream())
            return (None,) * 12
        gw1f, gw2f, gw3f = gw1p[:p1].sum(0), gw2p[:p2].sum(0), gw3p[:p3].sum(0)
        g1w, g2w, g3w, g4w = unpack_grads(gw1f, gw2f, gw3f, gw4p, ctx.scale, ctx.c1)
        return None, g1w, db1, g2w, db2, g3w, db3, g4w, db4, None, None, None


class dual_forward:
    """``with dual_forward(online_body, target_body, next_states):`` -- inside the context the first call of
    ``online_body`` also evaluates ``target_body(next_states)`` (one launch per layer for both networks, see
    ``forward_dual``) and the following call ``target_body(next_states)`` returns those features instead of
    recomputing them.  Used by the graph learner; everything else calls the bodies separately."""
    current = None

    def __init__(self, primary, companion, x_companion):
        self.primary, self.companion, self.x = primary, companion, x_companion
        self.features = []

    def __enter__(self):
        dual_forward.current = self
        return self

    def __exit__(self, *exc):
        dual_forward.current = None
        return False


def conv1_pair(state, next_state, w1f, b1, v1f, c1):
    """relu(conv1_w1f(state) + b1) and relu(conv1_v1f(next_state) + c1) in ONE launch (b2rl_conv1_u8_fwd_pair): the two
    ``RingFrames`` must be the same batch of one ring, ``next_state`` one ring row after ``state`` (n_step 1), so that the
    kernel reads each sample's five-frame window once.  Returns (x1, z1), conv2's space-to-depth(2) input rows."""
    s, n = state, next_state
    if not (isinstance(s, RingFrames) and isinstance(n, RingFrames)):
        raise ValueError("conv1_pair takes the RingFrames of a state and its next state")
    if n.first != s.first + 1:
        raise ValueError("conv1_pair: the next state must start one ring row after the state (n_step 1), got first %d and %d"
                         % (s.first, n.first))
    if (n.frames.data_ptr(), n.idx.data_ptr(), n.batch, n.row_bytes, n.frame_w, n.history) != \
            (s.frames.data_ptr(), s.idx.data_ptr(), s.batch, s.row_bytes, s.frame_w, s.history):
        raise ValueError("conv1_pair: the state and the next state must be the same batch of the same ring")
    e = lambda: torch.empty((s.batch * 100, 128), dtype=_bf16, device=s.device)
    x1, z1 = e(), e()
    _lib.call("b2rl_conv1_u8_fwd_pair", *s.args(), _lib.ptr(w1f), _lib.ptr(v1f), _lib.ptr(x1), _lib.ptr(z1), x1.stride(0),
              _lib.ptr(b1), _lib.ptr(c1), 1, 1, 20, _lib.stream())
    return x1, z1


class paired_conv1:
    """``with paired_conv1(online_body, target_body, state, next_state, scale):`` -- launches conv1 of the online body on
    ``state`` and of the target body on ``next_state`` as ONE kernel (``conv1_pair``) on the current stream; inside the
    context ``forward_only`` takes those outputs instead of launching conv1 for exactly these two (RingFrames, weights)
    pairs, so the two forwards may continue on different streams.  Every other conv1 (double-Q's online(next_state))
    launches its own kernel.  Used by the graph learner."""
    current = None

    def __init__(self, online, target, state, next_state, scale):
        pk, pt = packed_operands(online, scale, state.device), packed_operands(target, scale, state.device)
        x1, z1 = conv1_pair(state, next_state, pk.w1f, online.conv1.bias.detach(), pt.w1f, target.conv1.bias.detach())
        self.out = [(state, pk.w1f, x1), (next_state, pt.w1f, z1)]

    @staticmethod
    def take(x0, w1f):
        for x, w, y in paired_conv1.current.out:
            if x is x0 and w is w1f:
                return y
        return None

    def __enter__(self):
        paired_conv1.current = self
        return self

    def __exit__(self, *exc):
        paired_conv1.current = None
        return False


def packed_operands(body, scale, device):
    """The packed bf16 operands of ``body`` (built on first use), re-packed here unless the owner manages them
    (``body.auto_repack = False`` + ``body.repack(scale)`` after every parameter change)."""
    pk = getattr(body, "_packed", None)
    if pk is None:
        pk = body._packed = PackedWeights(body.conv1.in_channels, body.fc4.out_features, device)
    if getattr(body, "auto_repack", True) or pk.scale != float(scale):
        repack(body, scale)
    return pk


def nature_body(body, x0, scale):
    """``relu(fc4(flatten(relu(conv3(relu(conv2(relu(conv1(x * scale)))))))))`` for space-to-depth bf16 frames ``x0``.
    ``body`` is the NatureConvBody; its packed bf16 operands are refreshed here unless the owner manages them
    (``body.auto_repack = False`` + ``body.repack(scale)`` after every parameter change)."""
    if isinstance(x0, RingFrames):
        if not (_lib.CONV_SLAB and x0.history == 4 and x0.grid == 21 and dual_forward.current is None):
            x0 = x0.materialize()
    if not isinstance(x0, RingFrames) and not x0.is_contiguous(memory_format=torch.channels_last):
        x0 = x0.contiguous(memory_format=torch.channels_last)
    pk = packed_operands(body, scale, x0.device)
    c1, c2, c3, f4 = body.conv1, body.conv2, body.conv3, body.fc4
    d = dual_forward.current
    companion = None
    if d is not None:
        if body is d.companion and d.features and x0.data_ptr() == d.x.data_ptr():
            return d.features[0]                                   # computed alongside the primary network
        if body is d.primary and not d.features and torch.is_grad_enabled():
            o = d.companion
            xb = d.x if d.x.is_contiguous(memory_format=torch.channels_last) else d.x.contiguous(memory_format=torch.channels_last)
            pb = getattr(o, "_packed", None)
            if pb is None or getattr(o, "auto_repack", True) or pb.scale != float(scale):
                pb = repack(o, scale)
            if xb.shape == x0.shape and pb.n4 == pk.n4:
                companion = (xb, pb, tuple(m.bias.detach() for m in (o.conv1, o.conv2, o.conv3, o.fc4)), d.features)
    y4 = _NatureBody.apply(x0, c1.weight, c1.bias, c2.weight, c2.bias, c3.weight, c3.bias, f4.weight, f4.bias,
                           float(scale), pk, companion)
    if FUSED_BWD:
        mark_relu_features(y4)
    return y4


def repack(body, scale):
    pk = getattr(body, "_packed", None)
    if pk is None:
        dev = _lib.require_cuda(body.conv1.weight.device)       # the pack kernel reads the parameters in device memory
        pk = body._packed = PackedWeights(body.conv1.in_channels, body.fc4.out_features, dev)
    w = [m.weight.detach() for m in (body.conv1, body.conv2, body.conv3, body.fc4)]
    w = [t if t.is_contiguous() else t.contiguous() for t in w]
    pk.pack(w[0], w[1], w[2], w[3], scale)
    return pk
