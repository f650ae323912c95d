"""The convolution wgmma kernels of csrc/gemm.cu compared EXACTLY with a float64 reference, at the batch sizes where their
schedules actually run: several tiles per CTA (both MMA warpgroups of conv_slab_wgmma_kernel, its "MMA turn" barriers),
slab and weight-gradient rings that wrap, partial last tiles, row counts that are not multiples of 128 or 64.

Exactness by choice of data: the operands are small integers in bf16 (activations 0..7, ring pixels 0..15, weights and output
gradients in -2..2 or -1..1, integer biases), so every product is exact in fp32 and every partial sum is an integer.  While
sum |a*b| < 2**24 for every output element, fp32 accumulation is exact in ANY order -- MMA order, split-K partition, fp32
atomics, the shared-memory atomics of the bias gradient -- so each output has exactly one correct value: fp32 outputs equal
the float64 reference, bf16 outputs equal ``ref64.float().to(bfloat16)`` (one round-to-nearest-even on both sides).  The
checks are ``torch.equal``: a single wrong, missing, duplicated or stale k-tile, tap, row or stage fails.  Every case
asserts that precondition on its own data; ``test_exact_accumulation_calibration`` checks the premise itself on the plain GEMM.
One Gaussian-operand case per kernel keeps a precision regression (narrower accumulator, wrong rounding) from hiding behind
small integers.

The reference (row-shift convolution, weight gradient, epilogues, output maps) is plain torch in float64, written from the
kernel contracts in csrc/gemm.cu (``conv_gemm_impl``, ``epilogue_row``); the CPU tests at the end pin it against
``F.conv2d`` / autograd on NCHW tensors.  Every destination is pre-filled with a sentinel (bf16 -12345, NaN for fp32
partials) so stray or missing stores show up, and every bias-gradient buffer with nonzero integers so that accumulation
(not overwrite) is checked."""
import ctypes
import zlib
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

gpu = pytest.mark.gpu

F64, BF = torch.float64, torch.bfloat16
EXACT = 2.0 ** 24           # sum |a*b| below this: integer fp32 accumulation is exact in any order
SENT = -12345.0             # bf16 sentinel of the output buffers (-12352 after rounding); no case here produces it
BATCHES = [1, 37, 512, 2048]
MAX_STAGES = 6              # deepest operand ring of the slab / weight-gradient kernels
FRAME_W, HIST = 84, 4

# layer geometries on their grids: (input channels, output channels, taps, taps_x, grid width)
CONV1, CONV2, CONV3 = (64, 32, 4, 2, 21), (128, 64, 4, 2, 10), (64, 64, 9, 3, 10)


# ================================================================================================= float64 reference
def shifted(X, s):
    """Rows X[r + s]; rows outside [0, rows) read as zero (the TMA's out-of-bounds fill)."""
    out = torch.zeros_like(X)
    n = X.shape[0]
    if s >= 0:
        out[:n - s] = X[s:]
    else:
        out[-s:] = X[:n + s]
    return out


def tap_shift(t, taps_x, grid_w, sign=1):
    return sign * ((t // taps_x) * grid_w + t % taps_x)


def row_conv(X, W, taps, taps_x, grid_w, sign=1):
    """Y[r] = sum_t X[r + s_t] W_t^T with W = [n_out][taps * C] tap-major: forward (sign 1) and dgrad (sign -1)."""
    C = X.shape[1]
    Y = X.new_zeros((X.shape[0], W.shape[0]))
    for t in range(taps):
        Y.addmm_(shifted(X, tap_shift(t, taps_x, grid_w, sign)), W[:, t * C:(t + 1) * C].t())
    return Y


def row_wgrad(X, G, taps, taps_x, grid_w):
    """D[n, t*C + c] = sum_r G[r, n] X[r + s_t, c]."""
    return torch.cat([G.t() @ shifted(X, tap_shift(t, taps_x, grid_w)) for t in range(taps)], dim=1)


def out_index(out_map, rows, N, G=0, V=0, sub_c=0, device="cpu"):
    """(destination row, destination column, kept) of every element [rows][N] of a GEMM output: the row maps of
    epilogue_row.  1: G-grid -> space-to-depth(2) rows of the V x V part; 2: G-grid -> compact V x V; 3: space-to-depth(2)
    rows, columns (sub-position, channel) -> G-grid; 4: image rows, columns (position, channel) -> G-grid."""
    r = torch.arange(rows, device=device).view(-1, 1)
    n = torch.arange(N, device=device).view(1, -1)
    keep = torch.ones((rows, 1), dtype=torch.bool, device=device)
    if out_map == 0:
        drow, dcol = r, n
    elif out_map in (1, 2):
        b, rem = r // (G * G), r % (G * G)
        oy, ox = rem // G, rem % G
        keep = (oy < V) & (ox < V)
        if out_map == 1:
            h = V // 2
            drow, dcol = b * h * h + (oy // 2) * h + ox // 2, ((oy % 2) * 2 + ox % 2) * N + n
        else:
            drow, dcol = b * V * V + oy * V + ox, n
    elif out_map == 3:
        h = V // 2
        img, rem = r // (h * h), r % (h * h)
        sy, sx = rem // h, rem % h
        sub, cc = n // sub_c, n % sub_c
        drow, dcol = img * G * G + (2 * sy + sub // 2) * G + 2 * sx + sub % 2, cc
    else:
        pos, cc = n // sub_c, n % sub_c
        drow, dcol = r * G * G + (pos // V) * G + pos % V, cc
    shape = (rows, N)
    return drow.expand(shape), dcol.expand(shape), keep.expand(shape)


def place(Y, out_map, shape, fill, G=0, V=0, sub_c=0):
    """The destination buffer `shape` (pre-filled with `fill`) after the epilogue stored Y through `out_map`."""
    if fill == SENT:
        assert not bool((Y.float().to(BF) == SENT).any()), "the data produces the sentinel value"
    drow, dcol, keep = out_index(out_map, Y.shape[0], Y.shape[1], G, V, sub_c, Y.device)
    out = torch.full(shape, fill, dtype=Y.dtype, device=Y.device)
    out[drow[keep], dcol[keep]] = Y[keep]
    return out


def fold(colsum, mod):
    """Bias-gradient columns: column j goes to j % dbias_mod (dbias_mod 0: one per column)."""
    return colsum if mod == 0 else colsum.view(-1, mod).sum(0)


# --- parameter layouts (reference [Cout, Cin, kh, kw] / (c, h, w)-ordered fc4 columns) -> the tap-major GEMM operands
def pack_w1f(w1):      # [32][(ty, tx, frame, py, px)]: 8x8 / stride 4 = 2x2 taps over the space-to-depth(4) grid
    n, c = w1.shape[:2]
    return w1.reshape(n, c, 2, 4, 2, 4).permute(0, 2, 4, 1, 3, 5).reshape(n, 4 * c * 16)


def pack_w2f(w2):      # [64][(ty, tx, sy, sx, c)]: 4x4 / stride 2 = 2x2 taps over the space-to-depth(2) grid
    return w2.reshape(64, 32, 2, 2, 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(64, 512)


def pack_w2d(w2):      # [(sy, sx, c)][(ty, tx, n)]: conv2's dgrad
    return w2.reshape(64, 32, 2, 2, 2, 2).permute(3, 5, 1, 2, 4, 0).reshape(128, 256)


def pack_w3f(w3):      # [64][(dy, dx, c)]
    return w3.permute(0, 2, 3, 1).reshape(64, 576)


def pack_w3d(w3):      # [c][(dy, dx, n)]
    return w3.permute(1, 2, 3, 0).reshape(64, 576)


def pack_w4p(w4):      # fc4 columns in (h, w, c) order
    return w4.reshape(-1, 64, 7, 7).permute(0, 2, 3, 1).reshape(w4.shape[0], 3136)


def s2d4(frames):
    """[B, history, 84, 84] frames -> conv1's [B*21*21][16*history] space-to-depth(4) grid matrix, channel (frame, py, px)."""
    B, h = frames.shape[:2]
    return frames.reshape(B, h, 21, 4, 21, 4).permute(0, 2, 4, 1, 3, 5).reshape(B * 441, 16 * h)


def ring_grid(ring, idx, first):
    """conv1's input grid matrix for the frame stacks idx[b] + first .. + history - 1 of a uint8 ring [capacity][84*84]."""
    rows = (idx + first).view(-1, 1) + torch.arange(HIST, device=idx.device).view(1, -1)
    return s2d4(ring[rows].view(-1, HIST, FRAME_W, FRAME_W).to(F64))


# ================================================================================================= helpers
def bf(ref):
    """The bf16 value a kernel stores for an exact fp32 result."""
    return ref.float().to(BF)


def exact_ok(S, what):
    assert float(S.max()) < EXACT, "%s: sum |a*b| = %g breaks the exactness precondition" % (what, float(S.max()))


def assert_bf16_equal(got, ref, what):
    bad = got.float() != bf(ref).float()
    assert not bool(bad.any()), "%s: %d of %d elements differ, first at %s: got %g want %g" % (
        what, int(bad.sum()), bad.numel(), tuple(bad.nonzero()[0].tolist()), float(got[bad][0]), float(bf(ref)[bad][0]))


def assert_bf16_bounded(got, ref, S, K, what):
    """Per-element bound of an fp32 accumulation of K terms then one bf16 rounding: 2^-8 |ref| + K 2^-23 sum |a*b|."""
    err = (got.double() - ref).abs()
    tol = 2.0 ** -8 * ref.abs() + K * 2.0 ** -23 * S
    assert bool(torch.isfinite(got.float()).all()), what
    assert bool((err <= tol).all()), "%s: max excess %g" % (what, float((err - tol).max()))


def draw(gen, shape, kind, lo, hi):
    """bf16 operand: integers lo..hi ("int") or standard normals ("gauss")."""
    if kind == "gauss":
        return torch.randn(shape, generator=gen, device="cuda").to(BF)
    return torch.randint(lo, hi + 1, shape, generator=gen, device="cuda").to(BF)


def draw_mask(gen, shape):
    """Saved forward activations for the ReLU-gradient mask: 0.0, -0.0 and negative values as well as positive ones."""
    vals = torch.tensor([-2.0, -1.0, -0.0, 0.0, 1.0, 2.0], device="cuda")
    return vals[torch.randint(0, 6, shape, generator=gen, device="cuda")].to(BF)


def sentinel(shape):
    return torch.full(shape, SENT, dtype=BF, device="cuda")


def nan_partials(k, n_out, cols):
    return torch.full((k.sms, n_out, cols), float("nan"), device="cuda")


def check_partials(k, buf, n, ref, what, kind="int"):
    """Split-K partials: every CTA stored its whole block (no NaN left in partials[:n]) and nothing past it; the fp64 sum of
    partials[:n] is the reference (exact for integer data, 1e-5 normwise for Gaussian data)."""
    assert 1 <= n <= k.sms, (what, n)
    assert not bool(buf[:n].isnan().any()), "%s: a CTA left part of its partial block unwritten" % what
    assert bool(buf[n:].isnan().all()), "%s: stores past the %d partials" % (what, n)
    got = buf[:n].double().sum(0)
    if kind == "int":
        bad = got != ref
        assert not bool(bad.any()), "%s: %d of %d weight-gradient elements differ (max |err| %g)" % (
            what, int(bad.sum()), bad.numel(), float((got - ref).abs().max()))
    else:
        rel = float((got - ref).norm() / ref.norm())
        assert rel <= 1e-5, (what, rel)


# ------------------------------------------------------------------------------------------------- launcher schedules
def slab_schedule(rows, n_cta):
    """conv_slab_wgmma_kernel: CTA 0's tile count and warpgroup 1's share of it (min(SMs, tiles) CTAs, or SMs // 2 per
    operand set for the dual launch; CTA c takes tiles c, c + n_cta, ...; its i-th tile goes to warpgroup i % 2)."""
    tiles = -(-rows // 128)
    n = min(n_cta, tiles)
    per = -(-tiles // n)
    return per, per // 2


def taps_schedule(rows, ctas):
    """The weight-gradient taps kernels (conv1's, conv2 / conv3's): (CTAs = partials, 128-row k-blocks per CTA) on at most
    `ctas` CTAs, equal contiguous ranges."""
    from test_gpu_conv_taps_wgrad import BK, partition      # imported here: that module imports this one
    blocks = -(-rows // BK)
    return partition(rows, ctas), -(-blocks // min(blocks, ctas))


def gemm_k_tiles(M, N, K, block_n, sms):
    """gemm_wgmma_kernel: k-tiles that CTA 0 streams through its ring (min(SMs, tiles) CTAs over all tiles)."""
    tiles = -(-M // 128) * -(-N // block_n)
    n = min(sms, tiles)
    return -(-tiles // n) * -(-K // 64)


# ================================================================================================= fixtures
@pytest.fixture(scope="module")
def k():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import deeprl_b200 as rl
    from deeprl_b200 import _lib
    from deeprl_b200.network import nature_tc as tc
    rl.select_device(0)
    return SimpleNamespace(rl=rl, lib=_lib, tc=tc, sms=torch.cuda.get_device_properties(0).multi_processor_count)


def gen_for(*key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(key).encode()))


# ================================================================================================= 1. the premise
@gpu
@pytest.mark.parametrize("K", [64, 4096])
def test_exact_accumulation_calibration(k, K):
    """The wgmma fp32 accumulator sums bf16 integer products exactly while sum |a*b| < 2^24: half the products are large
    (positive, so the running sum climbs to ~2^23), half are small (+-1 .. +-21) and would be lost by any rounding."""
    gen = torch.Generator(device="cuda").manual_seed(K)
    M, N = 256, 128
    big = torch.randperm(K, generator=gen, device="cuda")[:K // 2]
    is_big = torch.zeros(K, dtype=torch.bool, device="cuda")
    is_big[big] = True
    sgn = lambda *s: torch.randint(0, 2, s, generator=gen, device="cuda") * 2 - 1
    a_small = torch.randint(1, 4, (M, K), generator=gen, device="cuda") * sgn(M, K)
    b_small = torch.randint(1, 8, (N, K), generator=gen, device="cuda") * sgn(N, K)
    if K == 64:      # 32 products up to 255 * 1024
        a_big = torch.randint(192, 256, (M, K), generator=gen, device="cuda")
        b_big = torch.tensor([768, 896, 1024], device="cuda")[torch.randint(0, 3, (N, K), generator=gen, device="cuda")]
    else:            # 2048 products up to 255 * 16
        a_big = torch.randint(128, 256, (M, K), generator=gen, device="cuda")
        b_big = torch.full((N, K), 16, device="cuda")
    a = torch.where(is_big, a_big, a_small).to(BF)
    b = torch.where(is_big, b_big, b_small).to(BF)
    assert torch.equal(a.double(), torch.where(is_big, a_big, a_small).double())      # the operands are exact in bf16
    assert torch.equal(b.double(), torch.where(is_big, b_big, b_small).double())
    S = a.double().abs() @ b.double().abs().t()
    exact_ok(S, "calibration")
    assert float(S.max()) > 2.0 ** 22.5, "the sums must reach about 2^23"
    got = k.rl.ops.gemm_bf16(a, b, out_dtype=torch.float32)
    ref = a.double() @ b.double().t()
    assert torch.equal(got.double(), ref), "max |err| %g" % float((got.double() - ref).abs().max())


# ================================================================================================= 2. forward (slab kernel)
FWD = {   # layer: geometry, output map, G, V, block_n, output columns, output rows per image
    "conv1": (CONV1, 1, 21, 20, 32, 128, 100),
    "conv2": (CONV2, 0, 0, 0, 64, 64, 100),
    "conv3": (CONV3, 2, 10, 7, 64, 64, 49),
}


def fwd_operands(layer, B, kind, gen):
    (C, n, taps, tx, gw), _, _, _, _, _, _ = FWD[layer]
    X = draw(gen, (B * gw * gw, C), kind, 0, 7)
    W = draw(gen, (n, taps * C), kind, -2, 2)
    b = draw(gen, (n,), kind, -30, 30).float()
    return X, W, b


def fwd_reference(layer, B, X, W, b):
    (C, n, taps, tx, gw), out_map, G, V, _, ncols, per_img = FWD[layer]
    v = row_conv(X.double(), W.double(), taps, tx, gw) + b.double()
    S = row_conv(X.double().abs(), W.double().abs(), taps, tx, gw) + b.double().abs()
    ref = place(torch.relu(v), out_map, (B * per_img, ncols), SENT, G, V)
    return ref, S, taps * C + 1


def fwd_call(k, layer, X, W, b, out):
    (C, n, taps, tx, gw), out_map, G, V, bn, _, _ = FWD[layer]
    k.tc.conv_gemm(0, X, W, n, taps, tx, gw, 1, out, bias=b, relu=True, out_map=out_map, G=G, V=V, block_n=bn)


@gpu
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("layer", list(FWD))
def test_forward_exact(k, layer, B):
    """conv_gemm forward, bias + ReLU + output map, with forward_only's arguments; every output row, garbage grid rows too."""
    gen = gen_for("fwd", layer, B)
    X, W, b = fwd_operands(layer, B, "int", gen)
    ref, S, _ = fwd_reference(layer, B, X, W, b)
    exact_ok(S, layer)
    out = sentinel(ref.shape)
    fwd_call(k, layer, X, W, b, out)
    torch.cuda.synchronize()
    assert_bf16_equal(out, ref, "%s forward B=%d" % (layer, B))


@gpu
@pytest.mark.parametrize("B", [37, 512])
@pytest.mark.parametrize("layer", list(FWD))
def test_forward_dual_exact(k, layer, B):
    """conv_gemm_dual (forward_dual): half the CTAs per operand set, different data in the two sets, both outputs exact."""
    (C, n, taps, tx, gw), out_map, G, V, bn, _, _ = FWD[layer]
    gen = gen_for("dual", layer, B)
    ops = [fwd_operands(layer, B, "int", gen) for _ in range(2)]
    refs = [fwd_reference(layer, B, *o) for o in ops]
    for ref, S, _ in refs:
        exact_ok(S, layer)
    outs = [sentinel(r[0].shape) for r in refs]
    (X, W, b), (X2, W2, b2) = ops
    k.tc.conv_gemm_dual(X, X2, W, W2, n, taps, tx, gw, outs[0], outs[1], b, b2, out_map=out_map, G=G, V=V, block_n=bn)
    torch.cuda.synchronize()
    for i in range(2):
        assert_bf16_equal(outs[i], refs[i][0], "%s dual forward B=%d, operand set %d" % (layer, B, i))


# ================================================================================================= 3. dgrad with the fused epilogues
DGRAD = ["conv3", "conv2", "fc4"]


def dgrad_case(k, layer, B, kind, gen, dbias_mod=None):
    """One dgrad GEMM with its fused epilogue, called as _backward_fused calls it, and its float64 reference: output and
    reference buffers, sum |a*b| per GEMM element, K, bias-gradient buffer, its reference and its sum of |terms|."""
    lib = k.lib
    if layer == "conv3":       # conv3 dgrad on the 10-grid, masked by relu(conv2), bias gradient of conv2
        mod = 64 if dbias_mod is None else dbias_mod
        g = draw(gen, (B * 100, 64), kind, -1, 1)
        w = draw(gen, (64, 576), kind, -2, 2)
        mask = draw_mask(gen, (B * 100, 64))
        v, S, K = row_conv(g.double(), w.double(), 9, 3, 10, -1), row_conv(g.double().abs(), w.double().abs(), 9, 3, 10, -1), 576
        out_map, out_shape, G, V, sub_c = 0, (B * 100, 64), 0, 0, 0

        def call(out, e):
            lib.call("b2rl_conv_gemm_bwd_bf16", lib.ptr(g), B * 100, 64, lib.ptr(w), 64, 9, 3, 10, lib.ptr(out), 64, 0, 0, 0,
                     ctypes.byref(e), 64, lib.stream())
    elif layer == "conv2":     # conv2 dgrad: space-to-depth(2) rows -> conv1's 21-grid, masked by relu(conv1)
        mod = 32
        g = draw(gen, (B * 100, 64), kind, -1, 1)
        w = draw(gen, (128, 256), kind, -2, 2)
        mask = draw_mask(gen, (B * 100, 128))
        v, S, K = row_conv(g.double(), w.double(), 4, 2, 10, -1), row_conv(g.double().abs(), w.double().abs(), 4, 2, 10, -1), 256
        out_map, out_shape, G, V, sub_c = 3, (B * 441, 32), 21, 20, 32

        def call(out, e):
            lib.call("b2rl_conv_gemm_bwd_bf16", lib.ptr(g), B * 100, 64, lib.ptr(w), 128, 4, 2, 10, lib.ptr(out), 32, 3, 21, 20,
                     ctypes.byref(e), 128, lib.stream())
    else:                      # fc4 dgrad: per-image positions -> conv3's 10-grid, masked by relu(conv3)
        mod, n4 = 64, 512
        g = draw(gen, (B, n4), kind, -1, 1)
        w = draw(gen, (n4, 3136), kind, -2, 2)
        mask = draw_mask(gen, (B, 3136))
        v, S, K = g.double() @ w.double(), g.double().abs() @ w.double().abs(), n4
        out_map, out_shape, G, V, sub_c = 4, (B * 100, 64), 10, 7, 64

        def call(out, e):
            lib.call("b2rl_gemm_bwd_bf16", lib.ptr(g), g.stride(0), lib.ptr(w), 1, w.stride(0), lib.ptr(out), 64, B, 3136, n4, 4,
                     10, 7, ctypes.byref(e), 128, lib.stream())
    keep = mask.double() > 0
    vm = torch.where(keep, v, torch.zeros_like(v))
    ref = place(vm, out_map, out_shape, SENT, G, V, sub_c)
    # dbias_mod 0 writes one bias per column: a buffer longer than N shows stray stores past it
    db0 = torch.randint(-1000, 1001, (128 if mod == 0 else mod,), generator=gen, device="cuda").float()
    db_ref, db_abs = db0.double(), db0.double().abs()
    db_ref[:v.shape[1] if mod == 0 else mod] += fold(vm.sum(0), mod)
    db_abs[:v.shape[1] if mod == 0 else mod] += fold(torch.where(keep, v.abs(), torch.zeros_like(v)).sum(0), mod)
    out = sentinel(out_shape)
    db = db0.clone()
    e = lib.bwd_epilogue(mask, db, mod, sub_c)
    call(out, e)
    torch.cuda.synchronize()
    return SimpleNamespace(out=out, ref=ref, S=S, K=K, db=db, db_ref=db_ref, db_abs=db_abs, mod=mod, out_map=out_map)


@gpu
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("layer", DGRAD)
def test_dgrad_epilogue_exact(k, layer, B):
    """dgrad GEMM + ReLU-gradient mask + bias gradient (dbias_mod 64 / 32 / 64) + scatter map, with _backward_fused's
    arguments.  Rows / columns of the grid that no tile covers keep the sentinel; the bias gradient is ADDED to the
    buffer's integers."""
    c = dgrad_case(k, layer, B, "int", gen_for("dgrad", layer, B))
    exact_ok(c.S, layer)
    exact_ok(c.db_abs, layer + " bias gradient")
    assert_bf16_equal(c.out, c.ref, "%s dgrad B=%d" % (layer, B))
    if c.out_map == 3:         # row / column 20 of the 21-grid: never stored
        grid = c.out.view(B, 21, 21, 32)
        assert bool((grid[:, 20] == SENT).all() and (grid[:, :, 20] == SENT).all())
    if c.out_map == 4:         # rows / columns 7-9 of the 10-grid: never stored
        grid = c.out.view(B, 10, 10, 64)
        assert bool((grid[:, 7:] == SENT).all() and (grid[:, :, 7:] == SENT).all())
    assert torch.equal(c.db.double(), c.db_ref), "%s bias gradient B=%d: max |err| %g" % (
        layer, B, float((c.db.double() - c.db_ref).abs().max()))


@gpu
@pytest.mark.parametrize("B", [37, 512])
def test_conv3_dgrad_per_column_bias_gradient(k, B):
    """dbias_mod 0: one bias per output column, added straight to global memory (no shared-memory fold)."""
    c = dgrad_case(k, "conv3", B, "int", gen_for("dgrad0", B), dbias_mod=0)
    exact_ok(c.S, "conv3")
    exact_ok(c.db_abs, "conv3 bias gradient")
    assert_bf16_equal(c.out, c.ref, "conv3 dgrad B=%d" % B)
    assert torch.equal(c.db[:64].double(), c.db_ref[:64])
    assert torch.equal(c.db[64:].double(), c.db_ref[64:]), "columns past N must not be touched"


# ================================================================================================= 4. weight gradients
WGRAD = {   # layer: geometry (conv1-3 as _backward_fused calls wgrad_partials)
    "conv1": CONV1, "conv2": CONV2, "conv3": CONV3,                 # the taps kernels: one partial per CTA
    "odd96": (64, 96, 9, 3, 10), "odd128": (64, 128, 9, 3, 10),     # the tap-addressing GEMM: one atomic partial
    "conv1_c8": (128, 32, 4, 2, 21),                                # conv1 of NatureConvBody(in_channels=8): likewise
}
TAPS_WGRAD = ("conv1", "conv2", "conv3")


def wgrad_case(k, layer, B, kind, gen):
    """nature_tc.wgrad_partials on the layer's geometry, its partial buffer NaN-filled before the kernel runs."""
    C, n, taps, tx, gw = WGRAD[layer]
    rows = B * gw * gw
    X = draw(gen, (rows, C), kind, 0, 7)
    Gr = draw(gen, (rows, n), kind, -1, 1)
    empty = torch.empty
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(torch, "empty", lambda *a, **kw: empty(*a, **kw).fill_(float("nan")))
        buf, cnt = k.tc.wgrad_partials(X, Gr, n, taps, tx, gw)
    torch.cuda.synchronize()
    ref = row_wgrad(X.double(), Gr.double(), taps, tx, gw)
    S = row_wgrad(X.double().abs(), Gr.double().abs(), taps, tx, gw)
    return buf, cnt, ref, S


@gpu
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("layer", list(WGRAD))
def test_wgrad_dispatch_exact(k, layer, B):
    """nature_tc.wgrad_partials, the dispatch the backward pass calls: conv1-3 on their taps kernels, every other geometry on
    the tap-addressing GEMM.  The partials, summed in fp64, equal the reference; the partial count is the taps launchers'
    partition over one CTA per SM, or 1 (one atomically accumulated partial)."""
    buf, n, ref, S = wgrad_case(k, layer, B, "int", gen_for("wgrad", layer, B))
    exact_ok(S, layer)
    gw = WGRAD[layer][4]
    assert n == (taps_schedule(B * gw * gw, k.sms)[0] if layer in TAPS_WGRAD else 1), (layer, B, n)
    check_partials(k, buf, n, ref, "%s wgrad B=%d" % (layer, B))


@gpu
@pytest.mark.parametrize("layer", ["conv1", "conv2", "conv3", "odd96"])
def test_wgrad_dispatch_gaussian(k, layer):
    """Batch 512 with Gaussian bf16 operands through nature_tc.wgrad_partials: the summed partials within 1e-5 normwise of
    float64."""
    case = "wgrad_" + layer
    buf, n, ref, _ = wgrad_case(k, layer, 512, "gauss", gen_for("gauss", case))
    check_partials(k, buf, n, ref, case, kind="gauss")


# ================================================================================================= 5. K1: conv1 from the uint8 ring
def k1_case(k, B, n_step, which, kind, gen):
    cap = 700
    ring = torch.randint(0, 256 if kind == "gauss" else 16, (cap, FRAME_W * FRAME_W), dtype=torch.uint8, generator=gen,
                         device="cuda")
    hi = cap - 1 - n_step
    idx = torch.randint(3, hi + 1, (B,), generator=gen, device="cuda")
    if B > 1:
        idx[B // 2] = idx[0]                       # duplicates in one batch
        idx[1] = 3                                 # oldest stacked frame of the state at ring row 0
        idx[B // 2 + 1] = hi                       # newest stacked frame of the next state at the last ring row
    else:
        idx[0] = 3 if which == 0 else hi
    first = which * n_step - (HIST - 1)
    rf = k.tc.RingFrames(ring, idx, first, FRAME_W * FRAME_W, FRAME_W, HIST)
    x0 = ring_grid(ring, idx, first)
    return rf, x0


@gpu
@pytest.mark.parametrize("which", [0, 1], ids=["state", "next_state"])
@pytest.mark.parametrize("n_step", [1, 3])
@pytest.mark.parametrize("B", [1, 37, 512])
def test_k1_from_ring_exact(k, B, n_step, which):
    """b2rl_conv1_u8_fwd and b2rl_conv1_u8_wgrad_partials against the fp64 reference built from the ring's own frames
    (not against the materialising kernels, which share the slab pipeline)."""
    lib = k.lib
    gen = gen_for("k1", B, n_step, which)
    rf, x0 = k1_case(k, B, n_step, which, "int", gen)
    w1f = draw(gen, (32, 256), "int", -1, 1)
    b1 = draw(gen, (32,), "int", -20, 20).float()
    v = row_conv(x0, w1f.double(), 4, 2, 21) + b1.double()
    exact_ok(row_conv(x0, w1f.double().abs(), 4, 2, 21) + b1.double().abs(), "K1 forward")
    ref = place(torch.relu(v), 1, (B * 100, 128), SENT, 21, 20)
    x1 = sentinel((B * 100, 128))
    lib.call("b2rl_conv1_u8_fwd", *rf.args(), lib.ptr(w1f), 32, lib.ptr(x1), x1.stride(0), lib.ptr(b1), 1, 1, 20, lib.stream())
    g1 = draw(gen, (B * 441, 32), "int", -1, 1)
    buf = nan_partials(k, 32, 256)
    cnt = ctypes.c_int32(0)
    lib.call("b2rl_conv1_u8_wgrad_partials", *rf.args(), lib.ptr(g1), 32, lib.ptr(buf), ctypes.byref(cnt), lib.stream())
    torch.cuda.synchronize()
    assert_bf16_equal(x1, ref, "K1 forward B=%d n_step=%d" % (B, n_step))
    wref = row_wgrad(x0, g1.double(), 4, 2, 21)
    exact_ok(row_wgrad(x0, g1.double().abs(), 4, 2, 21), "K1 wgrad")
    check_partials(k, buf, int(cnt.value), wref, "K1 wgrad B=%d n_step=%d" % (B, n_step))


# ================================================================================================= 6. Gaussian operands
GAUSS = ["fwd_conv1", "fwd_conv2", "fwd_conv3", "dgrad_conv3", "dgrad_conv2", "dgrad_fc4", "k1"]


@gpu
@pytest.mark.parametrize("case", GAUSS)
def test_gaussian_operands(k, case):
    """Batch 512 with Gaussian bf16 operands: |got - ref| <= 2^-8 |ref| + K 2^-23 sum|a*b| per element on forward and dgrad
    outputs, 1e-5 normwise on K1's summed weight-gradient partials (the other weight gradients: test_wgrad_dispatch_gaussian)."""
    B = 512
    gen = gen_for("gauss", case)
    kind, layer = case.split("_", 1) if "_" in case else (case, None)
    if kind == "fwd":
        X, W, b = fwd_operands(layer, B, "gauss", gen)
        ref, S, K = fwd_reference(layer, B, X, W, b)
        out = sentinel(ref.shape)
        fwd_call(k, layer, X, W, b, out)
        torch.cuda.synchronize()
        assert_bf16_bounded(out, ref, place(S, FWD[layer][1], ref.shape, 0.0, FWD[layer][2], FWD[layer][3]), K, case)
    elif kind == "dgrad":
        c = dgrad_case(k, layer, B, "gauss", gen)
        G, V, sub_c = {0: (0, 0, 0), 3: (21, 20, 32), 4: (10, 7, 64)}[c.out_map]
        S = place(c.S, c.out_map, c.ref.shape, 0.0, G, V, sub_c)
        written = place(torch.ones_like(c.S), c.out_map, c.ref.shape, 0.0, G, V, sub_c) > 0
        assert_bf16_bounded(c.out[written], c.ref[written], S[written], c.K, case)
        assert bool((c.out[~written] == SENT).all()), case
    else:
        lib = k.lib
        rf, x0 = k1_case(k, B, 1, 0, "gauss", gen)
        w1f = draw(gen, (32, 256), "gauss", 0, 0) * 0.01
        b1 = torch.randn(32, generator=gen, device="cuda")
        v = row_conv(x0, w1f.double(), 4, 2, 21) + b1.double()
        S = place(row_conv(x0, w1f.double().abs(), 4, 2, 21) + b1.double().abs(), 1, (B * 100, 128), 0.0, 21, 20)
        x1 = sentinel((B * 100, 128))
        lib.call("b2rl_conv1_u8_fwd", *rf.args(), lib.ptr(w1f), 32, lib.ptr(x1), x1.stride(0), lib.ptr(b1), 1, 1, 20,
                 lib.stream())
        g1 = draw(gen, (B * 441, 32), "gauss", 0, 0)
        buf = nan_partials(k, 32, 256)
        cnt = ctypes.c_int32(0)
        lib.call("b2rl_conv1_u8_wgrad_partials", *rf.args(), lib.ptr(g1), 32, lib.ptr(buf), ctypes.byref(cnt), lib.stream())
        torch.cuda.synchronize()
        assert_bf16_bounded(x1, place(torch.relu(v), 1, (B * 100, 128), SENT, 21, 20), S, 257, "K1 forward")
        check_partials(k, buf, int(cnt.value), row_wgrad(x0, g1.double(), 4, 2, 21), "K1 wgrad", kind="gauss")


# ================================================================================================= 7. tap-addressing fallback
@gpu
def test_tap_addressing_fallback_exact(k):
    """set_conv_slab(0): forward, dgrad and weight gradients on the tap-addressing gemm_wgmma_kernel (the path of any layer
    shape the slab kernel is not instantiated for), exact at batch 512."""
    B = 512
    k.lib.set_conv_slab(0)
    try:
        for layer in FWD:
            X, W, b = fwd_operands(layer, B, "int", gen_for("tap", layer))
            ref, S, _ = fwd_reference(layer, B, X, W, b)
            exact_ok(S, layer)
            out = sentinel(ref.shape)
            fwd_call(k, layer, X, W, b, out)
            torch.cuda.synchronize()
            assert_bf16_equal(out, ref, "%s forward, tap addressing" % layer)
        for layer in DGRAD:
            c = dgrad_case(k, layer, B, "int", gen_for("tap-dgrad", layer))
            exact_ok(c.S, layer)
            assert_bf16_equal(c.out, c.ref, "%s dgrad, tap addressing" % layer)
            assert torch.equal(c.db.double(), c.db_ref), layer
        for layer in ("conv1", "conv2", "conv3"):
            C, n, taps, tx, gw = WGRAD[layer]
            gen = gen_for("tap-wgrad", layer)
            X = draw(gen, (B * gw * gw, C), "int", 0, 7)
            Gr = draw(gen, (B * gw * gw, n), "int", -1, 1)
            parts, p = k.tc.wgrad_partials(X, Gr, n, taps, tx, gw)          # one atomically accumulated "partial"
            torch.cuda.synchronize()
            exact_ok(row_wgrad(X.double().abs(), Gr.double().abs(), taps, tx, gw), layer)
            assert p == 1 and torch.equal(parts[0].double(), row_wgrad(X.double(), Gr.double(), taps, tx, gw)), layer
    finally:
        k.lib.set_conv_slab(2)


# ================================================================================================= 8. teacher-forced body chain
def chain_params(gen, n4=512):
    """Sparse integer weights (1 in 3 nonzero, +-1) and biases in -1..1: with 0/1 frames and a sparse output gradient every
    layer of the body stays inside the exactness precondition up to batch 512 (about half of it at the weight gradients), and
    about half of every ReLU passes."""
    def w(*s):
        v = torch.randint(-1, 2, s, generator=gen, device="cuda").float()
        return v * (torch.randint(0, 2, s, generator=gen, device="cuda") == 0)
    b = lambda n: torch.randint(-1, 2, (n,), generator=gen, device="cuda").float()
    return (w(32, 4, 8, 8), w(64, 32, 4, 4), w(64, 64, 3, 3), w(n4, 3136)), (b(32), b(64), b(64), b(n4))


def chain_frames(gen, B):
    f = torch.randint(0, 2, (B, 4, FRAME_W, FRAME_W), generator=gen, device="cuda").double()
    return s2d4(f).to(BF).view(B, 21, 21, 64).permute(0, 3, 1, 2)        # channels_last [B, 64, 21, 21]


def packed_exact(tc, ws):
    packed = tc.pack_weights(*ws, 1.0)
    mine = (pack_w1f(ws[0]), pack_w2f(ws[1]), pack_w2d(ws[1]), pack_w3f(ws[2]), pack_w3d(ws[2]), pack_w4p(ws[3]))
    for name, got, want in zip(("w1f", "w2f", "w2d", "w3f", "w3d", "w4p"), packed, mine):
        assert torch.equal(got.double(), want.double()), "b2rl_nature_pack_weights: %s" % name
    return packed


def forward_reference(x0m, packed, biases, B, acts=None):
    """One layer at a time, in fp64, then the bf16 rounding each kernel's store applies.  With `acts` = the kernels' own
    (x1, y2, y3) every layer starts from the kernel's previous output (teacher forcing)."""
    w1f, w2f, _, w3f, _, w4p = (p.double() for p in packed)
    b1, b2, b3, b4 = (b.double() for b in biases)
    out, S = [], []
    x = x0m.double()
    for i, (w, b, geo, om, G, V, shape) in enumerate((
            (w1f, b1, CONV1, 1, 21, 20, (B * 100, 128)), (w2f, b2, CONV2, 0, 0, 0, (B * 100, 64)),
            (w3f, b3, CONV3, 2, 10, 7, (B * 49, 64)))):
        _, _, taps, tx, gw = geo
        S.append(row_conv(x.abs(), w.abs(), taps, tx, gw) + b.abs())
        out.append(bf(place(torch.relu(row_conv(x, w, taps, tx, gw) + b), om, shape, 0.0, G, V)))
        x = (acts[i] if acts is not None else out[-1]).double()
    x = x.view(B, 3136)
    S.append(x.abs() @ w4p.abs().t() + b4.abs())
    out.append(bf(torch.relu(x @ w4p.t() + b4)))
    return out, S


@gpu
@pytest.mark.parametrize("B", [37, 512])
def test_body_chain_teacher_forced(k, monkeypatch, B):
    """forward_only and _backward_fused on integer weights packed with scale 1.0: each layer (fc4 included) equals the
    reference applied to the kernel's own previous-layer output, and so do the weight and bias gradients -- this pins the
    call sites of nature_tc (arguments, buffers, maps), not only the kernels."""
    tc = k.tc
    gen = gen_for("chain", B)
    ws, biases = chain_params(gen)
    packed = packed_exact(tc, ws)
    x0 = chain_frames(gen, B)
    y4, (x0m, x1, y2, y3) = tc.forward_only(x0, packed, *biases)
    torch.cuda.synchronize()
    want, S = forward_reference(x0m, packed, biases, B, acts=(x1, y2, y3))
    for name, got, ref, s in zip(("conv1", "conv2", "conv3", "fc4"), (x1, y2, y3, y4), want, S):
        exact_ok(s, name)
        assert torch.equal(got, ref), "forward_only: %s differs in %d elements" % (name, int((got != ref).sum()))
    assert int((y3 > 0).sum()) > y3.numel() // 8 and int((y4 > 0).sum()) > y4.numel() // 8, "ReLUs must pass enough"
    # ---- backward, in _backward_fused's order; the dgrad outputs are seen where they enter the weight-gradient GEMMs
    seen = []
    real = tc.wgrad_partials

    def recording(X, G_rows, *a, **kw):
        seen.append(G_rows.clone())
        return real(X, G_rows, *a, **kw)

    monkeypatch.setattr(tc, "wgrad_partials", recording)
    gy4 = torch.randint(-1, 2, y4.shape, generator=gen, device="cuda")
    gy4 = (gy4 * (torch.randint(0, 8, y4.shape, generator=gen, device="cuda") == 0)).to(BF)      # 1 in 12 nonzero
    ctx = SimpleNamespace(saved_tensors=(x0m, x1, y2, y3, y4, packed[2], packed[4], packed[5]), params=(None,) * 8, ring=None)
    (gw1p, p1, gw2p, p2, gw3p, p3, gw4p), (db1, db2, db3, db4) = tc._backward_fused(ctx, gy4)
    torch.cuda.synchronize()
    g3, g2, g1 = seen
    d = lambda t: t.double()
    zero = lambda v, m: torch.where(d(m) > 0, v, torch.zeros_like(v))
    y3c = y3.view(B, 3136)
    g4 = zero(d(gy4), y4)
    assert torch.equal(d(db4), g4.sum(0)), "fc4 bias gradient"
    exact_ok(g4.abs().t() @ d(y3c).abs(), "fc4 wgrad")
    assert torch.equal(d(gw4p), g4.t() @ d(y3c)), "fc4 weight gradient"
    steps = (   # (dgrad output seen, its reference from the previous kernel output, sum |a*b|, bias gradient, dbias_mod)
        ("g3 (fc4 dgrad)", g3, zero(g4 @ d(packed[5]), y3c), g4.abs() @ d(packed[5]).abs(), 4, (10, 7, 64), db3, 64),
        ("g2 (conv3 dgrad)", g2, zero(row_conv(d(g3), d(packed[4]), 9, 3, 10, -1), y2),
         row_conv(d(g3).abs(), d(packed[4]).abs(), 9, 3, 10, -1), 0, (0, 0, 0), db2, 64),
        ("g1 (conv2 dgrad)", g1, zero(row_conv(d(g2), d(packed[2]), 4, 2, 10, -1), x1),
         row_conv(d(g2).abs(), d(packed[2]).abs(), 4, 2, 10, -1), 3, (21, 20, 32), db1, 32),
    )
    for name, got, vm, s, om, (G, V, sub_c), db, mod in steps:
        exact_ok(s, name)
        assert torch.equal(got, bf(place(vm, om, got.shape, 0.0, G, V, sub_c))), "%s gradient" % name
        assert torch.equal(d(db), fold(vm.sum(0), mod)), "%s bias gradient" % name
    for name, parts, n, X, Gr, geo in (("conv3", gw3p, p3, y2, g3, CONV3), ("conv2", gw2p, p2, x1, g2, CONV2),
                                       ("conv1", gw1p, p1, x0m, g1, CONV1)):
        _, _, taps, tx, gw = geo
        exact_ok(row_wgrad(d(X).abs(), d(Gr).abs(), taps, tx, gw), name + " wgrad")
        assert torch.equal(parts[:n].double().sum(0), row_wgrad(d(X), d(Gr), taps, tx, gw)), "%s weight gradient" % name


@gpu
@pytest.mark.parametrize("B", [37, 512])
def test_body_chain_dual(k, B):
    """forward_dual: two networks with different integer weights and frames, one launch per layer; the first network's
    layers teacher-forced as above, the second's features against its own exact layer-by-layer reference."""
    tc = k.tc
    gen = gen_for("chain-dual", B)
    nets = []
    for _ in range(2):
        ws, biases = chain_params(gen)
        nets.append((chain_frames(gen, B), packed_exact(tc, ws), biases))
    (x0, pa, ba), (x0b, pb, bb) = nets
    y4, (x0m, x1, y2, y3), z4 = tc.forward_dual(x0, pa, ba, x0b, pb, bb)
    torch.cuda.synchronize()
    want, S = forward_reference(x0m, pa, ba, B, acts=(x1, y2, y3))
    for name, got, ref, s in zip(("conv1", "conv2", "conv3", "fc4"), (x1, y2, y3, y4), want, S):
        exact_ok(s, name)
        assert torch.equal(got, ref), "forward_dual, first network: %s" % name
    x0bm = x0b.permute(0, 2, 3, 1).reshape(B * 441, 64)
    want_b, S_b = forward_reference(x0bm, pb, bb, B)
    for s in S_b:
        exact_ok(s, "second network")
    assert torch.equal(z4, want_b[3]), "forward_dual, second network's features"


# ================================================================================================= 9. the schedules are reached
@gpu
def test_batches_reach_the_schedules(k):
    """At the batches above, for every instantiation: some case gives warpgroup 1 of the slab kernel at least two tiles of a
    CTA (ping-pong and MMA-turn barriers run), and some case streams more than MAX_STAGES tiles or k-tiles through one CTA
    (every ring wraps, whatever stage count the launcher picks)."""
    sms = k.sms
    slab = {   # instantiation: (rows per image, CTAs per operand set, batches)
        "slab<32,F,F,2,2,1> conv1 fwd": (441, sms, BATCHES), "slab<64,F,F,2,2,2> conv2 fwd": (100, sms, BATCHES),
        "slab<64,F,F,3,3,1> conv3 fwd": (100, sms, BATCHES), "slab<64,T,F,3,3,1> conv3 dgrad": (100, sms, BATCHES),
        "slab<128,T,F,2,2,1> conv2 dgrad": (100, sms, BATCHES), "slab<32,F,T,2,2,1> K1 fwd": (441, sms, [1, 37, 512]),
        "dual conv1": (441, sms // 2, [37, 512]), "dual conv2": (100, sms // 2, [37, 512]),
        "dual conv3": (100, sms // 2, [37, 512]),
    }
    for name, (per_img, n_cta, batches) in slab.items():
        sched = [slab_schedule(B * per_img, n_cta) for B in batches]
        assert any(wg1 >= 2 for _, wg1 in sched), (name, sched)
        assert any(per > MAX_STAGES for per, _ in sched), (name, sched)
    assert gemm_k_tiles(2048, 3136, 512, 128, sms) > MAX_STAGES, "gemm<128,4,EXT> fc4 dgrad"
    for name in TAPS_WGRAD:
        gw = WGRAD[name][4]
        assert any(taps_schedule(B * gw * gw, sms)[1] > MAX_STAGES for B in (512, 2048)), name
        bench_ctas = sms if name == "conv1" else k.tc.SIDE_CTAS     # conv2 / conv3 run on the side branch's CTAs
        assert taps_schedule(512 * gw * gw, bench_ctas)[1] > MAX_STAGES, name + ": the bench batch wraps the ring"
    assert taps_schedule(512 * 441, sms)[1] > 4, "K1 wgrad (four operand stages)"


# ================================================================================================= 10. CPU: the reference itself
def test_reference_matches_conv2d_chain():
    """The row-shift forward / dgrad / wgrad formulas, the parameter packers and output maps 1-4 equal F.conv2d and autograd
    in float64 on NCHW tensors through the whole NatureConvBody geometry (conv1 8x8/4, conv2 4x4/2, conv3 3x3, fc4)."""
    torch.manual_seed(0)
    B = 2
    frames = torch.randn(B, 4, FRAME_W, FRAME_W, dtype=F64)
    w1, w2, w3 = (torch.randn(s, dtype=F64, requires_grad=True) for s in ((32, 4, 8, 8), (64, 32, 4, 4), (64, 64, 3, 3)))
    w4 = torch.randn(16, 3136, dtype=F64, requires_grad=True)
    a1 = F.conv2d(frames, w1, stride=4)
    a2 = F.conv2d(a1, w2, stride=2)
    a3 = F.conv2d(a2, w3)
    a4 = a3.flatten(1) @ w4.t()
    for a in (a1, a2, a3):
        a.retain_grad()
    gy4 = torch.randn_like(a4)
    a4.backward(gy4)
    nhwc = lambda a: a.detach().permute(0, 2, 3, 1)
    # forward: each layer's rows on its grid; the output maps feed the next layer
    x0 = s2d4(frames)
    x1 = place(row_conv(x0, pack_w1f(w1.detach()), 4, 2, 21), 1, (B * 100, 128), 0.0, 21, 20)
    y2 = row_conv(x1, pack_w2f(w2.detach()), 4, 2, 10)
    y3 = place(row_conv(y2, pack_w3f(w3.detach()), 9, 3, 10), 2, (B * 49, 64), 0.0, 10, 7)
    close = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-9)
    close(x1.view(B, 10, 10, 2, 2, 32).permute(0, 1, 3, 2, 4, 5).reshape(B, 20, 20, 32), nhwc(a1))
    close(y2.view(B, 10, 10, 64)[:, :9, :9], nhwc(a2))
    close(y3.view(B, 7, 7, 64), nhwc(a3))
    close(y3.view(B, 3136) @ pack_w4p(w4.detach()).t(), a4.detach())
    # dgrad: fc4 (map 4) -> conv3 (sign -1) -> conv2 (sign -1, map 3), on the grids
    g3 = place(gy4 @ pack_w4p(w4.detach()), 4, (B * 100, 64), 0.0, 10, 7, 64)
    close(g3.view(B, 10, 10, 64)[:, :7, :7], nhwc(a3.grad))
    g2 = row_conv(g3, pack_w3d(w3.detach()), 9, 3, 10, -1)
    close(g2.view(B, 10, 10, 64)[:, :9, :9], nhwc(a2.grad))
    g1 = place(row_conv(g2, pack_w2d(w2.detach()), 4, 2, 10, -1), 3, (B * 441, 32), 0.0, 21, 20, 32)
    close(g1.view(B, 21, 21, 32)[:, :20, :20], nhwc(a1.grad))
    # wgrad (the garbage grid rows carry zero gradient, as in the product)
    close(row_wgrad(x0, g1, 4, 2, 21), pack_w1f(w1.grad))
    close(row_wgrad(x1, g2, 4, 2, 10), pack_w2f(w2.grad))
    close(row_wgrad(y2, g3, 9, 3, 10), pack_w3f(w3.grad))
    close(gy4.t() @ y3.view(B, 3136), pack_w4p(w4.grad))


@pytest.mark.parametrize("out_map", [0, 1, 2, 3, 4])
def test_output_maps_are_permutations(out_map):
    """Each output map sends the elements it keeps to distinct destinations, and those are exactly the destination set the
    sentinel checks expect: all of x1 / y3 for maps 1 / 2, the 20 x 20 part of the 21-grid for map 3, the 7 x 7 part of the
    10-grid for map 4."""
    B = 3
    rows, N, G, V, sub_c, shape = {0: (B * 100, 64, 0, 0, 0, (B * 100, 64)), 1: (B * 441, 32, 21, 20, 0, (B * 100, 128)),
                                   2: (B * 100, 64, 10, 7, 0, (B * 49, 64)), 3: (B * 100, 128, 21, 20, 32, (B * 441, 32)),
                                   4: (B, 3136, 10, 7, 64, (B * 100, 64))}[out_map]
    drow, dcol, keep = out_index(out_map, rows, N, G, V, sub_c)
    flat = (drow[keep] * shape[1] + dcol[keep]).cpu()
    assert int(flat.unique().numel()) == int(flat.numel()), "two elements stored to one destination"
    hit = torch.zeros(shape[0] * shape[1], dtype=torch.bool)
    hit[flat] = True
    expect = torch.ones(shape, dtype=torch.bool)
    if out_map in (3, 4):
        expect = torch.zeros((B, G, G, shape[1]), dtype=torch.bool)
        expect[:, :V, :V] = True
    assert torch.equal(hit, expect.reshape(-1))
    if out_map in (1, 2):      # kept = the V x V part of the G-grid
        g = keep[:, 0].cpu().view(B, G, G)
        assert bool(g[:, :V, :V].all()) and int(g.sum()) == B * V * V
    else:
        assert bool(keep.all())
