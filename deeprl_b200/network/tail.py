"""Host side of ``csrc/tail.cu``: the tail of one gradient update (``loss.backward()``'s last step, ``clip_grad_norm_``,
``optimizer.step()`` -- DQN_agent.py:131-134) of a network with a wgmma ``NatureConvBody`` as TWO launches.

``NatureTail(opt, body, scale)`` binds a ``FlatOptimizer`` arena to the body's packed bf16 operands:

* ``reduce(...)`` (called by ``_NatureBody.backward`` while ``nature_tc.grad_sink(tail)`` is active) -- kernel A: split-K
  partials summed, GEMM layouts -> reference layouts, written into the ``.grad`` arena, bias gradients moved, sum of
  squares per unit.
* ``step(max_norm, grad_scale)`` -- kernel B: clip coefficient, RMSprop / Adam, gradient re-zeroed, updated weights written
  into the packed bf16 operands (no separate pack launch, no ``zero_grad`` memset).  With ``lr_dev`` set (a float32 device
  scalar) the kernel reads the learning rate there instead of ``opt.lr``.

The unit tables (int32 x 4 per unit, see the header of csrc/tail.cu) are built here once.
"""
import numpy as np
import torch

from .. import _lib

_f32 = torch.float32
U_PLAIN, U_W1, U_W2, U_W3, U_W4, U_B1, U_B2, U_B3, U_B4 = range(9)
PLAIN_CHUNK = 2048


def _plain_units(covered, n):
    """Units of kind 0 over the parts of [0, n) that ``covered`` (list of (offset, length)) leaves out."""
    out, pos = [], 0
    for off, ln in sorted(covered) + [(n, 0)]:
        while pos < off:
            k = min(PLAIN_CHUNK, off - pos)
            out.append((pos, k, U_PLAIN, 0))
            pos += k
        pos = max(pos, off + ln)
    return out


class NatureTail:
    def __init__(self, opt, body, scale):
        self.opt, self.body, self.scale = opt, body, float(scale)
        dev = opt.flat.device
        base = opt.flat.data_ptr()
        mods = (body.conv1, body.conv2, body.conv3, body.fc4)
        self.c1, self.n4 = body.conv1.in_channels, body.fc4.out_features

        def off(p):
            o = (p.data_ptr() - base) // 4
            if not (0 <= o < opt.n) or p.data_ptr() % 16:
                raise _lib.B2RLError("NatureTail: the body's parameters must live in the optimizer's arena")
            return int(o)

        ow = [off(m.weight) for m in mods]
        ob = [off(m.bias) for m in mods]
        rows = (32, 64, 64, self.n4)
        lens = (64 * self.c1, 512, 576, 3136)
        nb = (32, 64, 64, self.n4)
        pad4 = lambda k: (k + 3) // 4 * 4
        # kernel A: conv rows in 256-element segments first (the heavy units: they read every split-K partial), then fc4
        # rows, biases, and whatever else lives in the arena (the head's parameters)
        a_units, b_units, covered = [], [], []
        for layer in range(3):
            L = lens[layer]
            for n in range(rows[layer]):
                for seg in range((L + 255) // 256):
                    a_units.append((ow[layer] + n * L, min(256, L - seg * 256), U_W1 + layer, n | (seg << 16)))
        for n in range(self.n4):
            a_units.append((ow[3] + n * 3136, 3136, U_W4, n))
        for layer in range(4):
            a_units.append((ob[layer], nb[layer], U_B1 + layer, 0))
            covered.append((ow[layer], rows[layer] * lens[layer]))
            covered.append((ob[layer], pad4(nb[layer])))
            for n in range(rows[layer]):
                b_units.append((ow[layer] + n * lens[layer], lens[layer], U_W1 + layer, n))
            b_units.append((ob[layer], pad4(nb[layer]), U_PLAIN, 0))
        plain = _plain_units(covered, opt.n)
        # multi-GPU: the fc4 part (95 % of the gradient bytes, final right after the fc4 weight-gradient GEMM) is reduced into
        # the arena early and all-reduced while the convolution backward still runs; everything else follows at the end
        a4_units = [u for u in a_units if u[2] in (U_W4, U_B4)]
        arest_units = [u for u in a_units if u[2] not in (U_W4, U_B4)] + plain
        a_units += plain
        b_units += plain
        assert sum(u[1] for u in b_units) == opt.n, "unit table does not tile the arena"
        to_dev = lambda u: torch.from_numpy(np.asarray(u, dtype=np.int32).reshape(-1, 4)).to(dev)
        self.a_units, self.b_units = to_dev(a_units), to_dev(b_units)
        self.n_a, self.n_b = len(a_units), len(b_units)
        self.a4_units, self.arest_units = to_dev(a4_units), to_dev(arest_units)
        self.n_a4, self.n_arest = len(a4_units), len(arest_units)
        lo, hi = ow[3], ow[3] + self.n4 * 3136
        if ob[3] == hi:                                  # fc4.bias follows fc4.weight in the arena (parameter order of the body)
            hi = ob[3] + pad4(self.n4)
        self.early_slice = (lo, hi)
        self.late_slices = [(a, b) for a, b in ((0, lo), (hi, opt.n)) if b > a]
        self.split = False               # set by the owner (world_size > 1): backward calls reduce_w4 / reduce_rest
        self.early = None                # callable: the all-reduce of the early slice (enqueued right after reduce_w4)
        self.unit_sumsq = torch.zeros(self.n_a, dtype=_f32, device=dev)
        # bias-gradient accumulators of the dgrad epilogues / head backward: zero here, re-zeroed by kernel A after use
        self.db = torch.zeros(32 + 64 + 64 + self.n4, dtype=_f32, device=dev)
        self.db1, self.db2, self.db3, self.db4 = self.db[:32], self.db[32:96], self.db[96:160], self.db[160:]
        self.kind = {"rmsprop": 1 if opt.centered else 0, "adam": 2}[opt.kind]
        # clip_grad_norm_'s arguments of the NEXT step(): kernel A's last CTA already turns its unit partials into the
        # coefficient, so kernel B starts with one scalar load (set by the owner before the backward pass)
        self.max_norm, self.grad_scale = 0.0, 1.0
        # a float32 device scalar that replaces opt.lr in step() (a schedule the owner writes between graph replays), or None
        self.lr_dev = None

    def packed(self):
        from . import nature_tc
        pk = getattr(self.body, "_packed", None)
        if pk is None:
            pk = nature_tc.repack(self.body, self.scale)
        return pk

    def reduce(self, gw1p, p1, gw2p, p2, gw3p, p3, gw4p):
        o = self.opt
        _lib.call("b2rl_nature_grad_reduce", _lib.ptr(self.a_units), self.n_a, _lib.ptr(gw1p), int(p1), _lib.ptr(gw2p), int(p2),
                  _lib.ptr(gw3p), int(p3), _lib.ptr(gw4p), _lib.ptr(self.db1), _lib.ptr(self.db2), _lib.ptr(self.db3),
                  _lib.ptr(self.db4), self.c1, self.n4, self.scale, _lib.ptr(o.grad), _lib.ptr(self.unit_sumsq),
                  _lib.ptr(o.step_dev) if o.kind == "adam" else None, _lib.ptr(o.scratch), float(self.max_norm or 0.0),
                  float(self.grad_scale), _lib.stream())

    def _reduce(self, units, n, gw1p, p1, gw2p, p2, gw3p, p3, gw4p, stream=None):
        o = self.opt
        d = self.unit_sumsq                              # any valid address for the sources a partial table does not touch
        _lib.call("b2rl_nature_grad_reduce", _lib.ptr(units), n, _lib.ptr(d if gw1p is None else gw1p), int(p1 or 1),
                  _lib.ptr(d if gw2p is None else gw2p), int(p2 or 1), _lib.ptr(d if gw3p is None else gw3p), int(p3 or 1),
                  _lib.ptr(d if gw4p is None else gw4p), _lib.ptr(self.db1), _lib.ptr(self.db2), _lib.ptr(self.db3), _lib.ptr(self.db4),
                  self.c1, self.n4, self.scale, _lib.ptr(o.grad), _lib.ptr(self.unit_sumsq), None, None, 0.0, 1.0,
                  stream if stream is not None else _lib.stream())

    def reduce_w4(self, gw4p, stream=None):
        """Multi-GPU, early part: fc4's weight gradient (GEMM layout -> arena) and bias gradient."""
        self._reduce(self.a4_units, self.n_a4, None, 1, None, 1, None, 1, gw4p, stream)

    def reduce_rest(self, gw1p, p1, gw2p, p2, gw3p, p3):
        """Multi-GPU, late part: the convolution layers' gradients (+ Adam's step counter)."""
        self._reduce(self.arest_units, self.n_arest, gw1p, p1, gw2p, p2, gw3p, p3, None)
        if self.opt.kind == "adam":
            self.opt.step_dev.add_(1)

    def step(self, max_norm=0.0, grad_scale=1.0, reduced_elsewhere=False):
        """Clip + optimizer + bf16 operand pack.  ``reduced_elsewhere``: the gradient arena was all-reduced after ``reduce``
        (multi-GPU), so the norm is recomputed over the arena (one extra launch) instead of taken from the unit partials.
        Otherwise ``max_norm`` / ``grad_scale`` must be what ``self.max_norm`` / ``self.grad_scale`` held during ``reduce``."""
        o = self.opt
        pk = self.packed()
        if not reduced_elsewhere and (float(max_norm or 0.0), float(grad_scale)) != (float(self.max_norm or 0.0), float(self.grad_scale)):
            raise _lib.B2RLError("NatureTail.step: set tail.max_norm / tail.grad_scale before the backward pass")
        if reduced_elsewhere:
            _lib.call("b2rl_grad_norm", _lib.ptr(o.grad), o.n, float(grad_scale), float(max_norm or 0.0), _lib.ptr(o.scratch),
                      _lib.stream())
        a, b = (o.betas if o.kind == "adam" else (o.alpha, 0.0))
        _lib.call("b2rl_nature_fused_opt_lr", _lib.ptr(self.b_units), self.n_b, _lib.ptr(o.flat), _lib.ptr(o.grad),
                  _lib.ptr(o.s1), _lib.ptr(o.s2), self.kind, float(o.lr), _lib.ptr(self.lr_dev), float(a), float(b),
                  float(o.eps), float(max_norm or 0.0), float(grad_scale), None, self.n_a, _lib.ptr(o.scratch),
                  _lib.ptr(o.step_dev), self.c1, self.n4, self.scale, _lib.ptr(pk.w1f), _lib.ptr(pk.w2f), _lib.ptr(pk.w2d),
                  _lib.ptr(pk.w3f), _lib.ptr(pk.w3d), _lib.ptr(pk.w4p), 1, _lib.ptr(o.shadow), _lib.stream())
        pk.scale = self.scale
