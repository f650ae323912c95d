"""The CTA budget of the backward launchers (``b2rl_set_cta_budget``; ``nature_tc.wgrad_stream`` sets it for the dgrad chain
and for the weight gradients beside it), at the bench's batch of 512 on Gaussian operands:

* the dgrads (fc4 on the dense GEMM, conv3 and conv2 on the persistent slab kernel) give the same bits with a budget as on
  their full grids: a tile's arithmetic does not depend on which CTA runs it;
* their bias gradients and the weight gradients' split-K partial sums differ only by the order of their fp32 additions;
* every grid respects its budget, and with the budget cleared the launchers size their grids as they do without one.

Bound of the re-association check: two fp32 summation orders of the same n terms differ by at most about
n * 2**-24 * sum |term| (n = 51 200 rows here); the sums checked are far more accurate than that worst case, and the test
holds them to 1e-4 * sum |term|, with sum |term| bounded from the operands."""
import ctypes

import pytest
import torch

gpu = pytest.mark.gpu
B = 512
REASSOC = 1e-4


def _budget(n):
    from deeprl_b200 import _lib
    _lib.call("b2rl_set_cta_budget", int(n))


def _last_ctas():
    from deeprl_b200 import _lib
    n = ctypes.c_int32(-1)
    _lib.call("b2rl_last_grid_ctas", ctypes.byref(n))
    return n.value


@pytest.fixture(scope="module")
def ops():
    import deeprl_b200 as rl
    from deeprl_b200 import _lib
    rl.select_device(0)
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(11)
    r = lambda *s: torch.randn(s, generator=gen, device=dev).to(torch.bfloat16)
    t = dict(g4=r(B, 512), y3c=r(B, 3136), w4p=r(512, 3136) * 0.05, y2=r(B * 100, 64), x1=r(B * 100, 128),
             g3=r(B * 100, 64), g2=r(B * 100, 64), w3d=r(64, 576) * 0.05, w2d=r(128, 256) * 0.05)
    t["sms"] = torch.cuda.get_device_properties(dev).multi_processor_count
    yield t, _lib, dev
    _budget(0)


def _dgrads(t, _lib, dev):
    """The three dgrads of nature_tc._backward_fused: (outputs, bias gradients), fresh buffers each call."""
    z = lambda *s: torch.zeros(s, dtype=torch.bfloat16, device=dev)
    out, db, ctas = {}, {}, {}
    db["fc4"], db["conv3"], db["conv2"] = (torch.zeros(n, device=dev) for n in (64, 64, 32))
    out["fc4"] = z(B * 100, 64)
    e = _lib.bwd_epilogue(t["y3c"], db["fc4"], 64, 64)
    _lib.call("b2rl_gemm_bwd_bf16", _lib.ptr(t["g4"]), 512, _lib.ptr(t["w4p"]), 1, 3136, _lib.ptr(out["fc4"]), 64, B, 3136,
              512, 4, 10, 7, ctypes.byref(e), 128, _lib.stream())
    ctas["fc4"] = _last_ctas()
    out["conv3"] = z(B * 100, 64)
    e = _lib.bwd_epilogue(t["y2"], db["conv3"], 64, 0)
    _lib.call("b2rl_conv_gemm_bwd_bf16", _lib.ptr(t["g3"]), B * 100, 64, _lib.ptr(t["w3d"]), 64, 9, 3, 10,
              _lib.ptr(out["conv3"]), 64, 0, 0, 0, ctypes.byref(e), 64, _lib.stream())
    ctas["conv3"] = _last_ctas()
    out["conv2"] = z(B * 441, 32)
    e = _lib.bwd_epilogue(t["x1"], db["conv2"], 32, 32)
    _lib.call("b2rl_conv_gemm_bwd_bf16", _lib.ptr(t["g2"]), B * 100, 64, _lib.ptr(t["w2d"]), 128, 4, 2, 10,
              _lib.ptr(out["conv2"]), 32, 3, 21, 20, ctypes.byref(e), 128, _lib.stream())
    ctas["conv2"] = _last_ctas()
    torch.cuda.synchronize()
    return out, db, ctas


def _wgrads(t, dev):
    """fc4's weight gradient and the conv3 / conv2 split-K partial sums: ({name: fp32 gradient}, {name: (CTAs, partials)})."""
    from deeprl_b200.network import nature_tc
    from deeprl_b200.ops import gemm_bf16
    g, ctas = {}, {}
    g["fc4"] = gemm_bf16(t["g4"], t["y3c"], a_major="mn", b_major="mn", out_dtype=torch.float32, block_n=128)
    ctas["fc4"] = (_last_ctas(), None)
    for name, args in (("conv3", (t["y2"], t["g3"], 64, 9, 3, 10)), ("conv2", (t["x1"], t["g2"], 64, 4, 2, 10))):
        buf, p = nature_tc.wgrad_partials(*args)
        g[name] = buf[:p].sum(0)
        ctas[name] = (_last_ctas(), p)
    torch.cuda.synchronize()
    return g, ctas


def _terms_bound(G, X):
    """An upper bound of sum_r |G[r, n] X[r', c]| over any row pairing: the largest column sum of |G| times max |X|."""
    return float(G.float().abs().sum(0).max()) * float(X.float().abs().max())


@gpu
@pytest.mark.parametrize("main", [100, 84, 66])
def test_dgrad_bits_do_not_depend_on_the_budget(ops, main):
    t, _lib, dev = ops
    _budget(0)
    ref, ref_db, full = _dgrads(t, _lib, dev)
    _budget(main)
    out, db, ctas = _dgrads(t, _lib, dev)
    _budget(0)
    tiles = {"fc4": 4 * 25, "conv3": 400, "conv2": 400}
    for k in ref:
        assert full[k] == min(tiles[k], t["sms"]), (k, full[k])          # no budget: one CTA per SM, at most one per tile
        assert ctas[k] == min(tiles[k], main), (k, ctas[k])
        assert torch.equal(out[k], ref[k]), k
        # the bias gradient sums the masked dgrad output over the rows: sum |term| <= sum of |output| (with a margin for
        # the bf16 rounding of the stored output)
        col = out[k].float().abs().sum(0)
        bound = REASSOC * (1.01 * float(col.max()) + 1.0)
        assert float((db[k] - ref_db[k]).abs().max()) <= bound, k


@gpu
@pytest.mark.parametrize("side", [16, 32, 48])
def test_wgrad_partial_sums_within_fp32_reassociation(ops, side):
    t, _lib, dev = ops
    _budget(0)
    ref, full = _wgrads(t, dev)
    _budget(side)
    g, ctas = _wgrads(t, dev)
    _budget(0)
    assert full["fc4"][0] == min(100, t["sms"])
    for k, (n, p) in ctas.items():
        assert n <= side, (k, n, side)
        if p is not None:
            assert p <= full[k][1] and n % p == 0, (k, n, p, full[k])   # partials = CTAs per 128-column group
    operands = {"fc4": (t["g4"], t["y3c"]), "conv3": (t["g3"], t["y2"]), "conv2": (t["g2"], t["x1"])}
    for k, (G, X) in operands.items():
        err = float((g[k] - ref[k]).abs().max())
        assert err <= REASSOC * _terms_bound(G, X), (k, err)
        assert float(ref[k].abs().max()) > 0


@gpu
def test_no_budget_restores_the_full_grids(ops):
    t, _lib, dev = ops
    _budget(0)
    ref, ref_db, full = _dgrads(t, _lib, dev)
    wref, wfull = _wgrads(t, dev)
    _budget(24)
    _dgrads(t, _lib, dev), _wgrads(t, dev)
    _budget(0)
    out, db, ctas = _dgrads(t, _lib, dev)
    w, wctas = _wgrads(t, dev)
    assert ctas == full and wctas == wfull
    for k in ref:
        assert torch.equal(out[k], ref[k]) and torch.equal(w[k], wref[k]), k
    assert all(n <= t["sms"] for n, _ in wfull.values())


@gpu
def test_backward_budgets_from_wgrad_stream(ops):
    from deeprl_b200.network import nature_tc
    t, _lib, dev = ops
    s = torch.cuda.Stream()
    with nature_tc.wgrad_stream(s):
        assert nature_tc._budgets(dev) == (t["sms"] - nature_tc.SIDE_CTAS, nature_tc.SIDE_CTAS)
        with nature_tc.wgrad_stream(s, side_ctas=0):
            assert nature_tc._budgets(dev) == (0, 0)
    with nature_tc.wgrad_stream(None):
        assert nature_tc._budgets(dev) == (0, 0)
    assert nature_tc._budgets(dev) == (0, 0)
    with nature_tc.wgrad_stream(s, side_ctas=t["sms"]), pytest.raises(ValueError):
        nature_tc._budgets(dev)
    with nature_tc._cta_budget(8):
        nature_tc.wgrad_partials(t["y2"], t["g3"], 64, 9, 3, 10)
        assert _last_ctas() <= 8
    nature_tc.wgrad_partials(t["y2"], t["g3"], 64, 9, 3, 10)         # the context cleared the budget
    assert _last_ctas() > 8
