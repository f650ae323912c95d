"""Rainbow on the device (``config.device_rainbow``; deeprl_b200/csrc/rainbow.cu): one ``b2rl_rainbow_actor_step`` launch per
env step and ONE ``b2rl_rainbow_replay_update`` launch per gradient update of CategoricalDQN_agent.py:60-89 on
DQN_agent.py:101-138, for a RainbowNet on a two-layer FCBody whose four layers are all NoisyLinear or all nn.Linear.

CPU: the update's phase functions (csrc/rainbow_phases.h on dist_phases.h and a2c_phases.h, rainbow_sequence.inc) are compiled
for the host by tests/host_emul/rainbow_emul.cpp and run with the block's threads in sequence, with the noise given, against
the reference's recorded Rainbow updates (tests/golden/rainbow_agent.npz) and against oracle/rainbow.py RainbowOracle with
RMSprop.
GPU: the CUDA build of the same source through the C ABI and through the agent; the noise the kernels draw; the actor step.

Tolerances: fp32 sums in another order than torch's kernels, one RMSprop step per update: parameters to 1e-5 absolute."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import rainbow as rainbow_oracle  # noqa: E402

TANH, RELU = 0, 1
LAYERS = ("body.layers.0", "body.layers.1", "fc_advantage", "fc_value")
NOISY_NAMES, PLAIN_NAMES = ("weight_mu", "weight_sigma", "bias_mu", "bias_sigma"), ("weight", "bias")
P = ctypes.c_void_p


def keys_of(noisy):
    """The kernels' tensor order."""
    return [l + "." + p for l in LAYERS for p in (NOISY_NAMES if noisy else PLAIN_NAMES)]


def vp(x):
    return None if x is None else P(x.ctypes.data)


def layer_shapes(D, H1, H2, A, K):
    return [(D, H1), (H1, H2), (H2, A * K), (H2, K)]                      # (in, out) per layer


def noise_len(D, H1, H2, A, K):
    return sum(i + 2 * o for i, o in layer_shapes(D, H1, H2, A, K))


def noise_dict(vec, D, H1, H2, A, K):
    """A noise vector (per layer noise_in, noise_out_weight, noise_out_bias) as oracle/rainbow.py's dict."""
    out, o = {}, 0
    for l, (i, n) in zip(LAYERS, layer_shapes(D, H1, H2, A, K)):
        v = torch.as_tensor(np.asarray(vec[o:o + i + 2 * n], np.float32))
        out[l + "."] = (v[:i], v[i:i + n], v[i + n:])
        o += i + 2 * n
    return out


def transform(x):
    x = torch.as_tensor(x)
    return x.sign() * x.abs().sqrt()


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("rainbow_emul") / "rainbow_emul.so")
    subprocess.run(["g++", "-O2", "-fno-strict-aliasing", "-std=c++17", "-shared", "-fPIC", "-o", out,
                    os.path.join(ROOT, "tests", "host_emul", "rainbow_emul.cpp")], check=True)
    lib = ctypes.CDLL(out)
    i32, f32, f64 = ctypes.c_int32, ctypes.c_float, ctypes.c_double
    lib.rainbow_emul_update.argtypes = ([i32, i32, P, P, i32, f64, P, P, P] + [i32] * 6 + [P] * 6 + [f32] * 3
                                        + [i32, f32, i32, f64, f64, f32, P] + [f32] * 3 + [P] * 6 + [i32, i32])
    lib.rainbow_emul_noise_len.argtypes = [i32] * 6
    return lib


def arena(sd, keys):
    """FlatOptimizer's layout (ops.py): every tensor starts on a multiple of 4 elements."""
    offs, n = [], 0
    for k in keys:
        offs.append(n)
        n += (sd[k].numel() + 3) // 4 * 4
    flat = np.zeros(n, np.float32)
    for k, o in zip(keys, offs):
        flat[o:o + sd[k].numel()] = np.asarray(sd[k].detach()).ravel()
    return flat, np.asarray(offs, np.int32)


def unflatten(flat, offs, sd, keys):
    return {k: flat[o:o + sd[k].numel()].reshape(tuple(sd[k].shape)) for k, o in zip(keys, offs)}


class EmulState:
    """Online arena, target arena, RMSprop moments and step count, carried across updates."""

    def __init__(self, noisy, sd, target_sd=None):
        self.keys = keys_of(noisy)
        self.flat, self.off = arena(sd, self.keys)
        self.target = arena(target_sd if target_sd is not None else sd, self.keys)[0]
        self.sq, self.ga = np.zeros_like(self.flat), np.zeros_like(self.flat)
        self.step = np.zeros(1, np.int64)
        self.loss = np.zeros(1, np.float32)


def _batch_arrays(batch):
    s = np.ascontiguousarray(batch["state"])
    s2 = np.ascontiguousarray(batch["next_state"], dtype=s.dtype)
    a = np.ascontiguousarray(batch["action"], np.int64)
    r, m = (np.ascontiguousarray(batch[k], np.float32) for k in ("reward", "mask"))
    prob = batch.get("sampling_prob")
    return s, s2, a, r, m, None if prob is None else np.ascontiguousarray(prob, np.float32)


def emul_update(lib, st, noisy, gate, batch, H1, H2, cfg, noise=None, threads=512, reversed_=False):
    """One b2rl_rainbow_replay_update on the host.  noise: [2, noise_len] (target, online).  Returns (per-sample KL, priority,
    the noise arena the update wrote for the online module)."""
    s, s2, a, r, m, prob = _batch_arrays(batch)
    B, D = s.shape
    prio = np.zeros(B, np.float32) if prob is not None else None
    vec = np.zeros(B, np.float32)
    given = None if noise is None else np.ascontiguousarray(noise, np.float32)
    written = np.zeros(lib.rainbow_emul_noise_len(D, H1, H2, cfg["A"], cfg["K"], 1), np.float32) if noisy else None
    rc = lib.rainbow_emul_update(int(noisy), gate, vp(s), vp(s2), int(s.dtype == np.float64), cfg.get("coef", 1.0), vp(a), vp(r),
                                 vp(m), B, D, H1, H2, cfg["A"], cfg["K"], vp(st.flat), vp(st.target), vp(st.sq), vp(st.ga),
                                 vp(st.step), vp(st.off), cfg["lr"], cfg["alpha"], cfg["eps"], int(cfg["centered"]),
                                 cfg["discount"] ** cfg["n_step"], int(cfg["double"]), cfg["vmin"], cfg["vmax"], cfg["clip"],
                                 vp(prob), cfg.get("beta", 0.0), 0.01, 0.5, vp(prio), vp(vec), vp(st.loss), vp(given),
                                 vp(written), None, threads, int(reversed_))
    assert rc == 0
    return vec, prio, written


def _oracle(sd, tgt, cfg, gate):
    o = rainbow_oracle.RainbowOracle(
        {k: v.clone() for k, v in sd.items()}, cfg["A"],
        lambda p: torch.optim.RMSprop(p, cfg["lr"], alpha=cfg["alpha"], eps=cfg["eps"], centered=cfg["centered"]),
        cfg["discount"], n_step=cfg["n_step"], double_q=cfg["double"], gradient_clip=cfg["clip"],
        state_coef=cfg.get("coef", 1.0), atoms=np.linspace(cfg["vmin"], cfg["vmax"], cfg["K"]), v_min=cfg["vmin"],
        v_max=cfg["vmax"], replay_eps=0.01, replay_alpha=0.5, replay_beta=lambda: cfg.get("beta", 0.0),
        gate=torch.tanh if gate == TANH else F.relu)
    for k in o.target_sd:
        o.target_sd[k].copy_(tgt[k])
    return o


class _Tr:
    def __init__(self, **kw):
        self.__dict__.update(kw)


# ------------------------------------------------------------------------------------------------ golden records
GOLDEN_CFG = dict(lr=0.001, alpha=0.99, eps=1e-8, centered=False, clip=10.0, discount=0.99, n_step=3, A=2, K=50, vmin=-100.0,
                  vmax=100.0, double=True)
GOLDEN_DIMS = (4, 16, 16, 2, 50)


def golden_sd(g, flat):
    keys = [str(k) for k in g["keys"]]
    assert keys == keys_of(True)
    out, o = {}, 0
    for k in keys:
        shape = g["init." + k].shape
        n = int(np.prod(shape))
        out[k] = torch.from_numpy(np.asarray(flat[o:o + n]).reshape(shape).copy())
        o += n
    return out


def golden_batch(g, i):
    return {f: g["b_" + f][i] for f in ("state", "next_state", "action", "reward", "mask", "sampling_prob")}


def golden_states(g):
    """(online, target) state dicts before each recorded update."""
    init = {k: torch.from_numpy(g["init." + k]) for k in keys_of(True)}
    on, tg, out = init, init, []
    for i in range(g["kl"].shape[0]):
        out.append((on, tg))
        on = golden_sd(g, g["params"][i])
        if g["synced"][i]:
            tg = on
    return out


def check_golden_single_updates(g, update):
    """Each of the reference's recorded updates from its recorded online / target parameters, with the recorded noise: the
    per-sample KL and the priorities equal the recorded ones (1e-5 relative, 2e-6 absolute floor)."""
    assert g["noise"].shape[1] == noise_len(*GOLDEN_DIMS) and g["kl"].shape[0] >= 20
    worst = 0.0
    for i, (on, tg) in enumerate(golden_states(g)):
        st = EmulState(True, on, tg)
        cfg = dict(GOLDEN_CFG, beta=float(g["beta"][i]))
        vec, prio, _ = update(st, True, RELU, golden_batch(g, i), 16, 16, cfg, np.stack([g["target_noise"][i], g["noise"][i]]))
        np.testing.assert_allclose(vec, g["kl"][i], rtol=1e-5, atol=2e-6, err_msg=str(i))
        np.testing.assert_allclose(prio, g["priority"][i], rtol=1e-5, atol=2e-6, err_msg=str(i))
        worst = max(worst, float((np.abs(vec - g["kl"][i]) / np.maximum(np.abs(g["kl"][i]), 0.2)).max()))
    return worst


def test_golden_updates_emulated(emul, golden):
    g = golden("rainbow_agent")
    worst = check_golden_single_updates(g, lambda *a: emul_update(emul, *a))
    print("largest relative difference of the KL over the golden updates: %.3g" % worst)


# RMSprop's first steps move a parameter by about lr whatever the size of its gradient; with the reference's eps = 1e-8 a
# gradient near 1e-8 carries the fp32 rounding of its sum into the parameter, so consecutive updates are compared more loosely
# than single ones: 2e-4 absolute after 20 updates of lr 1e-3 (a parameter has then moved by up to 2e-2).
GOLDEN_CHAIN_ATOL = 2e-4


def check_golden_chain(g, update):
    sd0 = {k: torch.from_numpy(g["init." + k]) for k in keys_of(True)}
    st = EmulState(True, sd0)
    assert int(np.sum(g["synced"])) >= 3
    for i in range(g["kl"].shape[0]):
        cfg = dict(GOLDEN_CFG, beta=float(g["beta"][i]))
        update(st, True, RELU, golden_batch(g, i), 16, 16, cfg, np.stack([g["target_noise"][i], g["noise"][i]]))
        if g["synced"][i]:
            st.target[...] = st.flat
    want, want_t = golden_states(g)[-1][0], None
    want = golden_sd(g, g["params"][-1])
    last_sync = max(i for i in range(g["kl"].shape[0]) if g["synced"][i])
    want_t = golden_sd(g, g["params"][last_sync])
    got, got_t = unflatten(st.flat, st.off, sd0, st.keys), unflatten(st.target, st.off, sd0, st.keys)
    worst = 0.0
    for k in st.keys:
        err, err_t = float(np.abs(got[k] - want[k].numpy()).max()), float(np.abs(got_t[k] - want_t[k].numpy()).max())
        worst = max(worst, err, err_t)
        assert err <= GOLDEN_CHAIN_ATOL and err_t <= GOLDEN_CHAIN_ATOL, (k, err, err_t)
        assert np.abs(want[k].numpy() - sd0[k].numpy()).max() > 1e-3, k
    assert int(st.step[0]) == g["kl"].shape[0]
    return worst


def test_golden_twenty_consecutive_updates_emulated(emul, golden):
    """The recorded updates in sequence from the recorded init with the recorded noise and sync schedule: the 16 online tensors
    and the target equal the reference's after the last update (GOLDEN_CHAIN_ATOL)."""
    worst = check_golden_chain(golden("rainbow_agent"), lambda *a: emul_update(emul, *a))
    print("largest parameter difference to the reference after 20 updates: %.3g" % worst)


@pytest.mark.parametrize("noisy", [True, False])
def test_oracle_forward_is_rainbow_net(golden, noisy):
    """oracle/rainbow.py rainbow on the reference RainbowNet's recorded state_dict (the noise from its buffers) gives its outputs."""
    g = golden("rainbow")
    tag = "rb%d_" % int(noisy)
    sd = {k[len(tag) + 3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith(tag + "sd_")}
    p, lp = rainbow_oracle.rainbow(sd, torch.from_numpy(g[tag + "x"]), 4, 11, F.relu)
    np.testing.assert_allclose(p.numpy(), g[tag + "prob"], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(lp.numpy(), g[tag + "log_prob"], rtol=1e-5, atol=1e-6)
    if noisy:                                              # ... and the same with the noise passed in as vectors
        nz = {l + ".": tuple(sd[l + "." + b] for b in ("noise_in", "noise_out_weight", "noise_out_bias"))
              for l in ("body.layers.0", "fc_advantage", "fc_value")}
        p2, _ = rainbow_oracle.rainbow(sd, torch.from_numpy(g[tag + "x"]), 4, 11, F.relu, nz)
        np.testing.assert_allclose(p2.numpy(), g[tag + "prob"], rtol=1e-5, atol=1e-7)


# ------------------------------------------------------------------------------------------------ ragged shapes and the oracle
def smem_bytes(noisy, D, H1, H2, A, K, B, double):
    from deeprl_b200 import _lib
    return _lib.lib().b2rl_rainbow_smem_bytes(int(noisy), D, H1, H2, A, K, B, int(double))


def max_batch(noisy, D, H1, H2, A, K, double):
    B = 1
    while smem_bytes(noisy, D, H1, H2, A, K, B + 1, double) <= 227 * 1024:
        B += 1
    return B


CFG = dict(lr=1e-3, alpha=0.99, eps=1e-6, centered=False, discount=0.99, clip=5.0, n_step=1, double=False, per=False, coef=1.0,
           vmin=-100.0, vmax=100.0)
# (eps = 1e-6, not 1e-8: see test_dist_dqn_device.py)
CASES = [  # (noisy, gate, D, A, K, H1, H2, B, float64 states, cfg overrides)
    (True, RELU, 4, 2, 50, 64, 64, 32, True, dict(double=True, per=True, n_step=3, clip=10.0)),      # rainbow_feature
    (True, TANH, 11, 5, 21, 32, 48, 37, True, dict(double=True, per=True, centered=True, clip=1e6, n_step=3, coef=0.5)),
    (True, RELU, 7, 18, 2, 16, 24, 1, False, dict(per=True, clip=0.05, vmin=-3.0, vmax=3.0)),
    (True, TANH, 6, 2, 51, 8, 8, "max", False, dict(double=True, centered=True, clip=0.05, vmin=-10.0, vmax=10.0)),
    (True, RELU, 5, 5, 51, 24, 16, 10, True, dict(clip=1e6, n_step=3)),
    (False, RELU, 4, 2, 50, 64, 64, 32, True, dict(double=True, per=True, n_step=3, clip=10.0)),
    (False, TANH, 9, 5, 2, 40, 24, 37, False, dict(centered=True, clip=0.05, n_step=3, coef=0.25)),
    (False, RELU, 6, 2, 51, 8, 8, "max", True, dict(double=True, clip=1e6, vmin=-10.0, vmax=10.0)),
    (False, TANH, 5, 5, 50, 16, 24, 1, True, dict(per=True, centered=True, clip=1e6)),
    (False, RELU, 7, 18, 2, 24, 16, 10, False, dict(double=True, per=True, clip=0.05)),
]


def make_problem(noisy, D, A, K, H1, H2, B, f64, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale

    def net():
        sd = {}
        for l, (i, o) in zip(LAYERS, layer_shapes(D, H1, H2, A, K)):
            if noisy:
                sd.update({l + ".weight_mu": r(o, i, scale=i ** -0.5), l + ".weight_sigma": r(o, i, scale=0.4 * i ** -0.5),
                           l + ".bias_mu": r(o, scale=0.1), l + ".bias_sigma": r(o, scale=0.4 * o ** -0.5)})
            else:
                sd.update({l + ".weight": r(o, i, scale=i ** -0.5), l + ".bias": r(o, scale=0.1)})
        return sd

    sd, target = net(), net()
    dt = np.float64 if f64 else np.float32
    batch = dict(state=r(B, D, scale=2.0).double().numpy().astype(dt), next_state=r(B, D, scale=2.0).double().numpy().astype(dt),
                 action=torch.randint(0, A, (B,), generator=g).numpy(), reward=r(B, scale=3.0).numpy(),
                 mask=(torch.rand(B, generator=g) > 0.2).float().numpy(),
                 sampling_prob=(torch.rand(B, generator=g) * 0.01 + 1e-4).numpy())
    noise = (r(2, noise_len(D, H1, H2, A, K), scale=0.5).numpy() if noisy else None)
    return sd, target, batch, noise


def case_setup(case):
    noisy, gate, D, A, K, H1, H2, B, f64, over = CASES[case]
    cfg = dict(CFG, A=A, K=K, **over)
    if B == "max":
        B = max_batch(noisy, D, H1, H2, A, K, cfg["double"])
    assert 0 < smem_bytes(noisy, D, H1, H2, A, K, B, cfg["double"]) <= 227 * 1024      # (the emulation has no limit of its own)
    cfg["beta"] = 0.55 if cfg["per"] else 0.0
    sd0, tgt0, batch, noise = make_problem(noisy, D, A, K, H1, H2, B, f64, seed=900 + case)
    if not cfg["per"]:
        del batch["sampling_prob"]
    return noisy, gate, (D, H1, H2, A, K), cfg, sd0, tgt0, batch, noise


def run_case(lib, case, threads=512, reversed_=False):
    noisy, gate, dims, cfg, sd0, tgt0, batch, noise = case_setup(case)
    st = EmulState(noisy, sd0, tgt0)
    vec, prio, written = emul_update(lib, st, noisy, gate, batch, dims[1], dims[2], cfg, noise, threads, reversed_)
    return st, vec, prio, written


def oracle_update(case):
    noisy, gate, dims, cfg, sd0, tgt0, batch, noise = case_setup(case)
    o = _oracle(sd0, tgt0, cfg, gate)
    if noisy:
        o.target_noise, o.noise = noise_dict(noise[0], *dims), noise_dict(noise[1], *dims)
    tr = _Tr(**batch)
    if cfg["per"]:
        tr.idx = np.arange(len(batch["action"]))
    with torch.no_grad():
        vec = o.compute_loss(tr).numpy()
    prios = {}

    class Rep:
        def update_priorities(self, pairs):
            prios.update(dict(pairs))

    loss = o.update(tr, Rep())
    grads = {k: o.sd[k].grad.numpy().copy() for k in keys_of(noisy)}       # after clip_grad_norm_
    clipped = float(np.sqrt(sum((v.astype(np.float64) ** 2).sum() for v in grads.values())))
    prio = np.asarray([prios[i] for i in range(len(prios))], np.float32) if cfg["per"] else None
    return o, cfg, float(loss), vec, prio, clipped, grads, sd0, tgt0


def check_against_oracle(case, st, vec, prio, atol=1e-5):
    o, cfg, loss, v_want, p_want, clipped, grads, sd0, tgt0 = oracle_update(case)
    np.testing.assert_allclose(vec, v_want, rtol=1e-5, atol=2e-6)
    if cfg["per"]:
        np.testing.assert_allclose(prio, p_want, rtol=1e-5, atol=1e-6)
    got, got_t = unflatten(st.flat, st.off, sd0, st.keys), unflatten(st.target, st.off, sd0, st.keys)
    sq, ga = unflatten(st.sq, st.off, sd0, st.keys), unflatten(st.ga, st.off, sd0, st.keys)
    gmax = max(float(np.abs(v).max()) for v in grads.values())
    for k in st.keys:
        want = o.sd[k].detach().numpy()
        np.testing.assert_allclose(got[k], want, rtol=0, atol=atol, err_msg=k)
        assert np.abs(want - sd0[k].numpy()).max() > 1e-6, k                 # every tensor moved
        np.testing.assert_array_equal(got_t[k], tgt0[k].numpy(), err_msg=k)  # the target arena is only read
        # the gradient of this tensor (sigmas included), from the moments of the first RMSprop step: its magnitude from
        # square_avg = (1 - alpha) g^2, and where the moment is kept its sign too from grad_avg = (1 - alpha) g
        assert float(np.abs(grads[k]).max()) > 0, k
        np.testing.assert_allclose(np.sqrt(sq[k] / (1 - cfg["alpha"])), np.abs(grads[k]), rtol=1e-3, atol=1e-5 * gmax, err_msg=k)
        if cfg["centered"]:
            np.testing.assert_allclose(ga[k] / (1 - cfg["alpha"]), grads[k], rtol=1e-3, atol=1e-5 * gmax, err_msg=k)
    np.testing.assert_allclose(st.loss[0], loss, rtol=1e-5, atol=1e-7)
    assert int(st.step[0]) == 1
    return cfg, clipped


@pytest.mark.parametrize("case", range(len(CASES)))
def test_update_matches_oracle_emulated(emul, case):
    st, vec, prio, written = run_case(emul, case)
    cfg, clipped = check_against_oracle(case, st, vec, prio)
    if cfg["clip"] < 1.0:
        assert abs(clipped - cfg["clip"]) < 1e-4 * cfg["clip"]              # the clip was active
    elif cfg["clip"] >= 1e5:
        assert clipped < cfg["clip"]                                         # ... and here it was not
    noisy, _, dims, _, _, _, _, noise = case_setup(case)
    if noisy:                                                                # the noise arena: vectors, bias eps, weight eps
        check_noise_arena(written, noise[1], dims)


def check_noise_arena(written, vec, dims):
    """The arena an update wrote for the online module holds the noise vector and NoisyLinear.reset_noise's epsilons of it:
    f(x) to 1 ulp (torch's vectorised sqrt and sqrtf round differently in places), so weight_epsilon, the rounded product of
    two such factors, within 5e-7 relative."""
    nz = noise_len(*dims)
    np.testing.assert_array_equal(written[:nz], vec)
    nd = noise_dict(vec, *dims)
    beps = np.concatenate([transform(nd[l + "."][2]).numpy() for l in LAYERS])
    weps = np.concatenate([torch.outer(transform(nd[l + "."][1]), transform(nd[l + "."][0])).numpy().ravel() for l in LAYERS])
    np.testing.assert_allclose(written[nz:nz + beps.size], beps, rtol=2.4e-7, atol=0)
    np.testing.assert_allclose(written[nz + beps.size:], weps, rtol=5e-7, atol=0)


def test_cases_cover_the_shapes():
    setups = [case_setup(c) for c in range(len(CASES))]
    for noisy in (True, False):
        mine = [s for s in setups if s[0] == noisy]
        sizes = {s[6]["action"].shape[0] for s in mine}
        assert {1, 10, 32, 37} <= sizes and max(sizes) > 37, sizes
        assert {s[3]["A"] for s in mine} == {2, 5, 18}
        assert {2, 50, 51} <= {s[3]["K"] for s in mine}
        assert {s[1] for s in mine} == {TANH, RELU}
        assert {(s[3]["double"], s[3]["per"]) for s in mine} == {(False, False), (True, True), (False, True), (True, False)}
        assert {s[3]["centered"] for s in mine} == {True, False} and {s[3]["n_step"] for s in mine} == {1, 3}


@pytest.mark.parametrize("case", [1, 3, 6, 9])
def test_thread_order_and_count_do_not_change_the_result(emul, case):
    """Reversed thread order inside every phase, 64 and 37 threads instead of 512: bit-identical arenas (the race check)."""
    ref, v_ref, p_ref, w_ref = run_case(emul, case)
    for threads, rev in ((512, True), (64, False), (37, True)):
        got, v, p, w = run_case(emul, case, threads, rev)
        for k in ("flat", "target", "sq", "ga", "loss", "step"):
            assert np.array_equal(getattr(ref, k), getattr(got, k)), (threads, rev, k)
        assert np.array_equal(v_ref, v) and (p_ref is None or np.array_equal(p_ref, p))
        assert w_ref is None or np.array_equal(w_ref, w)


def test_kernels_have_no_spills_and_no_stack_frame(tmp_path):
    cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-o", str(tmp_path / "r.cubin"),
           os.path.join(ROOT, "deeprl_b200", "csrc", "rainbow.cu"), "-Xptxas", "-v"]
    out = subprocess.run(cmd, check=True, capture_output=True, text=True).stderr
    entries = out.split("Compiling entry function")[1:]
    names = [e.split("'")[1] for e in entries]
    # (NoisyLinear, nn.Linear) x (tanh, ReLU), the update and the actor step
    assert sum("rainbow_replay_update_kernel" in n for n in names) == 4, names
    assert sum("rainbow_actor_kernel" in n for n in names) == 4, names
    assert len(names) == 8, names
    for e in entries:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in e, e


def test_shared_memory_budget_accepts_the_launcher():
    launcher = smem_bytes(True, 4, 64, 64, 2, 50, 32, True)              # rainbow_feature: CartPole, batch 32, double_q
    assert launcher == 223552 and launcher <= 227 * 1024                 # the count DESIGN 5g states
    # double_q costs nothing: the online forward of the next states uses the rows the target's forward takes afterwards
    assert smem_bytes(True, 4, 64, 64, 2, 50, 32, False) == launcher
    assert 0 < smem_bytes(False, 4, 64, 64, 2, 50, 32, True) < launcher  # no noise vectors, half the norm partials
    assert smem_bytes(True, 4, 64, 64, 2, 50, 33, True) > launcher
    assert smem_bytes(True, 4, 64, 64, 2, 50, 512, True) > 227 * 1024
    for bad in ((2, 4, 64, 64, 2, 50, 32, 0), (1, 4, 64, 64, 2, 50, 0, 0), (1, 4, 64, 64, 1, 50, 32, 0),
                (0, 4, 64, 64, 2, 1, 32, 0), (1, 4, 64, 64, 2, 257, 32, 0), (1, 4, 129, 64, 2, 50, 32, 0),
                (1, 4, 64, 129, 2, 50, 32, 0), (0, 257, 64, 64, 2, 50, 32, 0), (1, 4, 64, 64, 33, 50, 32, 0),
                (1, 0, 64, 64, 2, 50, 32, 0)):
        assert smem_bytes(*bad) == 0, bad


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def rl():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import deeprl_b200 as rl
    rl.select_device(0)
    rl.Config.COMPUTE_DTYPE = torch.float32
    return rl


def cabi_update(st, noisy, gate, batch, H1, H2, cfg, noise=None, seed=0, counter=None, std=0.5):
    """emul_update through the CUDA build (b2rl_rainbow_replay_update); st is updated in place.  Without ``noise`` the kernel
    draws; ``counter`` (int64 device tensor) is then its Philox position.  Returns also the target network's noise vector."""
    from deeprl_b200 import _lib
    cu = lambda x: torch.as_tensor(np.ascontiguousarray(x)).cuda()
    t = {k: cu(getattr(st, k)) for k in ("flat", "target", "sq", "ga")}
    s, s2, a, r, m, prob = (None if x is None else cu(x) for x in _batch_arrays(batch))
    B, D = s.shape
    step, loss = torch.as_tensor(st.step).cuda(), torch.zeros((), device="cuda")
    vec = torch.zeros(B, device="cuda")
    prio = torch.zeros(B, device="cuda") if prob is not None else None
    dims = (D, H1, H2, cfg["A"], cfg["K"])
    nz = noise_len(*dims)
    written = torch.zeros(nz + sum(o + o * i for i, o in layer_shapes(*dims)), device="cuda") if noisy else None
    tnoise = torch.zeros(nz, device="cuda") if noisy else None
    given = None if noise is None else cu(np.asarray(noise, np.float32))
    counter = torch.zeros(1, dtype=torch.int64, device="cuda") if counter is None else counter
    _lib.call("b2rl_rainbow_replay_update", int(noisy), gate, _lib.ptr(s), _lib.ptr(s2), int(s.dtype == torch.float64),
              cfg.get("coef", 1.0), _lib.ptr(a), _lib.ptr(r), _lib.ptr(m), B, *dims, _lib.ptr(t["flat"]), _lib.ptr(t["target"]),
              _lib.ptr(t["sq"]), _lib.ptr(t["ga"]), _lib.ptr(step), _lib.ptr(torch.from_numpy(st.off)), cfg["lr"], cfg["alpha"],
              cfg["eps"], int(cfg["centered"]), cfg["discount"] ** cfg["n_step"], int(cfg["double"]), cfg["vmin"], cfg["vmax"],
              cfg["clip"], _lib.ptr(prob), cfg.get("beta", 0.0), 0.01, 0.5, _lib.ptr(prio), _lib.ptr(vec), _lib.ptr(loss), seed,
              std, _lib.ptr(given), _lib.ptr(written), _lib.ptr(tnoise), _lib.ptr(counter), _lib.stream())
    torch.cuda.synchronize()
    st.flat, st.target, st.sq, st.ga = (t[k].cpu().numpy() for k in ("flat", "target", "sq", "ga"))
    st.step, st.loss = step.cpu().numpy(), loss.reshape(1).cpu().numpy()
    st.target_noise = None if tnoise is None else tnoise.cpu().numpy()
    return vec.cpu().numpy(), None if prio is None else prio.cpu().numpy(), None if written is None else written.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(CASES)))
def test_cabi_update_matches_oracle(rl, case):
    """The CUDA build of the same phases through the C ABI, the noise given; the counter does not move."""
    noisy, gate, dims, cfg, sd0, tgt0, batch, noise = case_setup(case)
    st = EmulState(noisy, sd0, tgt0)
    counter = torch.full((1,), 77, dtype=torch.int64, device="cuda")
    vec, prio, written = cabi_update(st, noisy, gate, batch, dims[1], dims[2], cfg, noise, counter=counter)
    check_against_oracle(case, st, vec, prio)
    assert int(counter) == 77
    if noisy:
        check_noise_arena(written, noise[1], dims)
        np.testing.assert_array_equal(st.target_noise, noise[0])


@pytest.mark.gpu
def test_golden_updates_cabi(rl, golden):
    """test_golden_updates_emulated and test_golden_twenty_consecutive_updates_emulated through the CUDA build."""
    g = golden("rainbow_agent")
    worst = check_golden_single_updates(g, cabi_update)
    chain = check_golden_chain(g, cabi_update)
    print("(CUDA) largest relative KL difference %.3g, largest parameter difference after 20 updates %.3g" % (worst, chain))


@pytest.mark.gpu
def test_drawn_noise(rl):
    """The noise the update kernel draws: the written epsilons are reset_noise's of the written vectors; the same key and
    counter give the same vectors, the next launch (the advanced counter) other ones; an update advances the counter by
    2 noise_len; target and online vectors differ; the draws are N(0, std^2) (Kolmogorov-Smirnov, fixed key)."""
    from scipy import stats
    noisy, gate, dims, cfg, sd0, tgt0, batch, _ = case_setup(0)
    nz, std = noise_len(*dims), 0.5
    runs = []
    for start in (0, 0, None):
        counter = runs[-1][3] if start is None else torch.zeros(1, dtype=torch.int64, device="cuda")
        st = EmulState(noisy, sd0, tgt0)
        _, _, written = cabi_update(st, noisy, gate, batch, dims[1], dims[2], cfg, None, seed=1234, counter=counter, std=std)
        runs.append((written, st.target_noise, st.flat.copy(), counter))
        check_noise_arena(written, written[:nz], dims)
    assert int(runs[0][3]) == 2 * nz and int(runs[2][3]) == 4 * nz
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])
    assert np.array_equal(runs[0][2], runs[1][2])                           # ... and the same update
    assert not np.array_equal(runs[0][0][:nz], runs[2][0][:nz]) and not np.array_equal(runs[0][1], runs[2][1])
    assert not np.array_equal(runs[0][0][:nz], runs[0][1])
    draws = np.concatenate([runs[0][1], runs[0][0][:nz], runs[2][1], runs[2][0][:nz]])
    assert draws.size > 2000
    p = stats.kstest(draws / std, "norm").pvalue
    assert p > 0.01, p
    assert abs(float(draws.std()) - std) < 0.03 and abs(float(draws.mean())) < 0.03
    # another std scales the same draws
    st = EmulState(noisy, sd0, tgt0)
    _, _, w2 = cabi_update(st, noisy, gate, batch, dims[1], dims[2], cfg, None, seed=1234, std=0.25)
    np.testing.assert_allclose(w2[:nz], runs[0][0][:nz] * 0.5, rtol=1e-6)


def _rainbow_net(rl, noisy, gate, D, H, A, K, seed=5):
    torch.manual_seed(seed)
    net = rl.RainbowNet(A, K, rl.FCBody(D, (H, H), gate=torch.tanh if gate == TANH else F.relu, noisy_linear=noisy), noisy)
    with torch.no_grad():                                   # action values far enough apart to be visible
        for m in (net.fc_advantage, net.fc_value):
            (m.weight_mu if noisy else m.weight).normal_(0, 0.5)
    return net


def _actor(rl, noisy, gate, N, D, H, A, K, vmin=-10.0, vmax=10.0):
    from deeprl_b200 import _lib, ops
    from deeprl_b200.component.actor import rainbow_kernel_order
    net = _rainbow_net(rl, noisy, gate, D, H, A, K)
    opt = ops.FlatOptimizer.from_torch(torch.optim.RMSprop(net.parameters(), 1e-3), list(net.parameters()))
    off = torch.tensor([(t.data_ptr() - opt.flat.data_ptr()) // 4 for t in rainbow_kernel_order(net)], dtype=torch.int32)
    atoms = torch.tensor(np.linspace(vmin, vmax, K), dtype=torch.float32, device="cuda")
    nz = noise_len(D, H, H, A, K)

    def q_values(x):                                        # CategoricalDQNActor._q_tensor
        with torch.no_grad():
            return (net(x.float())["prob"] * atoms).sum(-1)

    def step(obs, counter, ncounter, seed, eps, given=None, noise=None):
        act, used = torch.empty((N, 1), device="cuda"), torch.zeros(nz, device="cuda")
        _lib.call("b2rl_rainbow_actor_step", int(noisy), gate, _lib.ptr(obs), 1.0, _lib.ptr(opt.flat), _lib.ptr(off), D, H, H, A,
                  K, N, vmin, vmax, eps, _lib.ptr(act), _lib.ptr(given), seed, _lib.ptr(counter), 0.5, _lib.ptr(noise),
                  _lib.ptr(used), _lib.ptr(ncounter), _lib.stream())
        torch.cuda.synchronize()
        return act[:, 0].long(), used

    return net, q_values, step


def _set_noise(net, vec, dims):
    """What NoisyLinear.reset_noise does, with the given vectors instead of drawn ones."""
    nd = noise_dict(vec, *dims)
    mods = dict(zip(LAYERS, list(net.body.layers) + [net.fc_advantage, net.fc_value]))
    with torch.no_grad():
        for l, m in mods.items():
            n_in, n_ow, n_ob = (v.to(m.noise_in.device) for v in nd[l + "."])
            m.noise_in.copy_(n_in), m.noise_out_weight.copy_(n_ow), m.noise_out_bias.copy_(n_ob)
            m.weight_epsilon.copy_(torch.outer(m.transform_noise(n_ow), m.transform_noise(n_in)))
            m.bias_epsilon.copy_(m.transform_noise(n_ob))


@pytest.mark.gpu
@pytest.mark.parametrize("N,gate,A,K", [(1, RELU, 2, 50), (5, TANH, 5, 51)])
def test_noisy_actor_step(rl, N, gate, A, K):
    """NoisyLinear: with given noise the action is the eager RainbowNet's argmax of sum prob * atoms under the same noise (no
    row within 1e-3 of a tie), whatever epsilon; no epsilon uniform is consumed; drawn noise advances the noise counter by
    noise_len, given noise does not; given actions are written through."""
    D, H = 6, 32
    dims = (D, H, H, A, K)
    net, q_values, step = _actor(rl, True, gate, N, D, H, A, K)
    rng = np.random.RandomState(3)
    counter = torch.full((1,), 5, dtype=torch.int64, device="cuda")
    ncounter = torch.zeros(1, dtype=torch.int64, device="cuda")
    for trial in range(4):
        vec = (rng.randn(noise_len(*dims)) * 0.5).astype(np.float32)
        _set_noise(net, vec, dims)
        cand = torch.randn(512, D, dtype=torch.float64, device="cuda")
        top = q_values(cand).topk(2, dim=1).values
        obs = cand[(top[:, 0] - top[:, 1]) > 1e-3][:N].contiguous()
        assert obs.shape[0] == N
        act, used = step(obs, counter, ncounter, 11, 1.0, noise=torch.from_numpy(vec).cuda())
        assert torch.equal(act, q_values(obs).argmax(1)) and np.array_equal(used.cpu().numpy(), vec)
        assert int(counter) == 5 and int(ncounter) == 0
    _, used1 = step(obs, counter, ncounter, 11, 1.0)
    assert int(ncounter) == noise_len(*dims) and int(counter) == 5
    _, used2 = step(obs, counter, ncounter, 11, 1.0)
    assert int(ncounter) == 2 * noise_len(*dims) and not torch.equal(used1, used2)
    ncounter.zero_()
    _, again = step(obs, counter, ncounter, 11, 1.0)
    assert torch.equal(used1, again)
    given = torch.randint(0, A, (N, 1), device="cuda").float()
    assert torch.equal(step(obs, counter, ncounter, 3, 0.5, given)[0], given[:, 0].long())


@pytest.mark.gpu
def test_plain_actor_step_is_epsilon_greedy(rl):
    """nn.Linear layers: epsilon = 0 is the eager argmax; epsilon = 1 gives dist_actor_kernel's actions for the same key and
    counter (the same uniforms of stream 17); the counter advances by 2 N and the noise counter stays."""
    from deeprl_b200 import _lib, ops
    from deeprl_b200.component.actor import dqn_kernel_order
    N, D, H, A, K = 64, 6, 32, 5, 51
    net, q_values, step = _actor(rl, False, RELU, N, D, H, A, K)
    cand = torch.randn(4096, D, dtype=torch.float64, device="cuda")
    top = q_values(cand).topk(2, dim=1).values
    obs = cand[(top[:, 0] - top[:, 1]) > 1e-3][:N].contiguous()
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    ncounter = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert torch.equal(step(obs, counter, ncounter, 11, 0.0)[0], q_values(obs).argmax(1)) and int(counter) == 2 * N
    cnet = rl.CategoricalNet(A, K, rl.FCBody(D, (H, H)))
    copt = ops.FlatOptimizer.from_torch(torch.optim.RMSprop(cnet.parameters(), 1e-3), list(cnet.parameters()))
    coff = torch.tensor([(t.data_ptr() - copt.flat.data_ptr()) // 4 for t in dqn_kernel_order(cnet)], dtype=torch.int32)
    ccounter = counter.clone()
    seen = set()
    for _ in range(20):
        act = step(obs, counter, ncounter, 11, 1.0)[0]
        cact = torch.empty((N, 1), device="cuda")
        _lib.call("b2rl_dist_dqn_actor_step", 0, RELU, _lib.ptr(obs), 1.0, _lib.ptr(copt.flat), _lib.ptr(coff), D, H, H, A, K, N,
                  -10.0, 10.0, 1.0, _lib.ptr(cact), None, 11, _lib.ptr(ccounter), _lib.stream())
        torch.cuda.synchronize()
        assert torch.equal(act, cact[:, 0].long())
        seen |= set(act.tolist())
    assert seen == set(range(A)) and int(counter) == int(ccounter) == 2 * N * 21 and int(ncounter) == 0


def _agent_cfg(rl, noisy=True, per=True, async_replay=False, device=True, **kw):
    c = rl.Config()
    c.merge(dict(tag=None, n_step=3))
    c.device_rainbow = device
    c.noisy_linear = noisy
    c.task_fn = lambda: rl.Task("CartPole-v0", seed=7)
    c.eval_env = c.task_fn()
    c.batch_size, c.discount = 16, 0.99
    c.optimizer_fn = lambda p: torch.optim.RMSprop(p, lr=1e-3, alpha=0.95, eps=0.01, centered=per)
    c.categorical_v_min, c.categorical_v_max, c.categorical_n_atoms = -100, 100, 50
    c.network_fn = lambda: rl.RainbowNet(c.action_dim, c.categorical_n_atoms,
                                         rl.FCBody(c.state_dim, (32, 32), noisy_linear=c.noisy_linear), c.noisy_linear)
    rk = dict(memory_size=512, batch_size=16, n_step=3, discount=0.99)
    c.replay_fn = lambda: rl.ReplayWrapper(rl.PrioritizedReplay if per else rl.UniformReplay, rk, async_replay)
    c.replay_eps, c.replay_alpha, c.replay_beta = 0.01, 0.5, rl.LinearSchedule(0.4, 1.0, 200)
    c.random_action_prob = rl.LinearSchedule(1.0, 0.1, 100)
    c.target_network_update_freq, c.exploration_steps = 5, 40
    c.sgd_update_frequency, c.gradient_clip, c.async_actor, c.double_q = 4, 10, False, True
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _params(net):
    return np.concatenate([p.detach().cpu().numpy().ravel() for p in net.parameters()])


def _noise_sequence(nz):
    """Network-level noise draw i of a run, the same for every agent that counts its draws."""
    return lambda i: (np.random.RandomState(5000 + i).randn(nz) * 0.5).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("per", [False, True])
@pytest.mark.parametrize("async_replay", [False, True])
def test_eager_and_device_agents_agree(rl, per, async_replay):
    """The same forced actions, noise sequence, replay seed and env seed: an eager agent (its networks' reset_noise reading
    the sequence: one vector per env step for the online network, then per update the target's and the online one's) and a
    device agent agree to 1e-4 on all parameters after 50 updates; afterwards the device agent's noise buffers are those of
    its last update, eval_step runs and save / load round-trips."""
    import deeprl_b200.agent.DQN_agent as dqn_mod
    rng = np.random.RandomState(0)
    forced = rng.randint(0, 2, size=100000)
    agents_ = []
    for device in (False, True):
        torch.manual_seed(1)
        agents_.append(rl.CategoricalDQNAgent(_agent_cfg(rl, True, per, async_replay, device)))
    eager, dev = agents_
    assert eager.device_dqn is None and type(dev.device_dqn).__name__ == "DeviceRainbow"
    dev.network.load_state_dict(eager.network.state_dict())
    dev.target_network.load_state_dict(eager.target_network.state_dict())
    init = _params(eager.network)
    dims = (4, 32, 32, 2, 50)
    nz = noise_len(*dims)
    assert dev.device_dqn.noise_len == nz
    seq = _noise_sequence(nz)
    k = [0, 0, 0, 0]                                           # actions eager / device, noise draws eager / device

    def forced_eager(eps, q):
        assert eps == 0
        a = forced[k[0]:k[0] + q.shape[0]]
        k[0] += q.shape[0]
        return a

    def reset_from_sequence(net):
        def reset_noise():
            _set_noise(net, seq(k[2]), dims)
            k[2] += 1
        return reset_noise

    eager.network.reset_noise = reset_from_sequence(eager.network)
    eager.target_network.reset_noise = reset_from_sequence(eager.target_network)
    last = {}

    def forced_noise(n):
        v = np.concatenate([seq(k[3] + j) for j in range(n)])
        k[3] += n
        last["v"] = v
        return v

    orig = dqn_mod.epsilon_greedy
    dqn_mod.epsilon_greedy = forced_eager
    try:
        def nxt():
            a = forced[k[1]:k[1] + 1]
            k[1] += 1
            return a
        dev.device_dqn.forced = nxt
        dev.device_dqn.forced_noise = forced_noise
        steps = 40 // 4 + 50
        for _ in range(steps):
            eager.step()
            dev.step()
    finally:
        dqn_mod.epsilon_greedy = orig
    torch.cuda.synchronize()
    assert k[2] == k[3] == 4 * steps + 2 * 50 and last["v"].size == 2 * nz
    ri, rd = getattr(eager.replay, "replay", eager.replay), getattr(dev.replay, "replay", dev.replay)
    assert ri.size() == rd.size()
    err = float(np.abs(_params(eager.network) - _params(dev.network)).max())
    err_t = float(np.abs(_params(eager.target_network) - _params(dev.target_network)).max())
    assert err <= 1e-4 and err_t <= 1e-4, (err, err_t)
    assert abs(float(eager.last_loss) - float(dev.last_loss)) <= 1e-4 * max(1.0, abs(float(eager.last_loss)))
    assert int(dev._flat.step_dev) == 50 and np.abs(_params(dev.network) - init).max() > 1e-4
    assert int(dev.device_dqn.noise_counter) == 0                # all noise was given: nothing drawn
    # the module's buffers are the online noise of the last update, which is also the eager network's
    want = last["v"][nz:]
    for m_dev, m_eager in zip(list(dev.network.body.layers) + [dev.network.fc_advantage, dev.network.fc_value],
                              list(eager.network.body.layers) + [eager.network.fc_advantage, eager.network.fc_value]):
        for b in ("noise_in", "noise_out_weight", "noise_out_bias", "weight_epsilon", "bias_epsilon"):
            np.testing.assert_allclose(getattr(m_dev, b).cpu().numpy(), getattr(m_eager, b).cpu().numpy(), rtol=5e-7, atol=0)
    np.testing.assert_array_equal(dev.device_dqn.noise[:nz].cpu().numpy(), want)
    state = [np.asarray([0.01, -0.02, 0.03, 0.04])]
    assert dev.eval_step(state).shape == (1,) and np.array_equal(dev.eval_step(state), eager.eval_step(state))
    eager.close()
    dev.close()


@pytest.mark.gpu
def test_save_and_load_round_trip(rl, tmp_path):
    """save() writes the arena's parameters and the noise buffers of the latest update; load() into another device agent
    restores them in place (the parameters stay views into the arenas)."""
    a = rl.CategoricalDQNAgent(_agent_cfg(rl))
    while a.total_steps <= a.config.exploration_steps + 16:
        a.step()
    torch.cuda.synchronize()
    assert float(a.device_dqn.noise.abs().max()) > 0 and int(a.device_dqn.noise_counter) > 0
    a.save(str(tmp_path / "rb"))
    b = rl.CategoricalDQNAgent(_agent_cfg(rl))
    b.load(str(tmp_path / "rb"))
    for (ka, va), (kb, vb) in zip(a.network.state_dict().items(), b.network.state_dict().items()):
        assert ka == kb and torch.equal(va, vb), ka
    assert torch.equal(a.device_dqn.noise, b.device_dqn.noise) and torch.equal(a.device_dqn.opt.flat, b.device_dqn.opt.flat)
    b.device_dqn._offsets()                                      # still in the arenas
    b.step()
    a.close()
    b.close()


def _launcher_agent(monkeypatch):
    import examples
    got = []
    monkeypatch.setattr(examples, "run_steps", got.append)
    examples.rainbow_feature(game="CartPole-v0", device_rainbow=True)
    return got[0]


@pytest.mark.gpu
def test_launcher_end_to_end(rl, monkeypatch):
    """rainbow_feature with its own configuration (NoisyLinear, batch 32, double_q, PER, n_step 3, clip 10, async actor, async
    replay) and the device flag, past its exploration steps: finite, varying losses; the noise counter moves; after a
    scheduled sync the target arena equals the online arena exactly, otherwise it is unchanged; one profiled step() lists
    sgd_update_frequency actor kernels, one update kernel, and besides them only the replay's kernels -- no normal_ / outer /
    elementwise noise kernel."""
    import time
    ag = _launcher_agent(monkeypatch)
    c, dev = ag.config, ag.device_dqn
    assert c.async_actor and c.noisy_linear and c.double_q and c.n_step == 3 and c.batch_size == 32 and c.gradient_clip == 10
    assert getattr(ag.replay, "async_", False) and type(dev).__name__ == "DeviceRainbow" and dev.noisy == 1
    assert (dev.D, dev.H1, dev.H2, dev.A, dev.K) == (4, 64, 64, 2, 50)
    losses_, syncs = [], 0
    while ag.total_steps <= c.exploration_steps + 4 * c.target_network_update_freq + 40:
        target = dev.target.clone()
        ag.step()
        torch.cuda.synchronize()
        if ag.total_steps / c.sgd_update_frequency % c.target_network_update_freq == 0:
            assert torch.equal(dev.target, dev.opt.flat)
            syncs += 1
        else:
            assert torch.equal(dev.target, target)
        if ag.last_loss is not None:
            losses_.append(float(ag.last_loss))
    assert syncs >= 2 and len(losses_) > 10 and all(np.isfinite(losses_)) and len(set(losses_)) > 1
    assert int(dev.noise_counter) >= dev.noise_len * (ag.total_steps + 2 * len(losses_)) and int(dev.counter) == 0

    actor = ag.actor                                            # (the actor thread runs ahead: test_dist_dqn_device.py)
    while True:
        while not actor._queue.full():
            time.sleep(0.001)
        n = actor._total_steps
        time.sleep(0.05)
        if actor._total_steps == n and actor._queue.full():
            break

    def step():
        n0 = actor._total_steps
        ag.step()
        while actor._total_steps < n0 + c.sgd_update_frequency:
            time.sleep(0.0005)
        time.sleep(0.01)
        assert actor._total_steps == n0 + c.sgd_update_frequency
        torch.cuda.synchronize()

    step()
    from _kernel_trace import profiled_kernels
    kernels = profiled_kernels(step, {"rainbow_actor_kernel": c.sgd_update_frequency, "rainbow_replay_update_kernel": 1,
                                     "feed_kernel": 1, "gather": 1, "sumtree_sample": 1, "direct_copy": 1})
    assert sum("rainbow_actor_kernel" in k for k in kernels) == c.sgd_update_frequency, kernels
    assert sum("rainbow_replay_update_kernel" in k for k in kernels) == 1, kernels
    others = [k for k in kernels if "rainbow_actor_kernel" not in k and "rainbow_replay_update_kernel" not in k]
    # the replay's own kernels (feed, sum-tree draw and update, gather) and its float64 -> float32 cast of the sampling
    # probabilities (replay.py _select_per); no torch noise, forward, backward or optimizer kernel
    foreign = [k for k in others if not k.startswith("b2rl::")]
    assert len(foreign) == 1 and "direct_copy" in foreign[0], others
    assert any("feed_kernel" in k for k in others) and any("gather" in k for k in others), others
    assert any("sumtree_sample" in k for k in others), others
    ag.close()


@pytest.mark.gpu
def test_unsupported_configurations_are_refused(rl):
    class OwnLoss(rl.CategoricalDQNAgent):
        def reduce_loss(self, loss):
            return loss.sum()

    C, Q, D_ = rl.CategoricalDQNAgent, rl.QuantileRegressionDQNAgent, rl.DQNAgent
    rb = lambda body, noisy=True, A=2, K=50: (lambda: rl.RainbowNet(A, K, body(), noisy))
    refused = [
        (C, dict(network_fn=lambda: rl.CategoricalNet(2, 50, rl.FCBody(4))), "CategoricalNet"),
        (C, dict(network_fn=rb(lambda: rl.NatureConvBody(in_channels=4, noisy_linear=True))), "NatureConvBody"),
        (C, dict(network_fn=rb(lambda: rl.FCBody(4, (64, 64, 64), noisy_linear=True))), "two-layer"),
        (C, dict(network_fn=rb(lambda: rl.FCBody(4, noisy_linear=False))), "not a mix"),
        (C, dict(network_fn=rb(lambda: rl.FCBody(4, noisy_linear=True), noisy=False)), "not a mix"),
        (C, dict(noisy_linear=False, network_fn=rb(lambda: rl.FCBody(4, noisy_linear=True))), "not a mix"),
        (C, dict(optimizer_fn=lambda p: torch.optim.Adam(p, 1e-3)), "Adam"),
        (C, dict(state_normalizer=rl.MeanStdNormalizer()), "MeanStdNormalizer"),
        (C, dict(history_length=4), "frame stacks"),
        (OwnLoss, {}, "reduce_loss"),
        (C, dict(batch_size=512), "shared memory"),
        (C, dict(network_fn=rb(lambda: rl.FCBody(4, noisy_linear=True), K=300)), "atoms 300"),
        (C, dict(network_fn=rb(lambda: rl.FCBody(4, (256, 64), noisy_linear=True))), "hidden 256"),
        (C, dict(device_c51=True), "device_rainbow and config.device_c51"),
        (C, dict(device_dqn=True), "device_rainbow and config.device_dqn"),
        (Q, dict(num_quantiles=20, network_fn=lambda: rl.QuantileNet(2, 20, rl.FCBody(4))), "QuantileRegressionDQNAgent"),
        (D_, dict(network_fn=lambda: rl.VanillaNet(2, rl.FCBody(4))), "DQNAgent"),
    ]
    for cls, kw, msg in refused:
        with pytest.raises(NotImplementedError, match=msg):
            cls(_agent_cfg(rl, **kw))
    # the other flags keep refusing a RainbowNet with their own messages
    with pytest.raises(NotImplementedError, match="device_c51: the network is a RainbowNet"):
        C(_agent_cfg(rl, device=False, device_c51=True))
    with pytest.raises(NotImplementedError, match="device_dqn: the network is a RainbowNet"):
        C(_agent_cfg(rl, device=False, device_dqn=True))
    for noisy in (True, False):                                   # the supported forms build, with the async actor too
        for async_actor in (False, True):
            ag = C(_agent_cfg(rl, noisy=noisy, async_actor=async_actor))
            assert ag.device_dqn is not None and ag.device_dqn.noisy == int(noisy)
            ag.step()
            ag.close()
