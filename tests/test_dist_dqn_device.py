"""C51 and QR-DQN on the device (``config.device_c51`` / ``config.device_qr``; deeprl_b200/csrc/dist_dqn.cu): one
``b2rl_dist_dqn_actor_step`` launch per env step and ONE ``b2rl_dist_dqn_replay_update`` launch per gradient update of
CategoricalDQN_agent.py:60-89 / QuantileRegressionDQN_agent.py:55-77, for a CategoricalNet or QuantileNet on a two-layer FCBody.

CPU: the update's phase functions (csrc/dist_phases.h on a2c_phases.h's HEAD = Q phases, dist_sequence.inc) are compiled for
the host by tests/host_emul/dist_emul.cpp and run with the block's threads in sequence, against the reference's recorded
losses (tests/golden/agent_steps.npz ``c51`` / ``qr``: the per-sample KL / the loss vector of each of 20 updates) and against
oracle/agents.py DQNFamilyOracle with RMSprop.
GPU: the CUDA build of the same source through the C ABI and through the agents; the actor step's epsilon-greedy.

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
from oracle import agents  # noqa: E402

TANH, RELU = 0, 1
C51, QR = 0, 1
HEAD = {C51: "fc_categorical", QR: "fc_quantiles"}
BODY = ["body.layers.0.weight", "body.layers.0.bias", "body.layers.1.weight", "body.layers.1.bias"]
KEYS = {k: BODY + [HEAD[k] + ".weight", HEAD[k] + ".bias"] for k in (C51, QR)}      # the kernels' tensor order
P = ctypes.c_void_p


def vp(x):
    return None if x is None else P(x.ctypes.data)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("dist_emul") / "dist_emul.so")
    subprocess.run(["g++", "-O2", "-fno-strict-aliasing", "-std=c++17", "-shared", "-fPIC", "-o", out,
                    os.path.join(ROOT, "tests", "host_emul", "dist_emul.cpp")], check=True)
    lib = ctypes.CDLL(out)
    i32, f32, f64 = ctypes.c_int32, ctypes.c_float, ctypes.c_double
    lib.dist_emul_update.argtypes = ([i32, i32, P, P, i32, f64, P, P, P] + [i32] * 6 + [P] * 6 + [f32] * 3
                                     + [i32, f32, i32, f64, f64, f32, P] + [f32] * 3 + [P] * 3 + [i32, i32])
    return lib


def arena(sd, keys):
    """FlatOptimizer's layout (ops.py): every tensor starts on a multiple of 4 elements."""
    offs, n = [], 0
    for k in keys:
        offs.append(n)
        n += (sd[k].numel() + 3) // 4 * 4
    flat = np.zeros(n, np.float32)
    for k, o in zip(keys, offs):
        flat[o:o + sd[k].numel()] = np.asarray(sd[k].detach() if torch.is_tensor(sd[k]) else sd[k]).ravel()
    return flat, np.asarray(offs, np.int32)


def unflatten(flat, offs, sd, keys):
    return {k: flat[o:o + sd[k].numel()].reshape(tuple(sd[k].shape)) for k, o in zip(keys, offs)}


class EmulState:
    """Online arena, target arena, RMSprop moments and step count, carried across updates."""

    def __init__(self, kind, sd, target_sd=None):
        self.keys = KEYS[kind]
        self.flat, self.off = arena(sd, self.keys)
        self.target = arena(target_sd if target_sd is not None else sd, self.keys)[0]
        self.sq, self.ga = np.zeros_like(self.flat), np.zeros_like(self.flat)
        self.step = np.zeros(1, np.int64)
        self.loss = np.zeros(1, np.float32)


def emul_update(lib, st, kind, gate, batch, H1, H2, cfg, threads=512, reversed_=False):
    """One b2rl_dist_dqn_replay_update on the host.  batch: dict of numpy arrays state / next_state (B, D; float32 or
    float64), action, reward, mask, and for PER sampling_prob.  Returns (loss vector, priority)."""
    s = np.ascontiguousarray(batch["state"])
    s2 = np.ascontiguousarray(batch["next_state"], dtype=s.dtype)
    B, D = s.shape
    a = np.ascontiguousarray(batch["action"], np.int64)
    r, m = (np.ascontiguousarray(batch[k], np.float32) for k in ("reward", "mask"))
    prob = batch.get("sampling_prob")
    prob = None if prob is None else np.ascontiguousarray(prob, np.float32)
    prio = np.zeros(B, np.float32) if prob is not None else None
    vec = np.zeros(B if kind == C51 else cfg["K"], np.float32)
    rc = lib.dist_emul_update(kind, gate, vp(s), vp(s2), int(s.dtype == np.float64), cfg.get("coef", 1.0), vp(a), vp(r), vp(m),
                              B, D, H1, H2, cfg["A"], cfg["K"], vp(st.flat), vp(st.target), vp(st.sq), vp(st.ga), vp(st.step),
                              vp(st.off), cfg["lr"], cfg["alpha"], cfg["eps"], int(cfg["centered"]),
                              cfg["discount"] ** cfg["n_step"], int(cfg["double"]), cfg["vmin"], cfg["vmax"], cfg["clip"],
                              vp(prob), cfg.get("beta", 0.0), 0.01, 0.5, vp(prio), vp(vec), vp(st.loss), threads,
                              int(reversed_))
    assert rc == 0
    return vec, prio


# ------------------------------------------------------------------------------------------------ golden records
GOLDEN = {"c51": dict(kind=C51, K=50), "qr": dict(kind=QR, K=20)}
GOLDEN_CFG = dict(lr=0.00025, alpha=0.95, eps=0.01, centered=True, clip=5.0, discount=0.99, n_step=1, A=2, vmin=-100.0,
                  vmax=100.0, double=False)


def golden_batch(g, pre, i):
    return {f: g[pre + "b_" + f][i] for f in ("state", "next_state", "action", "reward", "mask")}


def golden_sd(g, pre, flat):
    """The recorded parameter vector (keys order) as a state dict."""
    keys = [str(k) for k in g[pre + "keys"]]
    out, o = {}, 0
    for k in keys:
        shape = g[pre + "init." + k].shape
        n = int(np.prod(shape))
        out[k] = torch.from_numpy(np.asarray(flat[o:o + n]).reshape(shape).copy())
        o += n
    return out


def golden_synced(g, pre):
    """The updates after which the reference synced its target network (the recorded target changed)."""
    t = g[pre + "target"]
    init = np.concatenate([g[pre + "init." + str(k)].ravel() for k in g[pre + "keys"]])
    return [i for i in range(t.shape[0]) if not np.array_equal(t[i], t[i - 1] if i else init)]


@pytest.mark.parametrize("name", ["c51", "qr"])
def test_golden_losses_emulated(emul, golden, name):
    """Each of the reference's 20 recorded updates from its recorded online / target parameters before the update: the
    per-sample KL [16] (C51) / the loss vector [20] (QR) equal the recorded ones (1e-5 relative, 2e-6 absolute floor)."""
    g = golden("agent_steps")
    pre = name + "_"
    kind, K = GOLDEN[name]["kind"], GOLDEN[name]["K"]
    cfg = dict(GOLDEN_CFG, K=K)
    keys = [str(k) for k in g[pre + "keys"]]
    init = {k: torch.from_numpy(g[pre + "init." + k]) for k in keys}
    worst = 0.0
    for i in range(g[pre + "delta"].shape[0]):
        on = init if i == 0 else golden_sd(g, pre, g[pre + "params"][i - 1])
        tg = init if i == 0 else golden_sd(g, pre, g[pre + "target"][i - 1])
        st = EmulState(kind, on, tg)
        vec, _ = emul_update(emul, st, kind, RELU, golden_batch(g, pre, i), 32, 32, cfg)
        want = g[pre + "delta"][i]
        np.testing.assert_allclose(vec, want, rtol=1e-5, atol=2e-6, err_msg=str(i))
        worst = max(worst, float((np.abs(vec - want) / np.maximum(np.abs(want), 2e-6 / 1e-5)).max()))
    print("%s: largest relative difference of the loss over the 20 golden updates: %.3g" % (name, worst))


def _oracle(kind, sd, tgt, A, K, cfg, gate):
    o = agents.DQNFamilyOracle(
        {k: v.clone() for k, v in sd.items()}, "categorical" if kind == C51 else "quantile", "fc", A,
        lambda p: torch.optim.RMSprop(p, cfg["lr"], alpha=cfg["alpha"], eps=cfg["eps"], centered=cfg["centered"]),
        cfg["discount"], n_step=cfg["n_step"], double_q=cfg["double"], gradient_clip=cfg["clip"],
        state_coef=cfg.get("coef", 1.0), atoms=np.linspace(cfg["vmin"], cfg["vmax"], K) if kind == C51 else None,
        v_min=cfg["vmin"], v_max=cfg["vmax"], num_quantiles=K if kind == QR else None, replay_eps=0.01, replay_alpha=0.5,
        replay_beta=lambda: cfg.get("beta", 0.0), gate=torch.tanh if gate == TANH else F.relu)
    for k in o.target_sd:
        o.target_sd[k].copy_(tgt[k])
    return o


class _Tr:
    def __init__(self, **kw):
        self.__dict__.update(kw)


@pytest.mark.parametrize("name", ["c51", "qr"])
def test_golden_batches_twenty_updates_emulated(emul, golden, name):
    """20 consecutive updates from the recorded init on the recorded batches, the target synced on the recorded schedule,
    against the oracle with the same RMSprop: loss vector and loss after each update, online and target parameters (1e-5)."""
    g = golden("agent_steps")
    pre = name + "_"
    kind, K = GOLDEN[name]["kind"], GOLDEN[name]["K"]
    cfg = dict(GOLDEN_CFG, K=K)
    keys = [str(k) for k in g[pre + "keys"]]
    sd0 = {k: torch.from_numpy(g[pre + "init." + k]) for k in keys}
    st = EmulState(kind, sd0)
    o = _oracle(kind, sd0, sd0, 2, K, cfg, RELU)
    synced = golden_synced(g, pre)
    assert len(synced) >= 3, synced
    worst = 0.0
    for i in range(g[pre + "delta"].shape[0]):
        b = golden_batch(g, pre, i)
        vec, _ = emul_update(emul, st, kind, RELU, b, 32, 32, cfg)
        tr = _Tr(**b)
        with torch.no_grad():
            want = o.compute_loss(tr).numpy()
        loss = float(o.update(tr))
        np.testing.assert_allclose(vec, want, rtol=1e-5, atol=2e-6)
        np.testing.assert_allclose(st.loss[0], loss, rtol=1e-5, atol=1e-7)
        if i in synced:
            st.target[...] = st.flat
            o.sync_target()
        got, got_t = unflatten(st.flat, st.off, sd0, st.keys), unflatten(st.target, st.off, sd0, st.keys)
        for k in st.keys:
            err = float(np.abs(got[k] - o.sd[k].detach().numpy()).max())
            err_t = float(np.abs(got_t[k] - o.target_sd[k].numpy()).max())
            worst = max(worst, err, err_t)
            assert err <= 1e-5 and err_t <= 1e-5, (i, k, err, err_t)
    assert int(st.step[0]) == 20
    print("%s: largest parameter difference to the oracle over 20 updates: %.3g" % (name, worst))


# ------------------------------------------------------------------------------------------------ ragged shapes and the oracle
def max_batch(kind, D, H1, H2, A, K, double):
    from deeprl_b200 import _lib
    L = _lib.lib()
    B = 1
    while L.b2rl_dist_dqn_smem_bytes(kind, D, H1, H2, A, K, B + 1, int(double)) <= 227 * 1024:
        B += 1
    return B


CFG = dict(lr=1e-3, alpha=0.99, eps=1e-6, centered=False, discount=0.99, clip=5.0, n_step=1, double=False, per=False, coef=1.0,
           vmin=-100.0, vmax=100.0)
# (RMSprop's first step moves a parameter by about lr / sqrt(1 - alpha) whatever the size of its gradient, unless the gradient
# is near eps: with eps = 1e-8 a gradient of ~1e-8 carries the fp32 rounding of its sum into the parameter, so eps is 1e-6)
CASES = [  # (kind, gate, D, A, K, H1, H2, B, float64 states, cfg overrides)
    (C51, RELU, 4, 2, 50, 64, 64, 10, True, {}),                                                  # categorical_dqn_feature
    (C51, TANH, 11, 5, 20, 32, 48, 37, True, dict(double=True, per=True, centered=True, clip=1e6, n_step=3, coef=0.5)),
    (C51, RELU, 7, 18, 2, 16, 24, 1, False, dict(per=True, clip=0.05, vmin=-3.0, vmax=3.0)),
    (C51, TANH, 6, 18, 51, 8, 8, "max", False, dict(double=True, centered=True, clip=0.05, vmin=-10.0, vmax=10.0)),
    (C51, RELU, 4, 2, 51, 32, 32, "max", True, dict(double=True, per=True, clip=1e6, n_step=3, vmin=-10.0, vmax=10.0)),
    (QR, RELU, 4, 2, 20, 64, 64, 10, True, {}),                                                   # quantile_regression_dqn_feature
    (QR, TANH, 9, 5, 50, 40, 24, 37, False, dict(centered=True, clip=0.05, n_step=3, coef=0.25)),
    (QR, RELU, 5, 18, 2, 24, 32, 1, True, dict(centered=True, clip=1e6)),
    (QR, TANH, 6, 18, 51, 8, 8, "max", True, dict(clip=0.05)),
    (QR, RELU, 4, 2, 20, 64, 64, "max", False, dict(double=True, n_step=3, clip=1e6)),             # double_q: ignored
]


def make_problem(kind, D, A, K, H1, H2, B, f64, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale

    def net():
        return {"body.layers.0.weight": r(H1, D, scale=D ** -0.5), "body.layers.0.bias": r(H1, scale=0.1),
                "body.layers.1.weight": r(H2, H1, scale=H1 ** -0.5), "body.layers.1.bias": r(H2, scale=0.1),
                HEAD[kind] + ".weight": r(A * K, H2, scale=H2 ** -0.5), HEAD[kind] + ".bias": r(A * K, scale=0.1)}

    sd, target = net(), net()
    dt = np.float64 if f64 else np.float32
    batch = dict(state=r(B, D, scale=2.0).double().numpy().astype(dt), next_state=r(B, D, scale=2.0).double().numpy().astype(dt),
                 action=torch.randint(0, A, (B,), generator=g).numpy(), reward=r(B, scale=3.0).numpy(),
                 mask=(torch.rand(B, generator=g) > 0.2).float().numpy(),
                 sampling_prob=(torch.rand(B, generator=g) * 0.01 + 1e-4).numpy())
    return sd, target, batch


def case_setup(case):
    kind, gate, D, A, K, H1, H2, B, f64, over = CASES[case]
    cfg = dict(CFG, A=A, K=K, **over)
    if B == "max":
        B = max_batch(kind, D, H1, H2, A, K, cfg["double"])
    cfg["beta"] = 0.55 if cfg["per"] else 0.0
    sd0, tgt0, batch = make_problem(kind, D, A, K, H1, H2, B, f64, seed=700 + case)
    if not cfg["per"]:
        del batch["sampling_prob"]
    return kind, gate, H1, H2, cfg, sd0, tgt0, batch


def run_case(lib, case, threads=512, reversed_=False):
    kind, gate, H1, H2, cfg, sd0, tgt0, batch = case_setup(case)
    st = EmulState(kind, sd0, tgt0)
    vec, prio = emul_update(lib, st, kind, gate, batch, H1, H2, cfg, threads, reversed_)
    return st, vec, prio


def oracle_update(case):
    """One update by the oracle.  Returns (oracle, cfg, loss, loss vector, priorities, gradient norm after the clip, ...)."""
    kind, gate, H1, H2, cfg, sd0, tgt0, batch = case_setup(case)
    o = _oracle(kind, sd0, tgt0, cfg["A"], cfg["K"], cfg, gate)
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
    clipped = float(torch.sqrt(sum((p.grad.double() ** 2).sum() for p in o.params)))
    prio = np.asarray([prios[i] for i in range(len(prios))], np.float32) if cfg["per"] else None
    return o, cfg, float(loss), vec, prio, clipped, sd0, tgt0


def check_against_oracle(case, st, vec, prio, atol=1e-5):
    o, cfg, loss, v_want, p_want, clipped, sd0, tgt0 = oracle_update(case)
    np.testing.assert_allclose(vec, v_want, rtol=1e-5, atol=2e-6)
    if cfg["per"]:
        np.testing.assert_allclose(prio, p_want, rtol=1e-5, atol=1e-6)
    got, got_t = unflatten(st.flat, st.off, sd0, st.keys), unflatten(st.target, st.off, sd0, st.keys)
    sq, ga = unflatten(st.sq, st.off, sd0, st.keys), unflatten(st.ga, st.off, sd0, st.keys)
    for k in st.keys:
        want = o.sd[k].detach().numpy()
        np.testing.assert_allclose(got[k], want, rtol=0, atol=atol, err_msg=k)
        assert np.abs(want - sd0[k].numpy()).max() > 1e-6, k                 # every tensor moved
        np.testing.assert_array_equal(got_t[k], tgt0[k].numpy(), err_msg=k)  # the target arena is only read
        s = o.opt.state[o.sd[k]]
        np.testing.assert_allclose(sq[k], s["square_avg"].numpy(), rtol=2e-3, atol=1e-12, err_msg=k)
        if cfg["centered"]:
            np.testing.assert_allclose(ga[k], s["grad_avg"].numpy(), rtol=2e-3, atol=1e-8, err_msg=k)
    np.testing.assert_allclose(st.loss[0], loss, rtol=1e-5, atol=1e-7)
    assert int(st.step[0]) == 1
    return cfg, clipped


@pytest.mark.parametrize("case", range(len(CASES)))
def test_update_matches_oracle_emulated(emul, case):
    st, vec, prio = run_case(emul, case)
    cfg, clipped = check_against_oracle(case, st, vec, prio)
    if cfg["clip"] < 1.0:
        assert abs(clipped - cfg["clip"]) < 1e-4 * cfg["clip"]              # the clip was active
    elif cfg["clip"] >= 1e5:
        assert clipped < cfg["clip"]                                         # ... and here it was not


def test_cases_cover_the_shapes():
    setups = [case_setup(c) for c in range(len(CASES))]
    for kind in (C51, QR):
        sizes = {s[-1]["action"].shape[0] for s in setups if s[0] == kind}
        assert {1, 10, 37} <= sizes and max(sizes) > 37, sizes
        assert {s[4]["A"] for s in setups if s[0] == kind} == {2, 5, 18}
        assert {s[4]["K"] for s in setups if s[0] == kind} == {2, 20, 50, 51}
        assert {s[1] for s in setups if s[0] == kind} == {TANH, RELU}
    assert {(s[4]["double"], s[4]["per"]) for s in setups if s[0] == C51} == {(False, False), (True, True), (False, True),
                                                                               (True, False)}


@pytest.mark.parametrize("case", [1, 3, 6, 8])
def test_thread_order_and_count_do_not_change_the_result(emul, case):
    """Reversed thread order inside every phase, 64 and 37 threads instead of 512: bit-identical arenas (the race check)."""
    ref, v_ref, p_ref = run_case(emul, case)
    for threads, rev in ((512, True), (64, False), (37, True)):
        got, v, p = run_case(emul, case, threads, rev)
        for k in ("flat", "target", "sq", "ga", "loss", "step"):
            assert np.array_equal(getattr(ref, k), getattr(got, k)), (threads, rev, k)
        assert np.array_equal(v_ref, v) and (p_ref is None or np.array_equal(p_ref, p))


def test_kernels_have_no_spills_and_no_stack_frame(tmp_path):
    cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-o", str(tmp_path / "d.cubin"),
           os.path.join(ROOT, "deeprl_b200", "csrc", "dist_dqn.cu"), "-Xptxas", "-v"]
    out = subprocess.run(cmd, check=True, capture_output=True, text=True).stderr
    entries = out.split("Compiling entry function")[1:]
    names = [e.split("'")[1] for e in entries]
    # (C51, QR) x (tanh, ReLU), the update and the actor step
    assert sum("dist_replay_update_kernel" in n for n in names) == 4, names
    assert sum("dist_actor_kernel" in n for n in names) == 4, names
    assert len(names) == 8, names
    for e in entries:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in e, e


def test_shared_memory_budget_accepts_the_launchers():
    from deeprl_b200 import _lib
    L = _lib.lib()
    c51 = L.b2rl_dist_dqn_smem_bytes(C51, 4, 64, 64, 2, 50, 10, 0)         # categorical_dqn_feature: CartPole, batch 10
    qr = L.b2rl_dist_dqn_smem_bytes(QR, 4, 64, 64, 2, 20, 10, 0)           # quantile_regression_dqn_feature
    assert 0 < qr < c51 <= 227 * 1024, (c51, qr)
    assert L.b2rl_dist_dqn_smem_bytes(QR, 4, 64, 64, 2, 20, 10, 1) == qr   # QR ignores double_q
    assert L.b2rl_dist_dqn_smem_bytes(C51, 4, 64, 64, 2, 50, 10, 1) > c51
    assert L.b2rl_dist_dqn_smem_bytes(C51, 4, 64, 64, 2, 50, 512, 0) > 227 * 1024
    assert L.b2rl_dist_dqn_smem_bytes(QR, 4, 64, 64, 2, 20, 512, 0) > 227 * 1024
    for bad in ((2, 4, 64, 64, 2, 50, 10, 0), (C51, 4, 64, 64, 2, 50, 0, 0), (C51, 4, 64, 64, 1, 50, 10, 0),
                (QR, 4, 64, 64, 2, 1, 10, 0), (QR, 4, 64, 64, 2, 257, 10, 0), (C51, 4, 129, 64, 2, 50, 10, 0),
                (C51, 257, 64, 64, 2, 50, 10, 0), (QR, 4, 64, 64, 33, 20, 10, 0), (QR, 0, 64, 64, 2, 20, 10, 0)):
        assert L.b2rl_dist_dqn_smem_bytes(*bad) == 0, bad


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def rl():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import deeprl_b200 as rl
    rl.select_device(0)
    rl.Config.COMPUTE_DTYPE = torch.float32
    return rl


def cabi_update(st, kind, gate, batch, H1, H2, cfg):
    """emul_update through the CUDA build (b2rl_dist_dqn_replay_update); st is updated in place."""
    from deeprl_b200 import _lib
    cu = lambda x: torch.as_tensor(np.ascontiguousarray(x)).cuda()
    t = {k: cu(getattr(st, k)) for k in ("flat", "target", "sq", "ga")}
    b = {k: cu(v if k in ("state", "next_state", "action") else np.asarray(v, np.float32)) for k, v in batch.items()}
    b["state"], b["next_state"] = b["state"], b["next_state"].to(b["state"].dtype)
    b["action"] = b["action"].long()
    B = b["action"].shape[0]
    step, loss = torch.as_tensor(st.step).cuda(), torch.zeros((), device="cuda")
    vec = torch.zeros(B if kind == C51 else cfg["K"], device="cuda")
    per = "sampling_prob" in b
    prio = torch.zeros(B, device="cuda") if per else None
    off = torch.from_numpy(st.off)
    _lib.call("b2rl_dist_dqn_replay_update", kind, gate, _lib.ptr(b["state"]), _lib.ptr(b["next_state"]),
              int(b["state"].dtype == torch.float64), cfg.get("coef", 1.0), _lib.ptr(b["action"]), _lib.ptr(b["reward"]),
              _lib.ptr(b["mask"]), B, b["state"].shape[1], H1, H2, cfg["A"], cfg["K"], _lib.ptr(t["flat"]),
              _lib.ptr(t["target"]), _lib.ptr(t["sq"]), _lib.ptr(t["ga"]), _lib.ptr(step), _lib.ptr(off), cfg["lr"],
              cfg["alpha"], cfg["eps"], int(cfg["centered"]), cfg["discount"] ** cfg["n_step"], int(cfg["double"]), cfg["vmin"],
              cfg["vmax"], cfg["clip"], _lib.ptr(b.get("sampling_prob")), cfg.get("beta", 0.0), 0.01, 0.5, _lib.ptr(prio),
              _lib.ptr(vec), _lib.ptr(loss), _lib.stream())
    torch.cuda.synchronize()
    st.flat, st.target, st.sq, st.ga = (t[k].cpu().numpy() for k in ("flat", "target", "sq", "ga"))
    st.step, st.loss = step.cpu().numpy(), loss.reshape(1).cpu().numpy()
    return vec.cpu().numpy(), None if prio is None else prio.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(CASES)))
def test_cabi_update_matches_oracle(rl, case):
    """The CUDA build of the same phases through the C ABI."""
    kind, gate, H1, H2, cfg, sd0, tgt0, batch = case_setup(case)
    st = EmulState(kind, sd0, tgt0)
    vec, prio = cabi_update(st, kind, gate, batch, H1, H2, cfg)
    check_against_oracle(case, st, vec, prio)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c51", "qr"])
def test_golden_losses_cabi(rl, golden, name):
    """test_golden_losses_emulated through the CUDA build."""
    g = golden("agent_steps")
    pre = name + "_"
    kind, K = GOLDEN[name]["kind"], GOLDEN[name]["K"]
    cfg = dict(GOLDEN_CFG, K=K)
    keys = [str(k) for k in g[pre + "keys"]]
    init = {k: torch.from_numpy(g[pre + "init." + k]) for k in keys}
    worst = 0.0
    for i in range(g[pre + "delta"].shape[0]):
        on = init if i == 0 else golden_sd(g, pre, g[pre + "params"][i - 1])
        tg = init if i == 0 else golden_sd(g, pre, g[pre + "target"][i - 1])
        st = EmulState(kind, on, tg)
        vec, _ = cabi_update(st, kind, RELU, golden_batch(g, pre, i), 32, 32, cfg)
        want = g[pre + "delta"][i]
        np.testing.assert_allclose(vec, want, rtol=1e-5, atol=2e-6, err_msg=str(i))
        worst = max(worst, float((np.abs(vec - want) / np.maximum(np.abs(want), 2e-6 / 1e-5)).max()))
    print("%s (CUDA): largest relative difference of the loss over the 20 golden updates: %.3g" % (name, worst))


def _dist_actor(rl, kind, gate, N, D, H, A, K, vmin=-10.0, vmax=10.0, seed=5):
    from deeprl_b200 import _lib, ops
    from deeprl_b200.component.actor import dqn_kernel_order
    torch.manual_seed(seed)
    body = rl.FCBody(D, (H, H), gate=torch.tanh if gate == TANH else F.relu)
    net = rl.CategoricalNet(A, K, body) if kind == C51 else rl.QuantileNet(A, K, body)
    head = net.fc_categorical if kind == C51 else net.fc_quantiles
    with torch.no_grad():                                   # action values far enough apart to be visible
        head.weight.normal_(0, 0.5)
        head.bias.normal_(0, 0.5)
    opt = ops.FlatOptimizer.from_torch(torch.optim.RMSprop(net.parameters(), 1e-3), list(net.parameters()))
    off = torch.tensor([(t.data_ptr() - opt.flat.data_ptr()) // 4 for t in dqn_kernel_order(net)], dtype=torch.int32)
    atoms = torch.tensor(np.linspace(vmin, vmax, K), dtype=torch.float32, device="cuda")

    def q_values(x):                                        # CategoricalDQNActor / QuantileRegressionDQNActor._q_tensor
        with torch.no_grad():
            out = net(x.float())
        return (out["prob"] * atoms).sum(-1) if kind == C51 else out["quantile"].mean(-1)

    def step(obs, counter, seed, eps, given=None):
        act = torch.empty((N, 1), device="cuda")
        _lib.call("b2rl_dist_dqn_actor_step", kind, gate, _lib.ptr(obs), 1.0, _lib.ptr(opt.flat), _lib.ptr(off), D, H, H, A, K,
                  N, vmin, vmax, eps, _lib.ptr(act), _lib.ptr(given), seed, _lib.ptr(counter), _lib.stream())
        torch.cuda.synchronize()
        return act[:, 0].long()

    return q_values, step


@pytest.mark.gpu
@pytest.mark.parametrize("kind,gate,A,K", [(C51, RELU, 5, 51), (QR, TANH, 5, 20), (C51, TANH, 2, 50), (QR, RELU, 18, 2)])
def test_actor_step_epsilon_greedy(rl, kind, gate, A, K):
    """epsilon = 0: the argmax of the eager actor's action values on the same weights and states (no row within 1e-3 of a
    tie); epsilon = 1: uniform (Pearson chi-square below its 0.999 quantile at the fixed seed 11) and the same actions as
    dqn_actor_kernel's for the same key and counter; the counter advances by 2 N per step; given actions are written through."""
    from scipy import stats

    from deeprl_b200 import _lib
    N, D, H, steps = 64, 6, 32, 300
    q_values, step = _dist_actor(rl, kind, gate, N, D, H, A, K)
    cand = torch.randn(4096, D, dtype=torch.float64, device="cuda")
    top = q_values(cand).topk(2, dim=1).values
    obs = cand[(top[:, 0] - top[:, 1]) > 1e-3][:N].contiguous()
    assert obs.shape[0] == N
    greedy = q_values(obs).argmax(1)
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert torch.equal(step(obs, counter, 11, 0.0), greedy) and int(counter) == 2 * N
    # dqn_actor_kernel (b2rl_nstep_dqn_actor_step, VanillaNet) on the same key and counter: the same uniform draws
    vnet = rl.VanillaNet(A, rl.FCBody(D, (H, H)))
    vflat = torch.cat([p.detach().reshape(-1) for p in vnet.parameters()]).contiguous()
    sizes = [p.numel() for p in (vnet.body.layers[0].weight, vnet.body.layers[0].bias, vnet.body.layers[1].weight,
                                 vnet.body.layers[1].bias, vnet.fc_head.weight, vnet.fc_head.bias)]
    voff = torch.tensor(np.concatenate([[0], np.cumsum(sizes)[:-1]]), dtype=torch.int32)
    vcounter = counter.clone()
    counts = np.zeros(A)
    for _ in range(steps):
        act = step(obs, counter, 11, 1.0)
        vact = torch.empty((N, 1), device="cuda")
        _lib.call("b2rl_nstep_dqn_actor_step", RELU, _lib.ptr(obs), 1.0, _lib.ptr(vflat), _lib.ptr(voff), D, H, H, A, N, 1.0,
                  None, _lib.ptr(vact), None, 11, _lib.ptr(vcounter), _lib.stream())
        assert torch.equal(act, vact[:, 0].long())
        counts += np.bincount(act.cpu().numpy(), minlength=A)
    assert int(counter) == int(vcounter) == 2 * N * (1 + steps)
    exp_c = steps * N / A
    assert float(((counts - exp_c) ** 2 / exp_c).sum()) < stats.chi2.ppf(0.999, A - 1), counts
    given = torch.randint(0, A, (N, 1), device="cuda").float()
    assert torch.equal(step(obs, counter, 3, 0.5, given), given[:, 0].long()) and int(counter) == 2 * N * (1 + steps)


def _agent_cfg(rl, kind, per=False, async_replay=False, device=True, **kw):
    c = rl.Config()
    c.merge(dict(tag=None, n_step=1))
    setattr(c, "device_c51" if kind == C51 else "device_qr", device)
    c.task_fn = lambda: rl.Task("CartPole-v0", seed=7)
    c.eval_env = c.task_fn()
    c.batch_size, c.discount = 16, 0.99
    c.optimizer_fn = lambda p: torch.optim.RMSprop(p, lr=1e-3, alpha=0.95, eps=0.01, centered=per)
    if kind == C51:
        c.categorical_v_min, c.categorical_v_max, c.categorical_n_atoms = -100, 100, 50
        c.network_fn = lambda: rl.CategoricalNet(c.action_dim, c.categorical_n_atoms, rl.FCBody(c.state_dim, (32, 32)))
    else:
        c.num_quantiles = 20
        c.network_fn = lambda: rl.QuantileNet(c.action_dim, c.num_quantiles, rl.FCBody(c.state_dim, (32, 32)))
    rk = dict(memory_size=512, batch_size=16, n_step=1, discount=0.99)
    c.replay_fn = lambda: rl.ReplayWrapper(rl.PrioritizedReplay if per else rl.UniformReplay, rk, async_replay)
    c.replay_eps, c.replay_alpha, c.replay_beta = 0.01, 0.5, rl.LinearSchedule(0.4, 1.0, 200)
    c.random_action_prob = rl.LinearSchedule(1.0, 0.1, 100)
    c.target_network_update_freq, c.exploration_steps = 5, 40
    c.sgd_update_frequency, c.gradient_clip, c.async_actor, c.double_q = 4, 5, False, per
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _agent_cls(rl, kind):
    return rl.CategoricalDQNAgent if kind == C51 else rl.QuantileRegressionDQNAgent


def _params(net):
    return np.concatenate([p.detach().cpu().numpy().ravel() for p in net.parameters()])


@pytest.mark.gpu
@pytest.mark.parametrize("kind,per", [(C51, False), (C51, True), (QR, False)])
@pytest.mark.parametrize("async_replay", [False, True])
def test_eager_and_device_agents_agree(rl, kind, per, async_replay):
    """The same forced actions, replay seed and env seed: an eager and a device agent feed identical rings and draw identical
    indices; their online and target parameters agree to 1e-4 after 50 updates."""
    rng = np.random.RandomState(0)
    forced = rng.randint(0, 2, size=100000)
    agents_ = []
    for device in (False, True):
        torch.manual_seed(1)
        agents_.append(_agent_cls(rl, kind)(_agent_cfg(rl, kind, per, async_replay, device)))
    eager, dev = agents_
    assert eager.device_dqn is None and dev.device_dqn is not None
    dev.network.load_state_dict(eager.network.state_dict())
    dev.target_network.load_state_dict(eager.target_network.state_dict())
    init = _params(eager.network)
    k = [0, 0]

    def forced_eager(eps, q):
        a = forced[k[0]:k[0] + q.shape[0]]
        k[0] += q.shape[0]
        return a

    import deeprl_b200.agent.DQN_agent as dqn_mod
    orig = dqn_mod.epsilon_greedy
    dqn_mod.epsilon_greedy = forced_eager
    try:
        def nxt():
            a = forced[k[1]:k[1] + 1]
            k[1] += 1
            return a
        dev.device_dqn.forced = nxt
        steps = 40 // 4 + 50
        for _ in range(steps):
            eager.step()
            dev.step()
    finally:
        dqn_mod.epsilon_greedy = orig
    torch.cuda.synchronize()
    ri, rd = getattr(eager.replay, "replay", eager.replay), getattr(dev.replay, "replay", dev.replay)
    assert ri.size() == rd.size()
    err = float(np.abs(_params(eager.network) - _params(dev.network)).max())
    err_t = float(np.abs(_params(eager.target_network) - _params(dev.target_network)).max())
    assert err <= 1e-4 and err_t <= 1e-4, (err, err_t)
    assert abs(float(eager.last_loss) - float(dev.last_loss)) <= 1e-4 * max(1.0, abs(float(eager.last_loss)))
    assert int(dev._flat.step_dev) == steps - 10 and np.abs(_params(dev.network) - init).max() > 1e-4
    eager.close()
    dev.close()


def _launcher_agent(monkeypatch, kind):
    import examples
    got = []
    monkeypatch.setattr(examples, "run_steps", got.append)
    if kind == C51:
        examples.categorical_dqn_feature(game="CartPole-v0", device_c51=True)
    else:
        examples.quantile_regression_dqn_feature(game="CartPole-v0", device_qr=True)
    return got[0]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [C51, QR])
def test_launcher_end_to_end(rl, monkeypatch, kind):
    """categorical_dqn_feature / quantile_regression_dqn_feature with their own configuration (async actor, async replay) and
    the device flag: finite, varying losses; after every scheduled sync the target arena equals the online arena exactly,
    otherwise it is unchanged; one profiled step() past the exploration lists sgd_update_frequency actor kernels, one update
    kernel, and besides them only the replay's feed, draw and gather kernels."""
    import time
    ag = _launcher_agent(monkeypatch, kind)
    c, dev = ag.config, ag.device_dqn
    assert c.async_actor and getattr(ag.replay, "async_", False) and dev is not None
    losses_, syncs = [], 0
    while ag.total_steps <= c.exploration_steps + 4 * c.target_network_update_freq * 2:
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

    # The actor thread runs ahead: with its queue full it waits in put() with the next item made.  Once it is there, each
    # step() takes one item, the waiting one goes in, and the thread makes exactly one more item (sgd_update_frequency env
    # steps, each ending in a stream synchronise) before it waits again.
    actor = ag.actor
    while True:                                                 # reach that state
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
    kernels = profiled_kernels(step, {"dist_actor_kernel": c.sgd_update_frequency, "dist_replay_update_kernel": 1,
                                     "feed_kernel": 1, "gather": 1})
    assert sum("dist_actor_kernel" in k for k in kernels) == c.sgd_update_frequency, kernels
    assert sum("dist_replay_update_kernel" in k for k in kernels) == 1, kernels
    others = [k for k in kernels if "dist_actor_kernel" not in k and "dist_replay_update_kernel" not in k]
    assert all(k.startswith("b2rl::") for k in others), others          # no torch forward, backward or optimizer kernel
    assert any("feed_kernel" in k for k in others) and any("gather" in k for k in others), others
    ag.close()


@pytest.mark.gpu
def test_unsupported_configurations_are_refused(rl):
    class OwnLoss(rl.CategoricalDQNAgent):
        def reduce_loss(self, loss):
            return loss.sum()

    C, Q = rl.CategoricalDQNAgent, rl.QuantileRegressionDQNAgent
    refused = [
        (C, C51, dict(network_fn=lambda: rl.RainbowNet(2, 50, rl.FCBody(4), noisy_linear=False)), "RainbowNet"),
        (C, C51, dict(network_fn=lambda: rl.CategoricalNet(2, 50, rl.FCBody(4, noisy_linear=True))), "NoisyLinear"),
        (Q, QR, dict(network_fn=lambda: rl.QuantileNet(2, 20, rl.NatureConvBody(in_channels=4))), "NatureConvBody"),
        (C, C51, dict(network_fn=lambda: rl.CategoricalNet(2, 50, rl.FCBody(4, (64, 64, 64)))), "two-layer"),
        (Q, QR, dict(optimizer_fn=lambda p: torch.optim.Adam(p, 1e-3)), "Adam"),
        (C, C51, dict(state_normalizer=rl.MeanStdNormalizer()), "MeanStdNormalizer"),
        (Q, QR, dict(history_length=4), "frame stacks"),
        (Q, QR, dict(replay_fn=lambda: rl.ReplayWrapper(rl.PrioritizedReplay, dict(memory_size=512, batch_size=16), False)),
         "prioritized replay"),
        (OwnLoss, C51, {}, "reduce_loss"),
        (C, C51, dict(batch_size=4096), "shared memory"),
        (Q, QR, dict(network_fn=lambda: rl.QuantileNet(2, 300, rl.FCBody(4))), "quantiles 300"),
        (C, C51, dict(device_dqn=True), "device_dqn and config.device_c51"),
        (Q, QR, dict(device_dqn=True), "device_dqn and config.device_qr"),
    ]
    for cls, kind, kw, msg in refused:
        with pytest.raises(NotImplementedError, match=msg):
            cls(_agent_cfg(rl, kind, **kw))
    for kind in (C51, QR):                                        # the supported forms still build, with the async actor too
        for async_actor in (False, True):
            ag = _agent_cls(rl, kind)(_agent_cfg(rl, kind, async_actor=async_actor))
            assert ag.device_dqn is not None
            ag.close()
