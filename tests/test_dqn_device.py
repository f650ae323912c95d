"""Replay DQN on the device (``config.device_dqn``; deeprl_b200/csrc/a2c.cu): one ``b2rl_nstep_dqn_actor_step`` launch per env
step and ONE ``b2rl_dqn_replay_update`` launch per gradient update of DQN_agent.py:81-134, for a VanillaNet or DuelingNet on a
two-layer FCBody.

CPU: the update's phase functions (csrc/a2c_phases.h with HEAD = Q / DUEL + dqn_sequence.inc) are compiled for the host by
tests/host_emul/dqn_emul.cpp and run with the block's threads in sequence, against the reference's recorded updates
(tests/golden/agent_steps.npz ``dqn_uni`` / ``dqn_per``: delta, online AND target parameters after each of 20 updates) and
against oracle/agents.py DQNFamilyOracle.
GPU: the CUDA build of the same source through the C ABI and through ``DQNAgent``; the dueling actor step's epsilon-greedy.

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
VANILLA, DUELING = 0, 1
BODY = ["body.layers.0.weight", "body.layers.0.bias", "body.layers.1.weight", "body.layers.1.bias"]
KEYS = {VANILLA: BODY + ["fc_head.weight", "fc_head.bias"],                     # the kernels' tensor order
        DUELING: BODY + ["fc_advantage.weight", "fc_advantage.bias", "fc_value.weight", "fc_value.bias"]}
P = ctypes.c_void_p


def vp(x):
    return None if x is None else P(x.ctypes.data)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("dqn_emul") / "dqn_emul.so")
    subprocess.run(["g++", "-O2", "-fno-strict-aliasing", "-std=c++17", "-shared", "-fPIC", "-o", out,
                    os.path.join(ROOT, "tests", "host_emul", "dqn_emul.cpp")], check=True)
    lib = ctypes.CDLL(out)
    i32, f32, f64 = ctypes.c_int32, ctypes.c_float, ctypes.c_double
    lib.dqn_emul_update.argtypes = ([i32, i32, P, P, i32, f64, P, P, P] + [i32] * 5 + [P] * 6 + [f32] * 3
                                    + [i32, f32, i32, f32, P] + [f32] * 3 + [P] * 3 + [i32, i32])
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

    def __init__(self, head, sd, target_sd=None):
        self.keys = KEYS[head]
        self.flat, self.off = arena(sd, self.keys)
        self.target = arena(target_sd if target_sd is not None else sd, self.keys)[0]
        self.sq, self.ga = np.zeros_like(self.flat), np.zeros_like(self.flat)
        self.step = np.zeros(1, np.int64)
        self.loss = np.zeros(1, np.float32)


def emul_update(lib, st, head, gate, batch, H1, H2, cfg, threads=512, reversed_=False):
    """One b2rl_dqn_replay_update on the host.  batch: dict of numpy arrays state / next_state (B, D; float32 or float64),
    action, reward, mask, and for PER sampling_prob.  Returns (delta, priority)."""
    s = np.ascontiguousarray(batch["state"])
    s2 = np.ascontiguousarray(batch["next_state"], dtype=s.dtype)
    B, D = s.shape
    a = np.ascontiguousarray(batch["action"], np.int64)
    r, m = (np.ascontiguousarray(batch[k], np.float32) for k in ("reward", "mask"))
    prob = batch.get("sampling_prob")
    prob = None if prob is None else np.ascontiguousarray(prob, np.float32)
    prio = np.zeros(B, np.float32) if prob is not None else None
    delta = np.zeros(B, np.float32)
    rc = lib.dqn_emul_update(head, gate, vp(s), vp(s2), int(s.dtype == np.float64), cfg.get("coef", 1.0), vp(a), vp(r), vp(m),
                             B, D, H1, H2, cfg["A"], vp(st.flat), vp(st.target), vp(st.sq), vp(st.ga), vp(st.step), vp(st.off),
                             cfg["lr"], cfg["alpha"], cfg["eps"], int(cfg["centered"]), cfg["discount"] ** cfg["n_step"],
                             int(cfg["double"]), cfg["clip"], vp(prob), cfg.get("beta", 0.0), 0.01, 0.5, vp(prio), vp(delta),
                             vp(st.loss), threads, int(reversed_))
    assert rc == 0
    return delta, prio


# ------------------------------------------------------------------------------------------------ golden records
def golden_batch(g, pre, i):
    b = {f: g[pre + "b_" + f][i] for f in ("state", "next_state", "action", "reward", "mask")}
    if pre == "dqn_per_":
        b["sampling_prob"] = g[pre + "b_sampling_prob"][i]
    return b


GOLDEN_CFG = dict(lr=0.00025, alpha=0.95, eps=0.01, centered=True, clip=5.0, discount=0.99, n_step=1, A=2)


def synced_after(i):
    """The golden agents update once per step() from step 11 on (exploration 40, 4 env steps per step()) and sync the target
    when step() % 5 == 0 (DQN_agent.py:136-138, target_network_update_freq 5), so after updates 4, 9, 14 and 19."""
    return (11 + i) % 5 == 0


@pytest.mark.parametrize("name", ["dqn_uni", "dqn_per"])
def test_golden_updates_emulated(emul, golden, name):
    """The reference's 20 recorded updates (dqn_uni: VanillaNet, uniform replay; dqn_per: DuelingNet, double-Q, PER with beta
    from LinearSchedule(0.4, 1, 200) called once per update): the recorded delta, online and target parameters after every
    update; the priorities are (|delta| + 0.01)^0.5 of the recorded delta."""
    from deeprl_b200.utils.schedule import LinearSchedule
    g = golden("agent_steps")
    pre = name + "_"
    head = DUELING if name == "dqn_per" else VANILLA
    order = [str(k) for k in g[pre + "keys"]]
    sd0 = {k: torch.from_numpy(g[pre + "init." + k]) for k in order}
    st = EmulState(head, sd0)
    cfg = dict(GOLDEN_CFG, double=name == "dqn_per")
    beta = LinearSchedule(0.4, 1.0, 200)
    worst, syncs = 0.0, 0
    for i in range(g[pre + "delta"].shape[0]):
        batch = golden_batch(g, pre, i)
        if head == DUELING:
            cfg["beta"] = beta()
        delta, prio = emul_update(emul, st, head, RELU, batch, 32, 32, cfg)
        np.testing.assert_allclose(delta, g[pre + "delta"][i], rtol=1e-5, atol=5e-6)
        if prio is not None:
            np.testing.assert_allclose(prio, np.sqrt(np.abs(g[pre + "delta"][i]) + 0.01), rtol=1e-5, atol=1e-6)
        if synced_after(i):
            st.target[...] = st.flat
            syncs += 1
        got = unflatten(st.flat, st.off, sd0, st.keys)
        got_t = unflatten(st.target, st.off, sd0, st.keys)
        err = float(np.abs(np.concatenate([got[k].ravel() for k in order]) - g[pre + "params"][i]).max())
        err_t = float(np.abs(np.concatenate([got_t[k].ravel() for k in order]) - g[pre + "target"][i]).max())
        worst = max(worst, err, err_t)
        assert err <= 1e-5 and err_t <= 1e-5, (i, err, err_t)
    assert int(st.step[0]) == 20 and syncs == 4
    print("%s: largest online / target parameter difference over the 20 golden updates: %.3g" % (name, worst))


# ------------------------------------------------------------------------------------------------ ragged shapes and the oracle
def max_batch(head, D, H1, H2, A, double):
    from deeprl_b200 import _lib
    L = _lib.lib()
    B = 1
    while L.b2rl_dqn_replay_smem_bytes(head, D, H1, H2, A, B + 1, int(double)) <= 227 * 1024:
        B += 1
    return B


CFG = dict(lr=1e-3, alpha=0.99, eps=1e-8, centered=False, discount=0.99, clip=5.0, n_step=1, double=False, per=False, coef=1.0)
CASES = [  # (head, gate, D, A, H1, H2, B, float64 states, cfg overrides)
    (VANILLA, RELU, 4, 2, 64, 64, 10, True, {}),                                                  # dqn_feature
    (DUELING, TANH, 11, 3, 32, 48, 37, True, dict(double=True, per=True, centered=True, clip=1e6, n_step=3, coef=0.5)),
    (DUELING, RELU, 7, 5, 16, 24, 1, False, dict(per=True, clip=0.05)),
    (VANILLA, TANH, 11, 3, 32, 48, 37, True, dict(double=True, centered=True, clip=0.05, n_step=3)),
    (VANILLA, RELU, 4, 2, 64, 64, "max", True, dict(double=True, per=True, centered=True, clip=1e6)),
    (DUELING, TANH, 9, 4, 40, 24, 10, False, dict(clip=0.05, n_step=3, coef=0.25)),
    (DUELING, RELU, 5, 6, 24, 32, "max", True, dict(double=True, per=True, clip=0.05)),
    (VANILLA, TANH, 6, 32, 20, 28, 10, False, dict(per=True, centered=True, clip=1e6)),
]


def make_problem(head, D, A, H1, H2, B, f64, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale

    def net():
        sd = {"body.layers.0.weight": r(H1, D, scale=D ** -0.5), "body.layers.0.bias": r(H1, scale=0.1),
              "body.layers.1.weight": r(H2, H1, scale=H1 ** -0.5), "body.layers.1.bias": r(H2, scale=0.1)}
        if head == VANILLA:
            sd.update({"fc_head.weight": r(A, H2, scale=H2 ** -0.5), "fc_head.bias": r(A, scale=0.1)})
        else:
            sd.update({"fc_advantage.weight": r(A, H2, scale=H2 ** -0.5), "fc_advantage.bias": r(A, scale=0.1),
                       "fc_value.weight": r(1, H2, scale=H2 ** -0.5), "fc_value.bias": r(1, scale=0.1)})
        return sd

    sd, target = net(), net()
    dt = np.float64 if f64 else np.float32
    batch = dict(state=r(B, D, scale=2.0).double().numpy().astype(dt), next_state=r(B, D, scale=2.0).double().numpy().astype(dt),
                 action=torch.randint(0, A, (B,), generator=g).numpy(), reward=r(B).numpy(),
                 mask=(torch.rand(B, generator=g) > 0.2).float().numpy(),
                 sampling_prob=(torch.rand(B, generator=g) * 0.01 + 1e-4).numpy())
    return sd, target, batch


def case_setup(case):
    head, gate, D, A, H1, H2, B, f64, over = CASES[case]
    cfg = dict(CFG, A=A, **over)
    if B == "max":
        B = max_batch(head, D, H1, H2, A, cfg["double"])
    cfg["beta"] = 0.55 if cfg["per"] else 0.0
    sd0, tgt0, batch = make_problem(head, D, A, H1, H2, B, f64, seed=300 + case)
    if not cfg["per"]:
        del batch["sampling_prob"]
    return head, gate, H1, H2, cfg, sd0, tgt0, batch


def run_case(lib, case, threads=512, reversed_=False):
    head, gate, H1, H2, cfg, sd0, tgt0, batch = case_setup(case)
    st = EmulState(head, sd0, tgt0)
    delta, prio = emul_update(lib, st, head, gate, batch, H1, H2, cfg, threads, reversed_)
    return st, delta, prio


class _Tr:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def oracle_update(case):
    """DQN_agent.py:81-134 by the oracle.  Returns (oracle, loss, delta, priorities, gradient norm after the clip)."""
    head, gate, H1, H2, cfg, sd0, tgt0, batch = case_setup(case)
    gfn = torch.tanh if gate == TANH else F.relu
    o = agents.DQNFamilyOracle({k: v.clone() for k, v in sd0.items()}, "dueling" if head == DUELING else "vanilla", "fc",
                               cfg["A"], lambda p: torch.optim.RMSprop(p, cfg["lr"], alpha=cfg["alpha"], eps=cfg["eps"],
                                                                       centered=cfg["centered"]),
                               cfg["discount"], n_step=cfg["n_step"], double_q=cfg["double"], gradient_clip=cfg["clip"],
                               state_coef=cfg["coef"], replay_eps=0.01, replay_alpha=0.5, replay_beta=lambda: cfg["beta"],
                               gate=gfn)
    for k in o.target_sd:
        o.target_sd[k].copy_(tgt0[k])
    tr = _Tr(**batch)
    if cfg["per"]:
        tr.idx = np.arange(len(batch["action"]))
    with torch.no_grad():
        delta = o.compute_loss(tr).numpy()
    prios = {}

    class Rep:
        def update_priorities(self, pairs):
            prios.update(dict(pairs))

    loss = o.update(tr, Rep())
    clipped = float(torch.sqrt(sum((p.grad.double() ** 2).sum() for p in o.params)))
    prio = np.asarray([prios[i] for i in range(len(prios))], np.float32) if cfg["per"] else None
    return o, cfg, float(loss), delta, prio, clipped, sd0, tgt0


def check_against_oracle(case, st, delta, prio, atol=1e-5):
    o, cfg, loss, d_want, p_want, clipped, sd0, tgt0 = oracle_update(case)
    np.testing.assert_allclose(delta, d_want, rtol=1e-5, atol=5e-6)
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
    st, delta, prio = run_case(emul, case)
    cfg, clipped = check_against_oracle(case, st, delta, prio)
    if cfg["clip"] < 1.0:
        assert abs(clipped - cfg["clip"]) < 1e-4 * cfg["clip"]              # the clip was active
    elif cfg["clip"] >= 1e5:
        assert clipped < cfg["clip"]                                         # ... and here it was not


def test_cases_cover_the_batch_sizes():
    sizes = {case_setup(c)[-1]["action"].shape[0] for c in range(len(CASES))}
    assert {1, 10, 37} <= sizes and max(sizes) > 37, sizes


@pytest.mark.parametrize("case", [1, 3, 6])
def test_thread_order_and_count_do_not_change_the_result(emul, case):
    """Reversed thread order inside every phase, 64 and 37 threads instead of 512: bit-identical arenas (the race check)."""
    ref, d_ref, p_ref = run_case(emul, case)
    for threads, rev in ((512, True), (64, False), (37, True)):
        got, d, p = run_case(emul, case, threads, rev)
        for k in ("flat", "target", "sq", "ga", "loss", "step"):
            assert np.array_equal(getattr(ref, k), getattr(got, k)), (threads, rev, k)
        assert np.array_equal(d_ref, d) and (p_ref is None or np.array_equal(p_ref, p))


def _compile(src_root, out, ptxas=False):
    cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-o", str(out),
           os.path.join(src_root, "deeprl_b200", "csrc", "a2c.cu")] + (["-Xptxas", "-v"] if ptxas else [])
    return subprocess.run(cmd, check=True, capture_output=True, text=True).stderr


def test_kernels_have_no_spills_and_no_stack_frame(tmp_path):
    out = _compile(ROOT, tmp_path / "a2c.cubin", ptxas=True)
    entries = out.split("Compiling entry function")[1:]
    names = [e.split("'")[1] for e in entries]
    # (VanillaNet, DuelingNet) x (tanh, ReLU), the update and the actor step
    assert sum("dqn_replay_update_kernel" in n for n in names) == 4, names
    assert sum("16dqn_actor_kernel" in n for n in names) == 4, names
    for e in entries:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in e, e


def test_shared_memory_budget_accepts_the_launcher():
    from deeprl_b200 import _lib
    L = _lib.lib()
    feature = L.b2rl_dqn_replay_smem_bytes(0, 4, 64, 64, 2, 10, 0)         # dqn_feature: CartPole, batch 10
    assert 0 < feature <= 227 * 1024, feature
    assert L.b2rl_dqn_replay_smem_bytes(1, 4, 64, 64, 2, 32, 1) <= 227 * 1024
    assert L.b2rl_dqn_replay_smem_bytes(0, 4, 128, 128, 2, 512, 1) > 227 * 1024
    assert L.b2rl_dqn_replay_smem_bytes(0, 4, 64, 64, 2, 0, 0) == 0
    assert L.b2rl_dqn_replay_smem_bytes(2, 4, 64, 64, 2, 10, 0) == 0


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def rl():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import deeprl_b200 as rl
    rl.select_device(0)
    rl.Config.COMPUTE_DTYPE = torch.float32
    return rl


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(CASES)))
def test_cabi_update_matches_oracle(rl, case):
    """The CUDA build of the same phases through the C ABI."""
    from deeprl_b200 import _lib
    head, gate, H1, H2, cfg, sd0, tgt0, batch = case_setup(case)
    st = EmulState(head, sd0, tgt0)
    cu = lambda x: torch.as_tensor(np.ascontiguousarray(x)).cuda()
    t = {k: cu(getattr(st, k)) for k in ("flat", "target", "sq", "ga")}
    b = {k: cu(v if k in ("state", "next_state", "action") else np.asarray(v, np.float32)) for k, v in batch.items()}
    B = b["action"].shape[0]
    step, loss = torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros((), device="cuda")
    delta = torch.zeros(B, device="cuda")
    prio = torch.zeros(B, device="cuda") if cfg["per"] else None
    off = torch.from_numpy(st.off)
    _lib.call("b2rl_dqn_replay_update", head, gate, _lib.ptr(b["state"]), _lib.ptr(b["next_state"]),
              int(b["state"].dtype == torch.float64), cfg["coef"], _lib.ptr(b["action"]), _lib.ptr(b["reward"]),
              _lib.ptr(b["mask"]), B, b["state"].shape[1], H1, H2, cfg["A"], _lib.ptr(t["flat"]), _lib.ptr(t["target"]),
              _lib.ptr(t["sq"]), _lib.ptr(t["ga"]), _lib.ptr(step), _lib.ptr(off), cfg["lr"], cfg["alpha"], cfg["eps"],
              int(cfg["centered"]), cfg["discount"] ** cfg["n_step"], int(cfg["double"]), cfg["clip"],
              _lib.ptr(b.get("sampling_prob")), cfg["beta"], 0.01, 0.5, _lib.ptr(prio), _lib.ptr(delta), _lib.ptr(loss),
              _lib.stream())
    torch.cuda.synchronize()
    st.flat, st.target, st.sq, st.ga = (t[k].cpu().numpy() for k in ("flat", "target", "sq", "ga"))
    st.step, st.loss = step.cpu().numpy(), loss.reshape(1).cpu().numpy()
    check_against_oracle(case, st, delta.cpu().numpy(), None if prio is None else prio.cpu().numpy())


def _golden_cfg(rl, name, **kw):
    c = rl.Config()
    c.merge(dict(tag=None, n_step=1, device_dqn=True))
    c.task_fn = lambda: rl.Task("CartPole-v0", seed=3)
    c.eval_env = c.task_fn()
    c.history_length, c.batch_size, c.discount = 1, 16, 0.99
    body = lambda: rl.FCBody(c.state_dim, hidden_units=(32, 32))
    c.optimizer_fn = lambda p: torch.optim.RMSprop(p, lr=0.00025, alpha=0.95, eps=0.01, centered=True)
    c.network_fn = (lambda: rl.DuelingNet(c.action_dim, body())) if name == "dqn_per" else (lambda: rl.VanillaNet(c.action_dim, body()))
    cls = rl.PrioritizedReplay if name == "dqn_per" else rl.UniformReplay
    rk = dict(memory_size=256, batch_size=16, n_step=1, discount=0.99, history_length=1)
    c.replay_fn = lambda: rl.ReplayWrapper(cls, rk, False)
    c.replay_eps, c.replay_alpha = 0.01, 0.5
    c.replay_beta = rl.LinearSchedule(0.4, 1.0, 200)
    c.random_action_prob = rl.LinearSchedule(1.0, 0.1, 100)
    c.target_network_update_freq, c.exploration_steps = 5, 40
    c.sgd_update_frequency, c.gradient_clip, c.async_actor = 4, 5, False
    c.double_q = name == "dqn_per"
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _params(net):
    return np.concatenate([p.detach().cpu().numpy().ravel() for p in net.parameters()])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dqn_uni", "dqn_per"])
def test_agent_replays_the_golden_record(rl, golden, name):
    """DQNAgent with device_dqn, replay.sample patched to return the batches the reference drew: after each of the 20 steps
    with an update the recorded online and target parameters (1e-5), the targets synced by the agent's own schedule."""
    g = golden("agent_steps")
    pre = name + "_"
    ag = rl.DQNAgent(_golden_cfg(rl, name))
    keys = [str(k) for k in g[pre + "keys"]]
    with torch.no_grad():
        for net in (ag.network, ag.target_network):
            for k, p in net.state_dict().items():
                p.copy_(torch.from_numpy(g[pre + "init." + k]))
    fields = ["state", "action", "reward", "next_state", "mask"] + (["sampling_prob", "idx"] if name == "dqn_per" else [])
    TCls = rl.PrioritizedTransition if name == "dqn_per" else rl.Transition
    it = [0]

    def sample():
        i = it[0]
        it[0] += 1
        return TCls(*[torch.as_tensor(g[pre + "b_" + f][i], dtype=torch.int64 if f in ("action", "idx") else torch.float32,
                                      device="cuda").contiguous() for f in fields])

    got_prio = []
    ag.replay.sample = sample
    ag.replay.update_priorities = lambda info: got_prio.append(info[1].cpu().numpy())
    assert [n for n, _ in ag.network.named_parameters()] == keys
    worst = 0.0
    while it[0] < 20:
        before = it[0]
        ag.step()
        if it[0] == before:
            continue
        i = before
        err = float(np.abs(_params(ag.network) - g[pre + "params"][i]).max())
        err_t = float(np.abs(_params(ag.target_network) - g[pre + "target"][i]).max())
        worst = max(worst, err, err_t)
        assert err <= 1e-5 and err_t <= 1e-5, (i, err, err_t)
        assert ag.last_loss.dim() == 0 and torch.isfinite(ag.last_loss)
        if name == "dqn_per":
            np.testing.assert_allclose(got_prio[-1], np.sqrt(np.abs(g[pre + "delta"][i]) + 0.01), rtol=1e-5, atol=1e-6)
    assert int(ag._flat.step_dev) == 20
    print("%s: device agent vs golden record, largest parameter difference: %.3g" % (name, worst))
    ag.close()


def _dueling_actor(rl, gate, N, D, H, A, seed=5):
    from deeprl_b200 import _lib, ops
    from deeprl_b200.component.actor import dqn_kernel_order
    torch.manual_seed(seed)
    net = rl.DuelingNet(A, rl.FCBody(D, (H, H), gate=torch.tanh if gate == TANH else F.relu))
    with torch.no_grad():                                   # q-values far enough apart to be visible
        net.fc_advantage.weight.normal_(0, 0.5)
        net.fc_advantage.bias.normal_(0, 0.5)
    opt = ops.FlatOptimizer.from_torch(torch.optim.RMSprop(net.parameters(), 1e-3), list(net.parameters()))
    off = torch.tensor([(t.data_ptr() - opt.flat.data_ptr()) // 4 for t in dqn_kernel_order(net)], dtype=torch.int32)

    def step(obs, counter, seed, eps, given=None, state_out=None):
        act = torch.empty((N, 1), device="cuda")
        _lib.call("b2rl_nstep_dqn_actor_step", gate + 2, _lib.ptr(obs), 1.0, _lib.ptr(opt.flat), _lib.ptr(off), D, H, H, A, N,
                  eps, _lib.ptr(state_out), _lib.ptr(act), _lib.ptr(given), seed, _lib.ptr(counter), _lib.stream())
        torch.cuda.synchronize()
        return act[:, 0].long()

    return net, step


@pytest.mark.gpu
def test_dueling_actor_step_epsilon_greedy(rl):
    """The DuelingNet actor step: epsilon = 0 the argmax of a torch forward (no row within 1e-3 of a tie); epsilon = 1 uniform
    (Pearson chi-square below its 0.999 quantile at the fixed seed 11); epsilon = 0.25 the share of non-greedy actions within 5
    binomial standard errors of epsilon (A - 1) / A; the counter advances by 2 N per step; given actions are written through."""
    from scipy import stats
    N, D, H, A, steps = 64, 6, 32, 5, 1000
    net, step = _dueling_actor(rl, TANH, N, D, H, A)
    cand = torch.randn(4096, D, dtype=torch.float64, device="cuda")
    with torch.no_grad():
        q = net(cand.float())["q"]
    top = q.topk(2, dim=1).values
    obs = cand[(top[:, 0] - top[:, 1]) > 1e-3][:N].contiguous()
    assert obs.shape[0] == N
    with torch.no_grad():
        greedy = net(obs.float())["q"].argmax(1)
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    st = torch.empty((N, D), device="cuda")
    assert torch.equal(step(obs, counter, 11, 0.0, state_out=st), greedy) and int(counter) == 2 * N
    assert torch.equal(st, obs.float())
    counts = np.zeros(A)
    for _ in range(steps):
        counts += np.bincount(step(obs, counter, 11, 1.0).cpu().numpy(), minlength=A)
    exp_c = steps * N / A
    assert float(((counts - exp_c) ** 2 / exp_c).sum()) < stats.chi2.ppf(0.999, A - 1), counts
    eps, other = 0.25, 0
    for _ in range(steps):
        other += int((step(obs, counter, 11, eps) != greedy).sum())
    n, p = steps * N, eps * (A - 1) / A
    assert abs(other / n - p) < 5 * np.sqrt(p * (1 - p) / n), (other / n, p)
    assert int(counter) == 2 * N * (1 + 2 * steps)
    given = torch.randint(0, A, (N, 1), device="cuda").float()
    assert torch.equal(step(obs, counter, 3, 0.5, given), given[:, 0].long()) and int(counter) == 2 * N * (1 + 2 * steps)


def _eager_vs_device_cfg(rl, per, async_replay, device):
    c = rl.Config()
    c.merge(dict(tag=None, n_step=1, device_dqn=device))
    c.task_fn = lambda: rl.Task("CartPole-v0", seed=7)
    c.eval_env = c.task_fn()
    c.history_length, c.batch_size, c.discount = 1, 16, 0.99
    c.optimizer_fn = lambda p: torch.optim.RMSprop(p, lr=1e-3, alpha=0.95, eps=0.01, centered=per)
    c.network_fn = lambda: (rl.DuelingNet if per else rl.VanillaNet)(c.action_dim, rl.FCBody(c.state_dim, (32, 32)))
    rk = dict(memory_size=512, batch_size=16, n_step=1, discount=0.99, history_length=1)
    c.replay_fn = lambda: rl.ReplayWrapper(rl.PrioritizedReplay if per else rl.UniformReplay, rk, async_replay)
    c.replay_eps, c.replay_alpha, c.replay_beta = 0.01, 0.5, rl.LinearSchedule(0.4, 1.0, 200)
    c.random_action_prob = rl.LinearSchedule(1.0, 0.1, 100)
    c.target_network_update_freq, c.exploration_steps = 5, 40
    c.sgd_update_frequency, c.gradient_clip, c.async_actor, c.double_q = 4, 5, False, per
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("per", [False, True])
@pytest.mark.parametrize("async_replay", [False, True])
def test_eager_and_device_agents_agree(rl, per, async_replay):
    """The same forced actions, replay seed and env seed: an eager and a device agent feed identical rings and draw identical
    indices; their parameters agree to 1e-4 after 50 agent steps past the exploration."""
    rng = np.random.RandomState(0)
    forced = rng.randint(0, 2, size=100000)
    agents_ = []
    for device in (False, True):
        torch.manual_seed(1)
        ag = rl.DQNAgent(_eager_vs_device_cfg(rl, per, async_replay, device))
        agents_.append(ag)
    eager, dev = agents_
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
    assert int(dev._flat.step_dev) == steps - 10 and np.abs(_params(dev.network) - init).max() > 1e-4
    eager.close()
    dev.close()


def _launcher_agent(monkeypatch, **kw):
    import examples
    got = []
    monkeypatch.setattr(examples, "run_steps", got.append)
    examples.dqn_feature(game="CartPole-v0", device_dqn=True, **kw)
    return got[0]


@pytest.mark.gpu
@pytest.mark.parametrize("replay_cls", ["UniformReplay", "PrioritizedReplay"])
def test_launcher_end_to_end(rl, monkeypatch, replay_cls):
    """dqn_feature with device_dqn (async replay): finite, varying losses; after every scheduled sync the target arena equals
    the online arena exactly, otherwise it is unchanged; one profiled step() past the exploration lists
    sgd_update_frequency actor kernels, one update kernel, and besides them only the replay's feed, draw + gather (and for
    PER the priority update) kernels."""
    ag = _launcher_agent(monkeypatch, replay_cls=getattr(rl, replay_cls))
    c, dev = ag.config, ag.device_dqn
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
    from _kernel_trace import profiled_kernels
    kernels = profiled_kernels(lambda: (ag.step(), torch.cuda.synchronize()), dict(
        {"dqn_actor_kernel": c.sgd_update_frequency, "dqn_replay_update_kernel": 1, "feed_kernel": 1, "gather": 1},
        **({"direct_copy": 1, "sumtree_sample": 1} if replay_cls == "PrioritizedReplay" else {})))
    assert sum("dqn_actor_kernel" in k for k in kernels) == c.sgd_update_frequency, kernels
    assert sum("dqn_replay_update_kernel" in k for k in kernels) == 1, kernels
    others = [k for k in kernels if "dqn_actor_kernel" not in k and "dqn_replay_update_kernel" not in k]
    # the replay's own kernels (feed, index draw, gather, sum tree) and, for PER, its float64 -> float32 cast of the sampling
    # probabilities (replay.py _select_per); no torch forward, backward or optimizer kernel
    foreign = [k for k in others if not k.startswith("b2rl::")]
    assert len(foreign) == (replay_cls == "PrioritizedReplay") and all("direct_copy" in k for k in foreign), others
    assert any("feed_kernel" in k for k in others) and any("gather" in k for k in others), others
    if replay_cls == "PrioritizedReplay":
        assert any("sumtree_sample" in k for k in others), others
    ag.close()


@pytest.mark.gpu
def test_unsupported_configurations_are_refused(rl):
    def cfg(**kw):
        c = _golden_cfg(rl, "dqn_uni")
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    class OwnLoss(rl.DQNAgent):
        def reduce_loss(self, loss):
            return loss.pow(2).mean()

    refused = [
        (rl.CategoricalDQNAgent, dict(network_fn=lambda: rl.CategoricalNet(2, 51, rl.FCBody(4)), categorical_v_min=-10,
                                      categorical_v_max=10, categorical_n_atoms=51), "CategoricalNet"),
        (rl.QuantileRegressionDQNAgent, dict(network_fn=lambda: rl.QuantileNet(2, 20, rl.FCBody(4)), num_quantiles=20),
         "QuantileNet"),
        (rl.DQNAgent, dict(network_fn=lambda: rl.VanillaNet(2, rl.NatureConvBody(in_channels=4))), "NatureConvBody"),
        (rl.DQNAgent, dict(network_fn=lambda: rl.VanillaNet(2, rl.FCBody(4, noisy_linear=True))), "NoisyLinear"),
        (rl.DQNAgent, dict(network_fn=lambda: rl.VanillaNet(2, rl.FCBody(4, (64, 64, 64)))), "two-layer"),
        (rl.DQNAgent, dict(optimizer_fn=lambda p: torch.optim.Adam(p, 1e-3)), "Adam"),
        (rl.DQNAgent, dict(state_normalizer=rl.MeanStdNormalizer()), "MeanStdNormalizer"),
        (rl.DQNAgent, dict(async_actor=True), "async_actor"),
        (rl.DQNAgent, dict(history_length=4), "frame stacks"),
        (OwnLoss, {}, "reduce_loss"),
        (rl.DQNAgent, dict(batch_size=4096), "shared memory"),
    ]
    for cls, kw, msg in refused:
        with pytest.raises(NotImplementedError, match=msg):
            cls(cfg(**kw))
    ag = rl.DQNAgent(cfg())                                       # the supported form still builds
    ag.close()
