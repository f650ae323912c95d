"""n-step Q-learning on the device (``config.device_nstep_dqn``; deeprl_b200/csrc/a2c.cu): one ``b2rl_nstep_dqn_actor_step``
launch per env step and ONE ``b2rl_nstep_dqn_update`` launch for the rest of NStepDQN_agent.py:26-67, target sync included.

CPU: the update's phase functions (csrc/a2c_phases.h with HEAD = Q + nstep_sequence.inc) are compiled for the host by
tests/host_emul/nstep_emul.cpp and run with the block's threads in sequence, against the reference's recorded CartPole trajectory
(tests/golden/nstep.npz: online AND target parameters after each of 16 rollouts) and against oracle/agents.py nstep_dqn_update.
GPU: the CUDA build of the same source through the C ABI and through ``NStepDQNAgent``; the actor step's epsilon-greedy draws.

Tolerances: fp32 sums in another order than torch's CPU kernels, one RMSprop step per update: parameters to 1e-5 absolute."""
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
KEYS = ["body.layers.0.weight", "body.layers.0.bias", "body.layers.1.weight", "body.layers.1.bias", "fc_head.weight",
        "fc_head.bias"]                                       # the kernel's tensor order
T_G, N_G, FREQ = 5, 5, 12                                     # the golden record's rollout, workers and target sync period
F32P, I64P, I32P = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int32)


def fp(x):
    return x.ctypes.data_as(F32P)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("nstep_emul") / "nstep_emul.so")
    subprocess.run(["g++", "-O2", "-fno-strict-aliasing", "-std=c++17", "-shared", "-fPIC", "-o", out,
                    os.path.join(ROOT, "tests", "host_emul", "nstep_emul.cpp")], check=True)
    return ctypes.CDLL(out)


def arena(sd):
    """FlatOptimizer's layout (ops.py): every tensor starts on a multiple of 4 elements."""
    offs, n = [], 0
    for k in KEYS:
        offs.append(n)
        n += (sd[k].numel() + 3) // 4 * 4
    flat = np.zeros(n, np.float32)
    for k, o in zip(KEYS, offs):
        flat[o:o + sd[k].numel()] = sd[k].detach().numpy().ravel()
    return flat, np.asarray(offs, np.int32)


def unflatten(flat, offs, sd):
    return {k: flat[o:o + sd[k].numel()].reshape(tuple(sd[k].shape)) for k, o in zip(KEYS, offs)}


class EmulState:
    """Online arena, target arena, RMSprop moments and step count, carried across updates."""

    def __init__(self, sd, target_sd=None):
        self.flat, self.off = arena(sd)
        self.target = arena(target_sd if target_sd is not None else sd)[0]
        self.sq, self.ga = np.zeros_like(self.flat), np.zeros_like(self.flat)
        self.step = np.zeros(1, np.int64)
        self.loss = np.zeros(1, np.float32)


def emul_update(lib, st, gate, states, actions, rewards, masks, H1, H2, cfg, sync, threads=512, reversed_=False):
    """One b2rl_nstep_dqn_update on the host.  states (T+1,N,D), actions / rewards / masks (T,N)."""
    T, N, D = states.shape[0] - 1, states.shape[1], states.shape[2]
    s, a, r, m = (np.ascontiguousarray(np.asarray(x, np.float32)) for x in (states, actions, rewards, masks))
    rc = lib.nstep_emul_update(gate, fp(s), fp(a), fp(r), fp(m), T, N, D, H1, H2, cfg["A"], fp(st.flat), fp(st.target),
                               int(sync), fp(st.sq), fp(st.ga), st.step.ctypes.data_as(I64P), st.off.ctypes.data_as(I32P),
                               ctypes.c_float(cfg["lr"]), ctypes.c_float(cfg["alpha"]), ctypes.c_float(cfg["eps"]),
                               int(cfg["centered"]), ctypes.c_float(cfg["discount"]), ctypes.c_float(cfg["clip"]), fp(st.loss),
                               threads, int(reversed_))
    assert rc == 0


def flat_in(order, flat, off, sd):
    """The arena's tensors concatenated in ``order`` (the golden record's parameters() order)."""
    got = unflatten(flat, off, sd)
    return np.concatenate([got[k].ravel() for k in order])


# ------------------------------------------------------------------------------------------------ problems and the oracle
def make_problem(D, A, H1, H2, N, T, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale

    def net():
        return {"body.layers.0.weight": r(H1, D, scale=D ** -0.5), "body.layers.0.bias": r(H1, scale=0.1),
                "body.layers.1.weight": r(H2, H1, scale=H1 ** -0.5), "body.layers.1.bias": r(H2, scale=0.1),
                "fc_head.weight": r(A, H2, scale=H2 ** -0.5), "fc_head.bias": r(A, scale=0.1)}

    sd, target = net(), net()
    actions = torch.randint(0, A, (T, N), generator=g)
    states = r(T + 1, N, D)
    rewards = r(T, N)
    masks = (torch.rand(T, N, generator=g) > 0.2).float()
    return sd, target, states, actions, rewards, masks


CFG = dict(lr=1e-3, alpha=0.99, eps=1e-8, centered=False, discount=0.99, clip=5.0)
CASES = [  # (gate, D, A, H1, H2, N, T, sync, cfg overrides)
    (RELU, 4, 2, 64, 64, 5, 5, True, {}),                                       # n_step_dqn_feature (examples.py:408-424)
    (TANH, 11, 3, 32, 48, 3, 7, True, dict(centered=True, clip=1e6)),           # ragged, centered, the clip inactive
    (RELU, 11, 3, 32, 48, 3, 7, False, dict(centered=True, clip=0.05)),         # sync off (another target), the clip active
    (TANH, 11, 3, 32, 48, 3, 7, False, dict(lr=7e-4, clip=0.05)),
    (RELU, 11, 3, 32, 48, 3, 7, True, dict(discount=0.9, clip=1e6)),
]


def run_case(lib, case, threads=512, reversed_=False):
    gate, D, A, H1, H2, N, T, sync, over = CASES[case]
    cfg = dict(CFG, A=A, **over)
    sd0, tgt0, states, actions, rewards, masks = make_problem(D, A, H1, H2, N, T, seed=200 + case)
    st = EmulState(sd0, tgt0)
    emul_update(lib, st, gate, states.numpy(), actions.numpy(), rewards.numpy(), masks.numpy(), H1, H2, cfg, sync, threads,
                reversed_)
    return st, cfg, (gate, sync, sd0, tgt0, states, actions, rewards, masks)


def oracle_update(gate, sync, sd0, tgt0, states, actions, rewards, masks, cfg):
    """NStepDQN_agent.py:26-67 by the oracle: the sync inside the rollout (:48-50) copies the online parameters as they are
    before the update.  Returns (state dict, target state dict, optimizer, loss, gradient norm after the clip)."""
    sd = agents.leafify(sd0)
    tgt = {k: v.clone() for k, v in (sd0 if sync else tgt0).items()}
    params = [sd[k] for k in KEYS]
    opt = torch.optim.RMSprop(params, cfg["lr"], alpha=cfg["alpha"], eps=cfg["eps"], centered=cfg["centered"])
    gfn = torch.tanh if gate == TANH else F.relu
    _, loss = agents.nstep_dqn_update(sd, tgt, params, opt, states, actions, rewards.unsqueeze(-1), masks.unsqueeze(-1),
                                      cfg["discount"], cfg["clip"], gfn)
    clipped = float(torch.sqrt(sum((p.grad.double() ** 2).sum() for p in params)))
    return sd, tgt, opt, float(loss), clipped


def check_against_oracle(st, cfg, problem, atol=1e-5):
    gate, sync, sd0, tgt0 = problem[:4]
    sd, tgt, opt, loss, clipped = oracle_update(*problem, cfg)
    got, got_t = unflatten(st.flat, st.off, sd0), unflatten(st.target, st.off, sd0)
    sq, ga = unflatten(st.sq, st.off, sd0), unflatten(st.ga, st.off, sd0)
    for k in KEYS:
        want = sd[k].detach().numpy()
        np.testing.assert_allclose(got[k], want, rtol=0, atol=atol, err_msg=k)
        assert np.abs(want - sd0[k].numpy()).max() > 1e-5, k              # every tensor moved: not two untouched copies
        np.testing.assert_array_equal(got_t[k], tgt[k].numpy(), err_msg=k)  # synced: a copy; else untouched
        s = opt.state[sd[k]]
        np.testing.assert_allclose(sq[k], s["square_avg"].numpy(), rtol=2e-3, atol=1e-12, err_msg=k)
        if cfg["centered"]:
            np.testing.assert_allclose(ga[k], s["grad_avg"].numpy(), rtol=2e-3, atol=1e-8, err_msg=k)
    np.testing.assert_allclose(st.loss[0], loss, rtol=1e-5, atol=1e-6)
    assert int(st.step[0]) == 1
    if not sync:
        assert any(np.abs(tgt0[k].numpy() - sd0[k].numpy()).max() > 0.1 for k in KEYS)
    return clipped


# ------------------------------------------------------------------------------------------------ CPU: host emulation
def golden_rollout(g, it, state):
    sl = slice(it * T_G, (it + 1) * T_G)
    states = np.concatenate([state[None], g["next_states"][sl].astype(np.float32)])
    rewards = g["rewards"][sl].astype(np.float32)                           # tensor(): float32 (torch_utils.py:20-25)
    masks = (1 - g["dones"][sl].astype(np.int64)).astype(np.float32)
    sync = any((it * T_G + k + 1) % FREQ == 0 for k in range(T_G))        # NStepDQN_agent.py:48-50, per env step
    return states, g["actions"][sl], rewards, masks, sync


def test_golden_trajectory_emulated(emul, golden):
    """The reference's own n_step_dqn_feature record (CartPole, 5 workers, rollout 5, target sync every 12 env steps): 16
    consecutive updates with the recorded actions and env stream give the recorded online and target parameters."""
    g = golden("nstep")
    order = [str(k) for k in g["keys"]]
    sd0 = {k: torch.from_numpy(g["init." + k]) for k in KEYS}
    st = EmulState(sd0)
    cfg = dict(CFG, A=2)
    worst, syncs = 0.0, 0
    state = g["state0"].astype(np.float32)
    for it in range(g["params"].shape[0]):
        states, actions, rewards, masks, sync = golden_rollout(g, it, state)
        syncs += sync
        emul_update(emul, st, RELU, states, actions, rewards, masks, 64, 64, cfg, sync)
        err = float(np.abs(flat_in(order, st.flat, st.off, sd0) - g["params"][it]).max())
        err_t = float(np.abs(flat_in(order, st.target, st.off, sd0) - g["target_params"][it]).max())
        worst = max(worst, err, err_t)
        assert err <= 1e-5 and err_t <= 1e-5, (it, err, err_t)
        state = states[-1]
    assert int(st.step[0]) == 16 and syncs == 6
    print("largest online / target parameter difference over the 16 golden steps: %.3g" % worst)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_update_matches_oracle_emulated(emul, case):
    st, cfg, problem = run_case(emul, case)
    clipped = check_against_oracle(st, cfg, problem)
    if cfg["clip"] < 1.0:
        assert abs(clipped - cfg["clip"]) < 1e-4 * cfg["clip"]              # the clip was active
    elif cfg["clip"] >= 1e5:
        assert clipped < cfg["clip"]                                         # ... and here it was not


@pytest.mark.parametrize("case", [0, 2])
def test_thread_order_and_count_do_not_change_the_result(emul, case):
    """Reversed thread order inside every phase, 64 and 37 threads instead of 512: bit-identical arenas (the race check)."""
    ref, _, _ = run_case(emul, case)
    for threads, rev in ((512, True), (64, False), (37, True)):
        got, _, _ = run_case(emul, case, threads, rev)
        for k in ("flat", "target", "sq", "ga", "loss", "step"):
            assert np.array_equal(getattr(ref, k), getattr(got, k)), (threads, rev, k)


def test_kernels_have_no_spills_and_no_stack_frame(tmp_path):
    out = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                          os.path.join(ROOT, "deeprl_b200", "csrc", "a2c.cu"), "-o", str(tmp_path / "a2c.o")],
                         check=True, capture_output=True, text=True).stderr
    entries = out.split("Compiling entry function")[1:]
    names = [e.split("'")[1] for e in entries]
    # Q x (tanh, ReLU), the update and the actor step
    assert sum("nstep_dqn_update_kernel" in n for n in names) == 2, names
    assert sum("nstep_dqn_actor_kernel" in n for n in names) == 2, names
    for e in entries:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in e, e


def test_shared_memory_budget_accepts_the_launcher():
    from deeprl_b200 import _lib
    L = _lib.lib()
    feature = L.b2rl_nstep_dqn_smem_bytes(4, 64, 64, 2, 5, 5)              # n_step_dqn_feature: CartPole, 5 workers, rollout 5
    assert 0 < feature <= 227 * 1024, feature
    assert L.b2rl_nstep_dqn_smem_bytes(4, 128, 128, 2, 64, 20) > 227 * 1024
    assert L.b2rl_nstep_dqn_smem_bytes(4, 64, 64, 2, 0, 5) == 0


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
    gate, D, A, H1, H2, N, T, sync, over = CASES[case]
    cfg = dict(CFG, A=A, **over)
    sd0, tgt0, states, actions, rewards, masks = make_problem(D, A, H1, H2, N, T, seed=200 + case)
    st = EmulState(sd0, tgt0)
    cu = lambda x: torch.as_tensor(np.ascontiguousarray(np.asarray(x, np.float32))).cuda()
    t = dict(s=cu(states), a=cu(actions), r=cu(rewards), m=cu(masks), flat=cu(st.flat), target=cu(st.target), sq=cu(st.sq),
             ga=cu(st.ga))
    step, loss, off = torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros((), device="cuda"), torch.from_numpy(st.off)
    _lib.call("b2rl_nstep_dqn_update", gate, _lib.ptr(t["s"]), _lib.ptr(t["a"]), _lib.ptr(t["r"]), _lib.ptr(t["m"]), T, N, D,
              H1, H2, A, _lib.ptr(t["flat"]), _lib.ptr(t["target"]), int(sync), _lib.ptr(t["sq"]), _lib.ptr(t["ga"]),
              _lib.ptr(step), _lib.ptr(off), cfg["lr"], cfg["alpha"], cfg["eps"], int(cfg["centered"]), cfg["discount"],
              cfg["clip"], _lib.ptr(loss), _lib.stream())
    torch.cuda.synchronize()
    st.flat, st.target, st.sq, st.ga = (t[k].cpu().numpy() for k in ("flat", "target", "sq", "ga"))
    st.step, st.loss = step.cpu().numpy(), loss.reshape(1).cpu().numpy()
    check_against_oracle(st, cfg, (gate, sync, sd0, tgt0, states, actions, rewards, masks))


def _replay_task(g):
    class Replay:                                          # Task stand-in that replays the recorded env stream
        def __init__(self):
            self.k = 0
            self.state_dim, self.action_dim, self.name = 4, 2, "replayed"

        def reset(self):
            return list(g["state0"])

        def step(self, actions):
            k = self.k
            self.k += 1
            assert np.array_equal(np.asarray(actions), g["actions"][k])
            return (list(g["next_states"][k]), g["rewards"][k], g["dones"][k],
                    tuple({"episodic_return": None} for _ in range(N_G)))

        def close(self):
            pass

    return Replay


def _config(rl, task_fn, **kw):
    c = rl.Config()
    c.merge(dict(tag=None, device_nstep_dqn=True, **kw))
    c.num_workers = N_G
    c.task_fn = task_fn
    c.optimizer_fn = lambda p: torch.optim.RMSprop(p, 0.001)
    c.network_fn = lambda: rl.VanillaNet(2, rl.FCBody(4))
    c.random_action_prob = rl.LinearSchedule(0.6, 0.1, 200)
    c.discount, c.target_network_update_freq, c.rollout_length, c.gradient_clip = 0.99, FREQ, T_G, 5
    return c


def _params(net):
    return np.concatenate([p.detach().cpu().numpy().ravel() for p in net.parameters()])


@pytest.mark.gpu
def test_agent_replays_the_golden_record(rl, golden):
    """NStepDQNAgent with device_nstep_dqn on the reference's recorded CartPole stream, the recorded actions given to the actor
    step's parity mode: the recorded online and target parameters after each of the 16 steps (1e-5)."""
    g = golden("nstep")
    ag = rl.NStepDQNAgent(_config(rl, _replay_task(g)))
    with torch.no_grad():
        for net in (ag.network, ag.target_network):
            for k, p in net.state_dict().items():
                p.copy_(torch.from_numpy(g["init." + k]))
    ag.device_nstep_dqn.forced = lambda: g["actions"][ag.task.k]
    worst = 0.0
    for it in range(g["params"].shape[0]):
        ag.step()
        err = float(np.abs(_params(ag.network) - g["params"][it]).max())
        err_t = float(np.abs(_params(ag.target_network) - g["target_params"][it]).max())
        worst = max(worst, err, err_t)
        assert err <= 1e-5 and err_t <= 1e-5, (it, err, err_t)
        assert ag.last_loss.dim() == 0 and torch.isfinite(ag.last_loss)
    assert ag.total_steps == N_G * T_G * 16 and int(ag.optimizer.step_dev) == 16
    dev = ag.device_nstep_dqn
    for net, flat in ((ag.network, dev.opt.flat), (ag.target_network, dev.target)):
        for t, o in zip(dev.kernel_order(net), dev.off.tolist()):           # state_dict() is a view of the arena
            assert torch.equal(t.detach().reshape(-1), flat[o:o + t.numel()])
    print("device agent vs golden record, largest parameter difference: %.3g" % worst)


def _actor(rl, gate, N, D, H, A, seed=5):
    """A FlatOptimizer arena for one VanillaNet and a call of b2rl_nstep_dqn_actor_step on it."""
    from deeprl_b200 import _lib, ops
    torch.manual_seed(seed)
    net = rl.VanillaNet(A, rl.FCBody(D, (H, H), gate=torch.tanh if gate == TANH else F.relu))
    with torch.no_grad():                                   # q-values far enough apart to be visible
        net.fc_head.weight.normal_(0, 0.5)
        net.fc_head.bias.normal_(0, 0.5)
    tensors = [t for m in net.body.layers for t in (m.weight, m.bias)] + [net.fc_head.weight, net.fc_head.bias]
    opt = ops.FlatOptimizer.from_torch(torch.optim.RMSprop(net.parameters(), 1e-3), list(net.parameters()))
    off = torch.tensor([(t.data_ptr() - opt.flat.data_ptr()) // 4 for t in tensors], dtype=torch.int32)

    def step(obs, counter, seed, eps, given=None, scale=1.0):
        st = torch.empty((N, D), device="cuda")
        act = torch.empty((N, 1), device="cuda")
        _lib.call("b2rl_nstep_dqn_actor_step", gate, _lib.ptr(obs), scale, _lib.ptr(opt.flat), _lib.ptr(off), D, H, H, A, N,
                  eps, _lib.ptr(st), _lib.ptr(act), _lib.ptr(given), seed, _lib.ptr(counter), _lib.stream())
        torch.cuda.synchronize()
        return st, act[:, 0].long()

    return net, step


@pytest.mark.gpu
def test_actor_step_epsilon_greedy(rl):
    """epsilon = 0: the argmax of a torch forward of the same net (no row within 1e-3 of a tie); epsilon = 1: uniform frequencies
    (Pearson chi-square below the 0.999 quantile of its A - 1 degrees of freedom at the fixed seed 11); epsilon = 0.25: the share
    of non-greedy actions within 5 binomial standard errors of epsilon (A - 1) / A; the same seed and counter give the same
    actions; the counter advances by 2 N per step; given actions are written through and leave it alone; the state row is the
    rescaled observation."""
    from scipy import stats
    N, D, H, A, steps = 64, 6, 32, 5, 1000
    net, step = _actor(rl, RELU, N, D, H, A)
    cand = torch.randn(4096, D, dtype=torch.float64, device="cuda")
    with torch.no_grad():
        q = net(cand.float())["q"]
    top = q.topk(2, dim=1).values
    obs = cand[(top[:, 0] - top[:, 1]) > 1e-3][:N].contiguous()
    assert obs.shape[0] == N
    with torch.no_grad():
        greedy = net(obs.float())["q"].argmax(1)
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    st, a = step(obs, counter, 11, 0.0, scale=0.5)
    assert torch.equal(st, (0.5 * obs).float()) and int(counter) == 2 * N
    st, a = step(obs, counter, 11, 0.0)
    assert torch.equal(a, greedy) and int(counter) == 4 * N

    counts = np.zeros(A)
    for _ in range(steps):
        counts += np.bincount(step(obs, counter, 11, 1.0)[1].cpu().numpy(), minlength=A)
    exp_c = steps * N / A
    assert float(((counts - exp_c) ** 2 / exp_c).sum()) < stats.chi2.ppf(0.999, A - 1), counts

    eps, other = 0.25, 0
    for _ in range(steps):
        other += int((step(obs, counter, 11, eps)[1] != greedy).sum())
    n, p = steps * N, eps * (A - 1) / A
    assert abs(other / n - p) < 5 * np.sqrt(p * (1 - p) / n), (other / n, p)
    assert int(counter) == 2 * N * (2 + 2 * steps)

    c1, c2 = torch.full((1,), 77, dtype=torch.int64, device="cuda"), torch.full((1,), 77, dtype=torch.int64, device="cuda")
    assert torch.equal(step(obs, c1, 3, 0.5)[1], step(obs, c2, 3, 0.5)[1]) and int(c1) == 77 + 2 * N
    given = torch.randint(0, A, (N, 1), device="cuda").float()
    assert torch.equal(step(obs, c1, 3, 0.5, given)[1], given[:, 0].long()) and int(c1) == 77 + 2 * N


def _launcher_agent(monkeypatch, **kw):
    import examples
    got = []
    monkeypatch.setattr(examples, "run_steps", got.append)
    examples.n_step_dqn_feature(game="CartPole-v0", device_nstep_dqn=True, **kw)
    return got[0]


@pytest.mark.gpu
def test_launcher_end_to_end(rl, monkeypatch):
    """n_step_dqn_feature with device_nstep_dqn: finite, varying losses over 45 steps; after a step whose rollout reaches the sync
    schedule the target arena is the online arena as it was before that step, after any other step it is unchanged; one
    profiled step() is exactly T actor-step kernels and one update kernel, besides copies."""
    ag = _launcher_agent(monkeypatch)
    c, dev = ag.config, ag.device_nstep_dqn
    N, T = c.num_workers, c.rollout_length
    losses_, seen = [], set()
    for _ in range(45):
        k0 = ag.total_steps // N
        sync = any((k0 + k) % c.target_network_update_freq == 0 for k in range(1, T + 1))
        before, target = dev.opt.flat.clone(), dev.target.clone()
        ag.step()
        torch.cuda.synchronize()
        assert torch.equal(dev.target, before if sync else target), (k0, sync)
        seen.add(sync)
        losses_.append(ag.last_loss)
    assert seen == {True, False}
    assert all(bool(torch.isfinite(x)) for x in losses_) and ag.total_steps == 45 * N * T
    assert len(set(float(x) for x in losses_)) > 1
    torch.cuda.synchronize()
    # one warm-up cycle of the profiler, then the recorded step (events launched as the tracer starts can be missed)
    from _kernel_trace import profiled_kernels
    kernels = profiled_kernels(lambda: (ag.step(), torch.cuda.synchronize()),
                               {"nstep_dqn_actor_kernel": T, "nstep_dqn_update_kernel": 1})
    assert sum("nstep_dqn_actor_kernel" in k for k in kernels) == T, kernels
    assert sum("nstep_dqn_update_kernel" in k for k in kernels) == 1, kernels
    assert len(kernels) == T + 1, kernels
    ag.close()


@pytest.mark.gpu
def test_unsupported_configurations_are_refused(rl):
    def agent(**kw):
        c = _config(rl, lambda: rl.Task("CartPole-v0", num_envs=N_G, seed=0))
        c.eval_env = rl.Task("CartPole-v0", seed=0)
        for k, v in kw.items():
            setattr(c, k, v)
        return rl.NStepDQNAgent(c)

    refused = [
        (dict(network_fn=lambda: rl.VanillaNet(2, rl.NatureConvBody(in_channels=4))), "NatureConvBody"),
        (dict(network_fn=lambda: rl.DuelingNet(2, rl.FCBody(4))), "DuelingNet"),
        (dict(network_fn=lambda: rl.VanillaNet(2, rl.FCBody(4, noisy_linear=True))), "NoisyLinear"),
        (dict(network_fn=lambda: rl.VanillaNet(2, rl.FCBody(4, (64, 64, 64)))), "two-layer"),
        (dict(optimizer_fn=lambda p: torch.optim.Adam(p, 1e-3)), "Adam"),
        (dict(state_normalizer=rl.MeanStdNormalizer()), "MeanStdNormalizer"),
        (dict(num_workers=64, rollout_length=40), "shared memory"),
    ]
    for kw, msg in refused:
        with pytest.raises(NotImplementedError, match=msg):
            agent(**kw)
    ag = agent()                                                  # the supported form still builds
    ag.close()
