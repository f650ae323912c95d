"""A2C on the device (``config.device_a2c``; deeprl_b200/csrc/a2c.cu): one ``b2rl_a2c_actor_step`` launch per env step and
ONE ``b2rl_a2c_update`` launch for the rest of A2C_agent.py:22-64.

CPU: the update's phase functions (csrc/a2c_phases.h + a2c_sequence.inc) are compiled for the host by tests/host_emul and run
with the block's threads in sequence, against the reference's recorded CartPole trajectory (tests/golden/onpolicy.npz, the
categorical shared-trunk net of a2c_feature) and against restatements of A2C_agent.py:22-64 on torch-CPU (oracle/agents.py
a2c_update for the categorical net; ``a2c_update_gaussian`` below for the Gaussian separate-trunk net of a2c_continuous).
GPU: the CUDA build of the same source through the C ABI and through ``A2CAgent``; the actor step's sampling.

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
from oracle import agents, losses, nets  # noqa: E402

CAT, GAUSS = 0, 1
TANH, RELU = 0, 1
CAT_KEYS = ["phi_body.layers.0.weight", "phi_body.layers.0.bias", "phi_body.layers.1.weight", "phi_body.layers.1.bias",
            "fc_action.weight", "fc_action.bias", "fc_critic.weight", "fc_critic.bias"]
GAUSS_KEYS = ["actor_body.layers.0.weight", "actor_body.layers.0.bias", "actor_body.layers.1.weight", "actor_body.layers.1.bias",
              "critic_body.layers.0.weight", "critic_body.layers.0.bias", "critic_body.layers.1.weight",
              "critic_body.layers.1.bias", "fc_action.weight", "fc_action.bias", "fc_critic.weight", "fc_critic.bias", "std"]
F32P, I64P, I32P = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int32)


def fp(x):
    return x.ctypes.data_as(F32P)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("a2c_emul") / "a2c_emul.so")
    subprocess.run(["g++", "-O2", "-fno-strict-aliasing", "-std=c++17", "-shared", "-fPIC", "-o", out,
                    os.path.join(ROOT, "tests", "host_emul", "a2c_emul.cpp")], check=True)
    return ctypes.CDLL(out)


def arena(sd, keys):
    """FlatOptimizer's layout (ops.py): every tensor starts on a multiple of 4 elements; keys in the kernel's tensor order."""
    offs, n = [], 0
    for k in keys:
        offs.append(n)
        n += (sd[k].numel() + 3) // 4 * 4
    flat = np.zeros(n, np.float32)
    for k, o in zip(keys, offs):
        flat[o:o + sd[k].numel()] = sd[k].detach().numpy().ravel()
    return flat, np.asarray(offs, np.int32)


def unflatten(flat, offs, sd, keys):
    return {k: flat[o:o + sd[k].numel()].reshape(tuple(sd[k].shape)) for k, o in zip(keys, offs)}


class EmulState:
    """The arena, RMSprop moments and step count of one FlatOptimizer, carried across updates."""

    def __init__(self, sd, keys):
        self.keys = keys
        self.flat, self.off = arena(sd, keys)
        self.sq, self.ga = np.zeros_like(self.flat), np.zeros_like(self.flat)
        self.step = np.zeros(1, np.int64)
        self.loss = np.zeros(1, np.float32)


def emul_update(lib, st, head, gate, states, actions, rewards, masks, H1, H2, cfg, threads=512, reversed_=False):
    """One b2rl_a2c_update on the host.  states (T+1,N,D), actions (T,N) int or (T,N,A), rewards / masks (T,N)."""
    T, N, D = states.shape[0] - 1, states.shape[1], states.shape[2]
    A = cfg["A"]
    s, a, r, m = (np.ascontiguousarray(np.asarray(x, np.float32)) for x in (states, actions, rewards, masks))
    rc = lib.a2c_emul_update(head, int(head == CAT), gate, fp(s), fp(a), fp(r), fp(m), T, N, D, H1, H2, A, fp(st.flat), fp(st.sq),
                             fp(st.ga), st.step.ctypes.data_as(I64P), st.off.ctypes.data_as(I32P), ctypes.c_float(cfg["lr"]),
                             ctypes.c_float(cfg["alpha"]), ctypes.c_float(cfg["eps"]), int(cfg["centered"]),
                             ctypes.c_float(cfg["discount"]), ctypes.c_float(cfg["tau"]), int(cfg["use_gae"]),
                             ctypes.c_float(cfg["ent_w"]), ctypes.c_float(cfg["vw"]), ctypes.c_float(cfg["clip"]), fp(st.loss),
                             threads, int(reversed_))
    assert rc == 0


# ------------------------------------------------------------------------------------------------ problems and the oracle
def make_problem(head, D, A, H1, H2, N, T, seed, std_scale=0.3):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale
    if head == CAT:
        sd = {"phi_body.layers.0.weight": r(H1, D, scale=D ** -0.5), "phi_body.layers.0.bias": r(H1, scale=0.1),
              "phi_body.layers.1.weight": r(H2, H1, scale=H1 ** -0.5), "phi_body.layers.1.bias": r(H2, scale=0.1),
              "fc_action.weight": r(A, H2, scale=H2 ** -0.5), "fc_action.bias": r(A, scale=0.1),
              "fc_critic.weight": r(1, H2, scale=H2 ** -0.5), "fc_critic.bias": r(1, scale=0.1)}
        actions = torch.randint(0, A, (T, N), generator=g)
    else:
        sd = {}
        for body in ("actor_body", "critic_body"):
            sd.update({body + ".layers.0.weight": r(H1, D, scale=D ** -0.5), body + ".layers.0.bias": r(H1, scale=0.1),
                       body + ".layers.1.weight": r(H2, H1, scale=H1 ** -0.5), body + ".layers.1.bias": r(H2, scale=0.1)})
        sd.update({"fc_action.weight": r(A, H2, scale=0.5 * H2 ** -0.5), "fc_action.bias": r(A, scale=0.05),
                   "fc_critic.weight": r(1, H2, scale=H2 ** -0.5), "fc_critic.bias": r(1, scale=0.1), "std": r(A, scale=std_scale)})
        actions = r(T, N, A)
    states = r(T + 1, N, D)
    rewards = r(T, N)
    masks = (torch.rand(T, N, generator=g) > 0.2).float()
    return sd, states, actions, rewards, masks


def a2c_update_gaussian(sd, params, opt, states, actions, rewards, masks, discount, tau, entropy_weight,
                        value_loss_weight, gradient_clip, use_gae=True, gate=F.relu):
    """A2C_agent.py:22-64 for a GaussianActorCriticNet with separate actor / critic FCBody trunks (network_heads.py:173-214;
    ``a2c_continuous``, examples.py:384-404), one rollout whose env interaction is given: ``states`` (T+1,N,obs),
    ``actions`` (T,N,A), ``rewards``/``masks`` (T,N,1).  The companion of oracle/agents.py ``a2c_update`` (the categorical,
    shared-trunk net), built from the same oracle pieces.  Returns (adv, ret, loss)."""
    T = actions.shape[0]
    preds = [nets.gaussian_actor_critic(sd, states[t], actions[t], gate) for t in range(T)]      # :27-31, graphs kept
    last = nets.gaussian_actor_critic(sd, states[T], actions[T - 1], gate)                        # :38-41, only its v is used
    v = torch.stack([p["v"] for p in preds] + [last["v"]])
    adv, ret = losses.gae(rewards, masks, v.detach(), discount, tau, use_gae)                     # :43-53
    cat = lambda k: torch.cat([p[k] for p in preds], dim=0)
    loss = losses.a2c_loss(cat("log_pi_a"), cat("v"), ret.reshape(-1, 1), adv.reshape(-1, 1), cat("entropy"),
                           entropy_weight, value_loss_weight)                                      # :55-62
    opt.zero_grad()
    loss.backward()
    agents.clip_grad_norm(params, gradient_clip)                                                   # :63
    opt.step()                                                                                     # :64
    return adv, ret, loss.detach()


def oracle_update(head, gate, sd0, states, actions, rewards, masks, cfg):
    """One A2C_agent.py:22-64 update by the oracle; returns (state dict, optimizer, loss, gradient norm after the clip)."""
    keys = CAT_KEYS if head == CAT else GAUSS_KEYS
    sd = agents.leafify(sd0)
    params = [sd[k] for k in keys]
    opt = torch.optim.RMSprop(params, cfg["lr"], alpha=cfg["alpha"], eps=cfg["eps"], centered=cfg["centered"])
    gfn = torch.tanh if gate == TANH else F.relu
    r, m = rewards.unsqueeze(-1), masks.unsqueeze(-1)
    if head == CAT:
        T = actions.shape[0]
        with torch.no_grad():                               # the objective at the starting parameters (a2c_update returns none)
            preds = [nets.categorical_actor_critic(sd, states[t], actions[t], gfn) for t in range(T)]
            v = torch.stack([p["v"] for p in preds] + [nets.categorical_actor_critic(sd, states[T], None, gfn)["v"]])
            adv, ret = losses.gae(r, m, v, cfg["discount"], cfg["tau"], cfg["use_gae"])
            cat = lambda k: torch.cat([p[k] for p in preds], dim=0)
            loss = losses.a2c_loss(cat("log_pi_a"), cat("v"), ret.reshape(-1, 1), adv.reshape(-1, 1), cat("entropy"),
                                   cfg["ent_w"], cfg["vw"])
        assert cfg["use_gae"]
        agents.a2c_update(sd, params, opt, states, actions, r, m, cfg["discount"], cfg["tau"], cfg["ent_w"], cfg["vw"],
                          cfg["clip"], gfn)
    else:
        _, _, loss = a2c_update_gaussian(sd, params, opt, states, actions, r, m, cfg["discount"], cfg["tau"],
                                                cfg["ent_w"], cfg["vw"], cfg["clip"], cfg["use_gae"], gfn)
    clipped = float(torch.sqrt(sum((p.grad.double() ** 2).sum() for p in params)))     # the norm after clip_grad_norm_
    return sd, opt, float(loss), clipped


CFG = dict(lr=7e-4, alpha=0.99, eps=1e-8, centered=False, discount=0.99, tau=1.0, use_gae=True, ent_w=0.01, vw=1.0, clip=5.0)
CASES = [  # (head, gate, D, A, H1, H2, N, T, cfg overrides)
    (GAUSS, RELU, 17, 6, 64, 64, 16, 5, {}),                                            # a2c_continuous (examples.py:384-404)
    (GAUSS, TANH, 11, 3, 32, 48, 3, 7, dict(use_gae=False, vw=0.5, clip=1e6)),           # ragged, no GAE, the clip inactive
    (GAUSS, RELU, 11, 3, 32, 48, 3, 7, dict(centered=True, tau=0.95, clip=0.05)),        # ragged, centered, the clip active
    (CAT, TANH, 4, 2, 64, 64, 5, 5, dict(lr=1e-3, tau=0.95, clip=0.5)),                  # a2c_feature (examples.py:340-360)
    (CAT, RELU, 11, 3, 32, 48, 3, 7, dict(lr=1e-3, tau=0.95, clip=1e6, vw=2.0)),         # ragged categorical, the clip inactive
]


def run_case(lib, case, threads=512, reversed_=False):
    head, gate, D, A, H1, H2, N, T, over = CASES[case]
    cfg = dict(CFG, A=A, **over)
    sd0, states, actions, rewards, masks = make_problem(head, D, A, H1, H2, N, T, seed=100 + case)
    st = EmulState(sd0, CAT_KEYS if head == CAT else GAUSS_KEYS)
    emul_update(lib, st, head, gate, states.numpy(), actions.numpy(), rewards.numpy(), masks.numpy(), H1, H2, cfg, threads,
                reversed_)
    return st, cfg, (head, gate, sd0, states, actions, rewards, masks)


def check_against_oracle(st, cfg, problem, atol=1e-5):
    head, gate, sd0, states, actions, rewards, masks = problem
    sd, opt, loss, clipped = oracle_update(head, gate, sd0, states, actions, rewards, masks, cfg)
    got = unflatten(st.flat, st.off, sd0, st.keys)
    sq, ga = unflatten(st.sq, st.off, sd0, st.keys), unflatten(st.ga, st.off, sd0, st.keys)
    for k in st.keys:
        want = sd[k].detach().numpy()
        np.testing.assert_allclose(got[k], want, rtol=0, atol=atol, err_msg=k)
        assert np.abs(want - sd0[k].numpy()).max() > 1e-5, k              # every tensor moved: not two untouched copies
        s = opt.state[sd[k]]
        np.testing.assert_allclose(sq[k], s["square_avg"].numpy(), rtol=2e-3, atol=1e-12, err_msg=k)
        if cfg["centered"]:
            np.testing.assert_allclose(ga[k], s["grad_avg"].numpy(), rtol=2e-3, atol=1e-8, err_msg=k)
    np.testing.assert_allclose(st.loss[0], loss, rtol=1e-5, atol=1e-6)
    assert int(st.step[0]) == 1
    return clipped


# ------------------------------------------------------------------------------------------------ CPU: host emulation
def test_golden_trajectory_emulated(emul, golden):
    """The reference's own a2c_feature record (CartPole, 8 workers, rollout 5): 6 consecutive updates with the recorded actions
    and env stream give the recorded parameters after every step."""
    g = golden("onpolicy")
    sd0 = {k: torch.from_numpy(g["a2c_init." + k]) for k in CAT_KEYS}
    st = EmulState(sd0, CAT_KEYS)
    cfg = dict(CFG, A=2, lr=1e-3, tau=0.95, clip=0.5)
    T, worst = 5, 0.0
    state = g["a2c_state0"].astype(np.float32)
    for it in range(g["a2c_params"].shape[0]):
        sl = slice(it * T, (it + 1) * T)
        states = np.concatenate([state[None], g["a2c_next_states"][sl].astype(np.float32)])
        rewards = g["a2c_rewards"][sl].astype(np.float32)                       # tensor(): float32 (torch_utils.py:20-25)
        masks = (1 - g["a2c_dones"][sl].astype(np.int64)).astype(np.float32)
        emul_update(emul, st, CAT, TANH, states, g["a2c_actions"][sl], rewards, masks, 64, 64, cfg)
        flat = np.concatenate([st.flat[o:o + sd0[k].numel()] for k, o in zip(CAT_KEYS, st.off)])
        err = float(np.abs(flat - g["a2c_params"][it]).max())
        worst = max(worst, err)
        assert err <= 1e-5, (it, err)
        state = states[-1]
    assert int(st.step[0]) == 6
    print("largest parameter difference over the 6 golden steps: %.3g" % worst)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_update_matches_oracle_emulated(emul, case):
    st, cfg, problem = run_case(emul, case)
    clipped = check_against_oracle(st, cfg, problem)
    if cfg["clip"] < 1.0:
        assert abs(clipped - cfg["clip"]) < 1e-4 * cfg["clip"]              # the clip was active
    else:
        assert clipped < cfg["clip"]                                         # ... and here it was not


@pytest.mark.parametrize("case", [0, 3])
def test_thread_order_and_count_do_not_change_the_result(emul, case):
    """Reversed thread order inside every phase, and 64 instead of 512 threads: bit-identical arenas (the race check)."""
    ref, _, _ = run_case(emul, case)
    for threads, rev in ((512, True), (64, False), (37, True)):
        got, _, _ = run_case(emul, case, threads, rev)
        for k in ("flat", "sq", "ga", "loss", "step"):
            assert np.array_equal(getattr(ref, k), getattr(got, k)), (threads, rev, k)


def test_kernels_have_no_spills_and_no_stack_frame(tmp_path):
    out = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                          os.path.join(ROOT, "deeprl_b200", "csrc", "a2c.cu"), "-o", str(tmp_path / "a2c.o")],
                         check=True, capture_output=True, text=True).stderr
    entries = out.split("Compiling entry function")[1:]
    names = [e.split("'")[1] for e in entries]
    assert sum("a2c_update_kernel" in n for n in names) == 4 and sum("a2c_actor_kernel" in n for n in names) == 4, names
    for e in entries:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in e, e


def test_shared_memory_budget_accepts_the_launchers():
    from deeprl_b200 import _lib
    L = _lib.lib()
    cat = L.b2rl_a2c_smem_bytes(CAT, 1, 4, 64, 64, 2, 5, 5)                  # a2c_feature: CartPole, 5 workers, rollout 5
    gauss = L.b2rl_a2c_smem_bytes(GAUSS, 0, 17, 64, 64, 6, 16, 5)            # a2c_continuous: SyntheticCheetah, 16 workers
    assert 0 < cat <= 227 * 1024 and 0 < gauss <= 227 * 1024, (cat, gauss)
    assert L.b2rl_a2c_smem_bytes(GAUSS, 0, 17, 128, 128, 6, 64, 20) > 227 * 1024
    assert L.b2rl_a2c_smem_bytes(CAT, 0, 4, 64, 64, 2, 5, 5) == 0             # not an instantiated configuration


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
    head, gate, D, A, H1, H2, N, T, over = CASES[case]
    cfg = dict(CFG, A=A, **over)
    sd0, states, actions, rewards, masks = make_problem(head, D, A, H1, H2, N, T, seed=100 + case)
    st = EmulState(sd0, CAT_KEYS if head == CAT else GAUSS_KEYS)
    cu = lambda x: torch.as_tensor(np.ascontiguousarray(np.asarray(x, np.float32))).cuda()
    t = dict(s=cu(states), a=cu(actions), r=cu(rewards), m=cu(masks), flat=cu(st.flat), sq=cu(st.sq), ga=cu(st.ga))
    step, loss, off = torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros((), device="cuda"), torch.from_numpy(st.off)
    _lib.call("b2rl_a2c_update", head, int(head == CAT), gate, _lib.ptr(t["s"]), _lib.ptr(t["a"]), _lib.ptr(t["r"]),
              _lib.ptr(t["m"]), T, N, D, H1, H2, A, _lib.ptr(t["flat"]), _lib.ptr(t["sq"]), _lib.ptr(t["ga"]), _lib.ptr(step),
              _lib.ptr(off), cfg["lr"], cfg["alpha"], cfg["eps"], int(cfg["centered"]), cfg["discount"], cfg["tau"],
              int(cfg["use_gae"]), cfg["ent_w"], cfg["vw"], cfg["clip"], _lib.ptr(loss), _lib.stream())
    torch.cuda.synchronize()
    st.flat, st.sq, st.ga = (t[k].cpu().numpy() for k in ("flat", "sq", "ga"))
    st.step, st.loss = step.cpu().numpy(), loss.reshape(1).cpu().numpy()
    check_against_oracle(st, cfg, (head, gate, sd0, states, actions, rewards, masks))


def _replay_task(g, n):
    class Replay:                                          # Task stand-in that replays the recorded env stream
        def __init__(self):
            self.k = 0
            self.state_dim, self.action_dim, self.name = 4, 2, "replayed"

        def reset(self):
            return list(g["a2c_state0"])

        def step(self, actions):
            k = self.k
            self.k += 1
            assert np.array_equal(np.asarray(actions), g["a2c_actions"][k])
            return (list(g["a2c_next_states"][k]), g["a2c_rewards"][k], g["a2c_dones"][k],
                    tuple({"episodic_return": None} for _ in range(n)))

        def close(self):
            pass

    return Replay


def _a2c_feature_config(rl, n, task_fn, **kw):
    c = rl.Config()
    c.merge(dict(tag=None, device_a2c=True, **kw))
    c.num_workers = n
    c.task_fn = task_fn
    c.optimizer_fn = lambda p: torch.optim.RMSprop(p, 0.001)
    c.network_fn = lambda: rl.CategoricalActorCriticNet(4, 2, rl.FCBody(4, gate=torch.tanh))
    c.discount, c.use_gae, c.gae_tau, c.entropy_weight, c.rollout_length, c.gradient_clip = 0.99, True, 0.95, 0.01, 5, 0.5
    return c


@pytest.mark.gpu
def test_agent_replays_the_golden_record(rl, golden):
    """A2CAgent with device_a2c on the reference's recorded CartPole stream, the recorded actions given to the actor step's
    parity mode: the recorded parameters after each of the 6 steps (1e-5)."""
    g = golden("onpolicy")
    keys = [str(k) for k in g["a2c_keys"]]
    ag = rl.A2CAgent(_a2c_feature_config(rl, 8, _replay_task(g, 8)))
    with torch.no_grad():
        for k, p in ag.network.state_dict().items():
            p.copy_(torch.from_numpy(g["a2c_init." + k]))
    ag.device_a2c.forced = lambda: g["a2c_actions"][ag.task.k]
    worst = 0.0
    for it in range(g["a2c_params"].shape[0]):
        ag.step()
        flat = np.concatenate([p.detach().cpu().numpy().ravel() for p in ag.network.parameters()])
        err = float(np.abs(flat - g["a2c_params"][it]).max())
        worst = max(worst, err)
        assert err <= 1e-5, (it, err)
        assert ag.last_loss.dim() == 0 and torch.isfinite(ag.last_loss)
    assert ag.total_steps == 8 * 5 * 6 and int(ag.optimizer.step_dev) == 6 and len(keys) == 8
    print("device agent vs golden record, largest parameter difference: %.3g" % worst)


def _actor(rl, head, gate, N, D, H, A, seed=5):
    """A FlatOptimizer arena for one network and a call of b2rl_a2c_actor_step on it."""
    from deeprl_b200 import _lib, ops
    torch.manual_seed(seed)
    g = torch.tanh if gate == TANH else F.relu
    if head == CAT:
        net = rl.CategoricalActorCriticNet(D, A, rl.FCBody(D, (H, H), gate=g))
        tensors = [t for m in net.phi_body.layers for t in (m.weight, m.bias)]
    else:
        net = rl.GaussianActorCriticNet(D, A, actor_body=rl.FCBody(D, (H, H), gate=g), critic_body=rl.FCBody(D, (H, H), gate=g))
        tensors = [t for b in (net.actor_body, net.critic_body) for m in b.layers for t in (m.weight, m.bias)]
    with torch.no_grad():                                   # logits / means far enough from uniform / zero to be visible
        net.fc_action.weight.normal_(0, 0.5)
        net.fc_action.bias.normal_(0, 0.5)
    tensors += [net.fc_action.weight, net.fc_action.bias, net.fc_critic.weight, net.fc_critic.bias]
    if head == GAUSS:
        tensors.append(net.std)
    opt = ops.FlatOptimizer.from_torch(torch.optim.RMSprop(net.parameters(), 1e-3), list(net.parameters()))
    off = torch.tensor([(t.data_ptr() - opt.flat.data_ptr()) // 4 for t in tensors], dtype=torch.int32)
    acols = 1 if head == CAT else A

    def step(obs, counter, seed, given=None):
        st = torch.empty((N, D), device="cuda")
        act = torch.empty((N, acols), device="cuda")
        _lib.call("b2rl_a2c_actor_step", head, int(head == CAT), gate, _lib.ptr(obs), 1.0, _lib.ptr(opt.flat), _lib.ptr(off),
                  D, H, H, A, N, _lib.ptr(st), _lib.ptr(act), _lib.ptr(given), seed, _lib.ptr(counter), _lib.stream())
        torch.cuda.synchronize()
        return st, act

    return net, step


@pytest.mark.gpu
def test_actor_step_categorical_sampling(rl):
    """Inverse-CDF draws on Philox uniforms: the frequencies of 1000 steps x 64 rows agree with the softmax probabilities of each
    of 4 distinct rows (Pearson chi-square below the 0.999 quantile of its A - 1 = 4 degrees of freedom, 18.47, per row, with the
    fixed seed 11); the same seed and counter give the same actions; the counter advances by N per step; given actions are
    written through unchanged and do not advance it; the state row is the rescaled observation."""
    from scipy import stats
    N, D, H, A, steps = 64, 6, 32, 5, 1000
    net, step = _actor(rl, CAT, TANH, N, D, H, A)
    obs = torch.randn(4, D, dtype=torch.float64, device="cuda").repeat_interleave(N // 4, 0)
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    counts = np.zeros((N, A))
    for _ in range(steps):
        st, act = step(obs, counter, 11)
        a = act.cpu().numpy()[:, 0].astype(np.int64)
        counts[np.arange(N), a] += 1
    assert int(counter) == steps * N
    assert torch.equal(st, obs.float())
    with torch.no_grad():
        p = torch.softmax(net(obs.float())["log_pi_a"].new_tensor(
            torch.nn.functional.linear(net.phi_body(obs.float()), net.fc_action.weight, net.fc_action.bias).cpu().numpy()), -1)
    p = p.cpu().numpy()
    bound = stats.chi2.ppf(0.999, A - 1)
    for r in range(4):
        rows = slice(r * N // 4, (r + 1) * N // 4)
        obs_c, exp_c = counts[rows].sum(0), p[rows][0] * steps * (N // 4)
        chi2 = float(((obs_c - exp_c) ** 2 / exp_c).sum())
        assert chi2 < bound, (r, chi2, obs_c, exp_c)
    c1, c2 = torch.full((1,), 77, dtype=torch.int64, device="cuda"), torch.full((1,), 77, dtype=torch.int64, device="cuda")
    assert torch.equal(step(obs, c1, 3)[1], step(obs, c2, 3)[1]) and int(c1) == 77 + N
    given = torch.randint(0, A, (N, 1), device="cuda").float()
    assert torch.equal(step(obs, c1, 3, given)[1], given) and int(c1) == 77 + N


@pytest.mark.gpu
def test_actor_step_gaussian_sampling(rl):
    """mean + softplus(std) z: over 2000 steps x 16 rows of one observation the sample mean and std of every action dimension
    match the network's mean and softplus(std) (5 standard errors); same seed and counter, same actions; counter += N * A."""
    N, D, H, A, steps = 16, 17, 64, 6, 2000
    net, step = _actor(rl, GAUSS, RELU, N, D, H, A)
    with torch.no_grad():
        net.std.copy_(torch.linspace(-1.0, 1.0, A))
    obs = torch.randn(1, D, dtype=torch.float64, device="cuda").repeat(N, 1)
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    xs = []
    for _ in range(steps):
        xs.append(step(obs, counter, 21)[1].cpu().numpy())
    x = np.concatenate(xs)                                    # (steps * N, A)
    assert int(counter) == steps * N * A
    with torch.no_grad():
        out = net(obs.float()[:1])
    mean, sd = out["mean"][0].cpu().numpy(), F.softplus(net.std).detach().cpu().numpy()
    n = x.shape[0]
    assert np.all(np.abs(x.mean(0) - mean) < 5 * sd / np.sqrt(n)), (x.mean(0), mean)
    assert np.all(np.abs(x.std(0) - sd) < 5 * sd / np.sqrt(2 * n)), (x.std(0), sd)
    c1, c2 = torch.full((1,), 5, dtype=torch.int64, device="cuda"), torch.full((1,), 5, dtype=torch.int64, device="cuda")
    assert torch.equal(step(obs, c1, 8)[1], step(obs, c2, 8)[1])
    given = torch.randn(N, A, device="cuda")
    assert torch.equal(step(obs, c1, 8, given)[1], given) and int(c1) == 5 + N * A


def _launcher_agent(monkeypatch, name, **kw):
    import examples
    got = []
    monkeypatch.setattr(examples, "run_steps", got.append)
    getattr(examples, name)(device_a2c=True, **kw)
    return got[0]


@pytest.mark.gpu
@pytest.mark.parametrize("name,game", [("a2c_feature", "CartPole-v0"), ("a2c_continuous", "SyntheticCheetah-v0")])
def test_launchers_end_to_end(rl, monkeypatch, name, game):
    """The launchers' own configurations with device_a2c: a few dozen steps, finite losses, the step count; and in one profiled
    step() exactly T actor-step kernels and one update kernel -- no other kernel, only copies besides."""
    ag = _launcher_agent(monkeypatch, name, game=game)
    c = ag.config
    losses_ = []
    for _ in range(30):
        ag.step()
        losses_.append(ag.last_loss)
    assert all(bool(torch.isfinite(x)) for x in losses_) and ag.total_steps == 30 * c.num_workers * c.rollout_length
    assert len(set(float(x) for x in losses_)) > 1
    torch.cuda.synchronize()
    from _kernel_trace import profiled_kernels
    kernels = profiled_kernels(lambda: (ag.step(), torch.cuda.synchronize()),
                               {"a2c_actor_kernel": c.rollout_length, "a2c_update_kernel": 1}, warmup=False)
    assert sum("a2c_actor_kernel" in k for k in kernels) == c.rollout_length, kernels
    assert sum("a2c_update_kernel" in k for k in kernels) == 1, kernels
    assert len(kernels) == c.rollout_length + 1, kernels
    ag.close()


@pytest.mark.gpu
def test_unsupported_configurations_are_refused(rl):
    def agent(**kw):
        c = _a2c_feature_config(rl, 5, lambda: rl.Task("CartPole-v0", num_envs=5, seed=0))
        c.eval_env = rl.Task("CartPole-v0", seed=0)
        for k, v in kw.items():
            setattr(c, k, v)
        return rl.A2CAgent(c)

    with pytest.raises(NotImplementedError, match="FCBody phi_body"):
        agent(network_fn=lambda: rl.CategoricalActorCriticNet(4, 2, rl.NatureConvBody(in_channels=4)))
    with pytest.raises(NotImplementedError, match="Adam"):
        agent(optimizer_fn=lambda p: torch.optim.Adam(p, 1e-3))
    with pytest.raises(NotImplementedError, match="MeanStdNormalizer"):
        agent(state_normalizer=rl.MeanStdNormalizer())
    ag = agent()                                                  # the supported form still builds
    ag.close()
