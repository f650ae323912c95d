"""Data-parallel PPO (deeprl_b200/csrc/ppo_dp_sequence.inc): W ranks, each with its own rollout rows, advantage
normalisation and minibatch permutation; update k of every rank must be ONE step of the reference's non-shared PPO update
(PPO_agent.py:68-99) on the union of the ranks' k-th minibatches -- exactly, because every loss term is a mean over rows -- and
parameters, moments and step counts must be bit-identical on every rank.

CPU: the phase functions compiled for the host (tests/host_emul/ppo_dp_emul.cpp), W ranks in lockstep.  GPU: the CUDA
kernel through the C ABI with the W ranks as the W blocks of one cooperative launch on one device; across GPUs (>= 2 with
peer access) through
``PersistentPPOLearner`` and ``PPOAgent`` under torchrun (tests/_ppo_dp_ranks.py).  The oracle is ``union_oracle`` below."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import agents, losses, nets  # noqa: E402
from test_ppo_persistent import A_KEYS, C_KEYS, CASES, I32, I64, arena, batches_for, fp, make_problem  # noqa: E402

HYPER = dict(a_b1=0.9, a_b2=0.999, a_eps=1e-8, c_lr=1e-3, c_b1=0.9, c_b2=0.999, c_eps=1e-8, clip=0.2, ent_w=0.01)


def rank_problem(c, case, r):
    """Rank r's rollout for case `case`: rank 0 is test_ppo_persistent's problem; the others draw their own states, and their
    actions / old log-probs from the SAME initial network (so the ratios start near 1, as in a real rollout)."""
    sd0, *rest = make_problem(c["D"], c["A"], c["H1"], c["H2"], c["rows"], seed=case)
    if r == 0:
        return [sd0] + rest
    g = torch.Generator().manual_seed(1000 + 17 * case + r)
    rn = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale
    states = rn(c["rows"], c["D"])
    with torch.no_grad():
        out = nets.gaussian_actor_critic(sd0, states, torch.zeros(c["rows"], c["A"]))
        actions = out["mean"] + torch.nn.functional.softplus(sd0["std"]) * rn(c["rows"], c["A"])
        log_pi_old = nets.gaussian_actor_critic(sd0, states, actions)["log_pi_a"] + rn(c["rows"], 1, scale=0.05)
    return [sd0, states, actions, log_pi_old, rn(c["rows"], 1), rn(c["rows"], 1)]


def union_oracle(sd, a_opt, c_opt, problems, perms, target_kl):
    """PPO_agent.py:68-99 (non-shared representation) with the reference's own statements (oracle.agents.ppo_update), applied
    to explicit minibatches: update k trains on the concatenation of every rank's k-th minibatch.  Rank r's rows are
    r * rows + i of the concatenated rollout; each rank's advantages are normalised on their own (PPO_agent.py:66, rank-local).
    Returns the gate decisions."""
    rows = problems[0][1].shape[0]
    cat = lambda i: torch.cat([p[i] for p in problems])
    states, actions, log_pi_old, ret = cat(1), cat(2), cat(3), cat(4)
    adv = torch.cat([losses.normalize_advantage(p[5]) for p in problems])
    gates = []
    for k in range(perms[0].shape[0]):
        idx = torch.from_numpy(np.concatenate([r * rows + perms[r][k] for r in range(len(problems))])).long()
        out = nets.gaussian_actor_critic(sd, states[idx], actions[idx])
        pl, vl, kl = losses.ppo_losses(out["log_pi_a"], out["entropy"], out["v"], log_pi_old[idx], adv[idx], ret[idx],
                                       HYPER["clip"], HYPER["ent_w"])
        gates.append(bool(kl <= 1.5 * target_kl))
        if gates[-1]:
            a_opt.zero_grad()
            pl.backward()
            a_opt.step()
        c_opt.zero_grad()
        vl.backward()
        c_opt.step()
    return gates


class Setup:
    """W ranks' inputs in the one-device layout of b2rl_ppo_minibatch_updates_dp: every per-rank array is W consecutive
    copies; arenas start from rank 0's initial parameters on every rank."""

    def __init__(self, c, case, W, perm_seed=77):
        self.c, self.W = c, W
        self.problems = [rank_problem(c, case, r) for r in range(W)]
        sd0 = self.problems[0][0]
        self.sd0 = sd0
        a_flat, self.a_off = arena(sd0, A_KEYS)
        c_flat, self.c_off = arena(sd0, C_KEYS)
        self.a_n, self.c_n = a_flat.size, c_flat.size
        self.a_flat, self.c_flat = np.tile(a_flat, W), np.tile(c_flat, W)
        self.a_m, self.a_v, self.c_m, self.c_v = (np.zeros_like(x) for x in (self.a_flat, self.a_flat, self.c_flat, self.c_flat))
        self.a_step, self.c_step = np.zeros(W, np.int64), np.zeros(W, np.int64)
        self.stats = np.zeros(4 * W, np.float32)
        self.status = np.zeros(W, np.int64)
        f32 = lambda t: np.ascontiguousarray(t.numpy(), np.float32)
        self.st = np.concatenate([f32(p[1]) for p in self.problems])
        self.ac = np.concatenate([f32(p[2]) for p in self.problems])
        self.lp = np.concatenate([f32(p[3]).ravel() for p in self.problems])
        self.rt = np.concatenate([f32(p[4]).ravel() for p in self.problems])
        self.adv = np.concatenate([f32(losses.normalize_advantage(p[5])).ravel() for p in self.problems])
        self.set_perms(perm_seed)
        self.seq = 0

    def set_perms(self, seed):
        self.perms = [batches_for(self.c["rows"], self.c["epochs"], self.c["mb"], seed=seed + r) for r in range(self.W)]
        self.perm = np.ascontiguousarray(np.concatenate(self.perms))
        self.n_batches = self.perms[0].shape[0]

    def rank(self, r, key):
        x = getattr(self, key)
        n = x.size // self.W
        return x[r * n:(r + 1) * n]

    def oracle(self, state=None):
        if state is None:
            sd = agents.leafify(self.sd0)
            state = (sd, torch.optim.Adam([sd[k] for k in A_KEYS], self.c["a_lr"]),
                     torch.optim.Adam([sd[k] for k in C_KEYS], HYPER["c_lr"]))
        gates = union_oracle(*state, self.problems, self.perms, self.c["target_kl"])
        return state, gates

    def check(self, state, a_steps, total_batches):
        sd, a_opt, c_opt = state
        for r in range(self.W):
            assert int(self.rank(r, "c_step")[0]) == total_batches and int(self.rank(r, "a_step")[0]) == a_steps
            for keys, flat, off, opt, m, v in ((A_KEYS, "a_flat", self.a_off, a_opt, "a_m", "a_v"),
                                               (C_KEYS, "c_flat", self.c_off, c_opt, "c_m", "c_v")):
                for k, o in zip(keys, off):
                    want = sd[k].detach().numpy().ravel()
                    got = self.rank(r, flat)[o:o + want.size]
                    # Adam divides by sqrt(exp_avg_sq): a weight of a nearly saturated tanh unit turns rounding differences
                    # of its small gradient into visible steps (case 1 runs at 10x the examples' actor learning rate).  One such
                    # element per tensor was seen 2e-5..6e-5 off the fp32 oracle -- and ~3e-5 off a float64 one, as is the fp32
                    # oracle itself.  So: every element within 1e-4, and all but at most one per tensor within 2e-5.
                    np.testing.assert_allclose(got, want, rtol=0, atol=1e-4, err_msg=k)
                    assert int((np.abs(got - want) > 2e-5).sum()) <= 1, (k, np.sort(np.abs(got - want))[-3:])
                    assert np.abs(want - self.sd0[k].numpy().ravel()).max() > 1e-5 or a_steps == 0, k
                    if opt.state:
                        stt = opt.state[sd[k]]
                        np.testing.assert_allclose(self.rank(r, m)[o:o + want.size], stt["exp_avg"].numpy().ravel(), rtol=1e-3,
                                                   atol=1e-7, err_msg=k)
                        np.testing.assert_allclose(self.rank(r, v)[o:o + want.size], stt["exp_avg_sq"].numpy().ravel(),
                                                   rtol=2e-3, atol=1e-10, err_msg=k)

    def identical_across_ranks(self):
        for key in ("a_flat", "c_flat", "a_m", "a_v", "c_m", "c_v", "a_step", "c_step", "stats"):
            for r in range(1, self.W):
                assert np.array_equal(self.rank(0, key), self.rank(r, key)), key


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ppo_emul_dp") / "ppo_emul.so")
    emul_dir = os.path.join(ROOT, "tests", "host_emul")
    subprocess.run(["g++", "-O2", "-fno-strict-aliasing", "-std=c++17", "-shared", "-fPIC", "-o", out,
                    os.path.join(emul_dir, "ppo_emul.cpp"), os.path.join(emul_dir, "ppo_dp_emul.cpp")], check=True)
    return ctypes.CDLL(out)


def dp_region_floats(a_n, c_n):
    """ppo_phases.h ppo_dp_slot_floats: 128-byte flag header + two slots [actor | critic | 3 loss values], 16-byte aligned."""
    r4 = lambda n: (n + 3) // 4 * 4
    return 32 + 2 * (r4(a_n) + r4(c_n) + 4)


def run_emul_dp(lib, s, threads=512, reverse_ranks=False, reverse_threads=False, regions=None):
    c = s.c
    if regions is None:
        regions = np.zeros(s.W * dp_region_floats(s.a_n, s.c_n), np.float32)
    rc = lib.ppo_emul_minibatch_updates_dp(
        fp(s.st), fp(s.ac), fp(s.lp), fp(s.rt), fp(s.adv), c["D"], c["A"], c["H1"], c["H2"], c["mb"], s.perm.ctypes.data_as(I64),
        s.n_batches, fp(s.a_flat), fp(s.a_m), fp(s.a_v), s.a_step.ctypes.data_as(I64), s.a_off.ctypes.data_as(I32),
        fp(s.c_flat), fp(s.c_m), fp(s.c_v), s.c_step.ctypes.data_as(I64), s.c_off.ctypes.data_as(I32),
        ctypes.c_float(c["a_lr"]), ctypes.c_float(HYPER["a_b1"]), ctypes.c_float(HYPER["a_b2"]), ctypes.c_float(HYPER["a_eps"]),
        ctypes.c_float(HYPER["c_lr"]), ctypes.c_float(HYPER["c_b1"]), ctypes.c_float(HYPER["c_b2"]), ctypes.c_float(HYPER["c_eps"]),
        ctypes.c_float(HYPER["clip"]), ctypes.c_float(HYPER["ent_w"]), ctypes.c_float(1.5 * c["target_kl"]), fp(s.stats),
        c["rows"], s.a_n, s.c_n, s.W, fp(regions), ctypes.c_int64(dp_region_floats(s.a_n, s.c_n)), ctypes.c_int64(s.seq),
        s.status.ctypes.data_as(I64), threads, int(reverse_ranks), int(reverse_threads))
    assert rc == 0 and not s.status.any()
    s.seq += s.n_batches
    return regions


# ------------------------------------------------------------------------------------------------ CPU: host emulation
@pytest.mark.parametrize("W", [1, 2, 3, 4])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_dp_phase_functions_match_union_oracle(emul, case, W):
    c = CASES[case]
    s = Setup(c, case, W)
    run_emul_dp(emul, s)
    state, gates = s.oracle()
    s.check(state, sum(gates), s.n_batches)
    s.identical_across_ranks()
    assert int(s.stats[3]) == sum(gates)
    if case == 1:
        assert 0 < sum(gates) < len(gates)                       # the mean-kl gate was open for some updates and closed for others


@pytest.mark.parametrize("W", [2, 3])
@pytest.mark.parametrize("case", [0, 2])
def test_dp_no_dependence_on_rank_or_thread_order(emul, case, W):
    c = CASES[case]
    runs = []
    for rr, rt, nt in ((False, False, 512), (True, False, 512), (False, True, 512), (True, True, 64)):
        s = Setup(c, case, W)
        run_emul_dp(emul, s, threads=nt, reverse_ranks=rr, reverse_threads=rt)
        runs.append(s)
    for s in runs[1:]:
        for k in ("a_flat", "c_flat", "a_m", "a_v", "c_m", "c_v", "stats", "a_step", "c_step"):
            assert np.array_equal(getattr(runs[0], k), getattr(s, k)), k


@pytest.mark.parametrize("case", range(len(CASES)))
def test_dp_with_one_rank_is_the_single_process_kernel_bit_for_bit(emul, case):
    from test_ppo_persistent import run_emul
    c = CASES[case]
    s = Setup(c, case, 1)
    run_emul_dp(emul, s)
    ref = run_emul(emul, "ppo_emul_minibatch_updates", c, make_problem(c["D"], c["A"], c["H1"], c["H2"], c["rows"], seed=case), 512)
    for k in ("a_flat", "c_flat", "a_m", "a_v", "c_m", "c_v", "stats"):
        assert np.array_equal(getattr(s, k), ref[k]), k
    assert int(s.a_step[0]) == ref["a_step"] and int(s.c_step[0]) == ref["c_step"]


@pytest.mark.parametrize("W", [2, 3])
def test_dp_two_consecutive_calls_continue_the_sequence(emul, W):
    """Two iterations: the second call continues the sequence numbers (seq_base = updates so far) on the same exchange regions,
    with new permutations; it must match the union oracle run twice on the same optimizers."""
    c = CASES[2]
    s = Setup(c, 2, W)
    regions = run_emul_dp(emul, s)
    state, g1 = s.oracle()
    s.set_perms(178)
    run_emul_dp(emul, s, regions=regions)
    state, g2 = s.oracle(state)
    s.check(state, sum(g1) + sum(g2), 2 * s.n_batches)
    s.identical_across_ranks()
    flags = regions.view(np.int64).reshape(W, -1)[:, :W]
    assert (flags == 2 * s.n_batches).all()                      # every rank's flags hold the last global sequence number


# ------------------------------------------------------------------------------------------------ CPU: build checks
def _ptxas_and_sass(tmp_path):
    csrc = os.path.join(ROOT, "deeprl_b200", "csrc")
    cubin = str(tmp_path / "ppo.cubin")
    r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin", "-o",
                        cubin, os.path.join(csrc, "ppo_persistent.cu")], cwd=csrc, capture_output=True, text=True)
    if r.returncode != 0 and "not found" in r.stderr:
        pytest.skip("nvcc not available")
    assert r.returncode == 0, r.stderr[-3000:]
    props = {}
    for m in re.finditer(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill "
                         r"loads\n(?:ptxas info\s+: Used (\d+) registers)?", r.stderr):
        props[m.group(1)] = tuple(int(x) if x else None for x in m.groups()[1:])
    sass = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True, check=True).stdout
    return props, sass


@pytest.fixture(scope="module")
def built(tmp_path_factory):
    import shutil
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    return _ptxas_and_sass(tmp_path_factory.mktemp("ppo_cubin"))


def _kernel(props, name):
    hits = [v for k, v in props.items() if name in k]
    assert len(hits) == 1, (name, list(props))
    return hits[0]


def test_dp_kernel_has_no_stack_frame_and_no_spills(built):
    frame, st, ld, regs = _kernel(built[0], "ppo_dp_persistent_kernel")
    assert (frame, st, ld) == (0, 0, 0) and regs <= 128


def test_single_process_kernel_keeps_its_register_count_and_frame(built):
    """The single-process kernel is unchanged by the data-parallel form: 120 registers, no stack, no spills (sm_90a, -O3)."""
    assert _kernel(built[0], "ppo_minibatch_persistent_kernel") == (0, 0, 0, 120)


def test_dp_kernel_exchange_instructions(built):
    """fence.acq_rel.sys -> MEMBAR.ALL.SYS; st.release.sys / ld.acquire.sys of the 64-bit flags -> STG / LDG .64.STRONG.SYS;
    the peer-slot reads (ld.global.cg) -> LDG.E.STRONG.GPU, which is served by L2 / NVLink and never by a stale L1 line."""
    sass = built[1]
    i = sass.index("Function : _ZN4b2rl24ppo_dp_persistent_kernel")
    j = sass.find("Function : ", i + 10)
    body = sass[i:j if j > 0 else None]
    assert "MEMBAR.ALL.SYS" in body
    assert "STG.E.64.STRONG.SYS" in body, "system-scope release store of the flags"
    assert "LDG.E.64.STRONG.SYS" in body, "system-scope acquire load of the flags"
    assert "SR_GLOBALTIMER" in body and "NANOSLEEP" in body, "the wait backs off and is bounded by %globaltimer"
    assert body.count("LDG.E.STRONG.GPU") >= 4, "peer slots are read with L1-bypassing loads"
    assert "STL" not in body and "LDL" not in body


# ------------------------------------------------------------------------------------------------ GPU: one device, W blocks
def run_cuda_dp(s, regions=None):
    """The CUDA kernel through the C ABI: the W ranks as the W blocks of one cooperative launch (ranks_in_launch = W)."""
    from deeprl_b200 import _lib
    c, dev = s.c, torch.device("cuda", 0)
    cu = lambda x: torch.as_tensor(np.ascontiguousarray(x)).to(dev)
    t = {k: cu(getattr(s, k)) for k in ("st", "ac", "lp", "rt", "adv", "perm", "a_flat", "a_m", "a_v", "a_step", "c_flat", "c_m",
                                         "c_v", "c_step", "stats", "status")}
    rb = int(_lib.lib().b2rl_ppo_dp_region_bytes(s.a_n, s.c_n))
    assert rb == 4 * dp_region_floats(s.a_n, s.c_n)
    if regions is None:
        regions = torch.zeros(s.W * rb // 4, dtype=torch.float32, device=dev)
    table = (ctypes.c_void_p * s.W)(*[regions.data_ptr() + p * rb for p in range(s.W)])
    a_off, c_off = torch.from_numpy(s.a_off), torch.from_numpy(s.c_off)
    p = _lib.ptr
    _lib.call("b2rl_ppo_minibatch_updates_dp", p(t["st"]), p(t["ac"]), p(t["lp"]), p(t["rt"]), p(t["adv"]), c["D"], c["A"], c["H1"],
              c["H2"], c["mb"], p(t["perm"]), s.n_batches, p(t["a_flat"]), p(t["a_m"]), p(t["a_v"]), p(t["a_step"]), p(a_off),
              p(t["c_flat"]), p(t["c_m"]), p(t["c_v"]), p(t["c_step"]), p(c_off), c["a_lr"], HYPER["a_b1"], HYPER["a_b2"],
              HYPER["a_eps"], HYPER["c_lr"], HYPER["c_b1"], HYPER["c_b2"], HYPER["c_eps"], HYPER["clip"], HYPER["ent_w"],
              1.5 * c["target_kl"], p(t["stats"]), c["rows"], s.a_n, s.c_n, s.W, 0, table, s.seq, int(5e9), p(t["status"]), s.W,
              _lib.stream())
    torch.cuda.synchronize()
    for k in ("a_flat", "a_m", "a_v", "a_step", "c_flat", "c_m", "c_v", "c_step", "stats", "status"):
        setattr(s, k, t[k].cpu().numpy())
    assert not s.status.any(), s.status                           # no exchange timed out
    s.seq += s.n_batches
    return regions


def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


@pytest.mark.gpu
@pytest.mark.parametrize("W", [2, 3, 8])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_cuda_dp_one_device_matches_union_oracle(case, W):
    _gpu()
    c = CASES[case]
    s = Setup(c, case, W)
    run_cuda_dp(s)
    state, gates = s.oracle()
    s.check(state, sum(gates), s.n_batches)
    s.identical_across_ranks()
    assert int(s.stats[3]) == sum(gates)


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(CASES)))
def test_cuda_dp_with_one_rank_matches_the_single_process_kernel(case):
    _gpu()
    from deeprl_b200 import _lib
    c = CASES[case]
    s = Setup(c, case, 1)
    ref = Setup(c, case, 1)
    run_cuda_dp(s)
    dev = torch.device("cuda", 0)
    cu = lambda x: torch.as_tensor(np.ascontiguousarray(x)).to(dev)
    t = {k: cu(getattr(ref, k)) for k in ("st", "ac", "lp", "rt", "adv", "perm", "a_flat", "a_m", "a_v", "a_step", "c_flat", "c_m",
                                           "c_v", "c_step", "stats")}
    p = _lib.ptr
    _lib.call("b2rl_ppo_minibatch_updates", p(t["st"]), p(t["ac"]), p(t["lp"]), p(t["rt"]), p(t["adv"]), c["D"], c["A"], c["H1"],
              c["H2"], c["mb"], p(t["perm"]), ref.n_batches, p(t["a_flat"]), p(t["a_m"]), p(t["a_v"]), p(t["a_step"]),
              p(torch.from_numpy(ref.a_off)), p(t["c_flat"]), p(t["c_m"]), p(t["c_v"]), p(t["c_step"]), p(torch.from_numpy(ref.c_off)),
              c["a_lr"], HYPER["a_b1"], HYPER["a_b2"], HYPER["a_eps"], HYPER["c_lr"], HYPER["c_b1"], HYPER["c_b2"], HYPER["c_eps"],
              HYPER["clip"], HYPER["ent_w"], 1.5 * c["target_kl"], p(t["stats"]), _lib.stream())
    torch.cuda.synchronize()
    # every Adam site evaluates the update as the same explicit fmaf (ppo_phases.h adam_m / adam_v / adam_p), and 1/W = 1:
    # the two kernels agree bit for bit
    assert int(s.a_step[0]) == int(t["a_step"]) and int(s.c_step[0]) == int(t["c_step"])
    for k in ("a_flat", "c_flat", "a_m", "a_v", "c_m", "c_v", "stats"):
        assert np.array_equal(getattr(s, k), t[k].cpu().numpy()), k


@pytest.mark.gpu
@pytest.mark.parametrize("W", [2, 8])
def test_cuda_dp_two_consecutive_launches_continue(W):
    _gpu()
    c = CASES[2]
    s = Setup(c, 2, W)
    regions = run_cuda_dp(s)
    state, g1 = s.oracle()
    s.set_perms(178)
    regions = run_cuda_dp(s, regions)
    state, g2 = s.oracle(state)
    s.check(state, sum(g1) + sum(g2), 2 * s.n_batches)
    s.identical_across_ranks()
    rf = regions.view(torch.int64).view(W, -1)[:, :W].cpu().numpy()
    assert (rf == 2 * s.n_batches).all()


# ------------------------------------------------------------------------------------------------ GPU: >= 2 GPUs, torchrun
@pytest.mark.gpu
@pytest.mark.parametrize("what", ["learner", "agent"])
def test_data_parallel_across_gpus(what):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    n = min(torch.cuda.device_count(), 8)
    ok = all(torch.cuda.can_device_access_peer(a, b) for a in range(n) for b in range(n) if a != b)
    if not ok:
        pytest.skip("needs peer access between the GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n), "--master-addr", "127.0.0.1",
           "--master-port", "29547", os.path.join(ROOT, "tests", "_ppo_dp_ranks.py"), what]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ok=True" in r.stdout, r.stdout[-3000:]
