"""CPU-side tests (``-m "not gpu"``): the C-ABI library loads and exports every symbol include/b2rl.h declares
(no compute calls -- there is no GPU here), the ctypes signature table matches the header, and the host logic
(Config, schedules, normalizers, Task / envs, Storage, random_sample, A2C on the CPU device = BASELINE configs[0]).
"""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import deeprl_b200 as rl
from deeprl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_decls():
    hdr = open(os.path.join(ROOT, "include", "b2rl.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    out = {}
    for m in re.finditer(r"\b(?:int|void|int64_t|const char\*)\s+(b2rl_[a-z0-9_]+)\s*\(([^;]*?)\)\s*;", hdr, flags=re.S):
        args = [a.strip() for a in m.group(2).split(",") if a.strip() and a.strip() != "void"]
        out[m.group(1)] = args
    return out


def test_library_exports_every_declared_symbol():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    decl = _header_decls()
    assert len(decl) >= 20
    syms = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    exported = set(re.findall(r"\b(b2rl_[a-z0-9_]+)\b", syms))
    assert set(decl) <= exported, sorted(set(decl) - exported)
    L = _lib.lib()                      # dlopen + resolve every entry of the signature table
    assert L.b2rl_version() >= 100
    assert L.b2rl_last_error() is not None


def test_ctypes_signatures_match_header():
    decl = _header_decls()
    kinds = {"c_void_p": "p", "c_int": "i32", "c_long": "i64", "c_ulong": "u64", "c_float": "f32", "c_double": "f64"}
    for name, argtypes in _lib.SIGNATURES.items():
        assert name in decl, name
        assert len(argtypes) == len(decl[name]), (name, len(argtypes), len(decl[name]))
        for ct, c_arg in zip(argtypes, decl[name]):
            k = kinds[ct.__name__]
            if "*" in c_arg:
                assert k == "p", (name, c_arg)
            elif c_arg.startswith("int32_t"):
                assert k == "i32", (name, c_arg)
            elif c_arg.startswith("int64_t"):
                assert k == "i64", (name, c_arg)
            elif c_arg.startswith("uint64_t"):
                assert k == "u64", (name, c_arg)
            elif c_arg.startswith("float"):
                assert k == "f32", (name, c_arg)
            elif c_arg.startswith("double"):
                assert k == "f64", (name, c_arg)
            else:
                raise AssertionError((name, c_arg))


def test_device_components_refuse_cpu():
    rl.select_device(-1)
    with pytest.raises(_lib.B2RLError, match="no CPU fallback"):
        rl.UniformReplay(16, 4)
    with pytest.raises(_lib.B2RLError):
        rl.PrioritizedReplay(16, 4)
    with pytest.raises(_lib.B2RLError):
        rl.SumTree(16)


def test_schedules_and_normalizers():
    s = rl.LinearSchedule(1.0, 0.1, 9)
    vals = [s() for _ in range(12)]
    assert vals[0] == 1.0 and abs(vals[9] - 0.1) < 1e-12 and vals[11] == 0.1          # advances on every call, clamps
    up = rl.LinearSchedule(0.4, 1.0, 3)
    assert [round(up(), 6) for _ in range(5)] == [0.4, 0.6, 0.8, 1.0, 1.0]
    assert rl.ConstantSchedule(0.3)(5) == 0.3
    assert rl.LinearSchedule(0.5)() == 0.5
    x = np.array([[0, 128, 255]], np.uint8)
    assert np.allclose(rl.ImageNormalizer()(x), x / 255.0)
    assert list(rl.SignNormalizer()(np.array([-3.0, 0.0, 2.0]))) == [-1.0, 0.0, 1.0]
    n = rl.MeanStdNormalizer()
    rng = np.random.RandomState(0)
    data = [rng.randn(5, 3) * 4 + 2 for _ in range(50)]
    for d in data:
        out = n(d)
    assert np.abs(out).max() <= 10.0
    allx = np.concatenate(data)
    np.testing.assert_allclose(n.rms.mean[0], allx.mean(0), atol=1e-3)
    np.testing.assert_allclose(n.rms.var[0], allx.var(0), rtol=1e-3)
    n.set_read_only()
    before = n.rms.mean.copy()
    n(data[0] + 100)
    assert np.array_equal(before, n.rms.mean)
    st = n.state_dict()
    m2 = rl.MeanStdNormalizer()
    m2(data[0])
    m2.load_state_dict(st)
    assert np.array_equal(m2.rms.mean, n.rms.mean)


def test_config_and_misc():
    c = rl.Config()
    assert (c.categorical_n_atoms, c.optimization_epochs, c.mini_batch_size, c.async_actor, c.n_step) == (51, 4, 64, True, 1)
    assert isinstance(c.state_normalizer, rl.RescaleNormalizer) and c.gae_tau == 1.0 and c.double_q is False
    c.merge(dict(game="X", foo=3))
    assert c.foo == 3
    t = rl.Task("CartPole-v0", seed=1)
    c.eval_env = t
    assert (c.state_dim, c.action_dim, c.task_name) == (4, 2, "CartPole-v0")
    np.random.seed(0)
    rows = list(rl.random_sample(np.arange(10), 4))
    assert [len(r) for r in rows] == [4, 4, 2] and sorted(np.concatenate(rows)) == list(range(10))
    kw = dict(game="Breakout", run=2, lr=0.1)
    rl.generate_tag(kw)
    assert kw["tag"] == "Breakout-lr_0.1-run-2"
    np.random.seed(3)
    q = np.array([[0.1, 0.9], [0.8, 0.2]])
    assert list(rl.epsilon_greedy(0.0, q)) == [1, 0]
    assert rl.epsilon_greedy(0.0, q[0]) == 1


def test_task_and_envs():
    t = rl.Task("SyntheticAtari-v0", num_envs=3, seed=5)
    obs = t.reset()
    assert len(obs) == 3 and isinstance(obs[0], rl.LazyFrames) and np.asarray(obs[0]).shape == (4, 84, 84)
    assert np.asarray(obs[0]).dtype == np.uint8 and obs[0][-1].shape == (84, 84)
    o, r, d, info = t.step(np.array([0, 1, 2]))
    assert isinstance(o, tuple) and r.shape == (3,) and d.shape == (3,) and isinstance(info, tuple)
    assert set(info[0]) >= {"episodic_return"} and (t.state_dim, t.action_dim) == (4 * 84 * 84, 4)
    c = rl.Task("SyntheticCheetah-v0", num_envs=2, seed=1)
    c.reset()
    o, r, d, info = c.step(np.full((2, 6), 5.0))             # Box actions are clipped to [-1, 1] (envs.py:188)
    assert (c.state_dim, c.action_dim) == (17, 6) and np.asarray(o).shape == (2, 17)
    cp = rl.Task("CartPole-v0", seed=0)
    cp.reset()
    rets = []
    for _ in range(300):
        _, _, done, info = cp.step([1])
        if info[0]["episodic_return"] is not None:
            rets.append(info[0]["episodic_return"])
    assert rets and all(5 <= x <= 200 for x in rets)        # always pushing right falls over quickly; auto-reset works
    with pytest.raises(NotImplementedError):
        rl.Task("CartPole-v0", single_process=False)


def test_storage():
    s = rl.Storage(3)
    for i in range(3):
        s.feed(dict(reward=torch.full((2, 1), float(i)), mask=torch.ones(2, 1)))
    s.placeholder()
    assert s.v == [None] * 3
    e = s.extract(["reward", "mask"])
    assert e.reward.shape == (6, 1) and e.reward[:, 0].tolist() == [0, 0, 1, 1, 2, 2]          # t-major rows
    with pytest.raises(RuntimeError, match="Undefined key"):
        s.feed(dict(nope=1))


def test_a2c_feature_cartpole_8_workers_cpu():
    """BASELINE configs[0]: a2c_feature CartPole-v0, 8 parallel workers, CPU only (examples.py:340-360 wiring)."""
    rl.select_device(-1)
    rl.random_seed(0)
    c = rl.Config()
    c.merge(dict(tag=None))
    c.num_workers = 8
    c.task_fn = lambda: rl.Task("CartPole-v0", num_envs=c.num_workers, seed=0)
    c.eval_env = rl.Task("CartPole-v0", seed=0)
    c.optimizer_fn = lambda p: torch.optim.RMSprop(p, 0.001)
    c.network_fn = lambda: rl.CategoricalActorCriticNet(c.state_dim, c.action_dim, rl.FCBody(c.state_dim, gate=torch.tanh))
    c.discount, c.use_gae, c.gae_tau, c.entropy_weight, c.rollout_length, c.gradient_clip = 0.99, True, 0.95, 0.01, 5, 0.5
    c.max_steps, c.log_interval = 8 * 5 * 60, 0
    ag = rl.A2CAgent(c)
    rl.run_steps(ag)
    assert ag.total_steps == c.max_steps and torch.isfinite(ag.last_loss)
    assert len(ag.eval_step(c.eval_env.reset())) == 1


def test_a2c_cpu_matches_oracle_trajectory(golden):
    """The A2C statements of the product on the CPU device reproduce the reference's parameter trajectory when the
    env interaction is replayed from the golden record (atol 2e-6)."""
    rl.select_device(-1)
    g = golden("onpolicy")
    keys = [str(k) for k in g["a2c_keys"]]

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
            return list(g["a2c_next_states"][k]), g["a2c_rewards"][k], g["a2c_dones"][k], tuple({"episodic_return": None} for _ in range(8))

        def close(self):
            pass

    c = rl.Config()
    c.merge(dict(tag=None))
    c.num_workers = 8
    c.task_fn = Replay
    c.optimizer_fn = lambda p: torch.optim.RMSprop(p, 0.001)
    c.network_fn = lambda: rl.CategoricalActorCriticNet(4, 2, rl.FCBody(4, gate=torch.tanh))
    c.discount, c.use_gae, c.gae_tau, c.entropy_weight, c.rollout_length, c.gradient_clip = 0.99, True, 0.95, 0.01, 5, 0.5
    ag = rl.A2CAgent(c)
    ag.network.load_state_dict({k: torch.from_numpy(g["a2c_init." + k]) for k in keys})
    fwd = ag.network.forward

    def forced(obs, action=None):
        """The sampled actions are part of the record: the 5 rollout forwards of a step replay them; the bootstrap
        forward at the end of the rollout samples freely (only its value is used, A2C_agent.py:38-41)."""
        if action is None and forced.budget > 0:
            forced.budget -= 1
            action = torch.from_numpy(g["a2c_actions"][ag.task.k])
        return fwd(obs, action)

    ag.network.forward = forced
    for it in range(g["a2c_params"].shape[0]):
        forced.budget = 5
        ag.step()
        flat = np.concatenate([p.detach().numpy().ravel() for p in ag.network.parameters()])
        np.testing.assert_allclose(flat, g["a2c_params"][it], rtol=0, atol=2e-6)


# ------------------------------------------------------------------------------------------------ repository rules
def _py_files(root):
    for d, _, files in os.walk(root):
        for f in files:
            if f.endswith(".py"):
                yield os.path.join(d, f)


def test_product_never_imports_the_oracle_or_reads_the_reference():
    """oracle/ is test infrastructure: only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may import it,
    and nothing that runs on the GPU box may read /root/reference."""
    import ast
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for path in _py_files(os.path.join(root, "deeprl_b200")):
        tree = ast.parse(open(path).read())
        for node in ast.walk(tree):
            names = []
            if isinstance(node, ast.Import):
                names = [a.name for a in node.names]
            elif isinstance(node, ast.ImportFrom):
                names = [node.module or ""]
            assert not any(n == "oracle" or n.startswith("oracle.") for n in names), path
        assert "/root/reference" not in open(path).read(), path
    # bench.py: the oracle is imported inside the CPU arm only
    tree = ast.parse(open(os.path.join(root, "bench.py")).read())
    for fn in [n for n in tree.body if isinstance(n, ast.FunctionDef)]:
        uses = any(isinstance(n, ast.ImportFrom) and (n.module or "").startswith("oracle") for n in ast.walk(fn))
        assert uses == (fn.name == "make_cpu_agent"), fn.name
    entry = ast.parse(open(os.path.join(root, "__graft_entry__.py")).read())
    for fn in [n for n in entry.body if isinstance(n, ast.FunctionDef)]:
        uses = any(isinstance(n, ast.ImportFrom) and (n.module or "").startswith("oracle") for n in ast.walk(fn))
        assert not uses or fn.name == "smoke", fn.name


def test_bench_arms_on_a_cpu_only_host():
    """No GPU here: the product arm must refuse loudly (no CPU fallback), the reference arm must print ONE JSON line
    with the contract's keys and zero transfer bytes."""
    import json
    import subprocess
    import sys
    if torch.cuda.is_available():
        pytest.skip("CPU-host behaviour")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "bench.py", "--steps", "1", "--warmup", "1"], cwd=root, capture_output=True, text=True,
                       timeout=300)
    assert r.returncode != 0 and "no CPU fallback" in (r.stderr + r.stdout)
    r = subprocess.run([sys.executable, "bench.py", "--impl", "reference", "--steps", "1", "--warmup", "1"], cwd=root,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "updates/s" and d["higher_is_better"] is True and d["value"] > 0
    assert d["metric"].startswith("gradient-updates/sec")
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1


def test_wgmma_kernels_issue_mma_and_tma_directly():
    """SASS-level guard: the tensor-core GEMM kernels must contain HGMMA (wgmma.mma_async) and UTMALDG (TMA loads), the library
    must be built for sm_90, and the single-thread TMA producer must be entered through elect.sync -- behind a plain
    `lane == 0` test nvcc wraps the uniform-datapath TMA instructions in an ELECT / BRA.U.ANY loop."""
    import shutil
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    kernels = {}
    name = None
    for line in sass.splitlines():
        if "Function :" in line:
            name = line.split("Function :")[1].strip()
            kernels[name] = []
        elif name is not None:
            kernels[name].append(line)
    tc = {k: "\n".join(v) for k, v in kernels.items() if "wgmma_kernel" in k}
    assert len(tc) >= 9, sorted(kernels)[:5]                    # gemm x6, slab x7, wgrad x2 instantiations
    for k, body in tc.items():
        assert "HGMMA" in body and "UTMALDG" in body, k
        assert "BRA.U.ANY" not in body, "%s: uniform-datapath instructions are wrapped in ELECT loops again" % k
    assert "EF_CUDA_SM90" in sass
