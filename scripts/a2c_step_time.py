"""Agent steps per second of the rollout launchers' configurations, eager (the torch path of ``step()``) against the launcher's
device flag (one actor-step launch per env step, one update launch per rollout or gradient update: csrc/a2c.cu) --
``config.device_a2c`` for A2CAgent (a2c_feature, a2c_continuous), ``config.device_nstep_dqn`` for NStepDQNAgent
(n_step_dqn_feature), ``config.device_dqn`` for DQNAgent (dqn_feature, timed past its exploration steps), ``config.device_c51``
/ ``config.device_qr`` for CategoricalDQNAgent / QuantileRegressionDQNAgent (categorical_dqn_feature,
quantile_regression_dqn_feature: csrc/dist_dqn.cu, with the launchers' async actor), ``config.device_rainbow`` for
CategoricalDQNAgent on a noisy RainbowNet (rainbow_feature: csrc/rainbow.cu), ``config.cuda_graph`` for NStepDQNAgent on the
NatureConvBody (n_step_dqn_pixel on SyntheticAtari-v0: one GraphedQActor replay per env step, one GraphedNStepLearner replay per
rollout; both it and the eager side at bf16, plus the launcher's default fp32 eager side), and ``config.cuda_graph`` for A2CAgent
on the NatureConvBody the same way (a2c_pixel on SyntheticAtari-v0: one GraphedQActor replay per env step with the action drawn
on the device, one GraphedA2CLearner replay per rollout), and ``config.cuda_graph`` for PPOAgent on the NatureConvBody
(ppo_pixel: the same actor, one GraphedPPOPixelLearner replay per rollout for all its minibatch updates) -- in one process on one card, the sides alternated round by round.
For the pixel launchers the captured update alone is also timed: CUDA events around back-to-back replays of its graph; and the
first step of the graph side (which captures the actor's per-slot graphs) is timed alone, with the memory the caching
allocator reserved during it.  Also times the host envs alone (``task.step`` with fixed actions), so the share
left to the learner is visible.  Prints the card's name and power limit with the numbers.

    python scripts/a2c_step_time.py [--steps 300] [--rounds 5] [--only LAUNCHER[,LAUNCHER]] [--out DIR]

A side whose ``step()`` raises while it is warmed up is reported with its error and not timed (rainbow_feature's eager path:
its actor thread resets the NoisyLinear noise buffers in place while the learner's autograd graph holds them, and torch's
version check stops the backward).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (launcher, game, its device flag, the agent's name in the output keys)
CONFIGS = [("a2c_feature", "CartPole-v0", "device_a2c", "a2c"), ("a2c_continuous", "SyntheticCheetah-v0", "device_a2c", "a2c"),
           ("n_step_dqn_feature", "CartPole-v0", "device_nstep_dqn", "nstep_dqn"),
           ("dqn_feature", "CartPole-v0", "device_dqn", "dqn"),
           ("categorical_dqn_feature", "CartPole-v0", "device_c51", "c51"),
           ("quantile_regression_dqn_feature", "CartPole-v0", "device_qr", "qr"),
           ("rainbow_feature", "CartPole-v0", "device_rainbow", "rainbow"),
           ("n_step_dqn_pixel", "SyntheticAtari-v0", "cuda_graph", "nstep_dqn"),
           ("a2c_pixel", "SyntheticAtari-v0", "cuda_graph", "a2c"),
           ("ppo_pixel", "SyntheticAtari-v0", "cuda_graph", "ppo")]
# launchers timed at a given Config.COMPUTE_DTYPE per side (set around every step of that side): side -> dtype
DTYPES = {"n_step_dqn_pixel": {"eager": torch.bfloat16, "cuda_graph": torch.bfloat16, "eager_fp32": torch.float32},
          "a2c_pixel": {"eager": torch.bfloat16, "cuda_graph": torch.bfloat16, "eager_fp32": torch.float32},
          "ppo_pixel": {"eager": torch.bfloat16, "cuda_graph": torch.bfloat16, "eager_fp32": torch.float32}}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                  # noqa: BLE001
        q = "nvidia-smi unavailable (%s)" % e
    return "%s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q)


def make_agent(name, game, flag, on):
    import examples
    got = []
    run_steps = examples.run_steps
    examples.run_steps = got.append
    try:
        getattr(examples, name)(game=game, **{flag: on})
    finally:
        examples.run_steps = run_steps
    return got[0]


def timed(agent, steps, dtype=None):
    from deeprl_b200 import Config
    old = Config.COMPUTE_DTYPE
    Config.COMPUTE_DTYPE = dtype or old
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            agent.step()
        torch.cuda.synchronize()
        return steps / (time.perf_counter() - t0)
    finally:
        Config.COMPUTE_DTYPE = old


def update_replay_ms(agent, replays=400):
    """The captured rollout update alone: CUDA events around ``replays`` back-to-back replays of its graph (on the rollout
    staged last), milliseconds per replay."""
    g = agent._graph[0].graph
    for _ in range(20):
        g.replay()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(replays):
        g.replay()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / replays


def env_steps(agent):
    """Env steps per agent step: the rollout, or DQNAgent's sgd_update_frequency transitions."""
    from deeprl_b200 import DQNAgent
    return agent.config.sgd_update_frequency if isinstance(agent, DQNAgent) else agent.config.rollout_length


def past_exploration(agent):
    """DQNAgent: step until the gradient updates run, so that the timed steps include them."""
    from deeprl_b200 import DQNAgent
    if isinstance(agent, DQNAgent):
        while agent.total_steps <= agent.config.exploration_steps:
            agent.step()


def env_only(agent, steps):
    """task.step alone, env_steps * steps times, with the actions of one draw (what the host envs cost per agent step).  With
    an async actor its thread owns its task, so a new one is made."""
    from deeprl_b200 import CategoricalActorCriticNet, CategoricalNet, DuelingNet, QuantileNet, RainbowNet, VanillaNet
    c = agent.config
    a = (np.zeros(c.num_workers, dtype=np.int64)
         if isinstance(agent.network, (CategoricalActorCriticNet, VanillaNet, DuelingNet, CategoricalNet, QuantileNet, RainbowNet))
         else np.zeros((c.num_workers, c.action_dim), dtype=np.float32))
    own = hasattr(agent, "actor") and c.async_actor
    task = agent.task if hasattr(agent, "task") else c.task_fn() if own else agent.actor._task
    if own:
        task.reset()
    t0 = time.perf_counter()
    for _ in range(steps * env_steps(agent)):
        task.step(a)
    rate = steps / (time.perf_counter() - t0)
    if own:
        task.close()
    return rate


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--only", default=None, help="comma-separated launcher names (default: all of CONFIGS)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("a2c_step_time.py measures on a CUDA device; none is visible")
    import deeprl_b200 as rl
    rl.select_device(0)
    rl.random_seed(0)
    result = dict(card=card(), steps_per_round=args.steps, rounds=args.rounds, configs={})
    print(result["card"])
    only = None if args.only is None else set(args.only.split(","))
    if only is not None and not only <= {c[0] for c in CONFIGS}:
        raise SystemExit("--only: unknown launcher in %s" % sorted(only))
    for name, game, flag, unit in CONFIGS:
        if only is not None and name not in only:
            continue
        dtypes = DTYPES.get(name, {})
        agents = {"eager": make_agent(name, game, flag, False), flag: make_agent(name, game, flag, True)}
        if "eager_fp32" in dtypes:
            agents["eager_fp32"] = make_agent(name, game, flag, False)
        failed, first = {}, {}
        for k, ag in agents.items():
            try:
                past_exploration(ag)
                if k == "cuda_graph":                       # the first step captures the graphs
                    torch.cuda.synchronize()
                    torch.cuda.empty_cache()                # (graph capture empties the cache too)
                    m0 = torch.cuda.memory_reserved()
                    first = {"first_step_s": 1.0 / timed(ag, 1, dtypes.get(k)),
                             "first_step_reserved_mb": (torch.cuda.memory_reserved() - m0) / 2 ** 20}
                timed(ag, args.warmup, dtypes.get(k))
            except RuntimeError as e:
                failed[k] = "%s: %s" % (type(e).__name__, str(e).split(". Hint")[0])
        timed_agents = {k: ag for k, ag in agents.items() if k not in failed}
        rates = {k: [] for k in timed_agents}
        for _ in range(args.rounds):                        # alternated: all see the same host / card conditions
            for k, ag in timed_agents.items():
                rates[k].append(timed(ag, args.steps, dtypes.get(k)))
        env = env_only(agents[flag], args.steps)
        c = agents[flag].config
        med = {k: float(np.median(v)) for k, v in rates.items()}
        learner_ms = {k: 1e3 / med[k] - 1e3 / env for k in med}
        row = {"game": game, "num_workers": c.num_workers, "env_steps_per_agent_step": env_steps(agents[flag]), unit + "_steps_per_s": rates,
               "median_%s_steps_per_s" % unit: med,
               "speedup": med[flag] / med["eager"] if flag in med and "eager" in med else None,
               "env_only_%s_steps_per_s" % unit: env, "ms_per_step_besides_envs": learner_ms, "failed": failed}
        if dtypes:
            row["compute_dtype"] = {k: str(v) for k, v in dtypes.items()}
        if flag == "cuda_graph" and flag in timed_agents:
            row["update_replay_ms"] = update_replay_ms(agents[flag])
            row.update(first)
        result["configs"][name] = row
        print("%-18s %-20s N=%d env steps %d  %s;  envs alone %8.1f steps/s;  ms per step besides the envs: %s%s"
              % (name, game, c.num_workers, env_steps(agents[flag]),
                 "  ".join("%s %8.1f steps/s" % kv for kv in med.items()) + ("  (x%.2f)" % row["speedup"] if row["speedup"] else ""),
                 env, ", ".join("%s %.3f" % kv for kv in learner_ms.items()),
                 "".join(";  %s not timed (%s)" % kv for kv in failed.items())))
        if "update_replay_ms" in row:
            print("%-18s captured update alone: %.3f ms per replay" % (name, row["update_replay_ms"]))
            print("%-18s first step (captures): %.2f s, %.0f MB reserved" % (name, row["first_step_s"],
                                                                           row["first_step_reserved_mb"]))
        for ag in agents.values():
            ag.close()
    print(json.dumps(result))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "a2c_step_time.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
