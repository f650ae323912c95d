"""Agent steps per second of the replay pixel launchers (dqn_pixel, categorical_dqn_pixel, quantile_regression_dqn_pixel on
SyntheticAtari-v0, async replay as written) past their exploration steps: the captured path (``config.cuda_graph`` at bf16:
one GraphedQActor replay per env step, one GraphedDQNLearner replay per agent step with the feeds inside it) with
``async_actor`` on and off, the eager path at bf16 and at the launchers' default fp32, and the host envs alone (``task.step``
with fixed actions).  Also the captured update alone: CUDA events around back-to-back replays of its graphs on a ring larger
than the batch.  The launchers' 1e6-frame ring and 50 000 exploration steps are replaced by ``--memory`` and ``--explore``;
nothing else changes.  Each side is built, warmed past exploration and timed over ``--rounds`` consecutive windows
(``--steps`` agent steps on the captured sides, ``--eager-steps`` on the eager ones, ``--reps`` update replays), one side
at a time (the eager path reads ``Config.COMPUTE_DTYPE`` while it runs, on its actor thread too); the median and the
range over the windows are reported.  Prints the card's name and power limit with
the numbers (and writes them to ``--out``).

    python scripts/dqn_pixel_step_time.py [--steps 3000] [--eager-steps 300] [--reps 3000] [--rounds 3] [--explore 2000]
                                          [--memory 20000] [--only LAUNCHER[,...]] [--out DIR]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

LAUNCHERS = ("dqn_pixel", "categorical_dqn_pixel", "quantile_regression_dqn_pixel")
AGENTS = ("DQNAgent", "CategoricalDQNAgent", "QuantileRegressionDQNAgent")
SIDES = (("graph_async_actor", True, True, torch.bfloat16), ("graph_sync_actor", True, False, torch.bfloat16),
         ("eager_bf16", False, None, torch.bfloat16), ("eager_fp32", False, None, torch.float32))


def build(name, cuda_graph, async_actor, dtype, memory, explore):
    import examples
    import deeprl_b200 as rl
    rl.Config.COMPUTE_DTYPE = dtype
    got = []
    saved = {a: getattr(examples, a) for a in AGENTS + ("run_steps",)}
    for a in AGENTS:
        setattr(examples, a, lambda config, _c=saved[a]: got.append((_c, config)))
    examples.run_steps = lambda ag: None
    cwd = os.getcwd()
    os.chdir(tempfile.mkdtemp(prefix="dqn_pixel_time_"))             # the launcher's logger opens ./log
    try:
        getattr(examples, name)(game="SyntheticAtari-v0", cuda_graph=cuda_graph)
    finally:
        os.chdir(cwd)
        for a, v in saved.items():
            setattr(examples, a, v)
    cls, cfg = got[0]
    if name == "dqn_pixel":
        examples._replay(cfg, cfg.replay_cls, cfg.async_replay, memory_size=memory, n_step=cfg.n_step, discount=cfg.discount,
                         history_length=cfg.history_length)
    else:
        examples._replay(cfg, examples.UniformReplay, True, memory_size=memory, history_length=4)
    cfg.exploration_steps = explore
    if async_actor is not None:
        cfg.async_actor = async_actor
    np.random.seed(0), torch.manual_seed(0)
    return cls(cfg)


def warm(ag):
    while ag.total_steps <= ag.config.exploration_steps + 8 * ag.config.sgd_update_frequency:
        ag.step()                                                    # exploration, capture and a few updates
    torch.cuda.synchronize()


def agent_rate(ag, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        ag.step()
    float(ag.last_loss)                                              # ends in a synchronise
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def update_ms(lr, reps):
    """Back-to-back replays of the captured update (the staging buffer as the last step left it)."""
    for _ in range(10):
        lr.update()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        lr.update()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def env_rate(steps):
    import deeprl_b200 as rl
    task = rl.Task("SyntheticAtari-v0")
    task.reset()
    a = np.zeros(1, dtype=np.int64)
    t0 = time.perf_counter()
    for _ in range(steps * 4):
        task.step(a)
    return steps / (time.perf_counter() - t0)                        # agent steps (4 env steps each) per second


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3000)
    ap.add_argument("--eager-steps", type=int, default=300)
    ap.add_argument("--reps", type=int, default=3000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--explore", type=int, default=2000)
    ap.add_argument("--memory", type=int, default=20000)
    ap.add_argument("--only", default=",".join(LAUNCHERS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    from a2c_step_time import card
    import deeprl_b200 as rl
    rl.select_device(0)
    res = dict(card=card(), steps=args.steps, eager_steps=args.eager_steps, reps=args.reps, rounds=args.rounds,
               explore=args.explore, memory=args.memory, env_only_steps_per_s=round(env_rate(args.eager_steps), 1))
    print(res["card"])
    print("host envs alone: %.1f agent steps/s" % res["env_only_steps_per_s"])
    summary = lambda xs: dict(median=round(float(np.median(xs)), 4), min=round(min(xs), 4), max=round(max(xs), 4))
    for name in args.only.split(","):
        times = {"update_ms": []}
        for side, graph, async_actor, dtype in SIDES:
            # one side at a time: the eager path reads Config.COMPUTE_DTYPE while it runs, on its actor thread too
            ag = build(name, graph, async_actor, dtype, args.memory, args.explore)
            try:
                warm(ag)
                if graph and ag.graph_refusal is not None:
                    times[side + "_refusal"] = ag.graph_refusal
                times[side] = [agent_rate(ag, args.steps if graph else args.eager_steps) for _ in range(args.rounds)]
                if side == "graph_sync_actor" and ag._learner is not None:
                    times["update_ms"] = [update_ms(ag._learner, args.reps) for _ in range(args.rounds)]
            finally:
                ag.close()
                rl.Config.COMPUTE_DTYPE = torch.float32
        row = {k: (summary(v) if isinstance(v, list) and v else v) for k, v in times.items()}
        for side, *_ in SIDES:
            r = row[side]
            print("%-30s %-18s %8.1f agent steps/s (%.1f-%.1f)" % (name, side, r["median"], r["min"], r["max"]), flush=True)
        if row["update_ms"]:
            r = row["update_ms"]
            print("%-30s captured update    %8.4f ms (%.4f-%.4f)" % (name, r["median"], r["min"], r["max"]), flush=True)
        res[name] = row
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dqn_pixel_step_time.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
