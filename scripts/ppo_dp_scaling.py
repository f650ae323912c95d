"""Data-parallel PPO scaling (run under ``torchrun --nproc-per-node N``; N = 1 runs the single-process persistent kernel).

The bench.py PPO configuration per rank: 17-dim obs, 6 actions, hidden 64, 2048 x 16 rollout, 10 epochs x 64 minibatches on
synthetic envs seeded by rank.  Prints ONE JSON line: minibatch-phase updates/s per rank and aggregate (W x), whole-iteration
updates/s, the card and its power limit, and the per-phase cycle split of one data-parallel launch on rank 0 (including the
wait in the exchange).  Usage: torchrun --nproc-per-node N scripts/ppo_dp_scaling.py [iterations]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deeprl_b200 as rl  # noqa: E402
from deeprl_b200 import _lib, parallel  # noqa: E402

DP_PHASES = ["P1 fwd1", "P2 fwd2", "P3 heads", "P4 loss | critic bwd2", "P5 kl | critic bwd1", "P6 head bwd | prefetch",
             "P7 actor bwd2 | critic grads", "P8 actor bwd1", "P9 actor grads", "publish", "wait (exchange)", "reduce + Adam"]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=20).stdout.strip()
        name, watts = [x.strip() for x in out.split(",")]
        return name, watts
    except Exception:                                   # noqa: BLE001
        return torch.cuda.get_device_name(), "unknown"


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    world, rank, local = parallel.init()
    rl.select_device(local)
    rl.Config.COMPUTE_DTYPE = torch.float32
    seed = 1000 * rank
    torch.manual_seed(seed), np.random.seed(seed)
    c = rl.Config()
    c.merge(dict(tag=None))
    c.num_workers = 16
    c.task_fn = lambda: rl.Task("SyntheticCheetah-v0", num_envs=16, seed=seed)
    c.eval_env = rl.Task("SyntheticCheetah-v0", seed=seed)
    c.network_fn = lambda: rl.GaussianActorCriticNet(c.state_dim, c.action_dim, actor_body=rl.FCBody(c.state_dim, gate=torch.tanh),
                                                     critic_body=rl.FCBody(c.state_dim, gate=torch.tanh))
    c.actor_opt_fn = lambda p: torch.optim.Adam(p, 3e-4)
    c.critic_opt_fn = lambda p: torch.optim.Adam(p, 1e-3)
    c.discount, c.use_gae, c.gae_tau, c.gradient_clip = 0.99, True, 0.95, 0.5
    c.rollout_length, c.optimization_epochs, c.mini_batch_size, c.ppo_ratio_clip, c.target_kl = 2048, 10, 64, 0.2, 0.01
    c.state_normalizer = rl.MeanStdNormalizer()
    c.graph_minibatch = True
    ag = rl.PPOAgent(c)
    sgd = [0.0]
    inner = ag._graphed_epochs

    def timed(entries):
        torch.cuda.synchronize()
        t = time.perf_counter()
        inner(entries)
        torch.cuda.synchronize()
        sgd[0] += time.perf_counter() - t
    ag._graphed_epochs = timed
    ag.step()                                            # warm-up (learner construction, exchange rendezvous)
    torch.cuda.synchronize()
    mb = c.optimization_epochs * (c.rollout_length * c.num_workers // c.mini_batch_size)
    clocks = torch.zeros(2 + 12 * mb + 16, dtype=torch.int64, device=torch.device("cuda", local))
    sgd[0] = 0.0
    t0 = time.perf_counter()
    for i in range(iters):
        if i == iters - 1 and rank == 0:
            _lib.call("b2rl_ppo_set_phase_clocks", _lib.ptr(clocks))
        ag.step()
    torch.cuda.synchronize()
    _lib.call("b2rl_ppo_set_phase_clocks", None)
    dt = (time.perf_counter() - t0) / iters
    if world > 1:
        ag._graph.check_exchange()
    sgd_s = parallel.max_over_ranks(sgd[0] / iters, torch.device("cuda", local))
    dt = parallel.max_over_ranks(dt, torch.device("cuda", local))
    if rank == 0:
        name, watts = card()
        res = dict(metric="data-parallel PPO minibatch updates/s", world=world, iterations=iters, card=name, power_limit=watts,
                   minibatch_updates_per_iteration=mb, minibatch_phase_updates_per_s_per_rank=round(mb / sgd_s, 1),
                   minibatch_phase_updates_per_s_aggregate=round(world * mb / sgd_s, 1),
                   iteration_updates_per_s_per_rank=round(mb / dt, 1), iteration_updates_per_s_aggregate=round(world * mb / dt, 1),
                   seconds_per_iteration=round(dt, 3), minibatch_phase_seconds=round(sgd_s, 3))
        ck = clocks.cpu().numpy()
        n_ph = 12 if world > 1 else 9
        names = DP_PHASES if world > 1 else DP_PHASES[:8] + ["P9 actor update"]
        if ck[1 + n_ph * mb - 1] > 0:
            per = ck[1:1 + n_ph * mb].reshape(mb, n_ph) - np.concatenate([[ck[0]], ck[1:n_ph * mb]]).reshape(mb, n_ph)
            tot = per.sum(1).mean()
            res["cycles_per_update"] = round(float(tot), 0)
            res["phase_cycles_mean"] = {n: round(float(per[:, i].mean()), 0) for i, n in enumerate(names)}
            res["phase_share_pct"] = {n: round(100 * float(per[:, i].mean()) / tot, 1) for i, n in enumerate(names)}
        print(json.dumps(res), flush=True)
    ag.close()
    parallel.leave()


if __name__ == "__main__":
    main()
