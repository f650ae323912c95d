"""torchrun worker of tests/test_ppo_data_parallel.py::test_data_parallel_across_gpus (one process per GPU, peer access).

learner: PersistentPPOLearner on rank-seeded problems -> parameters bit-identical across ranks and equal to the union oracle.
agent:   PPOAgent, two iterations with a short rollout -> parameters bit-identical across ranks; after the first iteration rank
         0's parameters differ from a single-process PPOAgent with rank 0's seeds (the ranks really shared gradients).
agent_single OUT: the single-process run (no torchrun), parameters after one iteration saved to OUT."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def make_agent(rl, seed):
    torch.manual_seed(seed), np.random.seed(seed)
    c = rl.Config()
    c.merge(dict(tag=None))
    c.num_workers = 4
    c.task_fn = lambda: rl.Task("SyntheticCheetah-v0", num_envs=4, seed=seed)
    c.eval_env = rl.Task("SyntheticCheetah-v0", seed=seed)
    c.network_fn = lambda: rl.GaussianActorCriticNet(c.state_dim, c.action_dim, actor_body=rl.FCBody(c.state_dim, gate=torch.tanh),
                                                     critic_body=rl.FCBody(c.state_dim, gate=torch.tanh))
    c.actor_opt_fn = lambda p: torch.optim.Adam(p, 3e-4)
    c.critic_opt_fn = lambda p: torch.optim.Adam(p, 1e-3)
    c.discount, c.use_gae, c.gae_tau, c.gradient_clip = 0.99, True, 0.95, 0.5
    c.rollout_length, c.optimization_epochs, c.mini_batch_size, c.ppo_ratio_clip, c.target_kl = 64, 2, 64, 0.2, 0.01
    c.state_normalizer = rl.MeanStdNormalizer()
    c.graph_minibatch = True
    return rl.PPOAgent(c)


def flat_params(net):
    return torch.cat([p.detach().reshape(-1) for p in net.parameters()])


def main():
    what = sys.argv[1]
    import deeprl_b200 as rl
    if what == "agent_single":
        rl.select_device(0)
        rl.Config.COMPUTE_DTYPE = torch.float32
        ag = make_agent(rl, 1234)
        ag.step()
        torch.save(flat_params(ag.network).cpu(), sys.argv[2])
        return
    import torch.distributed as dist
    from deeprl_b200 import parallel
    world, rank, local = parallel.init()
    rl.select_device(local)
    rl.Config.COMPUTE_DTYPE = torch.float32
    dev = torch.device("cuda", local)
    ok = True
    if what == "learner":
        from deeprl_b200 import ops
        from deeprl_b200.learner import PersistentPPOLearner
        import test_ppo_data_parallel as T
        for case in (0, 1):
            c = T.CASES[case]
            s = T.Setup(c, case, world)
            net = rl.GaussianActorCriticNet(c["D"], c["A"], actor_body=rl.FCBody(c["D"], hidden_units=(c["H1"], c["H2"]), gate=torch.tanh),
                                            critic_body=rl.FCBody(c["D"], hidden_units=(c["H1"], c["H2"]), gate=torch.tanh))
            with torch.no_grad():
                for k, p in net.named_parameters():
                    p.copy_(s.sd0[k].reshape(p.shape))
            a = ops.FlatOptimizer.from_torch(torch.optim.Adam(net.actor_params, c["a_lr"]), net.actor_params)
            cr = ops.FlatOptimizer.from_torch(torch.optim.Adam(net.critic_params, T.HYPER["c_lr"]), net.critic_params)
            lr = PersistentPPOLearner(net, a, cr, c["rows"], c["D"], c["A"], c["mb"], T.HYPER["clip"], T.HYPER["ent_w"], c["target_kl"],
                                      s.n_batches, world=world, rank=rank)
            p = s.problems[rank]
            lr.buf["state"].copy_(p[1]), lr.buf["action"].copy_(p[2]), lr.buf["log_pi_a"].copy_(p[3]), lr.buf["ret"].copy_(p[4])
            lr.buf["advantage"].copy_(torch.from_numpy(s.rank(rank, "adv")).reshape(-1, 1))
            lr.run(lr.set_batches(list(s.perms[rank])))
            torch.cuda.synchronize()
            lr.check_exchange()
            mine = torch.cat([a.flat, cr.flat, a.s1, a.s2, cr.s1, cr.s2])
            allp = [torch.empty_like(mine) for _ in range(world)]
            dist.all_gather(allp, mine)
            same = all(torch.equal(allp[0], x) for x in allp)
            # against the union oracle: the Setup arrays take this rank's results for every rank (they are identical)
            for key, t in (("a_flat", a.flat), ("c_flat", cr.flat), ("a_m", a.s1), ("a_v", a.s2), ("c_m", cr.s1), ("c_v", cr.s2)):
                setattr(s, key, np.tile(t.cpu().numpy()[:getattr(s, key).size // world], world))
            s.a_step[:] = int(a.step_dev)
            s.c_step[:] = int(cr.step_dev)
            state, gates = s.oracle()
            try:
                s.check(state, sum(gates), s.n_batches)
                close = True
            except AssertionError as e:
                print("rank %d case %d: %s" % (rank, case, str(e)[:500]), flush=True)
                close = False
            print("rank %d case %d identical=%s oracle=%s actor_steps=%d/%d" % (rank, case, same, close, sum(gates), len(gates)),
                  flush=True)
            ok = ok and same and close
            lr.exchange.close()
    else:
        import subprocess
        import tempfile
        ag = make_agent(rl, 1234 + 7919 * rank)         # rank-local envs and seeds
        single = None
        if rank == 0:
            out = os.path.join(tempfile.mkdtemp(), "single.pt")
            env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "LOCAL_WORLD_SIZE",
                                                                    "MASTER_ADDR", "MASTER_PORT", "GROUP_RANK", "ROLE_RANK")}
            env["CUDA_VISIBLE_DEVICES"] = str(local)
            subprocess.run([sys.executable, os.path.abspath(__file__), "agent_single", out], env=env, check=True)
            single = torch.load(out)
        for it in range(2):
            ag.step()
            torch.cuda.synchronize()
            ag._graph.check_exchange()
            mine = flat_params(ag.network)
            allp = [torch.empty_like(mine) for _ in range(world)]
            dist.all_gather(allp, mine)
            same = all(torch.equal(allp[0], x) for x in allp)
            ok = ok and same
            if it == 0 and rank == 0:
                differs = not torch.equal(mine.cpu(), single)
                ok = ok and differs
                print("rank 0: differs from the single-process run=%s" % differs, flush=True)
            print("rank %d iteration %d identical=%s" % (rank, it, same), flush=True)
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("ok=%s" % bool(int(flag)), flush=True)
    parallel.leave()


if __name__ == "__main__":
    main()
