"""Golden fixture for the Rainbow update: ``CategoricalDQNAgent`` (CategoricalDQN_agent.py:27-89 on DQN_agent.py:101-138) of
the UNMODIFIED reference, imported through oracle/ref_shim.py in the build container, with a noisy ``RainbowNet`` on a noisy
two-layer ``FCBody``, RMSprop, prioritized replay, ``double_q`` and ``n_step`` 3 on a seeded synthetic task.
Writes tests/golden/rainbow_agent.npz: per gradient update the sampled batch (with ``sampling_prob``), beta, the noise both
networks drew in that update, the per-sample KL, the priorities handed to the replay, the online parameters afterwards and
whether the target network was synced afterwards.

Layouts: ``keys`` lists the 16 parameters in the device kernels' order (body.layers.0, body.layers.1, fc_advantage, fc_value;
each weight_mu, weight_sigma, bias_mu, bias_sigma); ``params`` rows are their concatenation.  A noise vector is, for the same
four layers in turn, noise_in, noise_out_weight, noise_out_bias."""
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle.ref_shim import import_reference  # noqa: E402

ref = import_reference()
from deeprl_b200.component.envs import Task as SynthTask  # noqa: E402  (host env, duck-typed for the reference)

torch.set_num_threads(1)
ref.select_device(-1)
LAYERS = ("body.layers.0", "body.layers.1", "fc_advantage", "fc_value")
KEYS = [l + "." + p for l in LAYERS for p in ("weight_mu", "weight_sigma", "bias_mu", "bias_sigma")]
UPDATES = 20


class NullLogger:
    def info(self, *a, **k): pass
    debug = warning = add_scalar = add_histogram = info


def flat_params(net):
    sd = net.state_dict()
    return np.concatenate([sd[k].detach().numpy().ravel() for k in KEYS])


def noise_vector(net):
    sd = net.state_dict()
    return np.concatenate([sd[l + "." + b].numpy().ravel() for l in LAYERS
                           for b in ("noise_in", "noise_out_weight", "noise_out_bias")])


np.random.seed(11), torch.manual_seed(11), random.seed(11)
c = ref.Config()
c.merge(dict(tag=None, n_step=3))
c.task_fn = lambda: SynthTask("CartPole-v0", seed=3)
c.eval_env = c.task_fn()
c.history_length, c.batch_size, c.discount, c.double_q, c.noisy_linear = 1, 16, 0.99, True, True
c.optimizer_fn = lambda p: torch.optim.RMSprop(p, 0.001)
c.categorical_v_min, c.categorical_v_max, c.categorical_n_atoms = -100, 100, 50
c.network_fn = lambda: ref.RainbowNet(c.action_dim, c.categorical_n_atoms,
                                      ref.FCBody(c.state_dim, hidden_units=(16, 16), noisy_linear=True), noisy_linear=True)
rk = dict(memory_size=256, batch_size=c.batch_size, n_step=c.n_step, discount=c.discount, history_length=1)
c.replay_fn = lambda: ref.ReplayWrapper(ref.PrioritizedReplay, rk, False)
c.replay_eps, c.replay_alpha = 0.01, 0.5
betas = []
schedule = ref.LinearSchedule(0.4, 1.0, 200)


def replay_beta():
    betas.append(schedule())
    return betas[-1]


c.replay_beta = replay_beta
c.random_action_prob = ref.LinearSchedule(1.0, 0.1, 100)
c.target_network_update_freq, c.exploration_steps = 5, 40
c.sgd_update_frequency, c.gradient_clip, c.async_actor = 4, 10, False
ag = ref.CategoricalDQNAgent(c)
ag.logger = NullLogger()
rec = dict(batches=[], kl=[], noise=[], target_noise=[], prio=[], params=[], synced=[])
orig_sample, orig_loss, orig_prio = ag.replay.sample, ag.compute_loss, ag.replay.update_priorities


def sample():
    t = orig_sample()
    rec["batches"].append(t)
    return t


def compute_loss(t):                                    # (called right after both reset_noise(), DQN_agent.py:116-119)
    rec["noise"].append(noise_vector(ag.network))
    rec["target_noise"].append(noise_vector(ag.target_network))
    kl = orig_loss(t)
    rec["kl"].append(kl.detach().numpy().copy())
    return kl


def update_priorities(info):
    info = list(info)
    rec["prio"].append(np.asarray([p for _, p in info], np.float32))
    return orig_prio(info)


ag.replay.sample, ag.compute_loss, ag.replay.update_priorities = sample, compute_loss, update_priorities
out = {"init." + k: v.detach().numpy().copy() for k, v in ag.network.state_dict().items() if k in KEYS}
while len(rec["params"]) < UPDATES:
    ag.step()
    if ag.total_steps > c.exploration_steps:
        rec["params"].append(flat_params(ag.network))
        rec["synced"].append(bool(np.array_equal(flat_params(ag.target_network), rec["params"][-1])))
assert len(rec["batches"]) == len(rec["kl"]) == len(rec["prio"]) == len(betas) == UPDATES and sum(rec["synced"]) >= 3
out["keys"] = np.asarray(KEYS)
for f in rec["batches"][0]._fields:
    out["b_" + f] = np.stack([np.asarray(getattr(b, f)) for b in rec["batches"]])
out.update(beta=np.asarray(betas, np.float64), kl=np.stack(rec["kl"]), priority=np.stack(rec["prio"]),
           noise=np.stack(rec["noise"]), target_noise=np.stack(rec["target_noise"]), params=np.stack(rec["params"]),
           synced=np.asarray(rec["synced"]))
path = os.path.join(HERE, "rainbow_agent.npz")
np.savez_compressed(path, **out)
print("rainbow_agent.npz %d arrays, %.1f KB" % (len(out), os.path.getsize(path) / 1024))
