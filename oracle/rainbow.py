"""TEST INFRASTRUCTURE -- functional torch-CPU restatement of the reference's Rainbow pieces: ``NoisyLinear`` in training mode
(network_utils.py:31-83), ``RainbowNet`` on an ``FCBody`` (network_heads.py:57-86, network_bodies.py:50-73) and
``CategoricalDQNAgent``'s update with them (CategoricalDQN_agent.py:60-89 on DQN_agent.py:115-134).  Driven by a
``state_dict`` with the reference's names like oracle/nets.py; the noise is passed in as tensors, so an update can be compared
with given noise.
"""
import torch
import torch.nn.functional as F

from .agents import DQNFamilyOracle

LAYERS = ("body.layers.0.", "body.layers.1.", "fc_advantage.", "fc_value.")


def transform_noise(x):                                                 # network_utils.py:81-83
    return x.sign().mul(x.abs().sqrt())


def noisy_or_linear(sd, x, prefix, noise=None):                         # network_utils.py:49-55 (training mode) / nn.Linear
    """``prefix`` names a NoisyLinear (``weight_mu`` ...) or an nn.Linear (``weight``).  ``noise``: this layer's
    (noise_in, noise_out_weight, noise_out_bias); without it the epsilons of the state dict's buffers are used."""
    if prefix + "weight_mu" not in sd:
        return F.linear(x, sd[prefix + "weight"], sd[prefix + "bias"])
    if noise is None:
        w_eps, b_eps = sd[prefix + "weight_epsilon"], sd[prefix + "bias_epsilon"]
    else:                                                               # reset_noise, network_utils.py:71-79
        w_eps, b_eps = torch.outer(transform_noise(noise[1]), transform_noise(noise[0])), transform_noise(noise[2])
    return F.linear(x, sd[prefix + "weight_mu"] + sd[prefix + "weight_sigma"] * w_eps,
                    sd[prefix + "bias_mu"] + sd[prefix + "bias_sigma"] * b_eps)


def rainbow(sd, x, action_dim, num_atoms, gate=F.relu, noise=None):
    """``noise``: dict layer prefix -> (noise_in, noise_out_weight, noise_out_bias) for the NoisyLinear layers.
    Returns (prob, log_prob), each [B, action_dim, num_atoms]."""
    nz = (lambda p: None) if noise is None else noise.get
    i = 0
    while "body.layers.%d.bias_mu" % i in sd or "body.layers.%d.bias" % i in sd:
        x = gate(noisy_or_linear(sd, x, "body.layers.%d." % i, nz("body.layers.%d." % i)))
        i += 1
    value = noisy_or_linear(sd, x, "fc_value.", nz("fc_value.")).view(-1, 1, num_atoms)
    adv = noisy_or_linear(sd, x, "fc_advantage.", nz("fc_advantage.")).view(-1, action_dim, num_atoms)
    q = value + (adv - adv.mean(1, keepdim=True))
    return F.softmax(q, dim=-1), F.log_softmax(q, dim=-1)


class RainbowOracle(DQNFamilyOracle):
    """``DQNFamilyOracle``'s categorical update with ``rainbow`` as the network.  ``sd`` holds the parameters only (every
    entry is trained).  ``noise`` / ``target_noise`` are the noise dicts of the next update, which the caller sets where
    the reference calls ``reset_noise()`` on the two networks (DQN_agent.py:116-118)."""

    def __init__(self, sd, action_dim, optimizer_fn, discount, **kw):
        DQNFamilyOracle.__init__(self, sd, "categorical", "fc", action_dim, optimizer_fn, discount, **kw)
        self.noise = self.target_noise = None

    def forward(self, sd, x):
        p, lp = rainbow(sd, x, self.A, self.atoms.numel(), self.gate, self.noise if sd is self.sd else self.target_noise)
        return dict(prob=p, log_prob=lp)
