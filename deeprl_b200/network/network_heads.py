#######################################################################
# This file restates an interface of ShangtongZhang/DeepRL, whose     #
# licence asks that the following declaration stay at the top:        #
#                                                                     #
# Copyright (C) 2017 Shangtong Zhang(zhangshangtong.cpp@gmail.com)    #
# Permission given to modify the code as long as you keep this        #
# declaration at the top                                              #
#######################################################################
"""Network heads returning the reference's output dicts (``deep_rl/network/network_heads.py``):
``VanillaNet``:11 / ``DuelingNet``:24 -> ``q``; ``CategoricalNet``:40 / ``RainbowNet``:57 -> ``prob, log_prob``;
``QuantileNet``:89 -> ``quantile``; ``GaussianActorCriticNet``:173 / ``CategoricalActorCriticNet``:217 ->
``action, log_pi_a, entropy, v[, mean]``.  Module and parameter names match the reference so its
``state_dict``s load.  Every ``forward`` accepts numpy or tensors (``tensor(x)``), outputs are float32.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ..utils import Config, tensor
from . import fused
from .network_bodies import DummyBody, _autocast
from .network_utils import BaseNet, NoisyLinear, layer_init


def _phi(body, x):
    if type(x).__name__ == "RingFrames":                  # not-materialised frame stacks (K1): the body reads the ring
        return body(x)
    x = tensor(x)
    if x.dtype == torch.uint8:
        x = x.float()
    return body(x)


class VanillaNet(nn.Module, BaseNet):
    def __init__(self, output_dim, body):
        super().__init__()
        self.fc_head = layer_init(nn.Linear(body.feature_dim, output_dim))
        self.body = body
        self.to(Config.DEVICE)

    def forward(self, x):
        phi = _phi(self.body, x)
        if fused.narrow_head_ok(phi, self.fc_head):
            return dict(q=fused.narrow_head(phi, self.fc_head))
        with _autocast():
            q = self.fc_head(phi)
        return dict(q=q.float())


class DuelingNet(nn.Module, BaseNet):
    def __init__(self, action_dim, body):
        super().__init__()
        self.fc_value = layer_init(nn.Linear(body.feature_dim, 1))
        self.fc_advantage = layer_init(nn.Linear(body.feature_dim, action_dim))
        self.body = body
        self.to(Config.DEVICE)

    def forward(self, x, to_numpy=False):
        phi = _phi(self.body, x)
        if fused.narrow_head_ok(phi, self.fc_advantage, self.fc_value):
            return dict(q=fused.narrow_head(phi, self.fc_advantage, self.fc_value))
        with _autocast():
            value = self.fc_value(phi).float()
            adv = self.fc_advantage(phi).float()
        q = value.expand_as(adv) + (adv - adv.mean(1, keepdim=True).expand_as(adv))
        return dict(q=q)


class CategoricalNet(nn.Module, BaseNet):
    def __init__(self, action_dim, num_atoms, body):
        super().__init__()
        self.fc_categorical = layer_init(nn.Linear(body.feature_dim, action_dim * num_atoms))
        self.action_dim, self.num_atoms = action_dim, num_atoms
        self.body = body
        self.to(Config.DEVICE)

    def forward(self, x):
        phi = _phi(self.body, x)
        if fused.dist_head_ok(phi, self.fc_categorical):           # wgmma GEMM + fused softmax / log_softmax (csrc/disthead.cu)
            log_prob, prob = fused.dist_head(phi, self.fc_categorical, self.action_dim, self.num_atoms, True)
            return dict(prob=prob, log_prob=log_prob)
        with _autocast():
            pre = self.fc_categorical(phi)
        pre = pre.float().view(-1, self.action_dim, self.num_atoms)
        return dict(prob=F.softmax(pre, dim=-1), log_prob=F.log_softmax(pre, dim=-1))


class RainbowNet(nn.Module, BaseNet):
    def __init__(self, action_dim, num_atoms, body, noisy_linear):
        super().__init__()
        if noisy_linear:
            self.fc_value = NoisyLinear(body.feature_dim, num_atoms)
            self.fc_advantage = NoisyLinear(body.feature_dim, action_dim * num_atoms)
        else:
            self.fc_value = layer_init(nn.Linear(body.feature_dim, num_atoms))
            self.fc_advantage = layer_init(nn.Linear(body.feature_dim, action_dim * num_atoms))
        self.action_dim, self.num_atoms = action_dim, num_atoms
        self.body = body
        self.noisy_linear = noisy_linear
        self.to(Config.DEVICE)

    def reset_noise(self):
        if self.noisy_linear:
            self.fc_value.reset_noise()
            self.fc_advantage.reset_noise()
            self.body.reset_noise()

    def forward(self, x):
        phi = _phi(self.body, x)
        with _autocast():
            value = self.fc_value(phi).float().view(-1, 1, self.num_atoms)
            adv = self.fc_advantage(phi).float().view(-1, self.action_dim, self.num_atoms)
        q = value + (adv - adv.mean(1, keepdim=True))
        return dict(prob=F.softmax(q, dim=-1), log_prob=F.log_softmax(q, dim=-1))


class QuantileNet(nn.Module, BaseNet):
    def __init__(self, action_dim, num_quantiles, body):
        super().__init__()
        self.fc_quantiles = layer_init(nn.Linear(body.feature_dim, action_dim * num_quantiles))
        self.action_dim, self.num_quantiles = action_dim, num_quantiles
        self.body = body
        self.to(Config.DEVICE)

    def forward(self, x):
        phi = _phi(self.body, x)
        if fused.dist_head_ok(phi, self.fc_quantiles):             # wgmma GEMMs (csrc/disthead.cu for the backward operand)
            q, _ = fused.dist_head(phi, self.fc_quantiles, self.action_dim, self.num_quantiles, False)
            return dict(quantile=q)
        with _autocast():
            quantiles = self.fc_quantiles(phi)
        return dict(quantile=quantiles.float().view(-1, self.action_dim, self.num_quantiles))


class _ActorCriticBase(nn.Module, BaseNet):
    def _build(self, state_dim, action_dim, phi_body, actor_body, critic_body):
        phi_body = phi_body if phi_body is not None else DummyBody(state_dim)
        actor_body = actor_body if actor_body is not None else DummyBody(phi_body.feature_dim)
        critic_body = critic_body if critic_body is not None else DummyBody(phi_body.feature_dim)
        self.phi_body, self.actor_body, self.critic_body = phi_body, actor_body, critic_body
        self.fc_action = layer_init(nn.Linear(actor_body.feature_dim, action_dim), 1e-3)
        self.fc_critic = layer_init(nn.Linear(critic_body.feature_dim, 1), 1e-3)

    def _trunk(self, obs):
        obs = tensor(obs)
        if obs.dtype == torch.uint8:
            obs = obs.float()
        phi = self.phi_body(obs)
        return self.actor_body(phi), self.critic_body(phi)


class GaussianActorCriticNet(_ActorCriticBase):
    def __init__(self, state_dim, action_dim, phi_body=None, actor_body=None, critic_body=None):
        super().__init__()
        self._build(state_dim, action_dim, phi_body, actor_body, critic_body)
        self.std = nn.Parameter(torch.zeros(action_dim))
        self.phi_params = list(self.phi_body.parameters())
        self.actor_params = list(self.actor_body.parameters()) + list(self.fc_action.parameters()) + self.phi_params
        self.actor_params.append(self.std)
        self.critic_params = list(self.critic_body.parameters()) + list(self.fc_critic.parameters()) + self.phi_params
        self.to(Config.DEVICE)

    def forward(self, obs, action=None):
        phi_a, phi_v = self._trunk(obs)
        mean = torch.tanh(self.fc_action(phi_a))
        v = self.fc_critic(phi_v)
        dist = torch.distributions.Normal(mean, F.softplus(self.std))
        if action is None:
            action = dist.sample()
        log_prob = dist.log_prob(action).sum(-1).unsqueeze(-1)
        entropy = dist.entropy().sum(-1).unsqueeze(-1)
        return dict(action=action, log_pi_a=log_prob, entropy=entropy, mean=mean, v=v)


class CategoricalActorCriticNet(_ActorCriticBase):
    def __init__(self, state_dim, action_dim, phi_body=None, actor_body=None, critic_body=None):
        super().__init__()
        self._build(state_dim, action_dim, phi_body, actor_body, critic_body)
        self.actor_params = list(self.actor_body.parameters()) + list(self.fc_action.parameters())
        self.critic_params = list(self.critic_body.parameters()) + list(self.fc_critic.parameters())
        self.phi_params = list(self.phi_body.parameters())
        self.to(Config.DEVICE)

    def forward(self, obs, action=None):
        phi_a, phi_v = self._trunk(obs)
        with _autocast():
            logits = self.fc_action(phi_a).float()
            v = self.fc_critic(phi_v).float()
        dist = torch.distributions.Categorical(logits=logits)
        if action is None:
            action = dist.sample()
        log_prob = dist.log_prob(action).unsqueeze(-1)
        entropy = dist.entropy().unsqueeze(-1)
        return dict(action=action, log_pi_a=log_prob, entropy=entropy, v=v)
