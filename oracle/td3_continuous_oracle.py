"""Restatement of cleanrl/td3_continuous_action.py's update in eager PyTorch (fp32, any device).  TEST INFRASTRUCTURE and
the eager arm of bench_td3_continuous.py.

* ``head_forward`` / ``head_backward``: the deterministic head of ``Actor.forward`` (td3_continuous_action.py:128-132)
  and autograd's chain through it, in the order the kernels use;
* ``smooth``: the target policy smoothing of :232-238, rounding for rounding;
* ``critic_loss``, ``actor_loss``: the pieces of the update (:239-256);
* ``EagerTD3``: the whole update with the reference's modules, autograd and torch.optim.Adam, its smoothing draw made
  by a caller-supplied ``noise(shape)``.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.sac_continuous_oracle import _Q, critic_forward, mlp_params  # noqa: F401  (re-exported for the tests)


def actor_trunk(params, x):
    """h2 of the actor's trunk and fc_mu's output z (params: fc1.w, fc1.b, fc2.w, fc2.b, fc_mu.w, fc_mu.b)."""
    w1, b1, w2, b2, wm, bm = params
    h = F.relu(F.linear(F.relu(F.linear(x, w1, b1)), w2, b2))
    return F.linear(h, wm, bm)


def head_forward(z, scale, bias):
    """(mu, y) of Actor.forward: y = tanh(z), mu = y * action_scale + action_bias."""
    y = torch.tanh(z)
    return y * scale + bias, y


def head_backward(y, scale, dmu):
    """d z of <dmu, mu>: autograd's mul backward (dmu * scale) then tanh_backward (* (1 - y^2))."""
    return (dmu * scale) * (1 - y * y)


def smooth(mu, eps, scale, policy_noise, noise_clip, low, high):
    """next_state_actions of td3_continuous_action.py:232-238 from the target actor's mu and the standard normals eps:
    a multiply, a clamp, a multiply, an add, a clamp to the scalar bounds."""
    clipped_noise = (eps * policy_noise).clamp(-noise_clip, noise_clip) * scale
    return (mu + clipped_noise).clamp(low, high)


def critic_loss(q1, q2, q1t, q2t, rewards, dones, gamma):
    """(y, qf1_loss, qf2_loss, dq1, dq2) of td3_continuous_action.py:241-247 (q* [B])."""
    y = rewards + (1 - dones) * gamma * torch.min(q1t, q2t)
    B = q1.numel()
    return y, F.mse_loss(q1, y), F.mse_loss(q2, y), (2.0 / B) * (q1 - y), (2.0 / B) * (q2 - y)


def actor_loss(q1_pi):
    return -q1_pi.mean()


class _Actor(nn.Module):
    def __init__(self, obs_dim, act_dim, scale, bias):
        super().__init__()
        self.fc1, self.fc2, self.fc_mu = nn.Linear(obs_dim, 256), nn.Linear(256, 256), nn.Linear(256, act_dim)
        self.register_buffer("action_scale", scale.clone())
        self.register_buffer("action_bias", bias.clone())

    def forward(self, x):
        x = F.relu(self.fc2(F.relu(self.fc1(x))))
        return torch.tanh(self.fc_mu(x)) * self.action_scale + self.action_bias


class EagerTD3:
    """The reference's update (td3_continuous_action.py:230-267) in eager PyTorch on ``device``: initialised from the
    flat parameters of the actor, the twin critics, the twin targets and the actor target."""

    def __init__(self, actor_flat, q_flat, qt_flat, actor_target_flat, obs_dim, act_dim, scale, bias, device,
                 learning_rate=3e-4, gamma=0.99, tau=0.005, policy_noise=0.2, noise_clip=0.5, policy_frequency=2,
                 low=-1.0, high=1.0):
        self.actor = _Actor(obs_dim, act_dim, scale, bias).to(device)
        self.target_actor = _Actor(obs_dim, act_dim, scale, bias).to(device)
        self.qs = [_Q(obs_dim, act_dim).to(device) for _ in range(4)]
        with torch.no_grad():
            torch.nn.utils.vector_to_parameters(actor_flat.to(device), self.actor.parameters())
            torch.nn.utils.vector_to_parameters(actor_target_flat.to(device), self.target_actor.parameters())
            n = sum(p.numel() for p in self.qs[0].parameters())
            for i, (flat, k) in enumerate(((q_flat, 0), (q_flat, 1), (qt_flat, 0), (qt_flat, 1))):
                torch.nn.utils.vector_to_parameters(flat[k * n:(k + 1) * n].to(device), self.qs[i].parameters())
        self.qf1, self.qf2, self.qf1_target, self.qf2_target = self.qs
        self.q_optimizer = torch.optim.Adam(list(self.qf1.parameters()) + list(self.qf2.parameters()), lr=learning_rate)
        self.actor_optimizer = torch.optim.Adam(list(self.actor.parameters()), lr=learning_rate)
        self.gamma, self.tau, self.pf = gamma, tau, policy_frequency
        self.policy_noise, self.noise_clip, self.low, self.high = policy_noise, noise_clip, low, high
        self.stats = {}

    def update(self, global_step, obs, actions, next_obs, rewards, dones, noise):
        with torch.no_grad():
            eps = noise(actions.shape)
            next_state_actions = smooth(self.target_actor(next_obs), eps, self.target_actor.action_scale,
                                        self.policy_noise, self.noise_clip, self.low, self.high)
            q1t, q2t = self.qf1_target(next_obs, next_state_actions), self.qf2_target(next_obs, next_state_actions)
            y = rewards.flatten() + (1 - dones.flatten()) * self.gamma * torch.min(q1t, q2t).view(-1)
        q1 = self.qf1(obs, actions).view(-1)
        q2 = self.qf2(obs, actions).view(-1)
        l1, l2 = F.mse_loss(q1, y), F.mse_loss(q2, y)
        self.q_optimizer.zero_grad()
        (l1 + l2).backward()
        self.q_optimizer.step()
        self.stats.update(qf1_values=q1.mean().item, qf2_values=q2.mean().item, qf1_loss=l1.item, qf2_loss=l2.item,
                          next_state_actions=next_state_actions, y=y)
        if global_step % self.pf == 0:
            al = -self.qf1(obs, self.actor(obs)).mean()
            self.actor_optimizer.zero_grad()
            al.backward()
            self.actor_optimizer.step()
            self.stats["actor_loss"] = al.item
            for src, dst in ((self.actor, self.target_actor), (self.qf1, self.qf1_target), (self.qf2, self.qf2_target)):
                for param, target_param in zip(src.parameters(), dst.parameters()):
                    target_param.data.copy_(self.tau * param.data + (1 - self.tau) * target_param.data)
