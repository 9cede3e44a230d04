"""Restatement of cleanrl/ddpg_continuous_action.py's update in eager PyTorch (fp32, any device).  TEST INFRASTRUCTURE
and the eager arm of bench_ddpg_continuous.py.

* the deterministic head and the actor loss are TD3's (``oracle.td3_continuous_oracle``, re-exported here);
* ``critic_loss``: the one-critic target, loss and gradient of ddpg_continuous_action.py:216-224;
* ``EagerDDPG``: the whole update with the reference's modules, autograd and torch.optim.Adam.  It draws nothing.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.td3_continuous_oracle import (  # noqa: F401  (re-exported for the tests)
    _Actor, _Q, actor_loss, actor_trunk, critic_forward, head_backward, head_forward, mlp_params)


def critic_loss(q, q_next, rewards, dones, gamma):
    """(y, qf1_loss, dq) of ddpg_continuous_action.py:219-224 (all [B]): y = r + (1 - d) gamma q_next, F.mse_loss(q, y)
    and its gradient (2 / B)(q - y)."""
    y = rewards + (1 - dones) * gamma * q_next
    return y, F.mse_loss(q, y), (2.0 / q.numel()) * (q - y)


class EagerDDPG:
    """The reference's update (ddpg_continuous_action.py:214-245) in eager PyTorch on ``device``: initialised from the
    flat parameters of the actor, qf1, qf1_target and the actor target."""

    def __init__(self, actor_flat, q_flat, qt_flat, actor_target_flat, obs_dim, act_dim, scale, bias, device,
                 learning_rate=3e-4, gamma=0.99, tau=0.005, policy_frequency=2):
        self.actor = _Actor(obs_dim, act_dim, scale, bias).to(device)
        self.target_actor = _Actor(obs_dim, act_dim, scale, bias).to(device)
        self.qf1, self.qf1_target = _Q(obs_dim, act_dim).to(device), _Q(obs_dim, act_dim).to(device)
        with torch.no_grad():
            for flat, net in ((actor_flat, self.actor), (actor_target_flat, self.target_actor), (q_flat, self.qf1),
                              (qt_flat, self.qf1_target)):
                n = sum(p.numel() for p in net.parameters())
                torch.nn.utils.vector_to_parameters(flat[:n].to(device), net.parameters())
        self.q_optimizer = torch.optim.Adam(list(self.qf1.parameters()), lr=learning_rate)
        self.actor_optimizer = torch.optim.Adam(list(self.actor.parameters()), lr=learning_rate)
        self.gamma, self.tau, self.pf = gamma, tau, policy_frequency
        self.stats = {}

    def update(self, global_step, obs, actions, next_obs, rewards, dones):
        with torch.no_grad():
            next_state_actions = self.target_actor(next_obs)
            qf1_next_target = self.qf1_target(next_obs, next_state_actions)
            y = rewards.flatten() + (1 - dones.flatten()) * self.gamma * qf1_next_target.view(-1)
        q1 = self.qf1(obs, actions).view(-1)
        l1 = F.mse_loss(q1, y)
        self.q_optimizer.zero_grad()
        l1.backward()
        self.q_optimizer.step()
        self.stats.update(qf1_values=q1.mean().item, qf1_loss=l1.item, next_state_actions=next_state_actions, y=y)
        if global_step % self.pf == 0:
            al = -self.qf1(obs, self.actor(obs)).mean()
            self.actor_optimizer.zero_grad()
            al.backward()
            self.actor_optimizer.step()
            self.stats["actor_loss"] = al.item
            for src, dst in ((self.actor, self.target_actor), (self.qf1, self.qf1_target)):
                for param, target_param in zip(src.parameters(), dst.parameters()):
                    target_param.data.copy_(self.tau * param.data + (1 - self.tau) * target_param.data)
