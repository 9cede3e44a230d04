"""Restatement of cleanrl/sac_continuous_action.py's update in eager PyTorch (fp32, any device).  TEST INFRASTRUCTURE and
the eager arm of bench_sac_continuous.py.

* ``head_forward`` / ``head_backward``: the tanh-Gaussian head of ``Actor.get_action`` (sac_continuous_action.py:139-151)
  and autograd's chain through it, restated step by step in the order the kernels use;
* ``critic_loss``, ``actor_loss``, ``temperature_step``: the pieces of the update (:257-297);
* ``EagerSAC``: the whole update with the reference's modules, autograd and torch.optim.Adam, its noise drawn by a
  caller-supplied ``noise(shape)`` in the reference's order (next_obs, then per actor step the actor and the autotune
  re-evaluation).
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn
import torch.nn.functional as F

LOG_STD_MAX = 2
LOG_STD_MIN = -5
_C = math.log(math.sqrt(2 * math.pi))


def mlp_params(flat, in_dim, out_dim, heads=1):
    """Views of one network's flat parameters (fc1.w, fc1.b, fc2.w, fc2.b, then per head w, b)."""
    out, off = [], 0
    for shape in [(256, in_dim), (256,), (256, 256), (256,)] + [(out_dim, 256), (out_dim,)] * heads:
        n = math.prod(shape)
        out.append(flat[off:off + n].view(shape))
        off += n
    return out, off


def critic_forward(params, x, a):
    w1, b1, w2, b2, w3, b3 = params
    h1 = F.relu(F.linear(torch.cat([x, a], 1), w1, b1))
    h2 = F.relu(F.linear(h1, w2, b2))
    return F.linear(h2, w3, b3)


def actor_head(params, x):
    w1, b1, w2, b2, wm, bm, ws, bs = params
    h = F.relu(F.linear(F.relu(F.linear(x, w1, b1)), w2, b2))
    return F.linear(h, wm, bm), F.linear(h, ws, bs)


def head_forward(mean, raw, eps, scale, bias):
    """(action, log_prob [B, 1], squashed mean, log_std) exactly as Actor.forward / get_action evaluate them."""
    log_std = torch.tanh(raw)
    log_std = LOG_STD_MIN + 0.5 * (LOG_STD_MAX - LOG_STD_MIN) * (log_std + 1)
    std = log_std.exp()
    x_t = mean + eps * std
    y_t = torch.tanh(x_t)
    action = y_t * scale + bias
    log_prob = -((x_t - mean) ** 2) / (2 * std ** 2) - std.log() - _C
    log_prob = log_prob - torch.log(scale * (1 - y_t.pow(2)) + 1e-6)
    return action, log_prob.sum(1, keepdim=True), torch.tanh(mean) * scale + bias, log_std


def head_backward(mean, raw, eps, scale, g, dpi):
    """(d mean, d raw_logstd) of g * log_pi + <dpi, action> per row (g [B, 1]), autograd's chain restated."""
    t = torch.tanh(raw)
    sd = (-5.0 + 3.5 * (t + 1)).exp()
    x = mean + eps * sd
    y = torch.tanh(x)
    u = x - mean
    nn_ = -(u * u)
    den = 2 * (sd * sd)
    qv = nn_ / den
    w2 = scale * (1 - y * y) + 1e-6
    g = g.expand_as(mean)
    g_w = -g / w2
    g_ysq = -(g_w * scale)
    g_y = dpi * scale + g_ysq * (2 * y)
    g_nn = g / den
    g_den = -(g * (qv / den))
    g_u = -g_nn * (2 * u)
    g_std = (g_den * 2) * (2 * sd)
    g_x = g_y * (1 - y * y) + g_u
    dm = g_x - g_u
    g_std = (g_x * eps + g_std) + (-g / sd)
    draw = ((g_std * sd) * 3.5) * (1 - t * t)
    return dm, draw


def critic_loss(q1, q2, q1t, q2t, next_logpi, rewards, dones, alpha, gamma):
    """(y, qf1_loss, qf2_loss, dq1, dq2) of sac_continuous_action.py:257-268 (q* [B])."""
    m = torch.min(q1t, q2t) - alpha * next_logpi
    y = rewards + (1 - dones) * gamma * m
    B = q1.numel()
    return y, F.mse_loss(q1, y), F.mse_loss(q2, y), (2.0 / B) * (q1 - y), (2.0 / B) * (q2 - y)


def actor_loss(log_pi, q1, q2, alpha):
    return ((alpha * log_pi) - torch.min(q1, q2)).mean()


def temperature_step(log_alpha, m, v, step, log_pi, target_entropy, lr, beta1=0.9, beta2=0.999, eps=1e-8):
    """One autotune step (sac_continuous_action.py:289-297) on detached tensors; returns (alpha_loss, log_alpha, m, v)."""
    la = log_alpha.clone().requires_grad_(True)
    loss = (-la.exp() * (log_pi + target_entropy)).mean()
    loss.backward()
    opt = torch.optim.Adam([la], lr=lr, betas=(beta1, beta2), eps=eps)
    opt.state[la] = {"step": torch.tensor(float(step - 1)), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
    opt.step()
    st = opt.state[la]
    return loss.detach(), la.detach(), st["exp_avg"], st["exp_avg_sq"]


class _Q(nn.Module):
    def __init__(self, obs_dim, act_dim):
        super().__init__()
        self.fc1, self.fc2, self.fc3 = nn.Linear(obs_dim + act_dim, 256), nn.Linear(256, 256), nn.Linear(256, 1)

    def forward(self, x, a):
        x = torch.cat([x, a], 1)
        return self.fc3(F.relu(self.fc2(F.relu(self.fc1(x)))))


class _Actor(nn.Module):
    def __init__(self, obs_dim, act_dim, scale, bias):
        super().__init__()
        self.fc1, self.fc2 = nn.Linear(obs_dim, 256), nn.Linear(256, 256)
        self.fc_mean, self.fc_logstd = nn.Linear(256, act_dim), nn.Linear(256, act_dim)
        self.register_buffer("action_scale", scale.clone())
        self.register_buffer("action_bias", bias.clone())

    def get_action(self, x, eps):
        h = F.relu(self.fc2(F.relu(self.fc1(x))))
        a, lp, m, _ = head_forward(self.fc_mean(h), self.fc_logstd(h), eps, self.action_scale, self.action_bias)
        return a, lp, m


class EagerSAC:
    """The reference's update (sac_continuous_action.py:255-304) in eager PyTorch on ``device``: initialised from the
    flat parameters of an actor, the twin critics and the twin targets."""

    def __init__(self, actor_flat, q_flat, qt_flat, obs_dim, act_dim, scale, bias, device, autotune=True, alpha=0.2,
                 q_lr=1e-3, policy_lr=3e-4, gamma=0.99, tau=0.005, policy_frequency=2, target_network_frequency=1):
        self.actor = _Actor(obs_dim, act_dim, scale, bias).to(device)
        self.qs = [_Q(obs_dim, act_dim).to(device) for _ in range(4)]
        with torch.no_grad():
            torch.nn.utils.vector_to_parameters(actor_flat.to(device), self.actor.parameters())
            n = sum(p.numel() for p in self.qs[0].parameters())
            for i, (flat, k) in enumerate(((q_flat, 0), (q_flat, 1), (qt_flat, 0), (qt_flat, 1))):
                torch.nn.utils.vector_to_parameters(flat[k * n:(k + 1) * n].to(device), self.qs[i].parameters())
        self.qf1, self.qf2, self.qf1_target, self.qf2_target = self.qs
        self.q_optimizer = torch.optim.Adam(list(self.qf1.parameters()) + list(self.qf2.parameters()), lr=q_lr)
        self.actor_optimizer = torch.optim.Adam(list(self.actor.parameters()), lr=policy_lr)
        self.autotune, self.gamma, self.tau = autotune, gamma, tau
        self.pf, self.tnf = policy_frequency, target_network_frequency
        self.target_entropy = -float(act_dim)
        self.log_alpha = torch.zeros(1, requires_grad=True, device=device)
        self.alpha = self.log_alpha.exp().item() if autotune else alpha
        self.a_optimizer = torch.optim.Adam([self.log_alpha], lr=q_lr)
        self.stats = {}

    def update(self, global_step, obs, actions, next_obs, rewards, dones, noise):
        with torch.no_grad():
            a2, lp2, _ = self.actor.get_action(next_obs, noise(actions.shape))
            q1t, q2t = self.qf1_target(next_obs, a2), self.qf2_target(next_obs, a2)
            m = torch.min(q1t, q2t) - self.alpha * lp2
            y = rewards.flatten() + (1 - dones.flatten()) * self.gamma * m.view(-1)
        q1 = self.qf1(obs, actions).view(-1)
        q2 = self.qf2(obs, actions).view(-1)
        l1, l2 = F.mse_loss(q1, y), F.mse_loss(q2, y)
        self.q_optimizer.zero_grad()
        (l1 + l2).backward()
        self.q_optimizer.step()
        self.stats.update(qf1_values=q1.mean().item, qf2_values=q2.mean().item, qf1_loss=l1.item, qf2_loss=l2.item)
        if global_step % self.pf == 0:
            for _ in range(self.pf):
                pi, log_pi, _ = self.actor.get_action(obs, noise(actions.shape))
                al = ((self.alpha * log_pi) - torch.min(self.qf1(obs, pi), self.qf2(obs, pi))).mean()
                self.actor_optimizer.zero_grad()
                al.backward()
                self.actor_optimizer.step()
                self.stats["actor_loss"] = al.item
                if self.autotune:
                    with torch.no_grad():
                        _, log_pi, _ = self.actor.get_action(obs, noise(actions.shape))
                    alpha_loss = (-self.log_alpha.exp() * (log_pi + self.target_entropy)).mean()
                    self.a_optimizer.zero_grad()
                    alpha_loss.backward()
                    self.a_optimizer.step()
                    self.alpha = self.log_alpha.exp().item()
                    self.stats["alpha_loss"] = alpha_loss.item
        if global_step % self.tnf == 0:
            for src, dst in ((self.qf1, self.qf1_target), (self.qf2, self.qf2_target)):
                for param, target_param in zip(src.parameters(), dst.parameters()):
                    target_param.data.copy_(self.tau * param.data + (1 - self.tau) * target_param.data)
