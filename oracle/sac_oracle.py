"""Discrete SAC oracle (cleanrl/sac_atari.py).  TEST INFRASTRUCTURE ONLY.

* ``critic_loss`` / ``actor_loss``: numpy fp32 restatements of the fused kernels (the soft-Q target, both critic losses
  and their head gradients; the actor loss, its logit gradient, the temperature loss and the one-element Adam step of
  log_alpha), in the reference's operation order.
* ``torch_critic`` / ``torch_actor``: the reference's own expressions (sac_atari.py:274-314) on head outputs, for autograd.
* ``TorchSAC``: the whole update as the reference runs it (cuDNN trunks, torch Adam) -- the eager arm of bench_sac.py.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32


def policy(logits):
    """(log_softmax, probs) of logits [n, A] in fp32."""
    x = np.asarray(logits, dtype=f32)
    t = x - x.max(1, keepdims=True)
    e = np.exp(t)
    s = e.sum(1, keepdims=True, dtype=f32)
    return (t - np.log(s)).astype(f32), (e / s).astype(f32)


def critic_loss(next_logits, q1t, q2t, q1, q2, actions, rewards, dones, gamma, alpha):
    """Returns (stats [qf1_values, qf2_values, qf1_loss, qf2_loss], y [B], dq1 [B, A], dq2 [B, A])."""
    lp, p = policy(next_logits)
    alpha, gamma = f32(alpha), f32(gamma)
    m = (p * (np.minimum(np.asarray(q1t, f32), np.asarray(q2t, f32)) - alpha * lp)).sum(1, dtype=f32)
    r = np.asarray(rewards, f32).reshape(-1)
    d = np.asarray(dones, f32).reshape(-1)
    y = (r + ((f32(1) - d) * gamma) * m).astype(f32)
    a = np.asarray(actions).reshape(-1).astype(np.int64)
    B = y.size
    i = np.arange(B)
    q1a, q2a = np.asarray(q1, f32)[i, a], np.asarray(q2, f32)[i, a]
    d1, d2 = q1a - y, q2a - y
    dq1 = np.zeros_like(np.asarray(q1, f32))
    dq2 = np.zeros_like(dq1)
    two_b = f32(2.0 / B)
    dq1[i, a] = two_b * d1
    dq2[i, a] = two_b * d2
    stats = np.array([q1a.mean(dtype=f32), q2a.mean(dtype=f32), (d1 * d1).mean(dtype=f32), (d2 * d2).mean(dtype=f32)], f32)
    return stats, y, dq1, dq2


def adam_one(p, g, m, v, step, lr, eps=1e-4, beta1=0.9, beta2=0.999):
    """torch.optim.Adam (single tensor) on fp32 scalars; the step scalars in double as torch computes them."""
    bc1 = 1.0 - beta1 ** step
    bc2 = 1.0 - beta2 ** step
    m = f32(m + f32(1 - beta1) * (f32(g) - m))
    v = f32(f32(v * f32(beta2)) + f32(f32(1 - beta2) * g) * f32(g))
    denom = f32(f32(np.sqrt(v) / f32(np.sqrt(bc2))) + f32(eps))
    p = f32(p + f32(-lr / bc1) * f32(m / denom))
    return p, m, v


def actor_loss(logits, q1, q2, alpha, target_entropy=None, log_alpha=None, m=0.0, v=0.0, step=1, lr=3e-4):
    """Returns (actor_loss, dlogits [B, A], alpha_loss, d log_alpha, (log_alpha, m, v) after the Adam step, new alpha).
    Without ``log_alpha`` (no autotune) the temperature outputs are None."""
    lp, p = policy(logits)
    B, A = p.shape
    alpha = f32(alpha)
    f = (alpha * lp - np.minimum(np.asarray(q1, f32), np.asarray(q2, f32))).astype(f32)
    loss = f32((p * f).sum(dtype=f32) / f32(B * A))
    dot = (p * f).sum(1, keepdims=True, dtype=f32)
    dl = (p * (f - dot) * f32(1.0 / (B * A))).astype(f32)
    if log_alpha is None:
        return loss, dl, None, None, None, None
    la = f32(log_alpha)
    ea = f32(np.exp(la))
    t = (lp + f32(target_entropy)).astype(f32)
    a_loss = f32((p * (-ea * t)).sum(dtype=f32) / f32(B * A))
    g = f32(-(f32(1.0 / (B * A)) * p * t).sum(dtype=f32) * ea)
    la2, m2, v2 = adam_one(la, g, f32(m), f32(v), step, lr)
    return loss, dl, a_loss, g, (la2, m2, v2), f32(np.exp(la2))


def target_entropy(A, scale=0.89):
    import torch
    return float(-scale * torch.log(1 / torch.tensor(A)))


def torch_critic(next_logits, q1t, q2t, q1_values, q2_values, actions, rewards, dones, gamma, alpha):
    """sac_atari.py:274-290 on head outputs; q*_values may require grad.  Returns (qf1_loss, qf2_loss, y, q1a, q2a)."""
    import torch
    import torch.nn.functional as F
    from torch.distributions.categorical import Categorical
    with torch.no_grad():
        dist = Categorical(logits=next_logits)
        probs, log_pi = dist.probs, F.log_softmax(next_logits, dim=1)
        m = (probs * (torch.min(q1t, q2t) - alpha * log_pi)).sum(dim=1)
        y = rewards.flatten() + (1 - dones.flatten()) * gamma * m
    a = actions.long().view(-1, 1)
    q1a = q1_values.gather(1, a).view(-1)
    q2a = q2_values.gather(1, a).view(-1)
    return F.mse_loss(q1a, y), F.mse_loss(q2a, y), y, q1a, q2a


def torch_actor(logits, q1, q2, alpha, log_alpha=None, target_entropy=None):
    """sac_atari.py:293-310 on head outputs; logits and log_alpha may require grad.  Returns (actor_loss, alpha_loss)."""
    import torch.nn.functional as F
    from torch.distributions.categorical import Categorical
    probs = Categorical(logits=logits).probs
    log_pi = F.log_softmax(logits, dim=1)
    loss = (probs * ((alpha * log_pi) - (q1.min(q2)))).mean()
    a_loss = None
    if log_alpha is not None:
        a_loss = (probs.detach() * (-log_alpha.exp() * (log_pi + target_entropy).detach())).mean()
    return loss, a_loss


class TorchSAC:
    """The reference's update (sac_atari.py:271-314) in eager PyTorch on the reference-shaped networks' ``conv``/``fc1``/
    head modules: cuDNN trunks, torch Adam (eps 1e-4), ``alpha`` read back with ``.item()`` every update."""

    def __init__(self, actor, qf1, qf2, qf1_target, qf2_target, A, q_lr=3e-4, policy_lr=3e-4, autotune=True, alpha=0.2):
        import torch
        self.nets = (actor, qf1, qf2, qf1_target, qf2_target)
        dev = next(actor.parameters()).device
        self.q_opt = torch.optim.Adam(list(qf1.parameters()) + list(qf2.parameters()), lr=q_lr, eps=1e-4)
        self.a_opt = torch.optim.Adam(list(actor.parameters()), lr=policy_lr, eps=1e-4)
        self.autotune = autotune
        self.te = target_entropy(A)
        self.log_alpha = torch.zeros(1, requires_grad=True, device=dev)
        self.alpha = self.log_alpha.exp().item() if autotune else alpha
        self.t_opt = torch.optim.Adam([self.log_alpha], lr=q_lr, eps=1e-4)

    @staticmethod
    def fwd(net, x):
        import torch.nn.functional as F
        h = F.relu(net.conv(x))
        h = F.relu(net.fc1(h))
        return (net.fc_q if hasattr(net, "fc_q") else net.fc_logits)(h)

    def update(self, obs, next_obs, actions, rewards, dones, gamma=0.99):
        import torch
        actor, qf1, qf2, qf1_target, qf2_target = self.nets
        obs, next_obs = obs.float() / 255.0, next_obs.float() / 255.0
        with torch.no_grad():
            nl = self.fwd(actor, next_obs)
            torch.distributions.Categorical(logits=nl).sample()
            q1t, q2t = self.fwd(qf1_target, next_obs), self.fwd(qf2_target, next_obs)
        l1, l2, _, _, _ = torch_critic(nl, q1t, q2t, self.fwd(qf1, obs), self.fwd(qf2, obs), actions, rewards, dones, gamma,
                                       self.alpha)
        self.q_opt.zero_grad()
        (l1 + l2).backward()
        self.q_opt.step()
        lo = self.fwd(actor, obs)
        torch.distributions.Categorical(logits=lo).sample()
        with torch.no_grad():
            q1, q2 = self.fwd(qf1, obs), self.fwd(qf2, obs)
        loss, a_loss = torch_actor(lo, q1, q2, self.alpha, self.log_alpha if self.autotune else None, self.te)
        self.a_opt.zero_grad()
        loss.backward()
        self.a_opt.step()
        if self.autotune:
            self.t_opt.zero_grad()
            a_loss.backward()
            self.t_opt.step()
            self.alpha = self.log_alpha.exp().item()
