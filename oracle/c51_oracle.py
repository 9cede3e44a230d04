"""C51 (cleanrl/c51_atari.py) restated twice, for the tests and the benchmark.  TEST INFRASTRUCTURE ONLY.

* numpy float32 oracle of ``QNetwork.get_action`` (c51_atari.py:131-138) and of the update's target projection,
  clamped cross-entropy and its gradient wrt the head logits (c51_atari.py:233-253, plus what ``loss.backward()``
  computes for the head);
* ``torch_update_loss``: the reference's own torch expressions, including its per-row ``index_add_`` loop, on any
  device -- the eager baseline of bench_c51.py and the autograd check of the oracle.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32


def softmax(x):
    """torch.softmax(x, dim=-1) in float32."""
    x = np.asarray(x, dtype=f32)
    e = np.exp(x - x.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def get_action(logits, atoms, action=None):
    """c51_atari.py:131-138 from the head logits [n, A * n_atoms]: (action [n], pmf of the action [n, n_atoms], q [n, A])."""
    atoms = np.asarray(atoms, dtype=f32)
    n, W = logits.shape
    Z = atoms.size
    pmfs = softmax(np.asarray(logits, dtype=f32).reshape(n, W // Z, Z))
    q = (pmfs * atoms).sum(2, dtype=f32)
    if action is None:
        action = q.argmax(1)
    action = np.asarray(action).reshape(-1).astype(np.int64)
    return action, pmfs[np.arange(n), action], q


def project(next_pmfs, rewards, dones, atoms, gamma, v_min, v_max):
    """Categorical projection of r + gamma * atoms * (1 - d) onto the atoms (c51_atari.py:235-250): target_pmfs [B, Z].
    np.add.at accumulates in index order like CPU index_add_: every d_m_l of a row, then every d_m_u."""
    atoms = np.asarray(atoms, dtype=f32)
    Z = atoms.size
    r = np.asarray(rewards, dtype=f32).reshape(-1, 1)
    d = np.asarray(dones, dtype=f32).reshape(-1, 1)
    next_atoms = r + (f32(gamma) * atoms)[None, :] * (f32(1) - d)
    tz = np.clip(next_atoms, f32(v_min), f32(v_max))
    delta_z = atoms[1] - atoms[0]
    b = (tz - f32(v_min)) / delta_z
    l = np.clip(np.floor(b), f32(0), f32(Z - 1))
    u = np.clip(np.ceil(b), f32(0), f32(Z - 1))
    d_m_l = (u + (l == u).astype(f32) - b) * next_pmfs
    d_m_u = (b - l) * next_pmfs
    target = np.zeros_like(next_pmfs, dtype=f32)
    for i in range(target.shape[0]):
        np.add.at(target[i], l[i].astype(np.int64), d_m_l[i])
        np.add.at(target[i], u[i].astype(np.int64), d_m_u[i])
    return target


def loss_and_grad(logits, next_logits, atoms, actions, rewards, dones, gamma, v_min, v_max):
    """(loss, q_values, dlogits [B, A * Z], target_pmfs [B, Z]) of one update (c51_atari.py:233-258).  q_values is the
    logged mean of (old_pmfs * atoms).sum(1) over the unclamped pmfs; dlogits is autograd's gradient (clamp passes
    the gradient on its closed interval, softmax backward y * (g - sum(g * y)), 1/B of the mean)."""
    atoms = np.asarray(atoms, dtype=f32)
    B, W = logits.shape
    Z = atoms.size
    _, next_pmfs, _ = get_action(next_logits, atoms)
    target = project(next_pmfs, rewards, dones, atoms, gamma, v_min, v_max)
    actions = np.asarray(actions).reshape(-1).astype(np.int64)
    _, old, _ = get_action(logits, atoms, actions)
    lo, hi = f32(1e-5), f32(1 - 1e-5)
    pc = np.clip(old, lo, hi)
    loss = (-(target * np.log(pc)).sum(-1, dtype=f32)).mean(dtype=f32)
    q_values = (old * atoms).sum(1, dtype=f32).mean(dtype=f32)
    g0 = f32(1) / f32(B)
    g = np.where((old >= lo) & (old <= hi), ((-g0) * target) / pc, f32(0)).astype(f32)
    dot = (g * old).sum(-1, keepdims=True, dtype=f32)
    dl = np.zeros((B, W // Z, Z), dtype=f32)
    dl[np.arange(B), actions] = old * (g - dot)
    return f32(loss), f32(q_values), dl.reshape(B, W), target


def torch_update_loss(logits, next_logits, atoms, actions, rewards, dones, gamma, v_min, v_max, n_atoms):
    """The reference's update expressions (c51_atari.py:131-138, 233-253) on head logits, with its Python loop of
    2 * B index_add_ calls.  ``logits`` may require grad: returns (loss, old_pmfs, target_pmfs)."""
    import torch

    def pmf_of(lg, action=None):
        n = lg.shape[0]
        pmfs = torch.softmax(lg.view(n, -1, n_atoms), dim=2)
        q_values = (pmfs * atoms).sum(2)
        if action is None:
            action = torch.argmax(q_values, 1)
        return action, pmfs[torch.arange(n), action]

    with torch.no_grad():
        _, next_pmfs = pmf_of(next_logits)
        next_atoms = rewards.view(-1, 1) + gamma * atoms * (1 - dones.view(-1, 1))
        delta_z = atoms[1] - atoms[0]
        tz = next_atoms.clamp(v_min, v_max)
        b = (tz - v_min) / delta_z
        l = b.floor().clamp(0, n_atoms - 1)
        u = b.ceil().clamp(0, n_atoms - 1)
        d_m_l = (u + (l == u).float() - b) * next_pmfs
        d_m_u = (b - l) * next_pmfs
        target_pmfs = torch.zeros_like(next_pmfs)
        for i in range(target_pmfs.size(0)):
            target_pmfs[i].index_add_(0, l[i].long(), d_m_l[i])
            target_pmfs[i].index_add_(0, u[i].long(), d_m_u[i])
    _, old_pmfs = pmf_of(logits, actions.flatten())
    loss = (-(target_pmfs * old_pmfs.clamp(min=1e-5, max=1 - 1e-5).log()).sum(-1)).mean()
    return loss, old_pmfs, target_pmfs
