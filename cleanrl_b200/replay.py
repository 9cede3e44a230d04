"""Device-resident replay ring for the DQN path (config 5).

Replaces the host-side numpy ``ReplayBuffer`` of cleanrl_utils/buffers.py:250-430 as dqn_atari.py uses it
(``optimize_memory_usage=True``: one uint8 frame ring, ``next_obs`` = slot ``(i+1) % size``, buffers.py:359-362,
:402).  Differences in mechanism, not in semantics:

* the ring lives in HBM (1 M x 28 224 B = 28 GB fits an 80 GB H100); ``add`` uploads the two 28 KB frames;
* ``sample`` draws the SAME index stream from numpy's global RNG (buffers.py:390-399: ``randint(1, size) + pos``
  when full, ``randint(0, pos)`` otherwise, then ``randint(0, n_envs)``) but returns ROW INDICES into the ring:
  the network kernels gather the frames themselves (no 2 x 231 MB host fancy-index + H2D per batch of 8192).
"""
from __future__ import annotations

import numpy as np
import torch


class DeviceReplayRing:
    def __init__(self, buffer_size, obs_shape, n_envs, device):
        self.buffer_size = max(int(buffer_size) // int(n_envs), 1)     # buffers.py:300 (size per env)
        self.n_envs = int(n_envs)
        self.device = device
        self.obs_shape = tuple(obs_shape)
        self.observations = torch.zeros((self.buffer_size, self.n_envs) + self.obs_shape, dtype=torch.uint8, device=device)
        self.actions = torch.zeros((self.buffer_size, self.n_envs), dtype=torch.int64, device=device)
        self.rewards = torch.zeros((self.buffer_size, self.n_envs), dtype=torch.float32, device=device)
        self.dones = torch.zeros((self.buffer_size, self.n_envs), dtype=torch.float32, device=device)
        self.pos = 0
        self.full = False

    def size(self):
        return self.buffer_size if self.full else self.pos

    @property
    def frames(self):
        """The ring as a flat list of frames [size * n_envs, 4, 84, 84] (row = slot * n_envs + env)."""
        return self.observations.view((self.buffer_size * self.n_envs,) + self.obs_shape)

    def add(self, obs, next_obs, action, reward, done, infos=None):
        """buffers.py:339-375."""
        dev = self.device
        self.observations[self.pos].copy_(torch.from_numpy(np.ascontiguousarray(obs)).to(torch.uint8), non_blocking=False)
        self.observations[(self.pos + 1) % self.buffer_size].copy_(
            torch.from_numpy(np.ascontiguousarray(next_obs)).to(torch.uint8), non_blocking=False)
        self.actions[self.pos].copy_(torch.as_tensor(np.asarray(action).reshape(self.n_envs), dtype=torch.int64))
        self.rewards[self.pos].copy_(torch.as_tensor(np.asarray(reward, dtype=np.float32).reshape(self.n_envs)))
        self.dones[self.pos].copy_(torch.as_tensor(np.asarray(done, dtype=np.float32).reshape(self.n_envs)))
        self.pos += 1
        if self.pos == self.buffer_size:
            self.full = True
            self.pos = 0

    def sample_indices(self, batch_size):
        """Host index draw, bit-identical to buffers.py:390-399 (numpy global RNG)."""
        if self.full:
            batch_inds = (np.random.randint(1, self.buffer_size, size=batch_size) + self.pos) % self.buffer_size
        else:
            batch_inds = np.random.randint(0, self.pos, size=batch_size)
        env_indices = np.random.randint(0, high=self.n_envs, size=(len(batch_inds),))
        return batch_inds, env_indices

    def sample(self, batch_size):
        """Returns dict(rows, next_rows: int64 device row indices into ``frames``; actions [B], rewards [B], dones [B])."""
        bi, ei = self.sample_indices(batch_size)
        rows = torch.from_numpy(bi * self.n_envs + ei).to(self.device)
        next_rows = torch.from_numpy(((bi + 1) % self.buffer_size) * self.n_envs + ei).to(self.device)
        return {"rows": rows, "next_rows": next_rows,
                "actions": self.actions.view(-1)[rows], "rewards": self.rewards.view(-1)[rows],
                "dones": self.dones.view(-1)[rows], "batch_inds": bi, "env_indices": ei}
