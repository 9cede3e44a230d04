"""Device-resident replay ring for the DQN path (config 5).

Replaces the host-side numpy ``ReplayBuffer`` of cleanrl_utils/buffers.py:250-430 as dqn_atari.py uses it
(``optimize_memory_usage=True``: one uint8 frame ring, ``next_obs`` = slot ``(i+1) % size``, buffers.py:359-362,
:402).  Differences in mechanism, not in semantics:

* the ring lives in HBM (1 M x 28 224 B = 28 GB fits an 80 GB H100); ``add`` uploads the two 28 KB frames;
* ``sample`` draws the SAME index stream from numpy's global RNG (buffers.py:390-399: ``randint(1, size) + pos``
  when full, ``randint(0, pos)`` otherwise, then ``randint(0, n_envs)``) but returns ROW INDICES into the ring:
  the network kernels gather the frames themselves (no 2 x 231 MB host fancy-index + H2D per batch of 8192).

``optimize_memory_usage=False`` is the layout sac_atari.py uses (buffers.py:301-303, 358-363, 217-225, 397-415): a
second device ring ``next_observations`` written from ``real_next_obs``, ``randint(0, size if full else pos)`` then the
env index, and ``sample`` rows that index both ``frames`` and ``next_frames``.  Both uint8 rings live in HBM (56.4 GB at
``buffer_size = 1e6``); a ring that does not fit in free device memory is an error at construction.

``obs_dtype=torch.float32`` with an ``action_shape`` is the layout sac_continuous_action.py uses (float32 observations,
float32 [act_dim] actions, ``optimize_memory_usage=False``): every (slot, env) is one packed row
``[obs | next_obs | action | reward | done]`` of one device tensor, so ``add`` is one host-to-device copy of a pinned
staging row; ``frames`` / ``next_frames`` / ``action_rows`` / ``reward_rows`` / ``done_rows`` are strided views of it.
"""
from __future__ import annotations

import numpy as np
import torch


class DeviceReplayRing:
    def __init__(self, buffer_size, obs_shape, n_envs, device, optimize_memory_usage=True, obs_dtype=torch.uint8,
                 action_shape=None):
        self.buffer_size = max(int(buffer_size) // int(n_envs), 1)     # buffers.py:300 (size per env)
        self.n_envs = int(n_envs)
        self.device = device
        self.obs_shape = tuple(obs_shape)
        self.optimize_memory_usage = bool(optimize_memory_usage)
        self.packed = None
        if obs_dtype == torch.float32:
            self._init_packed(action_shape)
            return
        if obs_dtype != torch.uint8 or action_shape is not None:
            raise ValueError("DeviceReplayRing: uint8 observations with int64 actions, or float32 observations with an "
                             "action_shape")
        shape = (self.buffer_size, self.n_envs) + self.obs_shape
        if not self.optimize_memory_usage:
            need = 2 * int(np.prod(shape))
            free = torch.cuda.mem_get_info(device)[0] if torch.device(device).type == "cuda" else need
            if need > free:
                raise RuntimeError(f"the replay buffer (observations and next_observations, uint8) needs {need / 1e9:.1f} GB "
                                   f"of device memory, {free / 1e9:.1f} GB are free: lower --buffer-size (it is not "
                                   "spilled to the host)")
        self.observations = torch.zeros(shape, dtype=torch.uint8, device=device)
        self.next_observations = None if self.optimize_memory_usage else torch.zeros(shape, dtype=torch.uint8, device=device)
        self.actions = torch.zeros((self.buffer_size, self.n_envs), dtype=torch.int64, device=device)
        self.rewards = torch.zeros((self.buffer_size, self.n_envs), dtype=torch.float32, device=device)
        self.dones = torch.zeros((self.buffer_size, self.n_envs), dtype=torch.float32, device=device)
        self.pos = 0
        self.full = False

    def _init_packed(self, action_shape):
        if self.optimize_memory_usage or action_shape is None:
            raise ValueError("DeviceReplayRing: float32 observations need optimize_memory_usage=False and an action_shape")
        self.obs_dim = int(np.prod(self.obs_shape))
        self.act_dim = int(np.prod(action_shape))
        self.action_shape = tuple(action_shape)
        od, ad = self.obs_dim, self.act_dim
        self.width = 2 * od + ad + 2
        need = 4 * self.buffer_size * self.n_envs * self.width
        free = torch.cuda.mem_get_info(self.device)[0] if torch.device(self.device).type == "cuda" else need
        if need > free:
            raise RuntimeError(f"the replay buffer needs {need / 1e9:.1f} GB of device memory, {free / 1e9:.1f} GB are "
                               "free: lower --buffer-size (it is not spilled to the host)")
        self.packed = torch.zeros((self.buffer_size, self.n_envs, self.width), dtype=torch.float32, device=self.device)
        rows = self.packed.view(-1, self.width)
        self.frames_view, self.next_frames_view = rows[:, :od], rows[:, od:2 * od]
        self.action_rows, self.reward_rows, self.done_rows = rows[:, 2 * od:2 * od + ad], rows[:, -2], rows[:, -1]
        self.observations = self.packed[..., :od].unflatten(-1, self.obs_shape)
        self.next_observations = self.packed[..., od:2 * od].unflatten(-1, self.obs_shape)
        self.actions = self.packed[..., 2 * od:2 * od + ad].unflatten(-1, self.action_shape)
        self.rewards, self.dones = self.packed[..., -2], self.packed[..., -1]
        pin = torch.cuda.is_available() and torch.device(self.device).type == "cuda"
        self._stage = torch.zeros((self.n_envs, self.width), dtype=torch.float32, pin_memory=pin)
        self._staged = torch.cuda.Event() if pin else None
        self.pos = 0
        self.full = False

    def size(self):
        return self.buffer_size if self.full else self.pos

    @property
    def frames(self):
        """The ring as a flat list of frames [size * n_envs, 4, 84, 84] (row = slot * n_envs + env)."""
        if self.packed is not None:
            return self.frames_view
        return self.observations.view((self.buffer_size * self.n_envs,) + self.obs_shape)

    @property
    def next_frames(self):
        """The frames ``next_rows`` index: ``frames`` itself, or the ``next_observations`` ring."""
        if self.packed is not None:
            return self.next_frames_view
        if self.optimize_memory_usage:
            return self.frames
        return self.next_observations.view((self.buffer_size * self.n_envs,) + self.obs_shape)

    def add(self, obs, next_obs, action, reward, done, infos=None):
        """buffers.py:339-375."""
        if self.packed is not None:
            return self._add_packed(obs, next_obs, action, reward, done)
        self.observations[self.pos].copy_(torch.from_numpy(np.ascontiguousarray(obs)).to(torch.uint8), non_blocking=False)
        nxt = self.observations[(self.pos + 1) % self.buffer_size] if self.optimize_memory_usage else \
            self.next_observations[self.pos]
        nxt.copy_(torch.from_numpy(np.ascontiguousarray(next_obs)).to(torch.uint8), non_blocking=False)
        self.actions[self.pos].copy_(torch.as_tensor(np.asarray(action).reshape(self.n_envs), dtype=torch.int64))
        self.rewards[self.pos].copy_(torch.as_tensor(np.asarray(reward, dtype=np.float32).reshape(self.n_envs)))
        self.dones[self.pos].copy_(torch.as_tensor(np.asarray(done, dtype=np.float32).reshape(self.n_envs)))
        self.pos += 1
        if self.pos == self.buffer_size:
            self.full = True
            self.pos = 0

    def _add_packed(self, obs, next_obs, action, reward, done):
        od, ad, st = self.obs_dim, self.act_dim, self._stage.numpy()
        if self._staged is not None:
            self._staged.synchronize()
        st[:, :od] = np.asarray(obs, dtype=np.float32).reshape(self.n_envs, od)
        st[:, od:2 * od] = np.asarray(next_obs, dtype=np.float32).reshape(self.n_envs, od)
        st[:, 2 * od:2 * od + ad] = np.asarray(action, dtype=np.float32).reshape(self.n_envs, ad)
        st[:, -2] = np.asarray(reward, dtype=np.float32).reshape(self.n_envs)
        st[:, -1] = np.asarray(done, dtype=np.float32).reshape(self.n_envs)
        self.packed[self.pos].copy_(self._stage, non_blocking=True)
        if self._stage.is_pinned():
            self._staged.record()                        # the next add waits for this copy before it rewrites the row
        self.pos += 1
        if self.pos == self.buffer_size:
            self.full = True
            self.pos = 0

    def sample_indices(self, batch_size):
        """Host index draw, bit-identical to buffers.py:390-399 / 217-225 (numpy global RNG)."""
        if not self.optimize_memory_usage:
            batch_inds = np.random.randint(0, self.buffer_size if self.full else self.pos, size=batch_size)
        elif self.full:
            batch_inds = (np.random.randint(1, self.buffer_size, size=batch_size) + self.pos) % self.buffer_size
        else:
            batch_inds = np.random.randint(0, self.pos, size=batch_size)
        env_indices = np.random.randint(0, high=self.n_envs, size=(len(batch_inds),))
        return batch_inds, env_indices

    def sample(self, batch_size):
        """Returns dict(rows: int64 device row indices into ``frames``, next_rows: into ``next_frames``; actions [B],
        rewards [B], dones [B])."""
        bi, ei = self.sample_indices(batch_size)
        rows = torch.from_numpy(bi * self.n_envs + ei).to(self.device)
        if self.optimize_memory_usage:
            next_rows = torch.from_numpy(((bi + 1) % self.buffer_size) * self.n_envs + ei).to(self.device)
        else:
            next_rows = rows
        if self.packed is not None:      # the kernels gather the sampled rows of frames / next_frames / *_rows
            return {"rows": rows, "next_rows": rows, "batch_inds": bi, "env_indices": ei}
        return {"rows": rows, "next_rows": next_rows,
                "actions": self.actions.view(-1)[rows], "rewards": self.rewards.view(-1)[rows],
                "dones": self.dones.view(-1)[rows], "batch_inds": bi, "env_indices": ei}
