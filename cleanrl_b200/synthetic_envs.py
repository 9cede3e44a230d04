"""Synthetic vector environments (host side, numpy).

The image this framework is built and measured in has no envpool / ALE /
gymnasium and no network, so real Breakout-v5 cannot run (SURVEY.md section 8d).
These classes supply deterministic, seeded stand-ins with the exact API surface
the reference loops touch:

* ``SyntheticAtariVec`` -- the gym-0.23 / envpool flavour used by
  ``ppo_atari_envpool.py`` (reference: cleanrl/ppo_atari_envpool.py:185-196,
  :237-247): ``reset() -> obs``, ``step(a) -> (obs, reward, done, info)`` with
  ``info = {"reward", "terminated", "lives"}``.
* ``SyntheticGymnasiumVec`` -- the gymnasium-0.29 flavour used by ``ppo.py`` /
  ``ppo_atari_multigpu.py`` / ``ppo_continuous_action.py``
  (reference: cleanrl/ppo.py:162-164,181,205-215): ``reset(seed=) -> (obs, info)``,
  ``step(a) -> (obs, reward, terminated, truncated, infos)`` with
  ``infos["final_info"]`` carrying ``{"episode": {"r", "l"}}``.

Two observation modes:

``fresh``  every env picks its next frame from a pool as a function of its own
           state and the action it received, so a wrong action changes every
           later observation (used for parity runs).
``pool``   whole pre-generated pinned batches are handed out round-robin at
           ~zero host cost (used for throughput runs; data = "synthetic").
``stack``  (Atari only) frame-stacked like envpool's ``stack_num=4`` observation
           (cleanrl/ppo_atari_envpool.py:185-196): planes 0..2 of an env's
           observation are planes 1..3 of its previous one, a done env comes back
           with four fresh planes.  Observations are strided zero-copy windows into
           one pinned frame ring (also ~zero host cost).

The environments own their ``np.random.Generator`` and never touch numpy's
global RNG (that one drives the minibatch shuffle, cleanrl/ppo.py:155,245).
"""
from __future__ import annotations

import numpy as np


class Discrete:
    """Minimal stand-in for gym.spaces.Discrete."""

    def __init__(self, n):
        self.n = int(n)
        self.shape = ()
        self.dtype = np.int64
        self._rng = np.random.default_rng(0)

    def seed(self, seed=None):
        self._rng = np.random.default_rng(seed)

    def sample(self):
        return int(self._rng.integers(0, self.n))

    def __repr__(self):
        return f"Discrete({self.n})"


class Box:
    """Minimal stand-in for gym.spaces.Box."""

    def __init__(self, low, high, shape, dtype):
        self.low = np.full(shape, low, dtype=dtype)
        self.high = np.full(shape, high, dtype=dtype)
        self.shape = tuple(shape)
        self.dtype = np.dtype(dtype)
        self._rng = np.random.default_rng(0)

    def seed(self, seed=None):
        self._rng = np.random.default_rng(seed)

    def sample(self):
        """Uniform in [low, high] from the space's own generator (bounded spaces only)."""
        if not (np.all(np.isfinite(self.low)) and np.all(np.isfinite(self.high))):
            raise ValueError("Box.sample: only bounded boxes can be sampled")
        return self._rng.uniform(self.low, self.high).astype(self.dtype)

    def __repr__(self):
        return f"Box({self.shape}, {self.dtype})"


def _alloc_host(shape, dtype, pinned):
    """Host buffer, page-locked when torch+CUDA is usable so H2D copies are async."""
    if pinned:
        import torch

        if torch.cuda.is_available():
            t = torch.empty(shape, dtype=getattr(torch, np.dtype(dtype).name), pin_memory=True)
            return t.numpy()
    return np.empty(shape, dtype=dtype)


class SyntheticAtariVec:
    """Breakout-shaped vector env: uint8 obs [N,4,84,84], Discrete(4) actions."""

    def __init__(self, num_envs, seed=1, mode="fresh", n_actions=4, obs_shape=(4, 84, 84),
                 pool=32, p_done=0.02, pinned=False):
        assert mode in ("fresh", "pool", "stack")
        self.num_envs = int(num_envs)
        self.mode = mode
        self.observation_space = Box(0, 255, obs_shape, np.uint8)
        self.action_space = Discrete(n_actions)
        self.p_done = float(p_done)
        self._rng = np.random.default_rng(seed)
        self._t = 0
        if mode == "fresh":
            self._frames = self._rng.integers(0, 256, size=(pool,) + tuple(obs_shape), dtype=np.uint8)
            self._idx = np.zeros(self.num_envs, dtype=np.int64)
            self._obs = _alloc_host((self.num_envs,) + tuple(obs_shape), np.uint8, pinned)
        elif mode == "stack":
            # frame ring [N, P+C-1, H, W]: the observation at time t is the window ring[:, w:w+C] with w = t mod P; planes
            # P..P+C-2 duplicate planes 0..C-2 so that the window after w = P-1 (w = 0) is again a shift by one plane
            C, H, W = obs_shape
            self._P = P = max(int(pool), 2 * C)
            self._ring = _alloc_host((self.num_envs, P + C - 1, H, W), np.uint8, pinned)
            self._bank = self._rng.integers(0, 256, size=(64, H, W), dtype=np.uint8)       # fresh planes for resets
            for q in range(P):
                self._ring[:, q] = self._rng.integers(0, 256, size=(self.num_envs, H, W), dtype=np.uint8)
            self._ring[:, P:] = self._ring[:, :C - 1]
        else:
            pool = min(int(pool), 8)
            self._batches = _alloc_host((pool, self.num_envs) + tuple(obs_shape), np.uint8, pinned)
            # fill in chunks; 29 MB per batch at N=1024
            for b in range(pool):
                self._batches[b] = self._rng.integers(
                    0, 256, size=(self.num_envs,) + tuple(obs_shape), dtype=np.uint8)
        self._lives = np.full(self.num_envs, 5, dtype=np.int32)

    # -- gym 0.23 API -------------------------------------------------------
    def reset(self, **kwargs):
        self._t = 0
        if self.mode == "fresh":
            self._idx = self._rng.integers(0, len(self._frames), size=self.num_envs)
            np.take(self._frames, self._idx, axis=0, out=self._obs)
            return self._obs
        if self.mode == "stack":
            return self._ring[:, 0:self.observation_space.shape[0]]
        return self._batches[0]

    def _step_stack(self, action):
        """``stack`` mode: same reward / done / lives model as below with the per-step randomness drawn in blocks of 64
        steps (a throughput env: its host cost should be a handful of numpy calls)."""
        n, C, P = self.num_envs, self.observation_space.shape[0], self._P
        j = self._t % 64
        if j == 0:
            self._blk_raw = self._rng.integers(0, 3, size=(64, n)).astype(np.float32)
            self._blk_done = self._rng.random((64, n)) < self.p_done
        self._t += 1
        raw = self._blk_raw[j] * (np.asarray(action).reshape(n) != 0)
        reward = np.sign(raw)
        done = self._blk_done[j]
        lives = self._lives - done
        game_over = lives <= 0
        info = {"reward": raw, "terminated": game_over.astype(np.int32), "lives": lives}
        self._lives = np.where(game_over, 5, lives).astype(np.int32)
        w = self._t % P
        idx = np.flatnonzero(done)
        if len(idx):
            # a done env returns a reset observation: the C-1 planes it would share with its previous observation get
            # fresh content (and so do their wrap-around duplicates)
            # (one contiguous copy of C-1 consecutive bank planes per reset env: numpy's fancy assignment is 5x slower)
            ring, bank = self._ring, self._bank
            starts = self._rng.integers(0, len(bank) - (C - 1), size=len(idx))
            wrap = w < C - 1 or w + C - 2 >= P
            for i, r in zip(idx.tolist(), starts.tolist()):
                ring[i, w:w + C - 1] = bank[r:r + C - 1]
                if wrap:
                    for jj in range(C - 1):
                        q = w + jj
                        if q < C - 1:
                            ring[i, q + P] = bank[r + jj]
                        elif q >= P:
                            ring[i, q - P] = bank[r + jj]
        return self._ring[:, w:w + C], reward, done, info

    def step(self, action):
        if self.mode == "stack":
            return self._step_stack(action)
        action = np.asarray(action).reshape(self.num_envs).astype(np.int64)
        self._t += 1
        n = self.num_envs
        raw = self._rng.integers(0, 3, size=n).astype(np.float32)  # raw game score 0,1,2
        raw *= (action != 0)                                           # NOOP never scores
        reward = np.sign(raw).astype(np.float32)                       # reward_clip=True
        done = self._rng.random(n) < self.p_done
        lost_life = done
        self._lives = np.where(lost_life, self._lives - 1, self._lives).astype(np.int32)
        game_over = self._lives <= 0
        info = {
            "reward": raw,
            "terminated": game_over.astype(np.int32),
            "lives": self._lives.copy(),
        }
        self._lives = np.where(game_over, 5, self._lives).astype(np.int32)
        if self.mode == "fresh":
            self._idx = (self._idx * 5 + action + 1 + self._t) % len(self._frames)
            np.take(self._frames, self._idx, axis=0, out=self._obs)
            obs = self._obs
        else:
            obs = self._batches[self._t % len(self._batches)]
        return obs, reward, done, info

    def close(self):
        pass


class SyntheticGymnasiumVec:
    """gymnasium-style vector env with float observations.

    ``kind="discrete"``: CartPole-shaped (obs f32 [N,4], Discrete(2)).
    ``kind="continuous"``: HalfCheetah-shaped (obs f32 [N,17] clipped to +-10, Box(6) actions).
    ``kind="atari"``: uint8 [N,4,84,84], Discrete(4) (for the multigpu script).
    """

    def __init__(self, num_envs, kind="discrete", obs_dim=None, act_dim=None, p_done=0.02, max_len=500):
        self.num_envs = int(num_envs)
        self.kind = kind
        if kind == "discrete":
            od = obs_dim or 4
            self.single_observation_space = Box(-np.inf, np.inf, (od,), np.float32)
            self.single_action_space = Discrete(act_dim or 2)
        elif kind == "continuous":
            od = obs_dim or 17
            self.single_observation_space = Box(-np.inf, np.inf, (od,), np.float32)
            self.single_action_space = Box(-1.0, 1.0, (act_dim or 6,), np.float32)
        elif kind in ("atari", "atari1"):     # atari1: FrameStack(1) as cleanrl/ppo_atari_lstm.py:105
            self.single_observation_space = Box(0, 255, (4 if kind == "atari" else 1, 84, 84), np.uint8)
            self.single_action_space = Discrete(act_dim or 4)
        else:
            raise ValueError(kind)
        self.observation_space = self.single_observation_space
        self.action_space = self.single_action_space
        self.p_done = float(p_done)
        self.max_len = int(max_len)
        self._rng = None
        self._ep_ret = np.zeros(self.num_envs, dtype=np.float64)
        self._ep_len = np.zeros(self.num_envs, dtype=np.int64)
        self._state = None

    def _draw_obs(self, act_term):
        n = self.num_envs
        shp = self.single_observation_space.shape
        if self.kind.startswith("atari"):
            return self._rng.integers(0, 256, size=(n,) + shp, dtype=np.uint8)
        self._state = 0.9 * self._state + 0.3 * self._rng.standard_normal((n,) + shp) + 0.05 * act_term
        return np.clip(self._state, -10, 10).astype(np.float32)

    def reset(self, seed=None, **kwargs):
        self._rng = np.random.default_rng(seed)
        self._ep_ret[:] = 0
        self._ep_len[:] = 0
        self._state = np.zeros((self.num_envs,) + self.single_observation_space.shape, dtype=np.float64)
        return self._draw_obs(0.0), {}

    def step(self, action):
        n = self.num_envs
        action = np.asarray(action)
        if self.kind == "continuous":
            act_term = np.clip(action, -1, 1).reshape(n, -1).mean(axis=1, keepdims=True)
            reward = np.clip(self._rng.standard_normal(n) + act_term[:, 0], -10, 10).astype(np.float32)
        else:
            a = action.reshape(n).astype(np.float64)
            act_term = (a - 0.5).reshape((n,) + (1,) * len(self.single_observation_space.shape))
            reward = np.ones(n, dtype=np.float32) if self.kind == "discrete" else \
                np.sign(self._rng.integers(0, 3, size=n) * (a != 0)).astype(np.float32)
        self._ep_ret += reward
        self._ep_len += 1
        terminated = self._rng.random(n) < self.p_done
        truncated = (self._ep_len >= self.max_len) & ~terminated
        done = terminated | truncated
        obs = self._draw_obs(act_term)
        infos = {}
        if done.any():
            final = np.empty(n, dtype=object)
            for i in np.nonzero(done)[0]:
                final[i] = {"episode": {"r": np.array([self._ep_ret[i]], dtype=np.float32),
                                        "l": np.array([self._ep_len[i]], dtype=np.int32)}}
            infos["final_info"] = final
            infos["_final_info"] = done.copy()
            fobs = np.empty(n, dtype=object)
            for i in np.nonzero(done)[0]:
                fobs[i] = obs[i].copy()
            infos["final_observation"] = fobs
            self._ep_ret[done] = 0
            self._ep_len[done] = 0
            if not self.kind.startswith("atari"):
                self._state[done] = 0
        return obs, reward, terminated, truncated, infos

    def close(self):
        pass


class CartPoleVec:
    """Vectorised CartPole-v1 dynamics (the classic cart-pole of Barto, Sutton & Anderson: Euler steps of 0.02 s,
    force +-10 N, failure beyond +-2.4 m or +-12 degrees, 500-step time limit) behind the gymnasium vector API with
    episode statistics in ``infos["final_info"]`` as ``RecordEpisodeStatistics`` + ``SyncVectorEnv`` deliver them
    (what cleanrl/ppo.py:210-215 reads).  Lets the PPO drop-in show a real learning curve without gymnasium
    installed (SURVEY 8d, config C1); host-side numpy, not part of the hot path."""

    GRAVITY, M_CART, M_POLE, HALF_LEN, FORCE, TAU = 9.8, 1.0, 0.1, 0.5, 10.0, 0.02
    X_LIMIT, THETA_LIMIT, MAX_STEPS = 2.4, 12 * 2 * np.pi / 360, 500

    def __init__(self, num_envs):
        self.num_envs = int(num_envs)
        self.single_observation_space = Box(-np.inf, np.inf, (4,), np.float32)
        self.single_action_space = Discrete(2)
        self.observation_space, self.action_space = self.single_observation_space, self.single_action_space
        self._rng = np.random.default_rng(0)
        self._s = np.zeros((self.num_envs, 4), dtype=np.float64)
        self._ret = np.zeros(self.num_envs, dtype=np.float64)
        self._len = np.zeros(self.num_envs, dtype=np.int64)

    def _fresh(self, k):
        return self._rng.uniform(-0.05, 0.05, size=(k, 4))

    def reset(self, seed=None, **kwargs):
        self._rng = np.random.default_rng(seed)
        self._s = self._fresh(self.num_envs)
        self._ret[:] = 0
        self._len[:] = 0
        return self._s.astype(np.float32), {}

    def step(self, action):
        a = np.asarray(action).reshape(self.num_envs)
        x, xd, th, thd = self._s.T
        force = np.where(a == 1, self.FORCE, -self.FORCE)
        total_m = self.M_CART + self.M_POLE
        pm_l = self.M_POLE * self.HALF_LEN
        cos, sin = np.cos(th), np.sin(th)
        tmp = (force + pm_l * thd * thd * sin) / total_m
        th_acc = (self.GRAVITY * sin - cos * tmp) / (self.HALF_LEN * (4.0 / 3.0 - self.M_POLE * cos * cos / total_m))
        x_acc = tmp - pm_l * th_acc * cos / total_m
        self._s = np.stack([x + self.TAU * xd, xd + self.TAU * x_acc, th + self.TAU * thd, thd + self.TAU * th_acc], axis=1)
        self._ret += 1.0
        self._len += 1
        terminated = (np.abs(self._s[:, 0]) > self.X_LIMIT) | (np.abs(self._s[:, 2]) > self.THETA_LIMIT)
        truncated = (self._len >= self.MAX_STEPS) & ~terminated
        done = terminated | truncated
        reward = np.ones(self.num_envs, dtype=np.float32)
        infos = {}
        if done.any():
            idx = np.nonzero(done)[0]
            final = np.empty(self.num_envs, dtype=object)
            fobs = np.empty(self.num_envs, dtype=object)
            for i in idx:
                final[i] = {"episode": {"r": np.array([self._ret[i]], dtype=np.float32),
                                        "l": np.array([self._len[i]], dtype=np.int32)}}
                fobs[i] = self._s[i].astype(np.float32)
            infos["final_info"], infos["_final_info"], infos["final_observation"] = final, done.copy(), fobs
            self._s[idx] = self._fresh(len(idx))          # auto-reset: the returned observation starts the next episode
            self._ret[idx] = 0
            self._len[idx] = 0
        return self._s.astype(np.float32), reward, terminated, truncated, infos

    def close(self):
        pass


class SyntheticProcgenVec:
    """Procgen-shaped vector env (gym3 / old-gym vector API as cleanrl/ppo_procgen.py:176-186,237-247 uses it after its
    wrappers): uint8 RGB frames [N, 64, 64, 3], Discrete(15) actions, ``reset() -> obs``, ``step(a) -> (obs, reward, done,
    info)`` with ``info`` a list of per-env dicts carrying ``{"episode": {"r", "l"}}`` when an episode ends.  The next frame
    of an env depends on its own step count and the action it received (a wrong action changes later observations)."""

    def __init__(self, num_envs, seed=0, n_actions=15, pool=32, p_done=0.02):
        self.num_envs = int(num_envs)
        self.observation_space = Box(0, 255, (64, 64, 3), np.uint8)
        self.action_space = Discrete(n_actions)
        self.single_observation_space, self.single_action_space = self.observation_space, self.action_space
        self.is_vector_env = True
        self._rng = np.random.default_rng(seed)
        self._frames = self._rng.integers(0, 256, size=(pool, 64, 64, 3), dtype=np.uint8)
        self._idx = np.zeros(self.num_envs, dtype=np.int64)
        self._ret = np.zeros(self.num_envs, dtype=np.float64)
        self._len = np.zeros(self.num_envs, dtype=np.int64)
        self.p_done = float(p_done)

    def reset(self, **kwargs):
        self._idx = self._rng.integers(0, len(self._frames), size=self.num_envs)
        self._ret[:] = 0
        self._len[:] = 0
        return self._frames[self._idx]

    def step(self, action):
        a = np.asarray(action).reshape(self.num_envs).astype(np.int64)
        reward = (self._rng.integers(0, 4, size=self.num_envs) == 0).astype(np.float32) * (a % 3 != 0)
        done = self._rng.random(self.num_envs) < self.p_done
        self._ret += reward
        self._len += 1
        info = [{} for _ in range(self.num_envs)]
        for i in np.nonzero(done)[0]:
            info[i] = {"episode": {"r": float(self._ret[i]), "l": int(self._len[i])}}
        self._ret[done] = 0
        self._len[done] = 0
        self._idx = (self._idx * 5 + a + 1) % len(self._frames)
        return self._frames[self._idx], reward, done, info

    def close(self):
        pass
