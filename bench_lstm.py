"""Recurrent PPO iteration benchmark (cleanrl/ppo_atari_lstm.py at its reference update settings: 4 epochs x 4 minibatches
of whole env sequences): one iteration of the drop-in loop of cleanrl_b200/ppo_atari_lstm.py -- a rollout of T steps over
N synthetic single-frame Atari-shaped envs carrying the LSTM state, GAE, then the update -- with the fp32 CUDA-core agent
and the bf16 tensor-core agent, the two arms alternating in one process.  Sizes: 8 envs x 128 steps (the reference
default, minibatches of 2 envs x 128 steps) and 256 x 128 (minibatches of 64 envs x 128 steps = 8 192 rows).  Rollout and
update are each timed with a device synchronise at both ends; library launches are counted per iteration; a separate
pass per arm records the per-kernel-family times (ProfScope events).  Prints one JSON line with the GPU name, power limit
and sampled SM clock.

    python bench_lstm.py [--iters 2] [--warmup 1] [--sizes 8x128,256x128]
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench import ClockSampler  # noqa: E402
from bench_c51 import _gpu_info  # noqa: E402
from cleanrl_b200 import _lib, ops  # noqa: E402
from cleanrl_b200.agents import LSTMAgent  # noqa: E402
from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec  # noqa: E402

EPOCHS, MINIBATCHES = 4, 4


class _Args:
    clip_coef, ent_coef, vf_coef, norm_adv, clip_vloss = 0.1, 0.01, 0.5, True, True


class Arm:
    """The loop of cleanrl_b200/ppo_atari_lstm.py (same calls, same order), one iteration per ``iteration()``."""

    def __init__(self, N, T, precision, dev):
        torch.manual_seed(1); np.random.seed(1)
        self.envs = SyntheticGymnasiumVec(N, kind="atari1")
        self.agent = LSTMAgent(self.envs).to(dev)
        self.agent.precision = precision
        self.flat = self.agent.flat
        self.N, self.T, self.dev = N, T, dev
        f32 = torch.float32
        self.obs = torch.zeros((T, N, 1, 84, 84), dtype=torch.uint8, device=dev)
        z = lambda dt=f32: torch.zeros((T, N), dtype=dt, device=dev)
        self.actions, self.logprobs, self.rewards, self.dones = z(torch.int64), z(), z(), z()
        self.values, self.advantages, self.returns = z(), z(), z()
        self.stats = torch.zeros(EPOCHS * MINIBATCHES, 16, dtype=f32, device=dev)
        self.rewards_h = torch.zeros((T, N), dtype=f32).pin_memory()
        o, _ = self.envs.reset(seed=1)
        self.next_obs = torch.from_numpy(np.ascontiguousarray(o)).to(dev)
        self.next_done = torch.zeros(N, dtype=f32, device=dev)
        self.state = (torch.zeros(1, N, 128, device=dev), torch.zeros(1, N, 128, device=dev))
        self.scratch = {}

    def iteration(self):
        ag, N, T, B, dev = self.agent, self.N, self.T, self.N * self.T, self.dev
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        initial_state = (self.state[0].clone(), self.state[1].clone())
        with torch.no_grad():
            for step in range(T):
                self.obs[step].copy_(self.next_obs)
                self.dones[step].copy_(self.next_done)
                action, logprob, _, value, self.state = ag.get_action_and_value(self.next_obs, self.state, self.next_done)
                self.values[step].copy_(value.flatten())
                self.actions[step].copy_(action)
                self.logprobs[step].copy_(logprob)
                o, r, term, trunc, _ = self.envs.step(action.cpu().numpy())
                self.rewards_h[step].copy_(torch.as_tensor(np.asarray(r, dtype=np.float32).reshape(-1)))
                self.next_obs = torch.from_numpy(np.ascontiguousarray(o)).to(dev)
                self.next_done = torch.from_numpy(np.logical_or(term, trunc).astype(np.float32)).to(dev)
            self.rewards.copy_(self.rewards_h, non_blocking=True)
            next_value = ag.get_value(self.next_obs, self.state, self.next_done).reshape(-1)
            ops.gae(self.rewards, self.values, self.dones, next_value, self.next_done, 0.99, 0.95, mode=1,
                    out=(self.advantages, self.returns))
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        b_obs = self.obs.reshape(-1, 1, 84, 84)
        b = {"actions": self.actions.view(B), "logprobs": self.logprobs.view(B), "advantages": self.advantages.view(B),
             "returns": self.returns.view(B), "values": self.values.view(B)}
        envinds, flatinds, per = np.arange(N), np.arange(B).reshape(T, N), N // MINIBATCHES
        k = 0
        for _ in range(EPOCHS):
            np.random.shuffle(envinds)
            for start in range(0, N, per):
                mbenv = envinds[start:start + per]
                mb_inds = torch.from_numpy(flatinds[:, mbenv].ravel()).to(dev)
                env_t = torch.from_numpy(mbenv).to(dev)
                st = (initial_state[0][:, env_t].contiguous(), initial_state[1][:, env_t].contiguous())
                logits, value = ag.forward_train(b_obs, mb_inds, st, self.dones.view(B))
                ag.loss_backward(logits, value, mb_inds, b, _Args, self.stats[k], self.scratch)
                self.flat.step += 1
                ops.clip_adam(self.flat.flat, self.flat.grad, self.flat.exp_avg, self.flat.exp_avg_sq, self.flat.step, 2.5e-4,
                              eps=1e-5, max_norm=0.5)
                ag.params_updated()
                k += 1
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        assert torch.isfinite(self.stats).all()
        return (t1 - t0) * 1e3, (t2 - t1) * 1e3


def _profile(arm):
    lib = _lib.load()
    lib.b200rl_profile_reset()
    lib.b200rl_profile_enable(1)
    arm.iteration()
    torch.cuda.synchronize()
    lib.b200rl_profile_enable(0)
    buf = ctypes.create_string_buffer(1 << 16)
    _lib.check(lib.b200rl_profile_summary(buf, 1 << 16), "profile_summary")
    return json.loads(buf.value.decode())


def _agreement(dev, S=128, n=32):
    """Fraction of sampled actions that agree between the two precisions over whole sequences: same weights, frames,
    done flags, initial state and sampling noise."""
    torch.manual_seed(7)
    env = SyntheticGymnasiumVec(1, kind="atari1")
    a32 = LSTMAgent(env).to(dev)
    a16 = LSTMAgent(env).to(dev)
    a16.load_state_dict(a32.state_dict())
    a16.precision = "bf16"
    A = a32.num_actions
    g = torch.Generator().manual_seed(11)
    obs = torch.randint(0, 256, (S * n, 1, 84, 84), dtype=torch.uint8, generator=g).to(dev)
    done = (torch.rand(S * n, generator=g) < 0.02).float().to(dev)
    state = tuple(torch.randn(1, n, 128, generator=g).to(dev) * 0.3 for _ in range(2))
    noise = torch.empty(S * n, A).exponential_(1, generator=g).to(dev)
    acts = []
    for ag in (a32, a16):
        ag.noise_fn = lambda n_, A_, d_: noise
        acts.append(ag.get_action_and_value(obs, state, done)[0])
    return float((acts[0] == acts[1]).double().mean())


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=2)
    p.add_argument("--warmup", type=int, default=1)
    p.add_argument("--sizes", default="8x128,256x128")
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lstm.py needs a CUDA device")
    dev = torch.device("cuda")
    lib = _lib.load()
    out = {"metric": "ppo_atari_lstm_iteration_ms", "update_epochs": EPOCHS, "num_minibatches": MINIBATCHES}
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    for size in a.sizes.split(","):
        N, T = (int(x) for x in size.split("x"))
        arms = {prec: Arm(N, T, prec, dev) for prec in ("fp32", "bf16")}
        for arm in arms.values():
            for _ in range(a.warmup):
                arm.iteration()
        res = {prec: [] for prec in arms}
        launches = {prec: [] for prec in arms}
        sampler.mark_begin()
        for _ in range(a.iters):
            for prec, arm in arms.items():          # alternate the arms
                l0 = lib.b200rl_launch_count()
                res[prec].append(arm.iteration())
                launches[prec].append(lib.b200rl_launch_count() - l0)
        sampler.mark_end()
        for prec, r in res.items():
            roll = float(np.median([x[0] for x in r]))
            upd = float(np.median([x[1] for x in r]))
            tot = roll + upd
            out[f"{size}_{prec}"] = {"iteration_ms": round(tot, 2), "rollout_ms": round(roll, 2), "update_ms": round(upd, 2),
                                     "env_steps_per_s": round(N * T / tot * 1e3, 1),
                                     "launches_per_iteration": int(np.median(launches[prec])),
                                     "kernels_ms": _profile(arms[prec])}
        del arms
        torch.cuda.empty_cache()
    out["action_agreement_bf16_vs_fp32"] = round(_agreement(dev), 4)
    out["clocks"] = sampler.stop()
    out["gpu"], out["power_limit"] = _gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
