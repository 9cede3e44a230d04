"""IMPALA-CNN PPO iteration benchmark (cleanrl/ppo_procgen.py at its reference update settings: 3 epochs x 8 minibatches):
one PPOEngine iteration -- a rollout of T steps over N synthetic procgen-shaped envs, then the update -- with the fp32
CUDA-core network and the bf16 tensor-core network, the two arms alternating in one process.  Sizes: 64 envs x 256 steps
(the reference default, minibatch 2048) and 512 x 256 (minibatch 16 384).  Rollout and update are each timed with a
device synchronise at both ends; a separate pass per arm records the per-kernel-family times (ProfScope events).
Prints one JSON line with the GPU name, power limit and sampled SM clock.

    python bench_procgen.py [--iters 2] [--warmup 1] [--sizes 64x256,512x256]
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
from bench import ClockSampler, ppo_args  # noqa: E402
from bench_c51 import _gpu_info  # noqa: E402
from cleanrl_b200 import _lib  # noqa: E402
from cleanrl_b200.agents import ImpalaAgent  # noqa: E402
from cleanrl_b200.ppo_engine import PPOEngine  # noqa: E402
from cleanrl_b200.synthetic_envs import SyntheticProcgenVec  # noqa: E402

MFLOP_PER_SAMPLE = 61.2       # forward pass, from the layer shapes; backward = 2x forward


def _args(N, T, precision):
    a = ppo_args(N, T, 1, precision)
    a.num_minibatches, a.update_epochs, a.gamma, a.gae_lambda = 8, 3, 0.999, 0.95
    a.clip_coef, a.ent_coef, a.learning_rate = 0.2, 0.01, 5e-4
    a.minibatch_size = a.batch_size // a.num_minibatches
    return a


class Arm:
    def __init__(self, N, T, precision, dev):
        torch.manual_seed(1); np.random.seed(1)
        self.env = SyntheticProcgenVec(N, seed=3)
        self.agent = ImpalaAgent(self.env).to(dev)
        self.agent.precision = precision
        self.eng = PPOEngine(self.agent, _args(N, T, precision), (64, 64, 3), np.uint8, N, dev, gae_mode=1)
        self.T, self.N = T, N
        self.obs, self.done = self.env.reset(), np.zeros(N, dtype=np.float32)

    def iteration(self):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for t in range(self.T):
            a = self.eng.policy_step(t, self.obs, self.done)
            self.obs, r, d, _ = self.env.step(a.copy())
            self.eng.record_reward(t, np.asarray(r, dtype=np.float32))
            self.done = np.asarray(d, dtype=np.float32)
        self.eng.finish_rollout(self.obs, self.done)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        st = self.eng.update(5e-4)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        assert np.isfinite(st["per_update"]).all()
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


def _agreement(dev, A=15, n=4096):
    """Fraction of sampled actions that agree between the two precisions: same weights, frames and sampling noise."""
    torch.manual_seed(7)
    env = SyntheticProcgenVec(1)
    a32 = ImpalaAgent(env).to(dev)
    a16 = ImpalaAgent(env).to(dev)
    a16.load_state_dict(a32.state_dict())
    a16.precision = "bf16"
    g = torch.Generator().manual_seed(11)
    obs = torch.randint(0, 256, (n, 64, 64, 3), dtype=torch.uint8, generator=g).to(dev)
    noise = torch.empty(n, A).exponential_(1, generator=g).to(dev)
    acts = []
    for ag in (a32, a16):
        ag.noise_fn = lambda n_, A_, d_: noise
        acts.append(ag.get_action_and_value(obs)[0])
    return float((acts[0] == acts[1]).double().mean())


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=2)
    p.add_argument("--warmup", type=int, default=1)
    p.add_argument("--sizes", default="64x256,512x256")
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_procgen.py needs a CUDA device")
    dev = torch.device("cuda")
    out = {"metric": "ppo_procgen_iteration_ms", "update_epochs": 3, "num_minibatches": 8}
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    for size in a.sizes.split(","):
        N, T = (int(x) for x in size.split("x"))
        arms = {prec: Arm(N, T, prec, dev) for prec in ("fp32", "bf16")}
        for arm in arms.values():
            for _ in range(a.warmup):
                arm.iteration()
        res = {prec: [] for prec in arms}
        sampler.mark_begin()
        for _ in range(a.iters):
            for prec, arm in arms.items():          # alternate the arms
                res[prec].append(arm.iteration())
        sampler.mark_end()
        B = N * T
        flop = MFLOP_PER_SAMPLE * 1e6 * (B + 3 * B * 3)      # rollout forward + 3 epochs of forward + backward
        for prec, r in res.items():
            roll = float(np.median([x[0] for x in r]))
            upd = float(np.median([x[1] for x in r]))
            tot = roll + upd
            out[f"{size}_{prec}"] = {"iteration_ms": round(tot, 2), "rollout_ms": round(roll, 2), "update_ms": round(upd, 2),
                                     "env_steps_per_s": round(B / tot * 1e3, 1),
                                     "network_tflops": round(flop / (tot * 1e-3) / 1e12, 2),
                                     "kernels_ms": _profile(arms[prec])}
        del arms
        torch.cuda.empty_cache()
    out["action_agreement_bf16_vs_fp32"] = round(_agreement(dev), 4)
    out["clocks"] = sampler.stop()
    out["gpu"], out["power_limit"] = _gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
