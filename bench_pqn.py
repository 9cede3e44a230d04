"""PQN (cleanrl/pqn.py) on one GPU: one JSON line.

* Update: one iteration's update (update_epochs 4 x num_minibatches 4) at the defaults (4 envs x 128 steps, M = 128) and
  at 1024 envs x 128 steps (M = 32 768), for the CartPole (4, 2) and (8, 4) shapes, as the captured per-epoch graphs, as
  eager launches of the same kernels, and as the reference's eager PyTorch update (autograd, clip_grad_norm_ and
  torch.optim.RAdam on the same card).  CUDA events, median over rounds that alternate the arms.
* The rollout step's latency (pinned packet upload, the act kernel, the action download) at n = 4 and n = 1024, the
  Q(lambda) kernel at 128 x 1024, the library launches per minibatch update, and the drop-in loop's env steps/s on
  ``synthetic_envs.CartPoleVec`` at the defaults.
* The card's name, power limit and SM clock (sampled before and after the timed work) are read in the same run.

    python bench_pqn.py [--rounds 10] [--e2e-steps 102400]
"""
from __future__ import annotations

import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np
import torch

from cleanrl_b200 import build, ops
from cleanrl_b200.agents import PQNQNetwork
from cleanrl_b200.pqn_engine import PQNEngine
from cleanrl_b200.synthetic_envs import Box, CartPoleVec, Discrete

DEV = torch.device("cuda")


def _env(n, d, A):
    env = CartPoleVec(n)
    env.single_observation_space = Box(-np.inf, np.inf, (d,), np.float32)
    env.single_action_space = Discrete(A)
    return env


def _args(n, T):
    return types.SimpleNamespace(num_steps=T, num_minibatches=4, update_epochs=4, max_grad_norm=10.0, gamma=0.99,
                                 q_lambda=0.65)


def _engine(n, T, d, A):
    torch.manual_seed(1)
    net = PQNQNetwork(_env(n, d, A)).to(DEV)
    eng = PQNEngine(net, _args(n, T), n, DEV)
    g = torch.Generator(device="cuda").manual_seed(0)
    eng.obs.copy_(torch.randn(eng.obs.shape, generator=g, device="cuda"))
    eng.actions.copy_(torch.randint(0, A, eng.actions.shape, generator=g, device="cuda"))
    eng.returns.copy_(torch.randn(eng.returns.shape, generator=g, device="cuda"))
    return net, eng


class EagerTorchUpdate:
    """pqn.py:226-240 restated: autograd through nn.Sequential, clip_grad_norm_ and torch.optim.RAdam."""

    def __init__(self, eng, d, A):
        torch.manual_seed(1)
        self.net = PQNQNetwork(_env(1, d, A)).network.to(DEV)
        self.opt = torch.optim.RAdam(self.net.parameters(), lr=2.5e-4)
        self.eng = eng

    def __call__(self):
        e = self.eng
        b_obs, b_actions, b_returns = e.obs, e.actions, e.returns.view(-1)
        b_inds = np.arange(e.B)
        for _ in range(e.epochs):
            np.random.shuffle(b_inds)
            for start in range(0, e.B, e.mbs):
                mb = torch.as_tensor(b_inds[start:start + e.mbs]).to(DEV)
                old_val = self.net(b_obs[mb]).gather(1, b_actions[mb].unsqueeze(-1)).squeeze()
                loss = torch.nn.functional.mse_loss(b_returns[mb], old_val)
                self.opt.zero_grad()
                loss.backward()
                torch.nn.utils.clip_grad_norm_(self.net.parameters(), 10.0)
                self.opt.step()


def _timed(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def update_arms(n, T, d, A, rounds):
    _, eng = _engine(n, T, d, A)
    eager = EagerTorchUpdate(eng, d, A)
    arms = {"graph_ms": lambda: eng.update(2.5e-4, use_graph=True),
            "eager_kernels_ms": lambda: eng.update(2.5e-4, use_graph=False),
            "eager_torch_ms": eager}
    for f in arms.values():
        f(); f()
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            res[k].append(_timed(f))
    return {k: round(float(np.median(v)), 4) for k, v in res.items()}


def launches_per_minibatch():
    _, eng = _engine(4, 128, 4, 2)
    lib = ops._lib.load()
    c0 = lib.b200rl_launch_count()
    eng.update(2.5e-4, use_graph=False)
    torch.cuda.synchronize()
    return (lib.b200rl_launch_count() - c0) / (eng.epochs * eng.nmb)


def step_latency_ms(n, reps=500):
    _, eng = _engine(n, 128, 4, 2)
    obs = np.random.default_rng(0).standard_normal((n, 4)).astype(np.float32)
    z = np.zeros(n, np.float32)
    for i in range(20):
        eng.policy_step(i % 128, obs, z, z, 0.5)
    t = time.perf_counter()
    for i in range(reps):
        eng.policy_step(i % 128, obs, z, z, 0.5)
    return (time.perf_counter() - t) / reps * 1e3


def qlambda_us(T=128, N=1024, reps=200):
    g = torch.Generator(device="cuda").manual_seed(0)
    r, v = torch.randn(T, N, generator=g, device="cuda"), torch.randn(T, N, generator=g, device="cuda")
    d = (torch.rand(T, N, generator=g, device="cuda") < 0.05).float()
    nv, nd, out = torch.randn(N, device="cuda"), torch.zeros(N, device="cuda"), torch.empty(T, N, device="cuda")
    f = lambda: ops.qlambda(r, v, d, nv, nd, 0.99, 0.65, returns=out)   # noqa: E731
    for _ in range(10):
        f()
    return _timed(f, reps) * 1e3


class _NullWriter:
    def __init__(self, *a, **k):
        pass

    def add_text(self, *a, **k):
        pass

    def add_scalar(self, *a, **k):
        pass

    def close(self):
        pass


def e2e_sps(steps):
    from cleanrl_b200 import pqn
    with contextlib.redirect_stdout(io.StringIO()):
        t = time.perf_counter()
        pqn.main(["--total-timesteps", str(steps)], writer_factory=_NullWriter,
                 env_factory=lambda a: CartPoleVec(a.num_envs))
        torch.cuda.synchronize()
    return steps / (time.perf_counter() - t)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--e2e-steps", type=int, default=102400)
    a = ap.parse_args()
    build.build()
    out = {"bench": "pqn", "gpu_before": gpu_info()}
    for n in (4, 1024):
        for d, A in ((4, 2), (8, 4)):
            out[f"update_n{n}_t128_{d}x{A}"] = update_arms(n, 128, d, A, a.rounds)
    out["launches_per_minibatch_update"] = launches_per_minibatch()
    out["rollout_step_ms_n4"] = round(step_latency_ms(4), 4)
    out["rollout_step_ms_n1024"] = round(step_latency_ms(1024), 4)
    out["qlambda_us_128x1024"] = round(qlambda_us(), 2)
    out["e2e_env_steps_per_s"] = round(e2e_sps(a.e2e_steps), 1)
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
