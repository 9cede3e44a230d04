"""RPO update (cleanrl/rpo_continuous_action.py:260-313) on one GPU: one JSON line.

Per iteration's update (``update_epochs x num_minibatches`` = 10 x 32 minibatch updates, the reference's defaults) at
num_envs 1 x 2048 steps (minibatch 64) and num_envs 64 (minibatch 4096), for HalfCheetah (17, 6) and Humanoid (376, 17)
shapes: the drop-in's update (PPOEngine.update with RPOAgent, host time included; CUDA events, median over rounds)
against the same update in eager PyTorch on the same card (autograd + torch.optim.Adam, one CPU z draw and
host-to-device copy per minibatch, as the reference); the host time of RPOAgent's per-epoch z draws and uploads per
iteration; library launches per minibatch update; and env steps per second of the drop-in's loop on the synthetic
HalfCheetah env.  The card's name and power limit are read in the same run.

    python bench_rpo_continuous.py [--rounds 3] [--e2e-iterations 4]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
import tempfile
import time
import types

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np
import torch
import torch.nn as nn
from torch.distributions.normal import Normal

from cleanrl_b200 import build, ops
from cleanrl_b200.agents import RPOAgent
from cleanrl_b200.ppo_engine import PPOEngine
from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec

DEV = torch.device("cuda")
T, NMB, EPOCHS = 2048, 32, 10


def _args():
    return types.SimpleNamespace(num_steps=T, num_minibatches=NMB, update_epochs=EPOCHS, gamma=0.99, gae_lambda=0.95,
                                 clip_coef=0.2, ent_coef=0.0, vf_coef=0.5, max_grad_norm=0.5, norm_adv=True,
                                 clip_vloss=True, target_kl=None, rpo_alpha=0.5)


def _setup(od, D, N):
    env = SyntheticGymnasiumVec(1, kind="continuous", obs_dim=od, act_dim=D)
    torch.manual_seed(1)
    agent = RPOAgent(env, 0.5).to(DEV)
    eng = PPOEngine(agent, _args(), (od,), np.float32, N, DEV)
    g = torch.Generator(device=DEV).manual_seed(2)
    eng.obs.copy_(torch.randn(eng.obs.shape, generator=g, device=DEV))
    eng.actions.copy_(torch.randn(eng.actions.shape, generator=g, device=DEV))
    eng.logprobs.copy_(torch.randn(eng.logprobs.shape, generator=g, device=DEV) * 0.2 - 0.92 * D)
    eng.values.copy_(torch.randn(eng.values.shape, generator=g, device=DEV))
    eng.advantages.copy_(torch.randn(eng.advantages.shape, generator=g, device=DEV))
    eng.returns.copy_(eng.advantages + eng.values)
    return env, agent, eng


class EagerRPO:
    """The reference's update loop in eager PyTorch: nn.Sequential MLPs, Normal(mean + z, std), autograd,
    clip_grad_norm_ and Adam, with z drawn on the CPU and copied to the device per minibatch."""

    def __init__(self, agent, eng):
        self.critic, self.actor_mean = copy.deepcopy(agent.critic), copy.deepcopy(agent.actor_mean)
        self.logstd = nn.Parameter(agent.actor_logstd.detach().clone())
        self.params = list(self.critic.parameters()) + list(self.actor_mean.parameters()) + [self.logstd]
        for q in self.params:           # own storage: the agent's parameters are views of its flat buffer
            q.data = q.data.clone()
        self.opt = torch.optim.Adam(self.params, lr=3e-4, eps=1e-5)
        B = eng.B
        self.b = {"obs": eng.obs.reshape(B, -1).clone(), "actions": eng.actions.reshape(B, -1).clone()}
        for k in ("logprobs", "advantages", "returns", "values"):
            self.b[k] = getattr(eng, k).reshape(B).clone()
        self.B, self.M = B, B // NMB

    def update(self):
        a, b, b_inds = _args(), self.b, np.arange(self.B)
        for _ in range(EPOCHS):
            np.random.shuffle(b_inds)
            for start in range(0, self.B, self.M):
                mb = torch.from_numpy(b_inds[start:start + self.M]).to(DEV)
                x = b["obs"][mb]
                mean = self.actor_mean(x)
                z = torch.FloatTensor(mean.shape).uniform_(-a.rpo_alpha, a.rpo_alpha).to(DEV)
                probs = Normal(mean + z, torch.exp(self.logstd.expand_as(mean)))
                newlogprob = probs.log_prob(b["actions"][mb]).sum(1)
                entropy = probs.entropy().sum(1)
                logratio = newlogprob - b["logprobs"][mb]
                ratio = logratio.exp()
                adv = b["advantages"][mb]
                adv = (adv - adv.mean()) / (adv.std() + 1e-8)
                pg_loss = torch.max(-adv * ratio, -adv * torch.clamp(ratio, 1 - a.clip_coef, 1 + a.clip_coef)).mean()
                nv = self.critic(x).view(-1)
                vu = (nv - b["returns"][mb]) ** 2
                vc = (b["values"][mb] + torch.clamp(nv - b["values"][mb], -a.clip_coef, a.clip_coef) - b["returns"][mb]) ** 2
                loss = pg_loss - a.ent_coef * entropy.mean() + 0.5 * torch.max(vu, vc).mean() * a.vf_coef
                self.opt.zero_grad()
                loss.backward()
                nn.utils.clip_grad_norm_(self.params, a.max_grad_norm)
                self.opt.step()


def _timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def update_arms(od, D, N, rounds):
    _, agent, eng = _setup(od, D, N)
    eager = EagerRPO(agent, eng)
    host = []
    orig = agent.begin_update_epoch

    def hook(*a):
        t = time.perf_counter()
        orig(*a)
        host.append(time.perf_counter() - t)
    agent.begin_update_epoch = hook
    arms = {"kernels": lambda: eng.update(3e-4), "eager_torch": eager.update}
    for f in arms.values():
        f()
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            res[k].append(_timed(f))
    lib = ops._lib.load()
    host.clear()
    c0 = lib.b200rl_launch_count()
    st = eng.update(3e-4)
    torch.cuda.synchronize()
    out = {f"{k}_ms": round(float(np.median(v)), 3) for k, v in res.items()}
    out["minibatch"] = eng.M
    out["z_draw_upload_host_ms_per_iteration"] = round(sum(host) * 1e3, 4)
    out["launches_per_minibatch"] = (lib.b200rl_launch_count() - c0) / st["num_updates"]
    return out


def e2e_sps(iterations):
    from cleanrl_b200 import rpo_continuous_action as S

    class W:
        def __init__(self, *a, **k): pass
        def add_text(self, *a, **k): pass
        def add_scalar(self, *a, **k): pass
        def close(self): pass
    marks = []
    argv = ["--synthetic-env", "--total-timesteps", str(T * iterations)]
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as d:
        os.chdir(d)
        try:
            S.main(argv, writer_factory=W, on_iteration=lambda it, eng, st: marks.append(time.perf_counter()))
        finally:
            os.chdir(cwd)
    return T * (len(marks) - 1) / (marks[-1] - marks[0])        # the first iteration (warm-up) is not timed


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--e2e-iterations", type=int, default=4)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rpo_continuous.py measures on a CUDA device; none is visible")
    build.build()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": smi[0].split(",")[-1].strip() if smi else None,
           "minibatch_updates_per_iteration": EPOCHS * NMB}
    for od, D in ((17, 6), (376, 17)):
        for N in (1, 64):
            out[f"update_obs{od}_act{D}_n{N}"] = update_arms(od, D, N, a.rounds)
    out["e2e_sps"] = round(e2e_sps(a.e2e_iterations), 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
