"""Continuous SAC update (cleanrl/sac_continuous_action.py:255-304) on one GPU: one JSON line.

Per-update time (CUDA events, median over alternated rounds; every update has actor steps on even global steps, so a
round is a critic-only update and an update with two actor + temperature steps) at B = 256 / 1024 for HalfCheetah
(17, 6) and Humanoid (376, 17) shapes, as the captured graph, as eager launches of the same kernels, and as the
reference's eager PyTorch update (oracle/sac_continuous_oracle.EagerSAC, autograd + torch.optim on the same GPU); the
library launches per update; the ``get_action`` latency at n = num_envs; and env steps per second of the drop-in's loop
after ``learning_starts`` on the synthetic HalfCheetah env, with the graph update against the eager PyTorch update.

    python bench_sac_continuous.py [--rounds 20] [--e2e-steps 2000]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np
import torch

from cleanrl_b200 import build, ops
from cleanrl_b200.agents import SACContinuousActor, SACContinuousState, SoftQNetworkMLP, sac_continuous_update
from cleanrl_b200.replay import DeviceReplayRing
from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
from oracle.sac_continuous_oracle import EagerSAC

DEV = torch.device("cuda")
ARGS = types.SimpleNamespace(policy_frequency=2, target_network_frequency=1, q_lr=1e-3, policy_lr=3e-4, gamma=0.99,
                             tau=0.005)


def _setup(od, D, num_envs=1, fill=20000):
    env = SyntheticGymnasiumVec(num_envs, kind="continuous", obs_dim=od, act_dim=D)
    torch.manual_seed(1)
    nets = [n.to(DEV) for n in (SACContinuousActor(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env),
                                 SoftQNetworkMLP(env), SoftQNetworkMLP(env))]
    nets[3].load_state_dict(nets[1].state_dict())
    nets[4].load_state_dict(nets[2].state_dict())
    st = SACContinuousState(*nets, DEV)
    rb = DeviceReplayRing(100000, (od,), num_envs, DEV, optimize_memory_usage=False, obs_dtype=torch.float32,
                          action_shape=(D,))
    g = np.random.default_rng(0)
    n = fill // num_envs
    rb.packed[:n].copy_(torch.from_numpy(g.standard_normal((n, num_envs, rb.width)).astype(np.float32)))
    rb.pos = n
    eager = EagerSAC(st.actor.flat.flat[:st.actor.flat.numel].clone(), st.q.flat[:st.q.numel].clone(),
                     st.qt.flat[:st.qt.numel].clone(), od, D, nets[0].action_scale, nets[0].action_bias, DEV)
    return env, st, rb, eager


def _noise(shape):
    return torch.empty(shape, device=DEV).normal_()


def _timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def update_arms(od, D, B, rounds):
    _, st, rb, eager = _setup(od, D)
    batches = [rb.sample(B) for _ in range(4)]
    step = [0]

    def arm(kind):
        def run():
            for s in (1, 2):                      # a critic-only update and one with actor steps
                step[0] += 1
                bt = batches[step[0] % 4]
                if kind == "eager_torch":
                    r = bt["rows"]
                    eager.update(s, rb.frames[r], rb.action_rows[r], rb.next_frames[r], rb.reward_rows[r], rb.done_rows[r],
                                 _noise)
                else:
                    sac_continuous_update(st, rb, bt, s, ARGS, graph=kind == "graph")
        return run

    arms = {k: arm(k) for k in ("graph", "eager_kernels", "eager_torch")}
    for f in arms.values():
        f(); f()
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            res[k].append(_timed(f, 5) / 2)
    lib = ops._lib.load()
    counts = []
    for s in (1, 2):
        c0 = lib.b200rl_launch_count()
        sac_continuous_update(st, rb, batches[0], s, ARGS, graph=False)
        counts.append(lib.b200rl_launch_count() - c0)
    torch.cuda.synchronize()
    out = {f"{k}_ms": round(float(np.median(v)), 4) for k, v in res.items()}
    out["launches_critic_only"], out["launches_with_actor"] = counts
    return out


def get_action_latency(num_envs=1, reps=200):
    env, st, _, _ = _setup(17, 6, num_envs, fill=num_envs)
    obs = np.random.default_rng(1).standard_normal((num_envs, 17)).astype(np.float32)

    def f():
        st.actor.get_action(torch.from_numpy(obs).to(DEV))[0].cpu()
    for _ in range(20):
        f()
    t = time.perf_counter()
    for _ in range(reps):
        f()
    return (time.perf_counter() - t) / reps * 1e3


def e2e_sps(steps, use_graph):
    env, st, rb, eager = _setup(17, 6, 1, fill=5000)
    np.random.seed(1)
    obs, _ = env.reset(seed=1)
    t0 = None
    for global_step in range(5000, 5000 + steps + 50):
        if global_step == 5050:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        if use_graph:
            actions = st.actor.get_action(torch.from_numpy(obs).to(DEV))[0].cpu().numpy()
        else:
            actions = eager.actor.get_action(torch.from_numpy(obs).to(DEV), _noise((1, 6)))[0].detach().cpu().numpy()
        next_obs, rewards, term, trunc, infos = env.step(actions)
        rb.add(obs, next_obs, actions, rewards, term, infos)
        obs = next_obs
        data = rb.sample(256)
        if use_graph:
            sac_continuous_update(st, rb, data, global_step, ARGS)
        else:
            r = data["rows"]
            eager.update(global_step, rb.frames[r], rb.action_rows[r], rb.next_frames[r], rb.reward_rows[r], rb.done_rows[r],
                         _noise)
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--rounds", type=int, default=20)
    p.add_argument("--e2e-steps", type=int, default=2000)
    a = p.parse_args()
    assert torch.cuda.is_available(), "bench_sac_continuous.py measures on a CUDA device"
    build.build()
    import subprocess
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": smi[0].split(",")[-1].strip() if smi else None}
    for od, D in ((17, 6), (376, 17)):
        for B in (256, 1024):
            out[f"update_obs{od}_act{D}_b{B}"] = update_arms(od, D, B, a.rounds)
    out["get_action_ms_n1"] = round(get_action_latency(1), 4)
    sps = {}
    for r in range(2):                            # alternated
        for k in (True, False):
            sps.setdefault(k, []).append(e2e_sps(a.e2e_steps, k))
    out["e2e_sps_graph"] = round(float(np.median(sps[True])), 1)
    out["e2e_sps_eager_torch"] = round(float(np.median(sps[False])), 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
