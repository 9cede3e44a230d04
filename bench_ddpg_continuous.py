"""DDPG update (cleanrl/ddpg_continuous_action.py:214-245) on one GPU: one JSON line.

Per-update time (CUDA events, median over alternated rounds; with the default policy_frequency 2 a round is a
critic-only update and an update with the actor step and the two target updates) at B = 256 / 1024 for HalfCheetah
(17, 6) and Humanoid (376, 17) shapes, as the captured graph, as eager launches of the same kernels, and as the
reference's eager PyTorch update (oracle/ddpg_continuous_oracle.EagerDDPG, autograd + torch.optim on the same GPU); the
library launches per update; the latency of the n = 1 actor forward with its exploration draw and host copy; and env
steps per second of the drop-in's loop after ``learning_starts`` on the synthetic HalfCheetah env, with the graph update
against the eager PyTorch update.  The card's name and power limit are read in the same run.

    python bench_ddpg_continuous.py [--rounds 20] [--e2e-steps 2000]
"""
from __future__ import annotations

import argparse
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
from cleanrl_b200.agents import DDPGActor, DDPGState, SoftQNetworkMLP, ddpg_update
from cleanrl_b200.replay import DeviceReplayRing
from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
from oracle.ddpg_continuous_oracle import EagerDDPG

DEV = torch.device("cuda")
ARGS = types.SimpleNamespace(policy_frequency=2, learning_rate=3e-4, gamma=0.99, tau=0.005, exploration_noise=0.1)


def _setup(od, D, fill=20000):
    env = SyntheticGymnasiumVec(1, kind="continuous", obs_dim=od, act_dim=D)
    torch.manual_seed(1)
    nets = [n.to(DEV) for n in (DDPGActor(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env), DDPGActor(env))]
    nets[3].load_state_dict(nets[0].state_dict())
    nets[2].load_state_dict(nets[1].state_dict())
    st = DDPGState(*nets, DEV)
    rb = DeviceReplayRing(100000, (od,), 1, DEV, optimize_memory_usage=False, obs_dtype=torch.float32,
                          action_shape=(D,))
    g = np.random.default_rng(0)
    rb.packed[:fill].copy_(torch.from_numpy(g.standard_normal((fill, 1, rb.width)).astype(np.float32)))
    rb.pos = fill
    flat = lambda f: f.flat[:f.numel].clone()   # noqa: E731
    eager = EagerDDPG(flat(st.actor.flat), flat(st.q), flat(st.qt), flat(st.target_actor.flat), od, D,
                      nets[0].action_scale, nets[0].action_bias, DEV)
    return env, st, rb, eager


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
            for s in (1, 2):                      # a critic-only update and one with the actor step
                step[0] += 1
                bt = batches[step[0] % 4]
                if kind == "eager_torch":
                    r = bt["rows"]
                    eager.update(s, rb.frames[r], rb.action_rows[r], rb.next_frames[r], rb.reward_rows[r],
                                 rb.done_rows[r])
                else:
                    ddpg_update(st, rb, bt, s, ARGS, graph=kind == "graph")
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
        ddpg_update(st, rb, batches[0], s, ARGS, graph=False)
        counts.append(lib.b200rl_launch_count() - c0)
    torch.cuda.synchronize()
    out = {f"{k}_ms": round(float(np.median(v)), 4) for k, v in res.items()}
    out["launches_critic_only"], out["launches_with_actor"] = counts
    return out


def actor_latency(reps=200):
    """The drop-in's rollout action at n = 1: actor forward, the [D] exploration draw, the host copy."""
    env, st, _, _ = _setup(17, 6, fill=1)
    obs = np.random.default_rng(1).standard_normal((1, 17)).astype(np.float32)

    def f():
        a = st.actor(torch.from_numpy(obs).to(DEV))
        a += torch.normal(0, st.actor.action_scale * ARGS.exploration_noise)
        a.cpu()
    for _ in range(20):
        f()
    t = time.perf_counter()
    for _ in range(reps):
        f()
    return (time.perf_counter() - t) / reps * 1e3


def e2e_sps(steps, use_graph):
    env, st, rb, eager = _setup(17, 6, fill=5000)
    np.random.seed(1)
    obs, _ = env.reset(seed=1)
    low, high = env.single_action_space.low, env.single_action_space.high
    t0 = None
    for global_step in range(5000, 5000 + steps + 50):
        if global_step == 5050:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        x = torch.from_numpy(obs).to(DEV)
        with torch.no_grad():
            actions = st.actor(x) if use_graph else eager.actor(x)
            actions += torch.normal(0, st.actor.action_scale * ARGS.exploration_noise)
        actions = actions.cpu().numpy().clip(low, high)
        next_obs, rewards, term, trunc, infos = env.step(actions)
        rb.add(obs, next_obs, actions, rewards, term, infos)
        obs = next_obs
        data = rb.sample(256)
        if use_graph:
            ddpg_update(st, rb, data, global_step, ARGS)
        else:
            r = data["rows"]
            eager.update(global_step, rb.frames[r], rb.action_rows[r], rb.next_frames[r], rb.reward_rows[r],
                         rb.done_rows[r])
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--rounds", type=int, default=20)
    p.add_argument("--e2e-steps", type=int, default=2000)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ddpg_continuous.py measures on a CUDA device; none is visible")
    build.build()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": smi[0].split(",")[-1].strip() if smi else None}
    for od, D in ((17, 6), (376, 17)):
        for B in (256, 1024):
            out[f"update_obs{od}_act{D}_b{B}"] = update_arms(od, D, B, a.rounds)
    out["actor_action_ms_n1"] = round(actor_latency(), 4)
    sps = {}
    for _ in range(2):                            # alternated
        for k in (True, False):
            sps.setdefault(k, []).append(e2e_sps(a.e2e_steps, k))
    out["e2e_sps_graph"] = round(float(np.median(sps[True])), 1)
    out["e2e_sps_eager_torch"] = round(float(np.median(sps[False])), 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
