"""C51 update benchmark: replay-ring sample + C51 update at batch 8192 on a ring of 65 536 frames, bf16 tensor-core
network, n_atoms = 51, for A = 4 (Breakout) and A = 18 (full action set).  In the same run it times the DQN update at
the same batch and a few updates of the eager torch restatement of the reference's update (oracle/c51_oracle.py, with
its per-row index_add_ loop) on the same GPU.  Times are CUDA events around a warmed-up loop.  Prints one JSON line
with the GPU name and power limit.

    python bench_c51.py [--batch 8192] [--steps 20] [--warmup 3] [--eager-steps 3]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from cleanrl_b200.agents import C51QNetwork, QNetworkAgent, c51_update, dqn_update  # noqa: E402
from cleanrl_b200.replay import DeviceReplayRing  # noqa: E402
from cleanrl_b200.synthetic_envs import Box, Discrete  # noqa: E402

RING = 65536
N_ATOMS = 51


def _envs(A):
    class E:
        single_observation_space = Box(0, 255, (4, 84, 84), np.uint8)
        single_action_space = Discrete(A)
    return E()


def _ring(dev, A):
    ring = DeviceReplayRing(RING, (4, 84, 84), 1, dev)
    ring.observations.random_(0, 256)
    ring.actions.random_(0, A); ring.rewards.normal_(); ring.dones.bernoulli_(0.02)
    ring.pos, ring.full = 0, True
    return ring


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(), "unknown"
    return name, power


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batch", type=int, default=8192)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--eager-steps", type=int, default=3)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_c51.py needs a CUDA device")
    dev = torch.device("cuda")
    torch.manual_seed(1); np.random.seed(1)
    B = a.batch
    out = {"metric": "c51_update_ms", "batch": B, "ring_frames": RING, "n_atoms": N_ATOMS, "precision": "bf16"}
    for A in (4, 18):
        ring = _ring(dev, A)
        q = C51QNetwork(_envs(A), n_atoms=N_ATOMS, v_min=-10, v_max=10).to(dev)
        t = C51QNetwork(_envs(A), n_atoms=N_ATOMS, v_min=-10, v_max=10).to(dev)
        q.precision = t.precision = "bf16"
        t.load_state_dict(q.state_dict())
        stats = torch.zeros(2, device=dev)
        out[f"c51_A{A}_ms"] = round(_time(lambda: c51_update(q, t, ring, ring.sample(B), 0.99, 2.5e-4, -10.0, 10.0, B,
                                                              stats=stats), a.steps, a.warmup), 3)
        assert np.isfinite(stats.cpu().numpy()).all()
        qd = QNetworkAgent(_envs(A)).to(dev)
        td = QNetworkAgent(_envs(A)).to(dev)
        qd.precision = td.precision = "bf16"
        td.load_state_dict(qd.state_dict())
        out[f"dqn_A{A}_ms"] = round(_time(lambda: dqn_update(qd, td, ring, ring.sample(B), 0.99, 1e-4, stats=stats),
                                          a.steps, a.warmup), 3)
        # eager torch restatement of the reference update (cuDNN trunk, per-row index_add_ loop, torch Adam)
        from oracle.c51_oracle import torch_update_loss
        torch.backends.cudnn.deterministic = True
        qe = C51QNetwork(_envs(A), n_atoms=N_ATOMS, v_min=-10, v_max=10).network.to(dev)
        te = C51QNetwork(_envs(A), n_atoms=N_ATOMS, v_min=-10, v_max=10).network.to(dev)
        atoms = torch.linspace(-10, 10, N_ATOMS, device=dev)
        opt = torch.optim.Adam(qe.parameters(), lr=2.5e-4, eps=0.01 / B)
        frames = ring.frames

        def eager():
            batch = ring.sample(B)
            obs, nxt = frames[batch["rows"]].float(), frames[batch["next_rows"]].float()
            with torch.no_grad():
                nl = te(nxt / 255.0)
            loss, _, _ = torch_update_loss(qe(obs / 255.0), nl, atoms, batch["actions"], batch["rewards"], batch["dones"],
                                           0.99, -10.0, 10.0, N_ATOMS)
            opt.zero_grad()
            loss.backward()
            opt.step()
        out[f"eager_A{A}_ms"] = round(_time(eager, a.eager_steps, 1), 3)
        del q, t, qd, td, qe, te, opt, ring
        torch.cuda.empty_cache()
    name, power = _gpu_info()
    out["gpu"], out["power_limit"] = name, power
    print(json.dumps(out))


if __name__ == "__main__":
    main()
