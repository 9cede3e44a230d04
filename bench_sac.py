"""Discrete-SAC update benchmark: one update (sample + the four steps of sac_atari.py:271-314) on a device ring of
16 384 frames in the reference's two-array layout, at batch 64 (the reference's default) and 1024, for A = 4 and 18.
Arms, alternated round by round after a warm-up of every arm: the bf16 update replayed as one CUDA graph, the same
update launched eagerly (``SACState.graph_max_batch`` picks between the two from these numbers), fp32 (CUDA-core
kernels) and the eager PyTorch restatement of the reference's update (oracle/sac_oracle.py: cuDNN trunks, torch Adam, ``alpha.item()`` every update) on the same GPU.  Times are CUDA events
around a loop of updates; each arm reports the median over rounds.  Also reports the library launches per bf16 update
and the latency of the n = 1 bf16 ``get_action`` of the rollout.  Prints one JSON line with the GPU name and power limit.

    python bench_sac.py [--steps 30] [--rounds 5] [--warmup 5]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_c51 import _envs, _gpu_info  # noqa: E402
from cleanrl_b200 import _lib  # noqa: E402
from cleanrl_b200.agents import SACActor, SACState, SoftQNetwork, sac_update  # noqa: E402
from cleanrl_b200.replay import DeviceReplayRing  # noqa: E402

RING = 16384


def _ring(dev, A):
    ring = DeviceReplayRing(RING, (4, 84, 84), 1, dev, optimize_memory_usage=False)
    ring.observations.random_(0, 256); ring.next_observations.random_(0, 256)
    ring.actions.random_(0, A); ring.rewards.normal_(); ring.dones.bernoulli_(0.02)
    ring.pos, ring.full = 0, True
    return ring


def _nets(A, dev, precision):
    nets = [SACActor(_envs(A))] + [SoftQNetwork(_envs(A)) for _ in range(4)]
    nets = [n.to(dev) for n in nets]
    nets[3].load_state_dict(nets[1].state_dict()); nets[4].load_state_dict(nets[2].state_dict())
    for n in nets:
        n.precision = precision
        n.flat
    return nets


def _time(fn, steps):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--warmup", type=int, default=5)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sac.py needs a CUDA device")
    dev = torch.device("cuda")
    torch.manual_seed(1); np.random.seed(1)
    torch.backends.cudnn.deterministic = True
    lib = _lib.load()
    out = {"metric": "sac_update_ms", "ring_frames": RING}
    for A in (4, 18):
        ring = _ring(dev, A)
        for B in (64, 1024):
            arms = {}
            for name, prec, graph in (("bf16_graph", "bf16", True), ("bf16_eager", "bf16", False), ("fp32", "fp32", False)):
                nets = _nets(A, dev, prec)
                st = SACState(A, dev)
                st.use_graph, st.graph_max_batch = graph, 1 << 30      # each arm forced, whatever the default choice
                arms[name] = (lambda nets=nets, st=st: sac_update(*nets, ring, ring.sample(B), st, 0.99, 3e-4, 3e-4))
            from oracle.sac_oracle import TorchSAC
            ref = [n.to(dev) for n in [SACActor(_envs(A))] + [SoftQNetwork(_envs(A)) for _ in range(4)]]
            eager = TorchSAC(*ref, A)
            frames, nframes = ring.frames, ring.next_frames

            def torch_arm(eager=eager):
                b = ring.sample(B)
                eager.update(frames[b["rows"]], nframes[b["next_rows"]], b["actions"], b["rewards"], b["dones"])
            arms["eager_torch"] = torch_arm
            for fn in arms.values():
                for _ in range(a.warmup):
                    fn()
            times = {k: [] for k in arms}
            for _ in range(a.rounds):
                for k, fn in arms.items():
                    times[k].append(_time(fn, a.steps))
            for k, v in times.items():
                out[f"A{A}_B{B}_{k}_ms"] = round(statistics.median(v), 4)
            torch.cuda.synchronize()
            n0 = lib.b200rl_launch_count()
            arms["bf16_eager"]()
            torch.cuda.synchronize()
            out[f"A{A}_B{B}_library_launches_per_update"] = int(lib.b200rl_launch_count() - n0)
            del arms, ref, eager
            torch.cuda.empty_cache()
        actor = _nets(A, dev, "bf16")[0]
        obs = torch.randint(0, 256, (1, 4, 84, 84), dtype=torch.uint8, device=dev)
        for _ in range(a.warmup):
            actor.get_action(obs)
        out[f"A{A}_get_action_n1_ms"] = round(statistics.median(
            [_time(lambda: actor.get_action(obs), a.steps) for _ in range(a.rounds)]), 4)
        del ring
        torch.cuda.empty_cache()
    name, power = _gpu_info()
    out["gpu"], out["power_limit"] = name, power
    print(json.dumps(out))


if __name__ == "__main__":
    main()
