"""Benchmark of cleanrl_b200/ppg_procgen.py: one policy iteration and the auxiliary phase, fp32 and bf16 alternating, next
to an eager-PyTorch restatement of the auxiliary minibatch update on the same GPU.

    python bench_ppg.py [--sizes 64x256x32,512x256x4] [--window-seconds 2]

A size is num_envs x num_steps x n_iteration.  The auxiliary buffer is filled directly with seeded synthetic frames,
returns and old logits (not by n_iteration rollouts).  The replayed bf16 arm (the drop-in's default) runs the WHOLE auxiliary phase (old-policy pass +
e_auxiliary epochs); every arm, and the bf16 update replayed as one CUDA graph, is also timed over windows of ``--window-seconds`` of auxiliary
minibatch updates, alternating, and
the fp32 / eager-PyTorch phase figures are those per-update times scaled to the phase's update count (``*_extrapolated``).
TFLOP/s are network arithmetic counted from shapes (61.2 MFLOP per forward sample, backward = 2x forward).  Prints one
JSON line with the GPU name, its power limit and the SM clocks sampled during the timed windows.
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
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench import ClockSampler  # noqa: E402
from bench_c51 import _gpu_info  # noqa: E402
from bench_procgen import MFLOP_PER_SAMPLE  # noqa: E402
from cleanrl_b200 import _lib, cli  # noqa: E402
from cleanrl_b200.agents import PPGAgent  # noqa: E402
from cleanrl_b200.ppg_engine import PPGEngine  # noqa: E402
from cleanrl_b200.synthetic_envs import SyntheticProcgenVec  # noqa: E402

A = 15


def _args(N, T, n_iteration, precision):
    a = cli.ppg_procgen_args()()
    a.num_envs, a.num_steps, a.n_iteration, a.precision = N, T, n_iteration, precision
    a.batch_size = N * T
    a.minibatch_size = a.batch_size // a.num_minibatches
    a.aux_batch_rollouts = N * n_iteration
    return a


def _fill(eng, seed=5):
    """Seeded synthetic buffer contents, generated on the device in slices."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    for t in range(eng.T):
        eng.aux_obs[t].copy_(torch.randint(0, 256, eng.aux_obs[t].shape, dtype=torch.uint8, device="cuda", generator=g))
    eng.aux_returns.copy_(torch.randn(eng.aux_returns.shape, device="cuda", generator=g))
    lg = torch.randn(eng.aux_pi.shape, device="cuda", generator=g) * 0.1
    eng.aux_pi.copy_(lg - lg.logsumexp(-1, keepdim=True))


class Arm:
    """One precision of the drop-in: a PPGEngine on the synthetic procgen env with a filled auxiliary buffer."""

    def __init__(self, N, T, n_iteration, precision, dev, replay=False, share=None):
        torch.manual_seed(1); np.random.seed(1)
        self.replay = replay
        self.env = SyntheticProcgenVec(N, seed=3)
        self.agent = PPGAgent(self.env).to(dev)
        self.agent.precision = precision
        self.eng = PPGEngine(self.agent, _args(N, T, n_iteration, precision), (64, 64, 3), N, dev, gae_mode=1)
        self.T, self.N = T, N
        self.obs, self.done = self.env.reset(), np.zeros(N, dtype=np.float32)
        if share is None:
            _fill(self.eng)
        else:                                              # read the other arm's auxiliary buffer instead of a second copy
            e = self.eng
            e.aux_obs, e.aux_returns, e.aux_pi = share.eng.aux_obs, share.eng.aux_returns, share.eng.aux_pi
            torch.cuda.empty_cache()
        self.cols = torch.arange(self.eng.Na, device=dev, dtype=torch.int64)
        self.k = 0

    def policy_iteration(self):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for t in range(self.T):
            a = self.eng.policy_step(t, self.obs, self.done)
            self.obs, r, d, _ = self.env.step(a.copy())
            self.eng.record_reward(t, np.asarray(r, dtype=np.float32))
            self.done = np.asarray(d, dtype=np.float32)
        self.eng.finish_rollout(self.obs, self.done)
        st = self.eng.update(5e-4)
        self.eng.store_rollout(1)
        torch.cuda.synchronize()
        assert np.isfinite(st["per_update"]).all()
        return (time.perf_counter() - t0) * 1e3

    def aux_updates(self, count):
        """``count`` auxiliary minibatch updates (forward, fused loss, backward, clip + Adam); ms per update."""
        e = self.eng
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if self.replay:
            e._aux_step_table(5e-4, min(count, e.aux_hyper.shape[0]))
        for j in range(count):
            start = (self.k * e.R) % e.Na
            if self.replay:
                e.aux_minibatch_replayed(self.cols[start:start + e.R], e.aux_hyper[j % e.aux_hyper.shape[0]], e.aux_stats[0])
            else:
                e.aux_minibatch(self.cols[start:start + e.R], 5e-4, e.aux_stats[0], True)
            self.k += 1
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / count

    def aux_phase(self):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = self.eng.aux_phase(5e-4)
        torch.cuda.synchronize()
        assert np.isfinite(out["per_minibatch"]).all()
        return (time.perf_counter() - t0) * 1e3


class _TorchNet(nn.Module):
    """The IMPALA-CNN with PPG's three heads in eager PyTorch (autograd, cuDNN): what a user of the reference runs."""

    def __init__(self):
        super().__init__()
        self.convs = nn.ModuleList()
        cin = 3
        for c in (16, 32, 32):
            self.convs.append(nn.ModuleList([nn.Conv2d(cin, c, 3, padding=1)] + [nn.Conv2d(c, c, 3, padding=1) for _ in range(4)]))
            cin = c
        self.fc = nn.Linear(2048, 256)
        self.actor, self.critic, self.aux_critic = nn.Linear(256, A), nn.Linear(256, 1), nn.Linear(256, 1)

    def forward(self, x):
        h = x.permute(0, 3, 1, 2) / 255.0
        for conv, a0, a1, b0, b1 in self.convs:
            h = F.max_pool2d(conv(h), 3, 2, 1)
            h = h + a1(F.relu(a0(F.relu(h))))
            h = h + b1(F.relu(b0(F.relu(h))))
        hid = F.relu(self.fc(F.relu(h.flatten(1))))
        return self.actor(hid), self.critic(hid.detach()), self.aux_critic(hid)


class TorchArm:
    def __init__(self, eng, dev):
        torch.manual_seed(1)
        self.e, self.net = eng, _TorchNet().to(dev)
        self.opt = torch.optim.Adam(self.net.parameters(), lr=5e-4, eps=1e-8)
        self.cols = torch.arange(eng.Na, device=dev, dtype=torch.int64)
        self.k = 0

    def aux_updates(self, count):
        from torch import distributions as td
        e = self.e
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(count):
            start = (self.k * e.R) % e.Na
            cols = self.cols[start:start + e.R]
            obs = e.aux_obs[:, cols].reshape(-1, 64, 64, 3).float()
            ret = e.aux_returns[:, cols].reshape(-1)
            old = td.Categorical(logits=e.aux_pi[:, cols].reshape(-1, A))
            lg, v, av = self.net(obs)
            kl = td.kl_divergence(old, td.Categorical(logits=lg)).mean()
            loss = 0.5 * ((av.view(-1) - ret) ** 2).mean() + kl + 0.5 * ((v.view(-1) - ret) ** 2).mean()
            loss.backward()
            nn.utils.clip_grad_norm_(self.net.parameters(), 0.5)
            self.opt.step()
            self.opt.zero_grad()
            self.k += 1
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / count


def _profile(arm, count=8):
    lib = _lib.load()
    lib.b200rl_profile_reset()
    lib.b200rl_profile_enable(1)
    arm.aux_updates(count)
    torch.cuda.synchronize()
    lib.b200rl_profile_enable(0)
    buf = ctypes.create_string_buffer(1 << 16)
    _lib.check(lib.b200rl_profile_summary(buf, 1 << 16), "profile_summary")
    return json.loads(buf.value.decode())


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--sizes", default="64x256x32,512x256x4")
    p.add_argument("--window-seconds", type=float, default=2.0, help="length of one timed window of auxiliary updates")
    p.add_argument("--rounds", type=int, default=3, help="timed windows per arm, alternating")
    p.add_argument("--policy-iters", type=int, default=3)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ppg.py needs a CUDA device")
    dev = torch.device("cuda")
    out = {"metric": "ppg_procgen_ms", "e_auxiliary": 6, "num_aux_rollouts": 4, "window_seconds": a.window_seconds, "rounds": a.rounds}
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    for size in a.sizes.split(","):
        N, T, n_it = (int(x) for x in size.split("x"))
        os.environ["CLEANRL_B200_PPG_AUX_GRAPH"] = "0"     # the fp32 / bf16 arms launch every update eagerly
        arms = {prec: Arm(N, T, n_it, prec, dev) for prec in ("fp32", "bf16")}
        torch_arm = TorchArm(arms["bf16"].eng, dev)
        # the same bf16 update replayed as one CUDA graph, on its own engine (the bf16 arm above launches eagerly)
        os.environ["CLEANRL_B200_PPG_AUX_GRAPH"] = "1"
        replay_arm = Arm(N, T, n_it, "bf16", dev, replay=True, share=arms["bf16"])
        every = dict(arms, bf16_replay=replay_arm, torch_eager=torch_arm)
        for arm in arms.values():                          # warm up every shape the timed windows use
            arm.policy_iteration()
        replay_arm.eng.aux_minibatch(replay_arm.cols[:replay_arm.eng.R], 5e-4, replay_arm.eng.aux_stats[0], True)
        counts = {}
        for k, arm in every.items():                       # warm up, then size each arm's window by time
            arm.aux_updates(3)
            counts[k] = max(8, int(a.window_seconds * 1e3 / arm.aux_updates(8)))
        replay_arm.eng.old_policy_pass()
        pol = {prec: [] for prec in arms}
        upd = {k: [] for k in every}
        sampler.mark_begin()
        for _ in range(a.policy_iters):
            for prec, arm in arms.items():
                pol[prec].append(arm.policy_iteration())
        for _ in range(a.rounds):
            for k, arm in every.items():
                upd[k].append(arm.aux_updates(counts[k]))
        phase_ms = replay_arm.aux_phase()                  # the drop-in's default path for bf16
        sampler.mark_end()
        e = arms["bf16"].eng
        rows = T * e.R
        n_upd = 6 * (e.Na // e.R)
        samples = T * e.Na
        flop_upd = MFLOP_PER_SAMPLE * 1e6 * 3 * rows
        flop_phase = MFLOP_PER_SAMPLE * 1e6 * samples * (1 + 6 * 3)
        flop_pol = MFLOP_PER_SAMPLE * 1e6 * N * T * (1 + 3)
        res = {"aux_minibatch_rows": rows, "aux_updates_per_phase": n_upd, "aux_buffer_gib": round(samples * 12288 / 2**30, 2)}
        for k in every:
            ms = float(np.median(upd[k]))
            res[k] = {"aux_update_ms": round(ms, 3), "updates_per_window": counts[k], "aux_update_windows_ms": [round(x, 3) for x in upd[k]],
                      "aux_samples_per_s": round(rows / ms * 1e3, 1), "aux_update_network_tflops": round(flop_upd / (ms * 1e-3) / 1e12, 2),
                      "aux_phase_ms_extrapolated": round(ms * n_upd, 1)}
        for prec in arms:
            ms = float(np.median(pol[prec]))
            res[prec].update({"policy_iteration_ms": round(ms, 2), "policy_env_steps_per_s": round(N * T / ms * 1e3, 1),
                              "policy_network_tflops": round(flop_pol / (ms * 1e-3) / 1e12, 2),
                              "aux_kernels_ms": _profile(arms[prec])})
        res["bf16_replay"].update({"aux_phase_ms": round(phase_ms, 1), "aux_phase_samples_per_s": round(samples * 6 / phase_ms * 1e3, 1),
                            "aux_phase_network_tflops": round(flop_phase / (phase_ms * 1e-3) / 1e12, 2)})
        out[size] = res
        del arms, torch_arm, replay_arm, every
        torch.cuda.empty_cache()
    out["clocks"] = sampler.stop()
    out["gpu"], out["power_limit"] = _gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
