#!/usr/bin/env python
"""Where a rollout step of the bf16 NatureCNN goes: one tensor-core policy step on the uint8 rollout slot (frame
conversion to space-to-depth rows, then ``NatureCNNAgent.sample_into``: conv1 on the integer tensor cores, conv2 -> conv3
in one kernel, fc, the heads and the categorical sampler), at the env batch of bench.py's rollout (n = 1024) and at the chunk sizes of
its end-to-end loop (256 and 512).

    python bench_rollout.py [--sizes 1024,512,256] [--reps 200] [--replays 2000]

Per size it reports
  * ``step_us``: the step replayed from one CUDA graph (as the engine replays it), device time per replay over
    ``--replays`` replays, no profiler;
  * ``launches``: per launch, microseconds with the library's CUDA-event profiler on (an eager pass of ``--reps`` steps),
    the bytes the profiler counts for it, and its floor: the larger of bytes over 3.35 TB/s (HBM3) and operations over
    989 TFLOP/s (dense bf16), both H100 SXM data-sheet figures, with the bound named.
Printed as one JSON line together with the card's name, its power limit and the SM clock sampled while the graph
replays.  Nothing is written to disk."""
import argparse
import ctypes
import json
import subprocess
import sys
import threading
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from cleanrl_b200 import _lib, build, ops  # noqa: E402
from cleanrl_b200.agents import NatureCNNAgent  # noqa: E402
from cleanrl_b200.synthetic_envs import SyntheticAtariVec  # noqa: E402

KERNELS = ("frames_to_s2d", "conv1_fwd", "conv23_fwd", "fc_fwd", "heads_fwd", "categorical_sample")
# a library built before conv2 and conv3 forward were fused reports them as two launches (A/B runs against it)
OLD_NAMES = {"conv23_fwd": ("conv2_fwd", "conv3_fwd")}
HBM_BPS, BF16_FLOPS = 3.35e12, 989e12


def smi(query):
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={query}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return [x.strip() for x in out.splitlines()[0].split(",")]
    except Exception:
        return None


class SmClock:
    """SM clock (MHz) sampled by nvidia-smi every 100 ms while the timed replays run."""

    def __init__(self):
        self.vals = []
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "--id=0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits",
                                          "-lms", "100"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for ln in self.proc.stdout:
            try:
                self.vals.append(float(ln.strip()))
            except ValueError:
                pass

    def stop(self):
        if self.proc is None:
            return None
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        return float(np.median(self.vals)) if self.vals else None


def measure(lib, n, reps, replays, dev):
    envs = SyntheticAtariVec(n, seed=1, mode="fresh", pool=1)          # only its spaces are used
    envs.single_observation_space, envs.single_action_space = envs.observation_space, envs.action_space
    torch.manual_seed(1)
    agent = NatureCNNAgent(envs).to(dev)
    agent.precision = "bf16"
    agent.flat
    g = torch.Generator().manual_seed(n)
    frames = torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8, generator=g).to(dev)
    rm = ops.alloc_u8_rollout_rows((n, 441, 64), dev)
    cm = torch.zeros((n, 64, 448), dtype=torch.uint8, device=dev)
    actions = torch.zeros(n, dtype=torch.int64, device=dev)
    logprobs = torch.zeros(n, dtype=torch.float32, device=dev)
    values = torch.zeros(n, dtype=torch.float32, device=dev)

    def step():
        ops.frames_to_s2d_u8(frames, rm, cm)
        agent.sample_into(rm, actions, logprobs, values)

    with torch.no_grad():
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        # per-launch times: an eager pass with the profiler's CUDA-event brackets
        lib.b200rl_profile_reset()
        lib.b200rl_profile_enable(1)
        for _ in range(reps):
            step()
        torch.cuda.synchronize()
        lib.b200rl_profile_enable(0)
        buf = ctypes.create_string_buffer(1 << 16)
        _lib.check(lib.b200rl_profile_summary(buf, 1 << 16), "profile_summary")
        prof = {r["name"]: r for r in json.loads(buf.value.decode())}
        # the step as the engine runs it: one captured graph, replayed
        agent._tc_plan()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        agent.pin_workspaces()
        for _ in range(20):
            graph.replay()
        torch.cuda.synchronize()
        clock = SmClock()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(replays):
            graph.replay()
        e1.record()
        torch.cuda.synchronize()
        sm_mhz = clock.stop()
    launches, floor_sum, eager_sum = {}, 0.0, 0.0
    for k in (m for k in KERNELS for m in ((k,) if k in prof else OLD_NAMES.get(k, (k,)))):
        r = prof[k]
        cnt = r["launches"]
        us = 1e3 * r["ms"] / cnt
        nbytes, flops = r["bytes"] / cnt, r["flops"] / cnt
        t_hbm, t_mma = 1e6 * nbytes / HBM_BPS, 1e6 * flops / BF16_FLOPS
        floor = max(t_hbm, t_mma)
        launches[k] = {"us": round(us, 2), "bytes": int(nbytes), "floor_us": round(floor, 2),
                       "bound": "hbm" if t_hbm >= t_mma else "bf16", "floor_share": round(floor / us, 3)}
        floor_sum += floor
        eager_sum += us
    return {"step_us": round(1e3 * e0.elapsed_time(e1) / replays, 2), "sm_mhz": sm_mhz,
            "eager_launch_sum_us": round(eager_sum, 2), "floor_sum_us": round(floor_sum, 2), "launches": launches}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--sizes", default="1024,512,256")
    ap.add_argument("--reps", type=int, default=200, help="eager profiled steps per size")
    ap.add_argument("--replays", type=int, default=2000, help="timed graph replays per size")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_rollout.py measures the H100 kernels: it needs a CUDA device")
    build.build()
    lib = _lib.load()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    info = smi("name,power.limit,clocks.max.sm")
    res = {"device": torch.cuda.get_device_name(dev),
           "power_limit_w": float(info[1]) if info else None, "sm_max_mhz": float(info[2]) if info else None,
           "unit": "us per step / per launch"}
    for n in (int(s) for s in a.sizes.split(",")):
        res[f"n{n}"] = measure(lib, n, a.reps, a.replays, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
