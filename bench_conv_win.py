#!/usr/bin/env python
"""Per-launch times of the convolutions and the fc layer of the bf16 NatureCNN (conv1 forward on the uint8 rollout, the
fused conv2 -> conv3 forward (conv23_fwd), the conv3 data gradient, the conv3 and conv2 weight gradients, conv21_bwd:
the conv2 data gradient fused with the conv1 weight gradient, and the fc Linear(3136, 512) forward, data gradient and
weight gradient) at the two batch sizes of a PPO iteration: n = 1024 (a rollout step) and n = 32 768 (a minibatch).

    python bench_conv_win.py [--reps R] [--sizes 1024,32768]

Each size runs forward + backward on uint8 space-to-depth rollout rows gathered through sorted minibatch indices (the
engine's path), with the library's per-launch CUDA-event profiler on.  Prints one JSON line: microseconds per launch
and the algorithmic bandwidth (the profiler's byte count of the launch over its time, GB/s), per size and kernel.
Nothing is written to disk."""
import argparse
import ctypes
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from cleanrl_b200 import _lib, build, ops  # noqa: E402

KERNELS = ("conv1_fwd", "conv23_fwd", "conv3_wgrad", "conv3_dgrad", "conv2_wgrad", "conv21_bwd", "fc_fwd", "fc_dgrad",
           "fc_wgrad")
# a library built before conv2 and conv3 forward were fused reports them as two launches (A/B runs against it)
OLD_NAMES = {"conv23_fwd": ("conv2_fwd", "conv3_fwd")}


def measure(lib, n, reps, dev):
    A = 4
    net = ops.NatureCNNBf16(A, dev)
    g = torch.Generator().manual_seed(n)
    flat = (torch.randn(net.param_count, generator=g) * 0.05).to(dev)
    B = 2 * n
    frames = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g).to(dev)
    obs, aux = ops.frames_to_s2d_u8(frames)
    del frames
    rows = torch.randperm(B, generator=g)[:n].sort().values.to(dev)
    dhead = (torch.randn(n, A + 1, generator=g) * 0.1).to(dev)
    grads = torch.zeros(net.param_count, dtype=torch.float32, device=dev)
    head = torch.empty(n, A + 1, dtype=torch.float32, device=dev)
    net.pack(flat)

    def step():
        net.forward(obs, rows, flat, head_out=head)
        net.backward(obs, rows, flat, dhead, grads, obs_aux=aux)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    lib.b200rl_profile_reset()
    lib.b200rl_profile_enable(1)
    for _ in range(reps):
        step()
    torch.cuda.synchronize()
    lib.b200rl_profile_enable(0)
    buf = ctypes.create_string_buffer(1 << 16)
    _lib.check(lib.b200rl_profile_summary(buf, 1 << 16), "profile_summary")
    prof = {r["name"]: r for r in json.loads(buf.value.decode())}
    names = [m for k in KERNELS for m in ((k,) if k in prof else OLD_NAMES.get(k, (k,)))]
    return {k: {"us": round(1e3 * prof[k]["ms"] / prof[k]["launches"], 2),
                "GB/s": round(prof[k]["bytes"] / (prof[k]["ms"] * 1e-3) / 1e9, 1)} for k in names}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sizes", default="1024,32768")
    a = ap.parse_args()
    build.build()
    lib = _lib.load()
    dev = torch.device("cuda:0")
    res = {"device": torch.cuda.get_device_name(dev), "unit": "us per launch, GB/s"}
    for n in (int(s) for s in a.sizes.split(",")):
        res[f"n{n}"] = measure(lib, n, a.reps, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
