"""Config 5 micro-benchmark: replay-ring sample + TD update at batch 8192 (BASELINE.json configs[4]).
Ring of 65536 frames resident in HBM; reports ms per (sample + update) and the reference-style host path
(numpy fancy-index gather of 2 x 231 MB + H2D) for comparison."""
import json
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
from cleanrl_b200 import build  # noqa: E402
from cleanrl_b200.agents import QNetworkAgent, dqn_update  # noqa: E402
from cleanrl_b200.replay import DeviceReplayRing  # noqa: E402
from cleanrl_b200.synthetic_envs import Box, Discrete  # noqa: E402

build.build()
B = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
SIZE = 65536


class E:
    single_observation_space = Box(0, 255, (4, 84, 84), np.uint8)
    single_action_space = Discrete(4)


dev = torch.device("cuda:0")
torch.manual_seed(1); np.random.seed(1)
out = {}
for precision in ("bf16", "fp32"):
    q, t = QNetworkAgent(E()).to(dev), QNetworkAgent(E()).to(dev)
    q.precision = t.precision = precision
    t.load_state_dict(q.state_dict())
    ring = DeviceReplayRing(SIZE, (4, 84, 84), 1, dev)
    ring.observations.random_(0, 256)
    ring.actions.random_(0, 4); ring.rewards.normal_(); ring.dones.bernoulli_(0.02)
    ring.pos, ring.full = 0, True
    stats = torch.zeros(2, device=dev)
    reps = 10 if precision == "bf16" else 2
    for _ in range(2):
        dqn_update(q, t, ring, ring.sample(B), 0.99, 1e-4, stats=stats)
    torch.cuda.synchronize()
    t0 = time.time()
    for _ in range(reps):
        dqn_update(q, t, ring, ring.sample(B), 0.99, 1e-4, stats=stats)
    torch.cuda.synchronize()
    ms = (time.time() - t0) / reps * 1e3
    flops = 4 * 2 * 9345536 * B   # target fwd + online fwd + bwd (2x)
    out[precision] = {"ms_per_sample_plus_update": round(ms, 3), "tflops": round(flops / (ms * 1e-3) / 1e12, 1),
                      "transitions_per_s": round(B / (ms * 1e-3))}
    del q, t, ring
    torch.cuda.empty_cache()
# reference-style host gather + H2D of the same batch (cleanrl_utils/buffers.py:397-415 data movement only)
host = np.random.randint(0, 256, (SIZE, 1, 4, 84, 84), dtype=np.uint8)
bi = np.random.randint(0, SIZE, B)
t0 = time.time()
for _ in range(3):
    o = torch.tensor(host[bi, 0], device=dev); n = torch.tensor(host[(bi + 1) % SIZE, 0], device=dev)
torch.cuda.synchronize()
out["reference_host_gather_h2d_ms"] = round((time.time() - t0) / 3 * 1e3, 2)
out["batch"] = B
print(json.dumps(out))
