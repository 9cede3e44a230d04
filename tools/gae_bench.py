"""GAE us/rollout (SURVEY.md 8d metric 2): our kernel vs the reference loop run with torch ops on the same GPU."""
import json
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from cleanrl_b200 import build, ops  # noqa: E402

build.build()


def ref_loop(r, v, d, nv, nd, gamma=0.99, lam=0.95):
    T = r.shape[0]
    adv = torch.zeros_like(r)
    last = 0
    for t in reversed(range(T)):
        if t == T - 1:
            nnt, nvs = 1.0 - nd, nv
        else:
            nnt, nvs = 1.0 - d[t + 1], v[t + 1]
        delta = r[t] + gamma * nvs * nnt - v[t]
        adv[t] = last = delta + gamma * lam * nnt * last
    return adv, adv + v


def timeit(fn, reps, flush=None):
    ts = []
    for _ in range(reps):
        if flush is not None:
            flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) * 1e3)
    return float(np.median(ts)), float(np.min(ts))


out = []
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
for T, N in [(128, 1024), (128, 4), (2048, 512), (123, 7), (128, 8192)]:
    r = torch.randint(-1, 2, (T, N), device="cuda").float()
    v = torch.randn(T, N, device="cuda")
    d = (torch.rand(T, N, device="cuda") < 0.02).float()
    nv = torch.randn(N, device="cuda")
    nd = (torch.rand(N, device="cuda") < 0.02).float()
    adv = torch.empty_like(r)
    ret = torch.empty_like(r)
    row = {"T": T, "N": N, "alg_bytes": 20 * T * N + 8 * N}
    for mode in (0, 1):
        f = lambda: ops.gae(r, v, d, nv, nd, 0.99, 0.95, mode=mode, out=(adv, ret))
        for _ in range(5):
            f()
        med, mn = timeit(f, 200)
        medc, _ = timeit(f, 50, flush)
        row[f"mode{mode}_us_warmL2"] = round(med, 2)
        row[f"mode{mode}_us_min"] = round(mn, 2)
        row[f"mode{mode}_us_coldL2"] = round(medc, 2)
        row[f"mode{mode}_GBs_cold"] = round(row["alg_bytes"] / (medc * 1e-6) / 1e9, 1)
    for _ in range(2):
        ref_loop(r, v, d, nv, nd)
    med, mn = timeit(lambda: ref_loop(r, v, d, nv, nd), 10)
    row["torch_loop_us"] = round(med, 1)
    out.append(row)
    print(json.dumps(row))
print(json.dumps(out, indent=1))
