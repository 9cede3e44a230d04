"""-m gpu: the tensor-core plans' host launchers must not change a bit of what the kernels compute.

tests/golden/tc_plan_bits.json holds SHA-256 digests of the head outputs, the flat gradient and (for the LSTM agent)
h / c out, on seeded inputs, for the cases the NatureCNN pipeline bits (test_gpu_conv_pipeline.py) do not cover: NatureCNN
wide heads (A = 305, C51-sized), NatureCNN at n = 9000 (the 128-column fc tile), IMPALA-CNN and the LSTM agent.  They
were recorded with a backward workspace larger than the plan asks for, so that no write past the requested size could
touch them.  Regenerate with `python tests/test_gpu_tc_plan_bits.py` on an H100, only when a change is MEANT to alter
the arithmetic."""
import hashlib
import json
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "tc_plan_bits.json"
CASES = ([("naturecnn", fmt, 305, n) for fmt in ("u8", "u8s2d") for n in (7, 300, 4099)] + [("naturecnn", "u8s2d", 6, 9000)]
         + [("impala", None, 15, n) for n in (1, 7, 300, 2049)]
         + [("lstm", (S, n), A, None) for A in (6, 23) for S, n in ((1, 7), (4, 8), (16, 64))])


def case_id(c):
    net, shape, A, n = c
    if net == "naturecnn":
        return f"naturecnn_{shape}_A{A}_n{n}"
    if net == "impala":
        return f"impala_A{A}_n{n}"
    return f"lstm_A{A}_S{shape[0]}_n{shape[1]}"


def build_case(net, shape, A, n, dev):
    """(plan, flat params, run_forward, run_backward(grads), outputs of the forward); every input drawn on the CPU.
    NatureCNN `shape` is the obs format (u8 NCHW frames, u8s2d rollout rows, bf16s2d frames); LSTM `shape` = (S, envs)."""
    from cleanrl_b200 import ops
    g = torch.Generator().manual_seed(sum(map(ord, case_id((net, shape, A, n)))))
    if net == "naturecnn":
        plan = ops.NatureCNNBf16(A, dev)
        flat = (torch.randn(plan.param_count, generator=g) * 0.05).to(dev)
        B = n + 5
        obs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g).to(dev)
        rows = torch.randperm(B, generator=g)[:n].to(dev)
        dhead = (torch.randn(n, A + 1, generator=g) * 0.1).to(dev)
        aux = None
        if shape == "u8s2d":
            obs, aux = ops.frames_to_s2d_u8(obs)
        elif shape == "bf16s2d":
            obs = ops.frames_to_s2d(obs)
        head = torch.empty(n, A + 1, dtype=torch.float32, device=dev)
        fwd = lambda: {"head": plan.forward(obs, rows, flat, head_out=head)}
        bwd = lambda grads: plan.backward(obs, rows, flat, dhead, grads, obs_aux=aux)
    elif net == "impala":
        plan = ops.ImpalaCNNBf16(A, dev)
        flat = (torch.randn(plan.param_count, generator=g) * 0.05).to(dev)
        B = n + 3
        obs = torch.randint(0, 256, (B, 64, 64, 3), dtype=torch.uint8, generator=g).to(dev)
        rows = torch.randperm(B, generator=g)[:n].to(dev)
        dhead = (torch.randn(n, A + 1, generator=g) * 0.1).to(dev)
        head = torch.empty(n, A + 1, dtype=torch.float32, device=dev)
        fwd = lambda: {"head": plan.forward(obs, rows, flat, head_out=head)}
        bwd = lambda grads: plan.backward(obs, rows, flat, dhead, grads)
    else:
        S, envs = shape
        M = S * envs
        plan = ops.LSTMAgentBf16(A, dev)
        flat = (torch.randn(plan.param_count, generator=g) * 0.05).to(dev)
        B = M + 13
        obs = torch.randint(0, 256, (B, 1, 84, 84), dtype=torch.uint8, generator=g).to(dev)
        rows = torch.randperm(B, generator=g)[:M].to(dev)
        done = (torch.rand(M, generator=g) < 0.25).float().to(dev)
        h0 = (torch.randn(envs, 128, generator=g) * 0.5).to(dev)
        c0 = (torch.randn(envs, 128, generator=g) * 0.5).to(dev)
        dhead = (torch.randn(M, A + 1, generator=g) * 0.1).to(dev)

        def fwd():
            head, h, c = plan.forward(obs, rows, S, envs, flat, h0, c0, done)
            return {"head": head, "h_out": h, "c_out": c}
        bwd = lambda grads: plan.backward(obs, rows, S, envs, flat, done, dhead, grads)
    plan.pack(flat)
    return plan, flat, fwd, bwd


def digest(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def compute(c, dev, ws_margin=0):
    """digests of the case's outputs; `ws_margin` > 0 hands the backward a workspace that many bytes larger"""
    net, shape, A, n = c
    plan, flat, fwd, bwd = build_case(net, shape, A, n, dev)
    out = fwd()
    if ws_margin:
        key = shape if net == "lstm" else (n,)
        plan._ws = torch.empty(plan._c("workspace_bytes")(*key, A) + ws_margin, dtype=torch.uint8, device=dev)
    grads = torch.zeros(plan.param_count, dtype=torch.float32, device=dev)
    bwd(grads)
    torch.cuda.synchronize()
    out["grads"] = grads
    assert all(bool(torch.isfinite(v).all()) for v in out.values())
    return {k: digest(v) for k, v in out.items()}


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_matches_recorded_bits(lib, c):
    want = json.loads(GOLDEN.read_text())[case_id(c)]
    got = compute(c, torch.device("cuda"))
    bad = [k for k in want if got[k] != want[k]]
    assert set(got) == set(want) and not bad, f"outputs differ from the recorded bits: {bad}"


if __name__ == "__main__":
    # recipe of tests/golden/tc_plan_bits.json (run on an H100 with the build whose bits are to be recorded)
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    from cleanrl_b200 import build
    build.build()
    rec = {case_id(c): compute(c, torch.device("cuda"), ws_margin=1 << 20) for c in CASES}
    GOLDEN.write_text(json.dumps(rec, indent=1, sort_keys=True) + "\n")
    print(f"wrote {GOLDEN}")
