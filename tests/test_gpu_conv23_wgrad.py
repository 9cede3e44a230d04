"""-m gpu: the conv2 and conv3 weight and bias gradients of the bf16 NatureCNN must keep their bits, from a split with a
single 128-row step up to the benchmarked 32 768-row minibatch, and must equal an fp64 sum of the same bf16 operands.

tests/golden/conv23_wgrad_bits.json holds SHA-256 digests of dW2, db2, dW3 and db3 (the flat-gradient slices, torch
layout) for seeded uint8 rollout rows.  n = 1 and 7 give splits of one step; 64, 300 and 4099 leave a partial last step
and a row count that is not a multiple of 128; 32 768 is the benchmarked minibatch.  Regenerate with
`python tests/test_gpu_conv23_wgrad.py` on an H100, only when a change is MEANT to alter the arithmetic."""
import hashlib
import json
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "conv23_wgrad_bits.json"
A = 6
# (n, rows gathered through a permutation of a larger rollout, or the rollout itself)
CASES = [(n, True) for n in (1, 7, 64, 300, 1024, 4099, 32768)] + [(300, False)]
# flat-gradient slices (NatureLayout in cleanrl_b200/csrc/net_tc.cu: conv1 w, b, conv2 w, b, conv3 w, b)
C2W, C2B = 32 * 4 * 8 * 8 + 32, 32 * 4 * 8 * 8 + 32 + 64 * 32 * 4 * 4
C3W = C2B + 64
C3B = C3W + 64 * 64 * 3 * 3
SLICES = {"dW2": (C2W, 64 * 32 * 16), "db2": (C2B, 64), "dW3": (C3W, 64 * 64 * 9), "db3": (C3B, 64)}


def case_id(n, gather):
    return f"n{n}" + ("" if gather else "_nogather")


def _setup(n, gather):
    from cleanrl_b200 import ops
    dev = torch.device("cuda")
    net = ops.NatureCNNBf16(A, dev)
    g = torch.Generator().manual_seed(3000 + n + (0 if gather else 1))
    flat = (torch.randn(net.param_count, generator=g) * 0.05).to(dev)
    B = n + 5 if gather else n
    frames = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g).to(dev)
    obs, aux = ops.frames_to_s2d_u8(frames)
    rows = torch.randperm(B, generator=g)[:n].to(dev) if gather else None
    dhead = (torch.randn(n, A + 1, generator=g) * 0.1).to(dev)
    net.pack(flat)
    grads = torch.zeros(net.param_count, dtype=torch.float32, device=dev)
    head = torch.empty(n, A + 1, dtype=torch.float32, device=dev)

    def run():
        net.forward(obs, rows, flat, head_out=head)
        net.backward(obs, rows, flat, dhead, grads, obs_aux=aux)
    return net, grads, run


def _digests(grads):
    return {k: hashlib.sha256(grads[o:o + m].contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()
            for k, (o, m) in SLICES.items()}


def _compute(n, gather):
    net, grads, run = _setup(n, gather)
    run()
    torch.cuda.synchronize()
    return _digests(grads)


def _check(got, c):
    want = json.loads(GOLDEN.read_text())[case_id(*c)]
    bad = [k for k in SLICES if got[k] != want[k]]
    assert not bad, f"{case_id(*c)}: differ from the recorded bits: {bad}"


@pytest.mark.parametrize("c", CASES, ids=lambda c: case_id(*c))
def test_conv23_wgrad_matches_recorded_bits(lib, c):
    _check(_compute(*c), c)


def test_conv23_wgrad_graph_replay_over_poisoned_workspace(lib):
    """A captured forward + backward, replayed after the backward workspace and the gradient were filled with NaN bit
    patterns, must write every element of the four gradients with the recorded bits: no partial may be read unwritten."""
    c = (1024, True)
    net, grads, run = _setup(*c)
    run()                                    # allocates the workspaces and sets the kernels' shared-memory attributes
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run()
    net.pin()
    for _ in range(2):
        net._ws.fill_(0xFF)
        grads.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        _check(_digests(grads), c)


def _views(acts, n):
    """act1, act2, dact3a, dact2a of the uint8-rollout activation workspace (NatureActs without x0)."""
    sizes = [("act1", 12800), ("act2", 5184), ("act3", 3136), ("hid", 512), ("dhid", 512), ("dact3a", 5184),
             ("dact3b", 7744), ("dact2a", 6400)]
    o, out = 0, {}
    for name, per in sizes:
        out[name] = acts[o:o + n * per]
        o += n * per
    return out


def test_conv23_wgrad_matches_fp64_sum_of_bf16_operands(lib):
    """dW and db against fp64 sums over the same bf16 operands (act1 / act2 windows and the dY grids the kernels read).
    The tolerance is a fraction of the sum of |products|: fp32 accumulation error, far below any misplaced tap,
    channel or row."""
    n = 300
    net, grads, run = _setup(n, True)
    run()
    torch.cuda.synchronize()
    v = _views(net.acts(n, 2).view(torch.bfloat16), n)
    x2 = v["act1"].view(n, 10, 10, 128).double()
    y2 = v["dact2a"].view(n, 10, 10, 64).double()[:, :9, :9]
    x3 = v["act2"].view(n, 9, 9, 64).double()
    y3 = v["dact3a"].view(n, 9, 9, 64).double()[:, :7, :7]
    ref2 = torch.zeros(64, 32, 4, 4, dtype=torch.float64, device=x2.device)
    abs2 = torch.zeros_like(ref2)
    for a in range(2):
        for b in range(2):
            xs = x2[:, a:a + 9, b:b + 9]
            s = torch.einsum("nyxq,nyxo->oq", xs, y2).view(64, 2, 2, 32)         # q = (py * 2 + px) * 32 + c
            t = torch.einsum("nyxq,nyxo->oq", xs.abs(), y2.abs()).view(64, 2, 2, 32)
            ref2[:, :, 2 * a:2 * a + 2, 2 * b:2 * b + 2] = s.permute(0, 3, 1, 2)
            abs2[:, :, 2 * a:2 * a + 2, 2 * b:2 * b + 2] = t.permute(0, 3, 1, 2)
    ref3 = torch.zeros(64, 64, 3, 3, dtype=torch.float64, device=x3.device)
    abs3 = torch.zeros_like(ref3)
    for ky in range(3):
        for kx in range(3):
            xs = x3[:, ky:ky + 7, kx:kx + 7]
            ref3[:, :, ky, kx] = torch.einsum("nyxc,nyxo->oc", xs, y3)
            abs3[:, :, ky, kx] = torch.einsum("nyxc,nyxo->oc", xs.abs(), y3.abs())
    refs = {"dW2": (ref2, abs2), "db2": (y2.sum((0, 1, 2)), y2.abs().sum((0, 1, 2))),
            "dW3": (ref3, abs3), "db3": (y3.sum((0, 1, 2)), y3.abs().sum((0, 1, 2)))}
    for k, (o, m) in SLICES.items():
        ref, mag = (t.reshape(-1) for t in refs[k])
        got = grads[o:o + m].double()
        assert float(mag.max()) > 0, k
        err = (got - ref).abs()
        assert bool((err <= 1e-4 * mag + 1e-9).all()), f"{k}: max error {float(err.max()):.3e}, largest |product| sum {float(mag.max()):.3e}"


if __name__ == "__main__":
    # recipe of tests/golden/conv23_wgrad_bits.json (run on an H100 with the build whose bits are to be recorded)
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    from cleanrl_b200 import build
    build.build()
    rec = {case_id(*c): _compute(*c) for c in CASES}
    out = Path(sys.argv[1]) if len(sys.argv) > 1 else GOLDEN
    out.write_text(json.dumps(rec, indent=1, sort_keys=True) + "\n")
    print(f"wrote {out}")
