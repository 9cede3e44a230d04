"""-m gpu: the fc layer of the bf16 NatureCNN (Linear(3136, 512) on tc_gemm_tma forward and data gradient, tc_wgrad_tma +
tc_fold_fc weight gradient) must stay bit-identical across changes to how those kernels tile and schedule their work:
at the batch sizes of a PPO iteration (n = 1024, a rollout step, and n = 32 768, a minibatch) and on both sides of the
n <= 8192 switch to the narrower forward tiles.

tests/golden/fc_gemm_bits.json holds SHA-256 digests of the hidden layer, its ReLU mask words, d(act3) on the 9x9 grid
and on the zero-padded 11x11 grid, the fc weight and bias gradients and the whole flat gradient for seeded inputs.  A
second test captures forward + backward as a CUDA graph, poisons the backward workspace and checks that the replay
reproduces the eager bits.  Regenerate with `python tests/test_gpu_fc_gemm_bits.py` on an H100, only when a change is
MEANT to alter the arithmetic."""
import hashlib
import json
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "fc_gemm_bits.json"
SIZES = (1024, 8192, 8193, 32768)
A = 4
FCW = 32 * 4 * 8 * 8 + 32 + 64 * 32 * 4 * 4 + 64 + 64 * 64 * 3 * 3 + 64    # NatureLayout.fcw; the bias follows


def _digest(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def _setup(n):
    from cleanrl_b200 import ops
    from cleanrl_b200.ops import NatureCNNBf16
    dev = torch.device("cuda")
    net = NatureCNNBf16(A, dev)
    g = torch.Generator().manual_seed(5000 + n)
    flat = (torch.randn(net.param_count, generator=g) * 0.05).to(dev)
    B = n + 5
    obs, aux = ops.frames_to_s2d_u8(torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g).to(dev))
    rows = torch.randperm(B, generator=g)[:n].sort().values.to(dev)
    dhead = (torch.randn(n, A + 1, generator=g) * 0.1).to(dev)
    grads = torch.zeros(net.param_count, dtype=torch.float32, device=dev)
    head = torch.empty(n, A + 1, dtype=torch.float32, device=dev)
    net.pack(flat)

    def step():
        net.forward(obs, rows, flat, head_out=head)
        net.backward(obs, rows, flat, dhead, grads, obs_aux=aux)
    return net, grads, step


def _outputs(net, n, grads):
    # NatureActs of the uint8 rollout (no x0), bf16 element offsets
    acts = net.acts(n, 2).view(torch.bfloat16)
    hid = n * (12800 + 5184 + 3136)
    dact3a = hid + 2 * n * 512
    dact3b = dact3a + n * 5184
    pad8 = lambda v: (v + 7) & ~7                                               # noqa: E731
    m4 = dact3b + n * (7744 + 6400 + 7744 + 14112) + pad8(n * 800) + pad8(n * 324) + pad8(n * 196)
    return {"hid": _digest(acts[hid:hid + n * 512]), "m4": _digest(acts[m4:m4 + n * 32]),
            "dact3a": _digest(acts[dact3a:dact3a + n * 5184]), "dact3b": _digest(acts[dact3b:dact3b + n * 7744]),
            "fc_w": _digest(grads[FCW:FCW + 512 * 3136]), "fc_b": _digest(grads[FCW + 512 * 3136:FCW + 512 * 3137]),
            "grads": _digest(grads)}


def _compute(n):
    net, grads, step = _setup(n)
    step()
    torch.cuda.synchronize()
    return _outputs(net, n, grads)


@pytest.mark.parametrize("n", SIZES)
def test_fc_gemm_matches_recorded_bits(lib, n):
    want = json.loads(GOLDEN.read_text())[f"n{n}"]
    got = _compute(n)
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, f"outputs differ from the recorded bits: {bad}"


@pytest.mark.parametrize("n", (1024, 8193))
def test_fc_gemm_graph_replay_after_poisoned_workspace(lib, n):
    net, grads, step = _setup(n)
    step()                                   # eager: allocates the workspaces the graph will reference
    torch.cuda.synchronize()
    want = _outputs(net, n, grads)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            step()
    torch.cuda.current_stream().wait_stream(s)
    net.pin()
    ws = net.workspace(n)
    ws.fill_(0xFF)                           # every partial the backward reads must be one it wrote
    grads.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    got = _outputs(net, n, grads)
    assert got == want, {k: got[k] == want[k] for k in got}


if __name__ == "__main__":
    # recipe of tests/golden/fc_gemm_bits.json (run on an H100 with the build whose bits are to be recorded)
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    from cleanrl_b200 import build
    build.build()
    rec = {f"n{n}": _compute(n) for n in SIZES}
    out = Path(sys.argv[1]) if len(sys.argv) > 1 else GOLDEN
    out.parent.mkdir(parents=True, exist_ok=True)
    out.write_text(json.dumps(rec, indent=1, sort_keys=True) + "\n")
    print(f"wrote {out}")
