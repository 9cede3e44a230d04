"""-m gpu: the backward of the bf16 NatureCNN on the uint8 space-to-depth rollout must stay bit-identical where the conv2
data gradient and the conv1 weight gradient split their work unevenly: batch sizes just below and above multiples of the
132 row splits, splits that own one or two images, and both sorted and unsorted minibatch gathers.

tests/golden/conv21_bwd_bits.json holds SHA-256 digests of d(act1) (fp16 x 2^12), the conv1 weight and bias gradients
and the whole flat gradient for seeded inputs.  A second test captures forward + backward as a CUDA graph, poisons the
backward workspace and checks that the replay reproduces the eager bits.  Regenerate with
`python tests/test_gpu_conv21_bwd_bits.py` on an H100, only when a change is MEANT to alter the arithmetic."""
import hashlib
import json
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "conv21_bwd_bits.json"
SIZES = (131, 133, 265, 4097, 8191)
ORDERS = ("sorted", "unsorted")
A = 6
C1 = 32 * 4 * 8 * 8           # conv1 weight elements; the bias follows (NatureLayout)


def _digest(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def _setup(n, order):
    from cleanrl_b200 import ops
    from cleanrl_b200.ops import NatureCNNBf16
    dev = torch.device("cuda")
    net = NatureCNNBf16(A, dev)
    g = torch.Generator().manual_seed(3000 + n + (order == "sorted"))
    flat = (torch.randn(net.param_count, generator=g) * 0.05).to(dev)
    B = n + 7
    obs, aux = ops.frames_to_s2d_u8(torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g).to(dev))
    rows = torch.randperm(B, generator=g)[:n]
    if order == "sorted":
        rows = rows.sort().values
    rows = rows.to(dev)
    dhead = (torch.randn(n, A + 1, generator=g) * 0.1).to(dev)
    grads = torch.zeros(net.param_count, dtype=torch.float32, device=dev)
    head = torch.empty(n, A + 1, dtype=torch.float32, device=dev)
    net.pack(flat)

    def step():
        net.forward(obs, rows, flat, head_out=head)
        net.backward(obs, rows, flat, dhead, grads, obs_aux=aux)
    return net, grads, step


def _outputs(net, n, grads):
    acts = net.acts(n, 2).view(torch.bfloat16)
    o = n * (12800 + 5184 + 3136 + 512 + 512 + 5184 + 7744 + 6400 + 7744)   # NatureActs.dact1 (no x0)
    return {"dact1": _digest(acts[o:o + n * 14112]), "conv1_w": _digest(grads[:C1]), "conv1_b": _digest(grads[C1:C1 + 32]),
            "grads": _digest(grads)}


def _compute(n, order):
    net, grads, step = _setup(n, order)
    step()
    torch.cuda.synchronize()
    return _outputs(net, n, grads)


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("n", SIZES)
def test_conv21_bwd_matches_recorded_bits(lib, n, order):
    want = json.loads(GOLDEN.read_text())[f"{order}_n{n}"]
    got = _compute(n, order)
    bad = [k for k in ("dact1", "conv1_w", "conv1_b", "grads") if got[k] != want[k]]
    assert not bad, f"outputs differ from the recorded bits: {bad}"


@pytest.mark.parametrize("n", (133, 4097))
def test_conv21_bwd_graph_replay_after_poisoned_workspace(lib, n):
    net, grads, step = _setup(n, "unsorted")
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
    # recipe of tests/golden/conv21_bwd_bits.json (run on an H100 with the build whose bits are to be recorded)
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    from cleanrl_b200 import build
    build.build()
    rec = {f"{order}_n{n}": _compute(n, order) for order in ORDERS for n in SIZES}
    out = Path(sys.argv[1]) if len(sys.argv) > 1 else GOLDEN
    out.parent.mkdir(parents=True, exist_ok=True)
    out.write_text(json.dumps(rec, indent=1, sort_keys=True) + "\n")
    print(f"wrote {out}")
