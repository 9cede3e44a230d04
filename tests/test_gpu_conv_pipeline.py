"""-m gpu: the bf16 NatureCNN forward and backward must stay bit-identical across kernel pipeline changes.

tests/golden/naturecnn_bf16_bits.json holds SHA-256 digests of the raw bytes of the head outputs, the conv activations
and every parameter gradient for seeded inputs at n in {1, 7, 300, 4099} (4099 leaves a partial last row split in the
conv weight gradients), for both the uint8 NCHW frames (bf16 conv1 window kernels) and the uint8 space-to-depth rollout
rows the engine stores (integer conv1 kernels); tests/golden/naturecnn_bf16_slices.npz holds some of those tensors at
n in {1, 7}.  Both were recorded with the kernels before the conv pipeline changes.  Regenerate them with
`python tests/test_gpu_conv_pipeline.py` on an H100, only when a change is MEANT to alter the arithmetic.

The same passes must also repeat bit for bit, and must give the same bits when replayed from a CUDA graph."""
import hashlib
import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "naturecnn_bf16_bits.json"
# the tensors themselves at the small sizes (head outputs, bias gradients, the first 1024 entries of every conv weight
# gradient): a mismatch then shows where and by how much the results differ
SLICES = Path(__file__).resolve().parent / "golden" / "naturecnn_bf16_slices.npz"
SLICE_SIZES = (1, 7)
SIZES = (1, 7, 300, 4099)
FORMATS = ("u8", "u8s2d")
A = 6


def _case(n, fmt, dev):
    """Seeded parameters, observations, minibatch gather and head gradient (all drawn on the CPU)."""
    from cleanrl_b200 import ops
    from cleanrl_b200.ops import NatureCNNBf16
    net = NatureCNNBf16(A, dev)
    g = torch.Generator().manual_seed(1000 + n)
    flat = (torch.randn(net.param_count, generator=g) * 0.05).to(dev)
    B = n + 5
    obs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g).to(dev)
    rows = torch.randperm(B, generator=g)[:n].to(dev)
    dhead = (torch.randn(n, A + 1, generator=g) * 0.1).to(dev)
    aux = None
    if fmt == "u8s2d":
        obs, aux = ops.frames_to_s2d_u8(obs)
    net.pack(flat)
    grads = torch.zeros(net.param_count, dtype=torch.float32, device=dev)
    head = torch.empty(n, A + 1, dtype=torch.float32, device=dev)
    return net, flat, obs, rows, dhead, aux, grads, head


def _run(net, flat, obs, rows, dhead, aux, grads, head):
    net.forward(obs, rows, flat, head_out=head)
    net.backward(obs, rows, flat, dhead, grads, obs_aux=aux)


def _outputs(net, n, fmt, grads, head):
    """Named byte views: head outputs, act1/act2/act3 of the workspace, and the flat gradient."""
    acts = net.acts(n, 0 if fmt == "u8" else 2).view(torch.bfloat16)
    o = n * 28224 if fmt == "u8" else 0           # uint8 NCHW input: the workspace starts with the space-to-depth frames
    out = {"head": head, "grads": grads}
    for name, size in (("act1", 12800), ("act2", 5184), ("act3", 3136)):
        out[name] = acts[o:o + n * size]
        o += n * size
    return {k: v.detach().clone() for k, v in out.items()}


def _slices(out):
    """name -> small fp32 array taken from the outputs (offsets of the flat parameter layout, include/b200rl.h)."""
    g = out["grads"].cpu().numpy()
    offs = {"c1w": 0, "c1b": 8192, "c2w": 8224, "c2b": 40992, "c3w": 41056, "c3b": 77920}
    res = {"head": out["head"].cpu().numpy(), "c1b": g[8192:8224], "c2b": g[40992:41056], "c3b": g[77920:77984]}
    for k in ("c1w", "c2w", "c3w"):
        res[k] = g[offs[k]:offs[k] + 1024]
    return res


def _digest(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def _compute(n, fmt, dev):
    case = _case(n, fmt, dev)
    _run(*case)
    torch.cuda.synchronize()
    return case, _outputs(case[0], n, fmt, case[6], case[7])


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("n", SIZES)
def test_matches_recorded_bits(lib, n, fmt):
    want = json.loads(GOLDEN.read_text())[f"{fmt}_n{n}"]
    _, got = _compute(n, fmt, torch.device("cuda"))
    assert bool(torch.isfinite(got["grads"]).all()) and bool(torch.isfinite(got["head"]).all())
    if n in SLICE_SIZES:
        rec = np.load(SLICES)
        for k, v in _slices(got).items():
            w = rec[f"{fmt}_n{n}_{k}"]
            assert np.array_equal(v, w), f"{k}: max |diff| {np.abs(v.astype(np.float64) - w).max():.3e}"
    bad = [k for k, v in got.items() if _digest(v) != want[k]]
    assert not bad, f"outputs differ from the recorded bits: {bad}"


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("n", (7, 4099))
def test_repeat_and_graph_replay_bit_identical(lib, n, fmt):
    dev = torch.device("cuda")
    case, first = _compute(n, fmt, dev)
    net, grads, head = case[0], case[6], case[7]
    grads.fill_(float("nan")); head.fill_(float("nan"))
    _run(*case)
    torch.cuda.synchronize()
    again = _outputs(net, n, fmt, grads, head)
    for k in first:
        assert torch.equal(first[k], again[k]), f"repeat differs: {k}"
    # capture forward + backward (the workspaces exist already) and replay into poisoned outputs
    net.pin()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            _run(*case)
    torch.cuda.current_stream().wait_stream(side)
    grads.fill_(float("nan")); head.fill_(float("nan"))
    # poison exactly the act1..act3 bytes that _outputs reads
    acts = net.acts(n, 0 if fmt == "u8" else 2)
    o = n * 28224 * 2 if fmt == "u8" else 0
    acts[o:o + n * (12800 + 5184 + 3136) * 2].fill_(0xFF)
    graph.replay()
    torch.cuda.synchronize()
    replayed = _outputs(net, n, fmt, grads, head)
    for k in first:
        assert torch.equal(first[k], replayed[k]), f"graph replay differs: {k}"


if __name__ == "__main__":
    # recipe of tests/golden/naturecnn_bf16_bits.json and naturecnn_bf16_slices.npz (run on an H100 with the build whose bits are to be recorded)
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    from cleanrl_b200 import build
    build.build()
    dev = torch.device("cuda")
    rec, arrs = {}, {}
    for fmt in FORMATS:
        for n in SIZES:
            _, out = _compute(n, fmt, dev)
            rec[f"{fmt}_n{n}"] = {k: _digest(v) for k, v in out.items()}
            if n in SLICE_SIZES:
                arrs.update({f"{fmt}_n{n}_{k}": v for k, v in _slices(out).items()})
    GOLDEN.write_text(json.dumps(rec, indent=1, sort_keys=True) + "\n")
    np.savez_compressed(SLICES, **arrs)
    print(f"wrote {GOLDEN} and {SLICES}")
