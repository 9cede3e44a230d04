"""-m gpu: the window convolutions (conv2/conv3 forward, conv3/conv2 data gradients) must stay bit-identical at the
batch sizes the benchmark runs and at sizes that leave partial and odd tile counts per CTA.

tests/golden/conv_win_bits.json holds SHA-256 digests of the raw bytes of act2, act3, their ReLU mask words, the data
gradients dact2a / dact2b / dact1 and the full flat gradient for seeded inputs, for both the uint8 NCHW frames and the
uint8 space-to-depth rollout rows (where dact1 is fp16 x 2^12).  The workspace offsets follow `NatureActs` in
cleanrl_b200/csrc/net_tc.cu.  Regenerate with `python tests/test_gpu_conv_win_sizes.py` on an H100, only when a change
is MEANT to alter the arithmetic."""
import hashlib
import json
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "conv_win_bits.json"
SIZES = (2, 3, 33, 1024, 1025, 32768)
FORMATS = ("u8", "u8s2d")
A = 6


def _pad8(v):
    return (v + 7) & ~7


def _views(acts, n, fmt):
    """name -> bf16-element slice of the activation workspace (the layout of NatureActs)."""
    sizes = [("x0", 28224 if fmt == "u8" else 0), ("act1", 12800), ("act2", 5184), ("act3", 3136), ("hid", 512),
             ("dhid", 512), ("dact3a", 5184), ("dact3b", 7744), ("dact2a", 6400), ("dact2b", 7744), ("dact1", 14112)]
    o, out = 0, {}
    for name, per in sizes:
        out[name] = acts[o:o + n * per]
        o += n * per
    o += _pad8(n * 100 * 4 * 2)                                   # m1
    out["m2"] = acts[o:o + n * 81 * 2 * 2]; o += _pad8(n * 81 * 2 * 2)
    out["m3"] = acts[o:o + n * 49 * 2 * 2]
    return out


KEYS = ("act2", "act3", "m2", "m3", "dact2a", "dact2b", "dact1")


def _compute(n, fmt):
    from cleanrl_b200 import ops
    from cleanrl_b200.ops import NatureCNNBf16
    dev = torch.device("cuda")
    net = NatureCNNBf16(A, dev)
    g = torch.Generator().manual_seed(2000 + n)
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
    net.forward(obs, rows, flat, head_out=head)
    net.backward(obs, rows, flat, dhead, grads, obs_aux=aux)
    torch.cuda.synchronize()
    acts = net.acts(n, 0 if fmt == "u8" else 2).view(torch.bfloat16)
    v = _views(acts, n, fmt)
    out = {k: v[k] for k in KEYS}
    out["grads"] = grads
    return {k: _digest(t) for k, t in out.items()}


def _digest(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("n", SIZES)
def test_conv_win_matches_recorded_bits(lib, n, fmt):
    want = json.loads(GOLDEN.read_text())[f"{fmt}_n{n}"]
    got = _compute(n, fmt)
    # report in data-flow order, so the first entry is the first tensor that differs
    bad = [k for k in KEYS + ("grads",) if got[k] != want[k]]
    assert not bad, f"outputs differ from the recorded bits (data-flow order): {bad}"


if __name__ == "__main__":
    # recipe of tests/golden/conv_win_bits.json (run on an H100 with the build whose bits are to be recorded)
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    from cleanrl_b200 import build
    build.build()
    rec = {f"{fmt}_n{n}": _compute(n, fmt) for fmt in FORMATS for n in SIZES}
    out = Path(sys.argv[1]) if len(sys.argv) > 1 else GOLDEN
    out.write_text(json.dumps(rec, indent=1, sort_keys=True) + "\n")
    print(f"wrote {out}")
