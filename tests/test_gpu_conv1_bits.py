"""-m gpu: conv1's forward output must stay bit-identical at the batch sizes the benchmark runs and at sizes that leave
one, an odd number of, or a partial last set of tiles per CTA.

tests/golden/conv1_bits.json holds SHA-256 digests of the raw bytes of act1 (bf16, 2x2 cells [n,100,128]) and its ReLU
mask words m1 ([n,100] x 4 uint32) for the seeded inputs of test_gpu_conv_win_sizes.py, for both the uint8 NCHW frames
and the uint8 space-to-depth rollout rows gathered through an unsorted index.  conv1's weight and bias gradients are
pinned by that test's digest of the full gradient.  The workspace offsets follow `NatureActs` in
cleanrl_b200/csrc/net_tc.cu.  Regenerate with `python tests/test_gpu_conv1_bits.py` on an H100, only when a change is
MEANT to alter the arithmetic."""
import hashlib
import json
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "conv1_bits.json"
SIZES = (2, 3, 33, 1024, 1025, 32768)
FORMATS = ("u8", "u8s2d")
KEYS = ("act1", "m1")
A = 6


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
    if fmt == "u8s2d":
        obs, _ = ops.frames_to_s2d_u8(obs)
    net.pack(flat)
    head = torch.empty(n, A + 1, dtype=torch.float32, device=dev)
    net.forward(obs, rows, flat, head_out=head)
    torch.cuda.synchronize()
    acts = net.acts(n, 0 if fmt == "u8" else 2).view(torch.bfloat16)
    # bf16-element offsets of NatureActs: x0 (u8 frames only), act1, ..., dact1, then m1
    o = n * (28224 if fmt == "u8" else 0)
    act1 = acts[o:o + n * 12800]
    o += n * (12800 + 5184 + 3136 + 512 + 512 + 5184 + 7744 + 6400 + 7744 + 14112)
    m1 = acts[o:o + n * 100 * 4 * 2]
    return {"act1": _digest(act1), "m1": _digest(m1)}


def _digest(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("n", SIZES)
def test_conv1_matches_recorded_bits(lib, n, fmt):
    want = json.loads(GOLDEN.read_text())[f"{fmt}_n{n}"]
    got = _compute(n, fmt)
    bad = [k for k in KEYS if got[k] != want[k]]
    assert not bad, f"outputs differ from the recorded bits: {bad}"


if __name__ == "__main__":
    # recipe of tests/golden/conv1_bits.json (run on an H100 with the build whose bits are to be recorded)
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    from cleanrl_b200 import build
    build.build()
    rec = {f"{fmt}_n{n}": _compute(n, fmt) for fmt in FORMATS for n in SIZES}
    out = Path(sys.argv[1]) if len(sys.argv) > 1 else GOLDEN
    out.write_text(json.dumps(rec, indent=1, sort_keys=True) + "\n")
    print(f"wrote {out}")
