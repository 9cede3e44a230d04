"""-m gpu: the fused conv2 -> conv3 forward (tc_conv23_fwd, one image per tile) must reproduce the bits of act2, act3 and
their ReLU mask words m2 / m3 where its per-image schedule differs between batch sizes: one image (one CTA, one busy
warpgroup), 131-133 and 263-265 images (one or two images per CTA on a 132-SM H100, partial last rounds per warpgroup),
8192 and 8193 images; through the minibatch gather of every input format, on the LSTM agent's trunk (S * n rows) and
when the forward is replayed from a CUDA graph after those regions of the activation workspace have been poisoned (a
stale row of the kernel's shared-memory act2 image, or a position it fails to store, then shows).

tests/golden/conv23_fwd_bits.json holds SHA-256 digests of the raw bytes, recorded with the forward that ran conv2 and
conv3 as two window-convolution launches.  The workspace offsets follow `NatureActs` in cleanrl_b200/csrc/net_tc.cu.
Regenerate with `python tests/test_gpu_conv23_fwd.py` on an H100, only when a change is MEANT to alter the arithmetic."""
import hashlib
import json
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "conv23_fwd_bits.json"
A = 6
KEYS = ("act2", "act3", "m2", "m3")
# (input format, n, gather through `rows`)
NATURE = ([("u8s2d", n, True) for n in (1, 131, 132, 133, 263, 264, 265, 8192, 8193)]
          + [("u8s2d", 265, False), ("u8", 133, True), ("bf16s2d", 264, True), ("bf16s2d", 1, False)])
LSTM = ((4, 33), (16, 64))
GRAPH_N = 1024


def nature_id(c):
    fmt, n, gather = c
    return f"naturecnn_{fmt}_n{n}" + ("_rows" if gather else "")


def lstm_id(c):
    return f"lstm_S{c[0]}_n{c[1]}"


def _views(acts, n, with_x0):
    """name -> bf16-element slice of the activation workspace (the layout of NatureActs)."""
    sizes = [("x0", 28224 if with_x0 else 0), ("act1", 12800), ("act2", 5184), ("act3", 3136), ("hid", 512),
             ("dhid", 512), ("dact3a", 5184), ("dact3b", 7744), ("dact2a", 6400), ("dact2b", 7744), ("dact1", 14112)]
    o, out = 0, {}
    for name, per in sizes:
        out[name] = acts[o:o + n * per]
        o += n * per
    pad8 = lambda v: (v + 7) & ~7
    o += pad8(n * 100 * 4 * 2)                                    # m1
    out["m2"] = acts[o:o + n * 81 * 2 * 2]; o += pad8(n * 81 * 2 * 2)
    out["m3"] = acts[o:o + n * 49 * 2 * 2]
    return out


def _digest(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def _nature(c, dev):
    """(forward closure, {key: workspace view}) of a seeded NatureCNN case; every input is drawn on the CPU."""
    from cleanrl_b200 import ops
    fmt, n, gather = c
    g = torch.Generator().manual_seed(sum(map(ord, nature_id(c))))
    net = ops.NatureCNNBf16(A, dev)
    flat = (torch.randn(net.param_count, generator=g) * 0.05).to(dev)
    B = n + 5 if gather else n
    obs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g).to(dev)
    rows = torch.randperm(B, generator=g)[:n].to(dev) if gather else None
    if fmt == "u8s2d":
        obs, _ = ops.frames_to_s2d_u8(obs)
    elif fmt == "bf16s2d":
        obs = ops.frames_to_s2d(obs)
    net.pack(flat)
    head = torch.empty(n, A + 1, dtype=torch.float32, device=dev)
    fwd = lambda: net.forward(obs, rows, flat, head_out=head)
    fwd()
    code = {"u8": 0, "bf16s2d": 1, "u8s2d": 2}[fmt]
    return fwd, _views(net.acts(n, code).view(torch.bfloat16), n, fmt == "u8")


def _lstm(c, dev):
    from cleanrl_b200 import ops
    S, envs = c
    M = S * envs
    g = torch.Generator().manual_seed(sum(map(ord, lstm_id(c))))
    net = ops.LSTMAgentBf16(A, dev)
    flat = (torch.randn(net.param_count, generator=g) * 0.05).to(dev)
    B = M + 13
    obs = torch.randint(0, 256, (B, 1, 84, 84), dtype=torch.uint8, generator=g).to(dev)
    rows = torch.randperm(B, generator=g)[:M].to(dev)
    done = (torch.rand(M, generator=g) < 0.25).float().to(dev)
    h0 = (torch.randn(envs, 128, generator=g) * 0.5).to(dev)
    c0 = (torch.randn(envs, 128, generator=g) * 0.5).to(dev)
    net.pack(flat)
    fwd = lambda: net.forward(obs, rows, S, envs, flat, h0, c0, done)
    fwd()
    return fwd, _views(net.acts(S, envs).view(torch.bfloat16), M, False)


def _digests(views):
    torch.cuda.synchronize()
    return {k: _digest(views[k]) for k in KEYS}


def _graph_replay(dev):
    """digests of a graph replay of the n = GRAPH_N rollout-row forward over a poisoned workspace"""
    fwd, views = _nature(("u8s2d", GRAPH_N, True), dev)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fwd()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fwd()
    for k in KEYS:
        views[k].view(torch.uint8).fill_(0xFF)                    # bf16 NaN, all mask bits set
    graph.replay()
    return _digests(views)


def _record(dev):
    rec = {nature_id(c): _digests(_nature(c, dev)[1]) for c in NATURE}
    rec.update({lstm_id(c): _digests(_lstm(c, dev)[1]) for c in LSTM})
    return rec


def _check(got, want):
    bad = [k for k in KEYS if got[k] != want[k]]
    assert not bad, f"outputs differ from the recorded bits (data-flow order): {bad}"


@pytest.mark.parametrize("c", NATURE, ids=nature_id)
def test_naturecnn_conv23_bits(lib, c):
    _check(_digests(_nature(c, torch.device("cuda"))[1]), json.loads(GOLDEN.read_text())[nature_id(c)])


@pytest.mark.parametrize("c", LSTM, ids=lstm_id)
def test_lstm_trunk_conv23_bits(lib, c):
    _check(_digests(_lstm(c, torch.device("cuda"))[1]), json.loads(GOLDEN.read_text())[lstm_id(c)])


def test_graph_replay_over_poisoned_workspace(lib):
    _check(_graph_replay(torch.device("cuda")), json.loads(GOLDEN.read_text())[nature_id(("u8s2d", GRAPH_N, True))])


if __name__ == "__main__":
    # recipe of tests/golden/conv23_fwd_bits.json (run on an H100 with the build whose bits are to be recorded); the
    # graph case's entry is an eager forward
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    from cleanrl_b200 import build
    build.build()
    dev = torch.device("cuda")
    rec = _record(dev)
    rec[nature_id(("u8s2d", GRAPH_N, True))] = _digests(_nature(("u8s2d", GRAPH_N, True), dev)[1])
    out = Path(sys.argv[1]) if len(sys.argv) > 1 else GOLDEN
    out.write_text(json.dumps(rec, indent=1, sort_keys=True) + "\n")
    print(f"wrote {out}")
