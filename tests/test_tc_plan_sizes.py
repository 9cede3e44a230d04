"""The host-side sizes of the tensor-core plans (NatureCNN, IMPALA-CNN, LSTM agent): parameter counts, packed-weight
bytes, activation bytes and layouts, backward workspace bytes.  These functions run without a GPU.

tests/golden/tc_plan_sizes.json holds every value over a grid of batch shapes and action counts, out-of-range arguments
(which return 0, -1 or an error) included.  The NatureCNN backward workspace was resized once on purpose, when its size
came to be built from the launches the backward makes: the fixture keeps the earlier values beside the current ones
(``naturecnn_workspace_bytes_before``).  Regenerate with `python tests/test_tc_plan_sizes.py`, only when a change is
MEANT to alter a size."""
import ctypes
import json
import sys
from pathlib import Path

GOLDEN = Path(__file__).resolve().parent / "golden" / "tc_plan_sizes.json"

NATURE_N = (0, 1, 7, 32, 64, 300, 1024, 4099, 32768)
NATURE_A = (0, 1, 2, 6, 23, 305, 2047, 2048)
IMPALA_N = (0, 1, 7, 300, 2049, 131072, 131073)
IMPALA_A = (0, 1, 15, 23, 24)
LSTM_SN = ((1, 0), (1, 7), (4, 8), (16, 64), (128, 8), (128, 1024), (256, 1024))
LSTM_A = (0, 1, 6, 23, 24)
OBS_FORMATS = (0, 1, 2)           # uint8 NCHW frames, bf16 space-to-depth, uint8 space-to-depth rollout rows
IMPALA_TENSORS, LSTM_TENSORS = 30, 13


def _layout(fn, shape, count):
    off = (ctypes.c_int64 * count)()
    return list(off) if fn(*shape, off) == 0 else None


def sizes(lib):
    """name -> value of every size function over the grid"""
    v = {}
    for A in NATURE_A:
        v[f"naturecnn_param_count/A={A}"] = lib.b200rl_naturecnn_param_count(A)
        v[f"naturecnn_bf16_packed_bytes/A={A}"] = lib.b200rl_naturecnn_bf16_packed_bytes(A)
    for n in NATURE_N:
        for f in OBS_FORMATS:
            v[f"naturecnn_bf16_acts_bytes/n={n}/fmt={f}"] = lib.b200rl_naturecnn_bf16_acts_bytes(n, f)
        for A in NATURE_A:
            v[f"naturecnn_bf16_workspace_bytes/n={n}/A={A}"] = lib.b200rl_naturecnn_bf16_workspace_bytes(n, A)
    for A in IMPALA_A:
        v[f"impala_param_count/A={A}"] = lib.b200rl_impala_param_count(A)
        v[f"impala_bf16_packed_bytes/A={A}"] = lib.b200rl_impala_bf16_packed_bytes(A)
    for n in IMPALA_N:
        v[f"impala_bf16_acts_bytes/n={n}"] = lib.b200rl_impala_bf16_acts_bytes(n)
        v[f"impala_bf16_acts_layout/n={n}"] = _layout(lib.b200rl_impala_bf16_acts_layout, (n,), IMPALA_TENSORS)
        for A in IMPALA_A:
            v[f"impala_bf16_workspace_bytes/n={n}/A={A}"] = lib.b200rl_impala_bf16_workspace_bytes(n, A)
    for A in LSTM_A:
        v[f"lstm_agent_param_count/A={A}"] = lib.b200rl_lstm_agent_param_count(A)
        v[f"lstm_agent_bf16_packed_bytes/A={A}"] = lib.b200rl_lstm_agent_bf16_packed_bytes(A)
    for S, n in LSTM_SN:
        v[f"lstm_agent_bf16_acts_bytes/S={S}/n={n}"] = lib.b200rl_lstm_agent_bf16_acts_bytes(S, n)
        v[f"lstm_agent_bf16_acts_layout/S={S}/n={n}"] = _layout(lib.b200rl_lstm_agent_bf16_acts_layout, (S, n), LSTM_TENSORS)
        for A in LSTM_A:
            v[f"lstm_agent_bf16_workspace_bytes/S={S}/n={n}/A={A}"] = lib.b200rl_lstm_agent_bf16_workspace_bytes(S, n, A)
    return v


def test_plan_sizes_match_the_recorded_values(lib):
    want = json.loads(GOLDEN.read_text())["sizes"]
    got = sizes(lib)
    assert set(got) == set(want)
    bad = {k: (got[k], want[k]) for k in want if got[k] != want[k]}
    assert not bad, f"{len(bad)} sizes differ (got, recorded): {dict(list(bad.items())[:10])}"


def test_naturecnn_workspace_resize_is_the_recorded_one():
    """The values before the resize are kept for every NatureCNN workspace size; out-of-range arguments still give 0."""
    rec = json.loads(GOLDEN.read_text())
    before, now = rec["naturecnn_workspace_bytes_before"], rec["sizes"]
    assert set(before) == {k for k in now if k.startswith("naturecnn_bf16_workspace_bytes/")}
    assert all((before[k] == 0) == (now[k] == 0) for k in before)


if __name__ == "__main__":
    # recipe of tests/golden/tc_plan_sizes.json: the current build's values; `--keep-before` keeps the recorded
    # naturecnn_workspace_bytes_before, otherwise they are taken from this build too
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    from cleanrl_b200 import _lib, build
    build.build()
    v = sizes(_lib.load())
    if "--keep-before" in sys.argv:
        before = json.loads(GOLDEN.read_text())["naturecnn_workspace_bytes_before"]
    else:
        before = {k: x for k, x in v.items() if k.startswith("naturecnn_bf16_workspace_bytes/")}
    GOLDEN.write_text(json.dumps({"sizes": v, "naturecnn_workspace_bytes_before": before}, indent=0, sort_keys=True) + "\n")
    print(f"wrote {GOLDEN}")
