"""-m gpu: every tensor-core backward stays inside the workspace its plan asks for.

The backward runs with a buffer 256 KiB longer than ``*_bf16_workspace_bytes`` and is told the requested size; the tail
is filled with a sentinel first and must be untouched afterwards.  A stage whose scratch the size function misses then
writes into the test's own allocation, where it is seen, rather than into a neighbouring tensor."""
import pytest
import torch

from test_gpu_tc_plan_bits import build_case

pytestmark = pytest.mark.gpu

TAIL, SENTINEL = 256 << 10, 0xA5
CASES = ([("naturecnn", fmt, A, n) for fmt in ("u8", "bf16s2d", "u8s2d") for A in (2, 6, 305) for n in (7, 32, 64, 300)]
         + [("impala", None, 15, n) for n in (1, 7, 64, 300)]
         + [("lstm", (S, n), 6, None) for S, n in ((1, 7), (4, 8), (8, 64))])


def _id(c):
    net, shape, A, n = c
    return f"lstm_S{shape[0]}_n{shape[1]}" if net == "lstm" else f"{net}_{shape or ''}_A{A}_n{n}"


@pytest.mark.parametrize("c", CASES, ids=_id)
def test_backward_stays_inside_its_workspace(lib, c):
    net, shape, A, n = c
    dev = torch.device("cuda")
    plan, flat, fwd, bwd = build_case(net, shape, A, n, dev)
    fwd()
    need = plan._c("workspace_bytes")(*(shape if net == "lstm" else (n,)), A)
    assert need > 0
    buf = torch.empty(need + TAIL, dtype=torch.uint8, device=dev)
    buf[need:].fill_(SENTINEL)
    plan._ws = buf[:need]                  # the plan passes ws.numel() = need as the workspace size
    grads = torch.zeros(plan.param_count, dtype=torch.float32, device=dev)
    bwd(grads)
    torch.cuda.synchronize()
    touched = (buf[need:] != SENTINEL).nonzero()
    assert touched.numel() == 0, f"backward wrote {int(touched.max()) + 1} bytes past the {need}-byte workspace"
