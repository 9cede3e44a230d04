"""-m gpu: a CUDA graph captured over a tensor-core agent's forward + backward bakes raw pointers into the plan's
activation AND backward workspaces.  After ``pin_workspaces()`` no later batch shape may free either kind, not even when
the backward workspace has to grow: the replay must still reproduce the eager result bit for bit."""
import weakref

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


class _Envs:
    def __init__(self, obs_shape, A):
        from cleanrl_b200.synthetic_envs import Box, Discrete
        self.single_observation_space = Box(0, 255, obs_shape, np.uint8)
        self.single_action_space = Discrete(A)


def _naturecnn(g):
    """NatureCNN on the uint8 space-to-depth rollout (the engine's default storage); batch = n rows"""
    from cleanrl_b200 import ops
    from cleanrl_b200.agents import NatureCNNAgent
    agent = NatureCNNAgent(_Envs((4, 84, 84), 6)).cuda()
    rm, cm = ops.frames_to_s2d_u8(torch.randint(0, 256, (600, 4, 84, 84), dtype=torch.uint8, generator=g).cuda())

    def train(n):
        rows = torch.randperm(600, generator=g)[:n].sort().values.cuda()
        return lambda: agent.forward_train(rm, rows, aux=cm)
    return agent, train


def _impala(g):
    from cleanrl_b200.agents import ImpalaAgent
    agent = ImpalaAgent(_Envs((64, 64, 3), 15)).cuda()
    obs = torch.randint(0, 256, (600, 64, 64, 3), dtype=torch.uint8, generator=g).cuda()

    def train(n):
        rows = torch.randperm(600, generator=g)[:n].cuda()
        return lambda: agent.forward_train(obs, rows)
    return agent, train


def _lstm(g):
    """the recurrent agent on sequences of S = 4 steps; batch = 4 * envs rows"""
    from cleanrl_b200.agents import LSTMAgent
    agent = LSTMAgent(_Envs((1, 84, 84), 6)).cuda()
    obs = torch.randint(0, 256, (600, 1, 84, 84), dtype=torch.uint8, generator=g).cuda()
    dones = (torch.rand(600, generator=g) < 0.1).float().cuda()

    def train(n):
        envs = n // 4
        rows = torch.randperm(600, generator=g)[:n].cuda()
        state = tuple(torch.randn(1, envs, 128, generator=g).cuda() * 0.5 for _ in range(2))
        return lambda: agent.forward_train(obs, rows, state, dones)
    return agent, train


@pytest.mark.parametrize("make", [_naturecnn, _impala, _lstm], ids=["naturecnn_u8", "impala", "lstm"])
def test_graph_workspaces_survive_a_larger_backward(lib, make):
    g = torch.Generator().manual_seed(7)
    torch.manual_seed(7)
    agent, train = make(g)
    agent.precision = "bf16"
    agent.flat
    n, big = 32, 512
    fwd = train(n)
    dhead, dl, dv = agent.alloc_head_grad(n, torch.device("cuda"))
    dl.copy_(torch.randn(dl.shape, generator=g) * 1e-2)
    dv.copy_(torch.randn(dv.shape, generator=g) * 1e-2)

    def fwd_bwd():
        lg, val = fwd()
        agent.backward(dhead)
        return lg, val

    lg, val = fwd_bwd()                      # eager: allocates the workspaces of this shape
    tc = agent._tc
    P = tc.param_count
    ref = (lg.clone(), val.clone(), agent.flat.grad[:P].clone())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        lg, val = fwd_bwd()
    agent.pin_workspaces()
    captured = [weakref.ref(t) for t in list(tc._acts.values()) + [tc._ws]]     # no strong reference from the test
    ptrs = [r().data_ptr() for r in captured]
    ws_bytes = tc._ws.numel()

    # a larger batch: a new activation workspace, and a backward workspace that must replace the captured one
    big_fwd = train(big)
    big_dhead, _, _ = agent.alloc_head_grad(big, torch.device("cuda"))
    big_dhead.normal_(0, 1e-2)
    big_fwd()
    agent.backward(big_dhead)
    torch.cuda.synchronize()
    assert tc._ws.numel() > ws_bytes, "the larger batch must grow the backward workspace"
    held = {t.data_ptr() for t in tc.__dict__.values() if isinstance(t, torch.Tensor)}
    for v in tc.__dict__.values():
        if isinstance(v, (list, tuple, dict)):
            held |= {t.data_ptr() for t in (v.values() if isinstance(v, dict) else v) if isinstance(t, torch.Tensor)}
    for r, p in zip(captured, ptrs):
        assert r() is not None and p in held, "a workspace referenced by the captured graph was freed"

    lg.fill_(float("nan")); val.fill_(float("nan")); agent.flat.grad[:P].fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(lg, ref[0]) and torch.equal(val, ref[1]) and torch.equal(agent.flat.grad[:P], ref[2])
