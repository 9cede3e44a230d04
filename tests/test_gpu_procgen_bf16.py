"""-m gpu: the IMPALA-CNN agent with ``precision = "bf16"`` (csrc/net_impala_tc.cu): forward and backward against a torch
model with the kernels' bf16 rounding points, against the fp64 reference, max-pool ties, determinism, the rows gather,
CUDA-graph replay, the engine's update / rollout graphs, the drop-in script and argument validation."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN
from test_gpu_procgen import _Envs, _Writer, _cpu_noise, _ref_forward

pytestmark = pytest.mark.gpu


class _RoundBf16(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return x.to(torch.bfloat16).float()

    @staticmethod
    def backward(ctx, g):
        return g.to(torch.bfloat16).float()     # the kernels store activation gradients in bf16 at the same tensors


def _r(x):
    return _RoundBf16.apply(x)


def _mirror_seq(p, i, h):
    """ConvSequence i in fp32 with the kernels' rounding points (input and output NCHW; seq0 takes the raw frames)."""
    c = F.conv2d(h, _r(p[f"network.{i}.conv.weight"]), None, padding=1)
    c = _r(c * (1.0 / 255.0) + p[f"network.{i}.conv.bias"].view(1, -1, 1, 1) if i == 0 else c + p[f"network.{i}.conv.bias"].view(1, -1, 1, 1))
    h = _r(F.max_pool2d(c, kernel_size=3, stride=2, padding=1))
    for b in (0, 1):
        pre = f"network.{i}.res_block{b}"
        y0 = _r(F.relu(F.conv2d(F.relu(h), _r(p[f"{pre}.conv0.weight"]), p[f"{pre}.conv0.bias"], padding=1)))
        h = _r(h + F.conv2d(y0, _r(p[f"{pre}.conv1.weight"]), p[f"{pre}.conv1.bias"], padding=1))
    return h


def _mirror_forward(p, x_nhwc):
    """IMPALA-CNN in fp32 with the kernels' rounding points: bf16 conv / fc weights, bf16 stored activations
    (conv output, relu(conv0), the residual stream, hidden), fp32 accumulation, fp32 heads."""
    h = x_nhwc.permute(0, 3, 1, 2).float()
    for i in range(3):
        h = _mirror_seq(p, i, h)
    hid = _r(F.relu(F.linear(F.relu(h.flatten(1)), _r(p["network.5.weight"]), p["network.5.bias"])))
    return F.linear(hid, p["actor.weight"], p["actor.bias"]), F.linear(hid, p["critic.weight"], p["critic.bias"])[:, 0]


class _Stored(torch.autograd.Function):
    """Forward: the tensor the kernels stored (so every ReLU mask and max-pool arg-max of the reference is the kernels'
    own); backward: the gradient rounded to bf16 as the kernels store it, times (stored > 0) when ``relu``."""

    @staticmethod
    def forward(ctx, pre, stored, relu):
        ctx.save_for_backward(stored)
        ctx.relu = relu
        return stored.clone()

    @staticmethod
    def backward(ctx, g):
        (stored,) = ctx.saved_tensors
        g = g.to(torch.bfloat16).float()
        if ctx.relu:
            g = g * (stored > 0)
        return g, None, None


def _nchw(t):
    return t.float().permute(0, 3, 1, 2).contiguous()


def _stored_forward(p, x_nhwc, T):
    """The network evaluated layer by layer on the kernels' stored forward tensors T (ImpalaCNNBf16.act_tensors):
    each layer's torch result is replaced by what the kernel stored, and the backward runs through torch's own conv,
    max-pool and linear gradients with the kernels' masks, arg-maxes and gradient rounding."""
    h = x_nhwc.permute(0, 3, 1, 2).float()
    for i in range(3):
        c = F.conv2d(h, _r(p[f"network.{i}.conv.weight"]), None, padding=1)
        c = c * (1.0 / 255.0) + p[f"network.{i}.conv.bias"].view(1, -1, 1, 1) if i == 0 else c + p[f"network.{i}.conv.bias"].view(1, -1, 1, 1)
        c = _Stored.apply(c, _nchw(T[f"c{i}"]), False)
        h = _Stored.apply(F.max_pool2d(c, kernel_size=3, stride=2, padding=1), _nchw(T[f"s0_{i}"]), False)
        for b in (0, 1):
            pre = f"network.{i}.res_block{b}"
            y0 = F.conv2d(F.relu(h), _r(p[f"{pre}.conv0.weight"]), p[f"{pre}.conv0.bias"], padding=1)
            y0 = _Stored.apply(y0, _nchw(T[f"y{b}_{i}"]), True)
            s = h + F.conv2d(y0, _r(p[f"{pre}.conv1.weight"]), p[f"{pre}.conv1.bias"], padding=1)
            if i == 2 and b == 1:
                h = _Stored.apply(s, _nchw(T["h0"].view(-1, 8, 8, 32)), True)        # relu(stream): the fc input
            else:
                h = _Stored.apply(s, _nchw(T[f"s{b + 1}_{i}"]), False)
    hid = _Stored.apply(F.linear(h.flatten(1), _r(p["network.5.weight"]), p["network.5.bias"]), T["hid"].float(), True)
    return F.linear(hid, p["actor.weight"], p["actor.bias"]), F.linear(hid, p["critic.weight"], p["critic.bias"])[:, 0]


def _agent(A, seed=2):
    from cleanrl_b200.agents import ImpalaAgent
    torch.manual_seed(seed)
    agent = ImpalaAgent(_Envs(A)).cuda()
    agent.precision = "bf16"
    agent.flat
    return agent


def _fwd_bwd(agent, obs, rows, gl, gv):
    lg, val = agent.forward_train(obs, rows)
    lg, val = lg.clone(), val.clone()
    n, A = lg.shape
    dhead, dl, dv = agent.alloc_head_grad(n, obs.device)
    dl.copy_(gl); dv.copy_(gv)
    agent.backward(dhead)
    return lg, val, agent.flat.grad.clone()


@pytest.fixture(autouse=True)
def _no_tf32():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


@pytest.mark.parametrize("n,B,A", [(6, 20, 15), (1, 3, 4), (33, 33, 15), (300, 300, 15), (2049, 2049, 15)])
def test_impala_bf16_vs_rounded_torch_and_fp64(lib, n, B, A):
    agent = _agent(A)
    g = torch.Generator().manual_seed(4)
    obs = torch.randint(0, 256, (B, 64, 64, 3), dtype=torch.uint8, generator=g)
    rows = torch.randperm(B, generator=g)[:n]
    gl = torch.randn(n, A, generator=g).cuda() / n
    gv = torch.randn(n, generator=g).cuda() / n
    lg, val, grad = _fwd_bwd(agent, obs.cuda(), rows.cuda(), gl, gv)
    torch.cuda.synchronize()
    # forward: an fp32 model with the kernels' rounding points, end to end (logits / value) and per sequence (each
    # sequence from the input the kernels stored for it, so that the check measures that sequence's kernels)
    p = {k: v.detach().clone() for k, v in agent.state_dict().items()}
    T = agent._tc.act_tensors(n)
    with torch.no_grad():
        logits, value = _mirror_forward(p, obs[rows].cuda())
        seqs = [_mirror_seq(p, 0, obs[rows].cuda().permute(0, 3, 1, 2).float()),
                _mirror_seq(p, 1, _nchw(T["s2_0"])), F.relu(_mirror_seq(p, 2, _nchw(T["s2_1"])))]
    for got, ref in [(_nchw(T["s2_0"]), seqs[0]), (_nchw(T["s2_1"]), seqs[1]), (_nchw(T["h0"].view(n, 8, 8, 32)), seqs[2]),
                     (lg, logits), (val, value)]:
        assert (got.float() - ref).abs().max() <= 1e-2 * max(ref.abs().max().item(), 1e-6)
    # backward: torch's gradients of the network evaluated on the kernels' stored tensors
    p = {k: v.detach().clone().requires_grad_(True) for k, v in agent.state_dict().items()}
    l2, v2 = _stored_forward(p, obs[rows].cuda(), T)
    assert (l2 - lg).abs().max() <= 1e-3 * max(lg.abs().max().item(), 1e-6)
    ((l2 * gl).sum() + (v2 * gv).sum()).backward()
    errs = {k: ((prm.grad - p[k].grad).norm() / max(p[k].grad.norm().item(), 1e-30)).item()
            for k, prm in agent.named_parameters()}
    assert max(errs.values()) <= 2e-2, errs
    if n <= 300:
        sd = {k: v.detach().cpu().double() for k, v in agent.state_dict().items()}
        l64, v64 = _ref_forward(sd, obs[rows])
        assert (lg.cpu().double() - l64).abs().max() <= 2e-2 * max(1.0, l64.abs().max().item())
        assert (val.cpu().double() - v64).abs().max() <= 2e-2 * max(1.0, v64.abs().max().item())


def test_maxpool_ties_route_to_first_maximum(lib):
    """seq0 conv with zero weights and a constant bias: every max-pool window of its output is all ties.  The gradient
    the kernels route to the conv output (the workspace's dc after the backward) must equal torch's max_pool2d backward
    of the same pooled gradient, i.e. go to the first maximum of each window in row-major order."""
    A, n = 15, 5
    agent = _agent(A)
    with torch.no_grad():
        agent.network[0].conv.weight.zero_()
        agent.network[0].conv.bias.fill_(0.25)
    agent.params_updated()
    g = torch.Generator().manual_seed(8)
    obs = torch.randint(0, 256, (n, 64, 64, 3), dtype=torch.uint8, generator=g)
    gl = torch.randn(n, A, generator=g).cuda()
    gv = torch.randn(n, generator=g).cuda()
    _fwd_bwd(agent, obs.cuda(), None, gl, gv)
    torch.cuda.synchronize()
    T = agent._tc.act_tensors(n)
    c0 = _nchw(T["c0"]).requires_grad_(True)
    assert (c0 == 0.25).all()
    dp = T["ga"][:, :32 * 32 * 16].float().view(n, 32, 32, 16).permute(0, 3, 1, 2)   # gradient of seq0's max-pool output
    assert dp.abs().amax() > 0
    F.max_pool2d(c0, kernel_size=3, stride=2, padding=1).backward(dp)
    ref = c0.grad.to(torch.bfloat16).float().permute(0, 2, 3, 1)
    got = T["dc"].float().view(n, 64, 64, 16)
    assert (got - ref).abs().max() <= 1e-2 * ref.abs().max()       # up to 4 windows summed in another order


def test_deterministic_rows_gather_and_graph_replay(lib):
    A, B, n = 15, 700, 512
    agent = _agent(A)
    g = torch.Generator().manual_seed(5)
    obs = torch.randint(0, 256, (B, 64, 64, 3), dtype=torch.uint8, generator=g).cuda()
    rows = torch.randperm(B, generator=g)[:n].cuda()
    gl = torch.randn(n, A, generator=g).cuda()
    gv = torch.randn(n, generator=g).cuda()
    a = _fwd_bwd(agent, obs, rows, gl, gv)
    b = _fwd_bwd(agent, obs, rows, gl, gv)
    c = _fwd_bwd(agent, obs[rows].contiguous(), None, gl, gv)
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, z)
    # capture forward + backward, poison outputs and activations, replay
    dhead, dl, dv = agent.alloc_head_grad(n, obs.device)
    dl.copy_(gl); dv.copy_(gv)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out = agent.forward_train(obs, rows)
        agent.backward(dhead)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        lg, val = agent.forward_train(obs, rows)
        agent.backward(dhead)
    agent.pin_workspaces()
    lg.fill_(float("nan")); agent.flat.grad.fill_(float("nan"))
    for buf in agent._tc._acts.values():
        buf.fill_(0x7F)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(lg, a[0]) and torch.equal(val, a[1]) and torch.equal(agent.flat.grad, a[2])


def _engine_run(update_graphs, cuda_graphs, iters=2):
    from bench import ppo_args
    from cleanrl_b200.ppo_engine import PPOEngine
    from cleanrl_b200.synthetic_envs import SyntheticProcgenVec
    dev = torch.device("cuda")
    N, T = 16, 16
    np.random.seed(5)
    agent = _agent(15, seed=5)
    args = ppo_args(N, T, iters, "bf16")
    eng = PPOEngine(agent, args, (64, 64, 3), np.uint8, N, dev, gae_mode=1, cuda_graphs=cuda_graphs)
    eng.update_graphs = update_graphs
    torch.manual_seed(9)
    env = SyntheticProcgenVec(N, seed=3)
    obs, done = env.reset(), np.zeros(N, dtype=np.float32)
    out = []
    for it in range(iters):
        for t in range(T):
            a = eng.policy_step(t, obs, done)
            obs, r, done, _ = env.step(a.copy())
            eng.record_reward(t, np.asarray(r, dtype=np.float32))
            done = np.asarray(done, dtype=np.float32)
        eng.finish_rollout(obs, done)
        roll = [getattr(eng, k).clone() for k in ("obs", "actions", "logprobs", "values")]
        st = eng.update(2.5e-4 * (1.0 - it / iters))
        out.append((roll, st["per_update"].copy(), eng.flat.flat.clone(), eng.flat.exp_avg.clone(), eng.flat.exp_avg_sq.clone()))
    return eng, out


def test_engine_graphs_equal_eager(lib):
    e_ref, ref = _engine_run(update_graphs=False, cuda_graphs=False)
    e_roll, roll = _engine_run(update_graphs=False, cuda_graphs=True)
    e_all, allg = _engine_run(update_graphs=True, cuda_graphs=True)
    assert len(e_all._upd_graphs) > 0 and len(e_roll._upd_graphs) == 0
    for it in range(len(ref)):
        for other in (roll, allg):
            for x, y in zip(ref[it][0], other[it][0]):
                assert torch.equal(x, y), f"rollout buffers differ in iteration {it}"
            assert np.array_equal(ref[it][1], other[it][1]), f"statistics differ in iteration {it}"
            for x, y in zip(ref[it][2:], other[it][2:]):
                assert torch.equal(x, y), f"parameters / Adam state differ in iteration {it}"


def test_procgen_script_bf16_vs_reference_run(lib):
    from cleanrl_b200 import ppo_procgen as S
    z = np.load(GOLDEN / "ppo_procgen_n8_t16_seed2.npz")
    argv = [a for a in z["argv"].tolist() if a != "--no-cuda"] + ["--synthetic-env", "--precision", "bf16"]
    snaps, writers = [], []

    def on_it(it, eng, st):
        snaps.append({k: getattr(eng, k).cpu().numpy().copy() for k in ("actions", "logprobs", "values")} | {"st": st})

    def hook(agent):
        agent.noise_fn = _cpu_noise

    def wf(path):
        w = _Writer(); writers.append(w); return w

    S.main(argv, writer_factory=wf, on_iteration=on_it, agent_hook=hook)
    n_it = z["actions"].shape[0]
    assert len(snaps) == n_it
    s = snaps[0]
    rel = lambda a, b: np.abs(a.astype(np.float64) - b.astype(np.float64)).max() / max(1.0, np.abs(b).max())
    assert (s["actions"] == z["actions"][0].astype(np.int64)).mean() >= 0.99
    for k in ("logprobs", "values"):
        assert rel(s[k], z[k][0]) <= 2e-2, (k, rel(s[k], z[k][0]))
    per = s["st"]["per_update"]
    for u in range(per.shape[0]):
        for col, key in ((0, "upd_pg_loss"), (1, "upd_v_loss"), (2, "upd_entropy_loss"), (6, "upd_loss")):
            ref = float(z[key][u])
            assert abs(per[u, col] - ref) <= (1e-2 if u == 0 else 5e-2) * max(1.0, abs(ref)), (u, key, per[u, col], ref)
    for it in range(1, n_it):
        assert np.isfinite(snaps[it]["values"]).all() and np.isfinite(snaps[it]["logprobs"]).all()
        assert (snaps[it]["actions"] == z["actions"][it].astype(np.int64)).mean() >= 0.5
    ours = {}
    for tag, v, step in writers[0].scalars:
        ours.setdefault(tag, []).append((step, v))
    for key in z.files:
        if key.startswith("tb/") and key != "tb/charts/SPS":
            tag, ref = key[3:], z[key]
            assert tag in ours, tag
            if not tag.startswith("charts/episodic"):
                assert np.array_equal(np.array(ours[tag])[:, 0], ref[:, 0]), tag


def test_argument_validation(lib):
    from cleanrl_b200 import _lib, ops
    L = _lib.load()
    A, n = 15, 4
    dev = torch.device("cuda")
    P = L.b200rl_impala_param_count(A)
    params = torch.zeros(P + 8, device=dev)
    packed = torch.zeros(L.b200rl_impala_bf16_packed_bytes(A) + 64, dtype=torch.uint8, device=dev)
    acts = torch.zeros(L.b200rl_impala_bf16_acts_bytes(n) + 512, dtype=torch.uint8, device=dev)
    obs = torch.zeros(n, 64, 64, 3, dtype=torch.uint8, device=dev)
    out = torch.zeros(n, A + 1, device=dev)
    launches = L.b200rl_launch_count()
    fwd = lambda o=obs.data_ptr(), nn=n, a=A, pr=params.data_ptr(), pk=packed.data_ptr(), ac=acts.data_ptr(), ho=out.data_ptr(): \
        L.b200rl_impala_bf16_forward(o, None, nn, a, pr, pk, ac, ho, None)
    assert fwd(o=None) == -1
    assert fwd(pk=None) == -1
    assert fwd(a=0) == -1 and fwd(a=24) == -1
    assert fwd(nn=(1 << 17) + 1) == -1
    assert fwd(pr=params.data_ptr() + 4) == -1
    assert fwd(ac=acts.data_ptr() + 16) == -1
    rows = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    assert L.b200rl_impala_bf16_forward(obs.data_ptr(), rows.data_ptr() + 4, n, A, params.data_ptr(), packed.data_ptr(),
                                        acts.data_ptr(), out.data_ptr(), None) == -1
    assert L.b200rl_impala_bf16_pack(params.data_ptr(), 0, packed.data_ptr(), None) == -1
    ws = torch.zeros(256, dtype=torch.uint8, device=dev)
    assert L.b200rl_impala_bf16_backward(obs.data_ptr(), None, n, A, params.data_ptr(), packed.data_ptr(), acts.data_ptr(),
                                         out.data_ptr(), params.data_ptr(), ws.data_ptr(), 256, None) == -4
    assert L.b200rl_launch_count() == launches
    assert L.b200rl_impala_bf16_packed_bytes(24) == 0 and L.b200rl_impala_param_count(0) == -1
    agent = _agent(A)
    with pytest.raises(ValueError):
        agent.get_value(torch.zeros(2, 3, 64, 64, dtype=torch.uint8, device=dev))
    with pytest.raises(ValueError):
        agent.get_value(torch.zeros(2, 84, 84, 3, dtype=torch.uint8, device=dev))
    with pytest.raises(ValueError):
        ops.ImpalaCNNBf16(24, dev)
