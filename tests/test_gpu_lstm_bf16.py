"""The recurrent agent (cleanrl/ppo_atari_lstm.py) on the tensor cores (``precision = "bf16"``): single-frame conv1, the
shared NatureCNN trunk, W_ih as a wide head, the one-launch recurrence in both directions, heads.

Checked against an fp32 torch model that rounds where the kernels round (bf16 operands, fp32 accumulation, c and the gate
math in fp32), against the fp64 reference network, and bitwise against itself; plus the drop-in script against the
reference run.  The argument-validation test runs without a GPU."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN

SHAPES = [(1, 1, 4), (5, 3, 4), (16, 2, 6), (128, 2, 4), (128, 17, 18), (1, 1024, 4)]
DONES = ["none", "all", "random"]


class _Envs:
    def __init__(self, A):
        from cleanrl_b200.synthetic_envs import Box, Discrete
        self.single_observation_space = Box(0, 255, (1, 84, 84), np.uint8)
        self.single_action_space = Discrete(A)


def _cpu_noise(n, A, device):
    return torch.empty(n, A, dtype=torch.float32).exponential_(1).to(device)


def _agent(A, seed=3):
    from cleanrl_b200.agents import LSTMAgent
    torch.manual_seed(seed)
    agent = LSTMAgent(_Envs(A)).cuda()
    agent.precision = "bf16"
    agent.flat
    return agent


def _inputs(S, n, done_kind, seed=5):
    """frames in a larger buffer + the gather rows, done [S*n], random (h0, c0)"""
    g = torch.Generator().manual_seed(seed)
    B = S * n + 13
    obs = torch.randint(0, 256, (B, 1, 84, 84), dtype=torch.uint8, generator=g)
    rows = torch.randperm(B, generator=g)[:S * n]
    done = {"none": torch.zeros(S * n), "all": torch.ones(S * n),
            "random": (torch.rand(S * n, generator=g) < 0.25).float()}[done_kind]
    h0 = torch.randn(n, 128, generator=g) * 0.5
    c0 = torch.randn(n, 128, generator=g) * 0.5
    return obs.cuda(), rows.cuda(), done.cuda(), h0.cuda(), c0.cuda()


def _rb(x):
    """round to bf16 in the forward, identity in the backward"""
    return x + (x.to(torch.bfloat16).to(x.dtype) - x).detach()


def _act1_nchw(a):         # [M, 10, 10, 128] 2x2 cells (class (py, px), 32 channels) -> [M, 32, 20, 20]
    M = a.shape[0]
    return a.view(M, 10, 10, 2, 2, 32).permute(0, 5, 1, 3, 2, 4).reshape(M, 32, 20, 20)


def _model(p, x, done, h0, c0, S, n, rounding, masks=None):
    """The network on frames x [M, 1, 84, 84] (float).  rounding=True: bf16 operands where the kernels round them;
    masks: the kernels' own ReLU masks (dict of 0/1 tensors) instead of relu.  Returns a dict of tensors."""
    rb = _rb if rounding else (lambda t: t)
    W = {k: rb(v) if k.endswith("weight") and not k.startswith(("actor", "critic")) else v for k, v in p.items()}

    def act(y, key):
        return y * masks[key] if masks is not None else torch.relu(y)
    a1 = rb(act(F.conv2d(x, W["network.0.weight"], stride=4) / 255.0 + p["network.0.bias"].view(1, -1, 1, 1), "a1"))
    a2 = rb(act(F.conv2d(a1, W["network.2.weight"], p["network.2.bias"], stride=2), "a2"))
    a3 = rb(act(F.conv2d(a2, W["network.4.weight"], p["network.4.bias"], stride=1), "a3"))
    feats = rb(act(F.linear(a3.flatten(1), W["network.7.weight"], p["network.7.bias"]), "feats"))
    gx = F.linear(feats, W["lstm.weight_ih_l0"], p["lstm.bias_ih_l0"])
    h, c = h0, c0
    dd = done.view(S, n, 1).to(x.dtype)
    hs = []
    for t in range(S):
        hm = rb((1 - dd[t]) * h)
        c = (1 - dd[t]) * c
        gates = gx[t * n:(t + 1) * n] + F.linear(hm, W["lstm.weight_hh_l0"], p["lstm.bias_hh_l0"])
        i, f, g, o = gates.chunk(4, dim=1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
        h = torch.sigmoid(o) * torch.tanh(c)
        hs.append(h)
    hseq = rb(torch.cat(hs))
    logits = F.linear(hseq, p["actor.weight"], p["actor.bias"])
    value = F.linear(hseq, p["critic.weight"], p["critic.bias"])[:, 0]
    return dict(feats=feats, gx=gx, hseq=hseq, h=h, c=c, logits=logits, value=value)


def _params(agent, dtype):
    return {k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in agent.state_dict().items()}


def _close(a, b, tol):
    a, b = a.detach().double(), b.detach().double()
    return (a - b).abs().max().item() <= tol * max(b.abs().max().item(), 1e-6)


def _run(agent, obs, rows, done, h0, c0, S, n):
    full_done = torch.zeros(obs.shape[0], device="cuda").index_copy_(0, rows, done)
    lg, val = agent.forward_train(obs, rows, (h0.view(1, n, 128), c0.view(1, n, 128)), full_done)
    return lg, val


@pytest.mark.gpu
@pytest.mark.parametrize("done_kind", DONES)
@pytest.mark.parametrize("S,n,A", SHAPES)
def test_forward_vs_rounding_model_and_fp64(lib, S, n, A, done_kind):
    """feats, gx, every h_t, (h_S, c_S), logits and value within 1e-2 of the rounding model (of each tensor's maximum);
    logits and value within 2e-2 of the fp64 reference."""
    agent = _agent(A)
    obs, rows, done, h0, c0 = _inputs(S, n, done_kind)
    x = obs[rows].float()
    hseq_k, (hS, cS) = agent.get_states(obs, (h0.view(1, n, 128), c0.view(1, n, 128)), done, rows=rows)
    lg, val = [v.clone() for v in agent._heads(hseq_k)]
    t = agent._tc.act_tensors(S, n)
    torch.cuda.synchronize()
    with torch.no_grad():
        m = _model(_params(agent, torch.float32), x, done, h0, c0, S, n, True)
        r = _model(_params(agent, torch.float64), x.double(), done, h0.double(), c0.double(), S, n, False)
    assert _close(t["feats"].float(), m["feats"], 1e-2)
    assert _close(t["gx"], m["gx"], 1e-2)
    assert _close(t["hseq"].float(), m["hseq"], 1e-2)
    assert _close(hS[0], m["h"], 1e-2) and _close(cS[0], m["c"], 1e-2)
    assert _close(lg, m["logits"], 1e-2) and _close(val, m["value"], 1e-2)
    scale = lambda v: max(1.0, v.abs().max().item())
    assert (lg.double() - r["logits"]).abs().max().item() <= 2e-2 * scale(r["logits"])
    assert (val.double() - r["value"]).abs().max().item() <= 2e-2 * scale(r["value"])


def _kernel_masks(t, M):
    return dict(a1=(_act1_nchw(t["act1"]) > 0).float(), a2=(t["act2"].permute(0, 3, 1, 2) > 0).float(),
                a3=(t["act3"].permute(0, 3, 1, 2) > 0).float(), feats=(t["feats"] > 0).float())


@pytest.mark.gpu
@pytest.mark.parametrize("S,n,A", SHAPES)
def test_backward_vs_autograd(lib, S, n, A):
    """Every parameter gradient within 2e-2 relative L2 of autograd through the rounding model, with the kernels' own ReLU
    masks (an independent model flips masks at near-zero pre-activations, DESIGN §2); cosine >= 0.99 against the fp64
    reference at S = 16."""
    agent = _agent(A)
    obs, rows, done, h0, c0 = _inputs(S, n, "random")
    M = S * n
    g = torch.Generator().manual_seed(9)
    gl = torch.randn(M, A, generator=g).cuda() * 0.1
    gv = torch.randn(M, generator=g).cuda() * 0.1
    _run(agent, obs, rows, done, h0, c0, S, n)
    masks = _kernel_masks(agent._tc.act_tensors(S, n), M)
    dhead, dl, dv = agent.alloc_head_grad(M, torch.device("cuda"))
    dl.copy_(gl); dv.copy_(gv)
    agent.backward(dhead)
    torch.cuda.synchronize()
    x = obs[rows].float()
    p = _params(agent, torch.float32)
    m = _model(p, x, done, h0, c0, S, n, True, masks)
    ((m["logits"] * gl).sum() + (m["value"] * gv).sum()).backward()
    for k, prm in agent.named_parameters():
        got, ref = prm.grad.double(), p[k].grad.double()
        err = ((got - ref).norm() / ref.norm().clamp_min(1e-30)).item()
        assert err <= 2e-2, (k, err)
    if S == 16:
        p64 = _params(agent, torch.float64)
        r = _model(p64, x.double(), done, h0.double(), c0.double(), S, n, False)
        ((r["logits"] * gl.double()).sum() + (r["value"] * gv.double()).sum()).backward()
        for k, prm in agent.named_parameters():
            cos = F.cosine_similarity(prm.grad.double().flatten(), p64[k].grad.flatten(), dim=0).item()
            assert cos >= 0.99, (k, cos)


@pytest.mark.gpu
def test_bitwise_repeat_gather_rows_and_graph_replay(lib):
    """Repeated calls are identical; the rows gather equals a materialised obs[rows]; a sequence over n envs equals the
    envs run one at a time; forward + backward captured in a CUDA graph and replayed after the activations are poisoned
    equal the eager launches."""
    S, n, A = 16, 5, 6
    agent = _agent(A)
    tc = agent._tc_plan()
    obs, rows, done, h0, c0 = _inputs(S, n, "random")
    flat, M = agent._flat.flat, S * n
    dhead = torch.randn(M, A + 1, generator=torch.Generator().manual_seed(2)).cuda() * 0.1

    def once(o, r, d=done, hh=h0, cc=c0, nn_=n, grads=None):
        out = [v.clone() for v in tc.forward(o, r, S, nn_, flat, hh, cc, d)]
        if grads is not None:
            tc.backward(o, r, S, nn_, flat, d, dhead, grads)
        return out
    g1, g2 = torch.zeros_like(flat), torch.zeros_like(flat)
    a = once(obs, rows, grads=g1)
    b = once(obs, rows, grads=g2)
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and torch.equal(g1, g2)
    c = once(obs[rows].contiguous(), None)
    assert all(torch.equal(x, y) for x, y in zip(a, c))
    head_seq = a[0].view(S, n, A + 1)
    for e in range(n):
        r_e = rows.view(S, n)[:, e].contiguous()
        h_e, c_e, d_e = h0[e:e + 1].contiguous(), c0[e:e + 1].contiguous(), done.view(S, n)[:, e].contiguous()
        one = [v.clone() for v in tc.forward(obs, r_e, S, 1, flat, h_e, c_e, d_e)]
        assert torch.equal(one[0], head_seq[:, e]) and torch.equal(one[1], a[1][e:e + 1]) and torch.equal(one[2], a[2][e:e + 1])
    # CUDA graph: static buffers, capture, poison the workspace, replay
    head, hS, cS = (torch.empty_like(a[0]), torch.empty_like(a[1]), torch.empty_like(a[2]))
    g3 = torch.zeros_like(flat)
    tc.forward(obs, rows, S, n, flat, h0, c0, done, head, hS, cS)        # allocate workspaces outside the capture
    tc.backward(obs, rows, S, n, flat, done, dhead, g3)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            tc.forward(obs, rows, S, n, flat, h0, c0, done, head, hS, cS)
            tc.backward(obs, rows, S, n, flat, done, dhead, g3)
    torch.cuda.current_stream().wait_stream(s)
    tc.pin()
    ws = tc.acts(S, n)
    t = tc.act_tensors(S, n)
    for k in ("act1", "act2", "act3", "feats", "gx", "hseq", "hm", "save", "cm", "dgates"):
        t[k].fill_(float("nan") if t[k].is_floating_point() else 0)
    head.fill_(float("nan")); g3[:tc.param_count].fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert ws.data_ptr() == tc.acts(S, n).data_ptr()
    assert torch.equal(head, a[0]) and torch.equal(hS, a[1]) and torch.equal(cS, a[2]) and torch.equal(g3, g1)


@pytest.mark.gpu
def test_rollout_steps_equal_training_forward(lib):
    """Logits and value of S = 1 rollout calls carrying (h, c) equal the training forward over the whole sequence."""
    S, n, A = 16, 3, 6
    agent = _agent(A)
    obs, rows, done, h0, c0 = _inputs(S, n, "random")
    lg, val = [v.clone() for v in _run(agent, obs, rows, done, h0, c0, S, n)]
    state = (h0.view(1, n, 128), c0.view(1, n, 128))
    for t in range(S):
        r_t = rows[t * n:(t + 1) * n]
        hseq, state = agent.get_states(obs[r_t], state, done[t * n:(t + 1) * n])
        l_t, v_t = agent._heads(hseq)
        assert _close(l_t, lg[t * n:(t + 1) * n], 1e-5) and _close(v_t, val[t * n:(t + 1) * n], 1e-5), t


@pytest.mark.gpu
def test_bf16_branch_rejects_other_observations(lib):
    agent = _agent(4)
    state = (torch.zeros(1, 2, 128, device="cuda"), torch.zeros(1, 2, 128, device="cuda"))
    with pytest.raises(ValueError, match="uint8 frames"):
        agent.get_states(torch.zeros(2, 1, 84, 84, device="cuda"), state, torch.zeros(2, device="cuda"))
    with pytest.raises(ValueError, match="uint8 frames"):
        agent.get_states(torch.zeros(2, 4, 84, 84, dtype=torch.uint8, device="cuda"), state, torch.zeros(2, device="cuda"))


class _Writer:
    def __init__(self, *a, **k):
        self.scalars = []
    def add_text(self, *a, **k): pass
    def add_scalar(self, tag, v, step): self.scalars.append((tag, float(np.asarray(v).reshape(-1)[0]), int(step)))
    def close(self): pass


@pytest.mark.gpu
def test_lstm_script_bf16_vs_reference_run(lib):
    """ppo_atari_lstm.py --precision bf16 vs the unmodified reference script (same CPU noise): iteration 1 >= 99 % of the
    actions agree and logprobs / values / advantages / returns within 2e-2; update 1's losses within 1e-2, the other 15
    within 5e-2; later iterations >= 50 % agreement; TensorBoard tags and steps identical."""
    from cleanrl_b200 import ppo_atari_lstm as S
    z = np.load(GOLDEN / "ppo_atari_lstm_n8_t16_seed4.npz")
    argv = [a for a in z["argv"].tolist() if a != "--no-cuda"] + ["--synthetic-env", "--precision", "bf16"]
    snaps, writers = [], []

    def on_it(it, state, st):
        assert state["agent"].precision == "bf16"
        snaps.append({k: state[k].cpu().numpy().copy() for k in
                      ("actions", "logprobs", "values", "rewards", "dones", "advantages", "returns")} | {"st": st})

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
    for k in ("logprobs", "values", "advantages", "returns"):
        assert rel(s[k], z[k][0]) <= 2e-2, (k, rel(s[k], z[k][0]))
    per = s["st"]["per_update"]
    assert per.shape[0] == 16
    for u in range(16):
        for col, key in ((0, "upd_pg_loss"), (1, "upd_v_loss"), (2, "upd_entropy_loss"), (6, "upd_loss")):
            ref = float(z[key][u])
            assert abs(per[u, col] - ref) <= (1e-2 if u == 0 else 5e-2) * max(1.0, abs(ref)), (u, key, per[u, col], ref)
    for it in range(1, n_it):
        assert (snaps[it]["actions"] == z["actions"][it].astype(np.int64)).mean() >= 0.5
    ours = {}
    for tag, v, step in writers[0].scalars:
        ours.setdefault(tag, []).append((step, v))
    for key in z.files:
        if not key.startswith("tb/") or key == "tb/charts/SPS" or key.startswith("tb/charts/episodic"):
            continue
        tag = key[3:]
        assert tag in ours, tag
        assert np.array_equal(np.array(ours[tag])[:, 0], z[key][:, 0]), tag


@pytest.mark.parametrize("S,n,A", [(16, 2, 6)])
def test_argument_validation_without_gpu(lib, S, n, A):
    """The recurrent-agent entry points reject bad arguments before any CUDA call (testable on a CPU-only machine)."""
    import ctypes
    p = 1 << 20                                           # an aligned, never-dereferenced address
    fwd, bwd = lib.b200rl_lstm_agent_bf16_forward, lib.b200rl_lstm_agent_bf16_backward

    def f(**kw):
        a = dict(obs=p, rows=None, S=S, n=n, A=A, params=p, packed=p, h0=p, c0=p, done=p, acts=p, head=p, h=p, c=p)
        a.update(kw)
        return fwd(*a.values(), None)

    def b(**kw):
        a = dict(obs=p, rows=None, S=S, n=n, A=A, params=p, packed=p, done=p, acts=p, dhead=p, grads=p, ws=p, wsb=1 << 40)
        a.update(kw)
        return bwd(*a.values(), None)
    for call in (f, b):
        for kw, msg in (({"obs": None}, b"null"), ({"params": None}, b"null"), ({"A": 0}, b"outside"),
                        ({"A": 24}, b"outside"), ({"S": 0}, b"S="), ({"n": 0}, b"S="), ({"S": 1 << 9, "n": 1 << 9}, b"S="),
                        ({"S": -1}, b"S="), ({"rows": p + 4}, b"misaligned"), ({"obs": p + 8}, b"misaligned")):
            assert call(**kw) == -1, (call.__name__, kw)
            assert msg in lib.b200rl_last_error(), (kw, lib.b200rl_last_error())
    assert f(h0=p + 8) == -1 and b"misaligned" in lib.b200rl_last_error()
    assert b(wsb=16) == -4                                 # workspace too small
    assert lib.b200rl_lstm_agent_bf16_pack(None, A, p, None) == -1
    assert lib.b200rl_lstm_agent_bf16_pack(p, 24, p, None) == -1
    assert lib.b200rl_lstm_agent_bf16_acts_bytes(0, 4) == 0 and lib.b200rl_lstm_agent_bf16_acts_bytes(1 << 9, 1 << 9) == 0
    assert lib.b200rl_lstm_agent_bf16_workspace_bytes(S, n, 0) == 0 and lib.b200rl_lstm_agent_bf16_packed_bytes(30) == 0
    off = (ctypes.c_int64 * 13)()
    assert lib.b200rl_lstm_agent_bf16_acts_layout(S, n, off) == 0 and len(set(off)) == 13 and min(off) == 0
    assert lib.b200rl_lstm_agent_param_count(A) == 2048 + 32 + 32768 + 64 + 36864 + 64 + 3136 * 512 + 512 + \
        512 * 512 + 512 * 128 + 1024 + (A + 1) * 129
